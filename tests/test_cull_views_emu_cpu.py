"""hnb_batch_cull_views's kernels (hnb_static_kernels.cu: k_cull_plan, k_cull_views_test<FAST>, k_cull_views_scan,
k_cull_views_write) under the CPU thread emulation of tests/static_emu.py. Every view's visible entries and draw args
equal the numpy restatement tests/cull_ref.py for its own frustum, bit for bit; d_visible, d_args and d_frusta hold the
views stacked with poisoned gaps between their slices, and every buffer sits between poisoned guards. One view, and any
view of a larger call, equals what the single-view kernels write byte for byte. The host's part (where `position` sits
in the slab's columns, the stacked layout, the scratch layout) is restated here."""
import ctypes as C

import numpy as np
import pytest

from tests import static_emu as S
from tests.cull_ref import ref_cull
from tests.helpers import Instance, RefWorld
from tests.kernel_emu import claim
from tests.static_emu import churned

pytestmark = pytest.mark.timeout(900)

VIEWS_DRIVER = r"""
extern "C" void semu_batch_cull_views(const CullViewsArgs* a, int fast, uint32_t grid) {
    CullViewsArgs d = *a;
    emu_run([&] { k_cull_plan(d.c); }, 1, DO_THREADS);
    if (fast) emu_run([&] { k_cull_views_test<true>(d); }, grid, DO_THREADS, 4);
    else emu_run([&] { k_cull_views_test<false>(d); }, grid, DO_THREADS, 4);
    emu_run([&] { k_cull_views_scan(d); }, d.c.src.max_instances * d.views, DO_THREADS, 8);
    emu_run([&] { k_cull_views_write(d); }, grid, DO_THREADS, 4);
}
extern "C" void semu_batch_cull_one(const CullArgs* a, int fast, uint32_t grid) {
    CullArgs d = *a;
    emu_run([&] { k_cull_plan(d); }, 1, DO_THREADS);
    if (fast) emu_run([&] { k_cull_test<true>(d); }, grid, DO_THREADS, 4);
    else emu_run([&] { k_cull_test<false>(d); }, grid, DO_THREADS, 4);
    emu_run([&] { k_cull_scan(d); }, d.src.max_instances, DO_THREADS, 8);
    emu_run([&] { k_cull_write(d); }, grid, DO_THREADS, 4);
}
extern "C" uint32_t semu_sizeof_cull_views_args(void) { return sizeof(CullViewsArgs); }
extern "C" uint32_t semu_cull_tile(void) { return DO_TILE; }
extern "C" uint32_t semu_cull_max_views(void) { return HNB_BATCH_CULL_MAX_VIEWS; }
"""


class BoundsArgs(C.Structure):
    """hnb::BoundsArgs (hnb_static_kernels.h)"""
    _fields_ = [("batch_info", C.c_void_p), ("spawners", C.c_void_p), ("metadata", C.c_void_p), ("num_spawners", C.c_uint32),
                ("num_metadata", C.c_uint32), ("ping", C.c_void_p), ("pong", C.c_void_p), ("claim", C.c_void_p),
                ("capacity_rows", C.c_uint32), ("max_instances", C.c_uint32), ("col", C.c_void_p * 3), ("col_words", C.c_uint32 * 3),
                ("col_lane", C.c_uint32 * 3), ("acc", C.c_void_p), ("out", C.c_void_p)]


class CullArgs(C.Structure):
    """hnb::CullArgs (hnb_static_kernels.h)"""
    _fields_ = [("src", BoundsArgs), ("frusta", C.c_void_p), ("src_list", C.c_void_p), ("visible", C.c_void_p), ("args", C.c_void_p),
                ("draw_args", C.c_void_p), ("num_draw_args", C.c_uint32), ("mask", C.c_void_p), ("prefix", C.c_void_p),
                ("info", C.c_void_p), ("total_tiles", C.c_void_p), ("max_tiles", C.c_uint32)]


class CullViewsArgs(C.Structure):
    """hnb::CullViewsArgs (hnb_static_kernels.h)"""
    _fields_ = [("c", CullArgs), ("views", C.c_uint32), ("frustum_rows", C.c_uint32), ("visible_rows", C.c_uint32),
                ("args_rows", C.c_uint32)]


MASK_WORDS = 128
GUARD = 64
POISON = np.uint32(0xA5A5A5A5)
NAN = np.uint32(0x7FC00000)
# rows between consecutive views' slices: visible entries, frusta (NaN planes: a view that read them would see nothing)
# and args rows
VISIBLE_GAP, FRUSTUM_GAP, ARGS_GAP = 37, 2, 3


@pytest.fixture(scope="module")
def clib():
    lib = S.build(VIEWS_DRIVER)
    for f in ("semu_batch_cull_views", "semu_batch_cull_one"):
        getattr(lib, f).argtypes = [C.c_void_p, C.c_int, C.c_uint32]
        getattr(lib, f).restype = None
    for f in ("semu_sizeof_cull_views_args", "semu_cull_tile", "semu_cull_max_views"):
        getattr(lib, f).restype = C.c_uint32
    assert lib.semu_sizeof_cull_views_args() == C.sizeof(CullViewsArgs)
    assert lib.semu_cull_tile() == 32 * MASK_WORDS
    assert lib.semu_cull_max_views() == 8
    return lib


def default_cut(stride, sector=False):
    plan, off = [], 0
    for w in S.physical_widths(stride, sector):
        plan.append((off, w))
        off += w
    return plan


C5_OWN = [(0, 16), (16, 8), (24, 4), (28, 4)]
SPLIT = [(0, 8), (8, 4), (12, 4), (16, 16)]
LAYOUTS = {
    "32-default": (8, default_cut(32), 0, True),
    "32-c5-own": (8, C5_OWN, 0, True),
    "32-split": (8, SPLIT, 0, False),
    "32-unaligned": (8, default_cut(32), 1, False),
    "32-sector": (8, default_cut(32, True), 0, True),
    "32-sector-second-half": (8, default_cut(32, True), 4, True),
    "48-default": (12, default_cut(48), 4, True),
}


def guarded(data, poison):
    buf = np.full(len(data) + 2 * GUARD, poison, dtype=data.dtype)
    buf[GUARD:GUARD + len(data)] = data
    return buf


def position_columns(plan, pos_word):
    where = []
    for k in range(3):
        byte = 4 * (pos_word + k)
        p = next(i for i, (off, w) in enumerate(plan) if off <= byte < off + w)
        where.append((p, plan[p][1] // 4, (byte - plan[p][0]) // 4))
    fast = where[0][0] == where[2][0] and where[0][2] % 4 == 0 and where[0][1] % 4 == 0
    return where, fast


def stacked(views, rows, per_view, gap, poison):
    """`views` slices of `rows` rows (each `per_view` = a list of arrays, or None for poison), `gap` poisoned rows apart."""
    width = rows + gap
    out = np.full(views * width, poison, dtype=np.uint32)
    for v in range(views):
        if per_view is not None:
            out[v * width:v * width + rows] = per_view[v]
    return out


class Device:
    """A RefWorld's slab in the device's layout under `plan`, a draw-args table, every buffer between poisoned guards,
    and what one hnb_batch_cull_views (or, through `single`, hnb_batch_cull) call over it enqueues."""

    def __init__(self, ref, plan, pos_word, claims=(0, 0), draw_rows=None, rng=None):
        self.ref, self.plan, self.pos_word = ref, plan, pos_word
        self.planes = [guarded(np.ascontiguousarray(ref.particles[:, off // 4:(off + w) // 4]).reshape(-1), NAN) for off, w in plan]
        self.lists = [guarded(np.ascontiguousarray(ref.indirect[:, c]), np.uint32(0xFFFFFFF0)) for c in range(2)]
        self.claims = guarded(np.array(claims, dtype=np.uint64), np.uint64(claim(0, 1 << 30)))
        self.spawners = (type(ref.spawners[0]) * len(ref.spawners)).from_buffer_copy(bytes(ref.spawners))
        self.metadata = (type(ref.metadata[0]) * len(ref.metadata)).from_buffer_copy(bytes(ref.metadata))
        self.batch_infos = (type(ref.batch_infos[0]) * len(ref.batch_infos)).from_buffer_copy(bytes(ref.batch_infos))
        rng = rng or np.random.default_rng(0)
        rows = len(ref.spawners) if draw_rows is None else draw_rows
        self.draw_args = guarded(rng.integers(0, 1 << 32, 5 * rows, dtype=np.uint64).astype(np.uint32), POISON)

    def list(self, c):
        return self.lists[c][GUARD:-GUARD]

    def table(self):
        return self.draw_args[GUARD:-GUARD]

    def run(self, lib, batch, frusta, src=None, count=None, grid=3, num_spawners=None, num_metadata=None, visible=None,
            single=False):
        """([d_visible of each view], [d_args rows of each view], fast). `frusta` is (views, instances, 6, 4); `visible`
        each view's d_visible before the call (poison by default). `single`: one view through the single-view kernels."""
        bi = self.batch_infos[batch]
        count = bi.prefix_sum_count if count is None else count
        views = len(frusta)
        assert not single or views == 1
        rows = self.ref.slab_rows
        where, fast = position_columns(self.plan, self.pos_word)
        max_tiles = rows // lib.semu_cull_tile() + count
        frustum_rows, args_rows = count + FRUSTUM_GAP, count + ARGS_GAP
        out = guarded(stacked(views, rows, visible, VISIBLE_GAP, POISON), POISON)
        args = guarded(stacked(views, 5 * count, None, 5 * ARGS_GAP, POISON), POISON)
        f = np.asarray(frusta, dtype=np.float32).reshape(views, -1, 24)[:, :count].view(np.uint32)
        frusta_buf = guarded(stacked(views, 24 * count, f.reshape(views, -1), 24 * FRUSTUM_GAP, NAN), NAN)
        src_buf = None if src is None else guarded(np.ascontiguousarray(src, dtype=np.uint32), POISON)
        scratch = guarded(np.full(views * (MASK_WORDS + 1) * max_tiles + 8 * count + 1, 0x5A5A5A5A, dtype=np.uint32), POISON)
        base = scratch[GUARD:]
        v = CullViewsArgs()
        a = v.c
        s = a.src
        s.batch_info = C.addressof(self.batch_infos[batch])
        s.spawners, s.metadata = C.addressof(self.spawners), C.addressof(self.metadata)
        s.num_spawners = len(self.spawners) if num_spawners is None else num_spawners
        s.num_metadata = len(self.metadata) if num_metadata is None else num_metadata
        s.ping, s.pong = self.lists[0][GUARD:].ctypes.data, self.lists[1][GUARD:].ctypes.data
        s.claim = self.claims[GUARD:].ctypes.data
        s.capacity_rows, s.max_instances = rows, count
        for k, (p, words, lane) in enumerate(where):
            s.col[k], s.col_words[k], s.col_lane[k] = self.planes[p][GUARD:].ctypes.data, words, lane
        a.frusta = frusta_buf[GUARD:].ctypes.data
        a.src_list = None if src_buf is None else src_buf[GUARD:].ctypes.data
        a.visible, a.args = out[GUARD:].ctypes.data, args[GUARD:].ctypes.data
        a.draw_args, a.num_draw_args = self.draw_args[GUARD:].ctypes.data, len(self.table()) // 5
        a.mask = base.ctypes.data
        a.prefix = base[views * MASK_WORDS * max_tiles:].ctypes.data
        a.info = base[views * (MASK_WORDS + 1) * max_tiles:].ctypes.data
        a.total_tiles = base[views * (MASK_WORDS + 1) * max_tiles + 8 * count:].ctypes.data
        a.max_tiles = max_tiles
        v.views, v.frustum_rows, v.visible_rows, v.args_rows = views, frustum_rows, rows + VISIBLE_GAP, args_rows
        inputs = [frusta_buf] + ([] if src_buf is None else [src_buf])
        state = self.state() + [x.copy() for x in inputs]
        if single:
            lib.semu_batch_cull_one(C.byref(a), int(fast), grid)
        else:
            lib.semu_batch_cull_views(C.byref(v), int(fast), grid)
        for k, (x, y) in enumerate(zip(state, self.state() + inputs)):
            np.testing.assert_array_equal(x, y, err_msg=f"the cull modified buffer {k}")
        for name, buf in (("d_visible", out), ("d_args", args), ("the scratch", scratch)):
            assert (buf[:GUARD] == POISON).all() and (buf[-GUARD:] == POISON).all(), f"stores outside {name}"
        vis, arg = out[GUARD:-GUARD].reshape(views, -1), args[GUARD:-GUARD].reshape(views, -1)
        assert (vis[:, rows:] == POISON).all(), "stores into the gap after a view's entries"
        assert (arg[:, 5 * count:] == POISON).all(), "stores into the args rows past a view's instances"
        return list(vis[:, :rows]), [x[:5 * count].reshape(-1, 5) for x in arg], fast

    def state(self):
        tables = [np.frombuffer(bytes(t), dtype=np.uint32).copy() for t in (self.spawners, self.metadata, self.batch_infos)]
        return [p.copy() for p in self.planes] + [l.copy() for l in self.lists] + [self.claims.copy(), self.draw_args.copy()] + tables


def random_world(rng, stride_words, caps, alive, pos_word=0, batches=None, scale=100.0):
    """Instances back to back, instance j with alive[j] live particles through a permuted list in column j & 1."""
    insts, off = [], 0
    for c in caps:
        insts.append(Instance(off, c))
        off += c
    ref = RefWorld(max(off, 1), stride_words, insts, batches=batches)
    ref.particles[:] = rng.integers(0, 1 << 32, ref.particles.shape, dtype=np.uint64).astype(np.uint32)
    ref.particles[:, pos_word:pos_word + 3] = (rng.standard_normal((ref.slab_rows, 3)) * scale).astype(np.float32).view(np.uint32)
    for j, n in enumerate(alive):
        churned(rng, ref, j, n, w=j & 1)
    return ref


def random_frusta(rng, views, count, scale=100.0):
    """Per view and instance, six planes of random unit normals, each passing most of a cloud of N(0, scale) points: a few
    to most visible, and different in every view. (views, count, 6, 4) float32."""
    f = rng.standard_normal((views, max(count, 1), 6, 3))
    f /= np.linalg.norm(f, axis=3, keepdims=True)
    d = rng.uniform(0.2, 1.8, (views, max(count, 1), 6, 1)) * scale
    return np.concatenate([f, d], axis=3).astype(np.float32)


def check(dev, lib, ref, batch, frusta, grid=3, src=None, **kw):
    """Every view against ref_cull for its own frusta."""
    got, args, fast = dev.run(lib, batch, frusta, src=src, grid=grid, **kw)
    for v in range(len(frusta)):
        want, want_args = ref_cull(ref, batch, dev.pos_word, frusta[v], np.full(ref.slab_rows, POISON, dtype=np.uint32),
                                   dev.table(), src=src, count=kw.get("count"), num_spawners=kw.get("num_spawners"),
                                   num_metadata=kw.get("num_metadata"))
        np.testing.assert_array_equal(got[v], want, err_msg=f"view {v}: visible entries (poison marks rows that must not be written)")
        np.testing.assert_array_equal(args[v], want_args, err_msg=f"view {v}: draw args")
    return got, args, fast


def mixed_world(rng, layout, tile):
    stride_words, plan, pos_word, want_fast = LAYOUTS[layout]
    caps = [40, 8, 3, tile + 10, tile, tile + 40, 3 * tile + 500, 90]
    alive = [20, 0, 1, tile - 1, tile, tile + 1, 3 * tile + 123, 77]
    ref = random_world(rng, stride_words, caps, alive, pos_word, batches=[[0], list(range(1, 8))])
    return ref, Device(ref, plan, pos_word, rng=rng), want_fast


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_every_layout(clib, layout):
    """Sizes across the tile boundary in one batch behind a batch of one: 0, 1, tile - 1, tile, tile + 1, several tiles, a
    small one; lists permuted after deaths, in alternating columns. Every position layout, the fast one included, with
    three views that see different parts."""
    rng = np.random.default_rng(len(layout) * 31)
    ref, dev, want_fast = mixed_world(rng, layout, clib.semu_cull_tile())
    _, args, fast = check(dev, clib, ref, 1, random_frusta(rng, 3, 7))
    assert fast == want_fast
    assert len({a[:, 1].tobytes() for a in args}) == 3, "the views see different counts"


@pytest.mark.parametrize("views", [1, 2, 3, 8])
@pytest.mark.parametrize("layout", ["32-c5-own", "32-split"])
def test_view_counts(clib, layout, views):
    """1, 2, 3 and the most views, on the fast layout and on position split over columns."""
    rng = np.random.default_rng(views * 5 + len(layout))
    ref, dev, _ = mixed_world(rng, layout, clib.semu_cull_tile())
    check(dev, clib, ref, 1, random_frusta(rng, views, 7))


@pytest.mark.parametrize("layout", ["32-default", "32-split"])
def test_each_view_is_the_single_view_call(clib, layout):
    """One view, and each view of a call of three, writes byte for byte what the single-view kernels write for its
    frusta, over visible buffers that held random words before the call."""
    rng = np.random.default_rng(len(layout))
    ref, dev, _ = mixed_world(rng, layout, clib.semu_cull_tile())
    frusta = random_frusta(rng, 3, 7)
    before = [rng.integers(0, 1 << 32, ref.slab_rows, dtype=np.uint64).astype(np.uint32) for _ in range(3)]
    got, args, _ = dev.run(clib, 1, frusta, visible=before)
    for v in range(3):
        one, one_args, _ = dev.run(clib, 1, frusta[v:v + 1], visible=before[v:v + 1], single=True)
        alone, alone_args, _ = dev.run(clib, 1, frusta[v:v + 1], visible=before[v:v + 1])
        for g, a in ((got[v], args[v]), (alone[0], alone_args[0])):
            assert g.tobytes() == one[0].tobytes() and a.tobytes() == one_args[0].tobytes()


@pytest.mark.parametrize("grid", [1, 2, 5])
def test_any_grid_and_many_instances(clib, grid):
    """300 instances of uneven sizes (one staging of the plan's scan is 256), two of several tiles, at any grid."""
    rng = np.random.default_rng(grid)
    tile = clib.semu_cull_tile()
    caps = [int(c) for c in rng.integers(1, 30, 300)]
    caps[17], caps[280] = 2 * tile + 9, tile + 1
    alive = [int(rng.integers(0, c + 1)) for c in caps]
    alive[17], alive[280] = 2 * tile + 9, tile + 1
    ref = random_world(rng, 8, caps, alive)
    check(Device(ref, C5_OWN, 0, rng=rng), clib, ref, 0, random_frusta(rng, 3, 300), grid=grid)


@pytest.mark.parametrize("size", ["small", "large"])
@pytest.mark.parametrize("claimed", ["all", "part", "none"])
def test_identity_claims(clib, size, claimed):
    """Column W is the identity under a claim over all, part or none of the live rows; claimed entries are poisoned with
    dead slots, whose positions would change the result."""
    rng = np.random.default_rng(7)
    tile = clib.semu_cull_tile()
    n = 1500 if size == "small" else 2 * tile + 100
    first, cap = 40, n + 300
    ref = random_world(rng, 8, [first, cap, 30], [10, 0, 7])
    md = ref.metadata[1]
    md.alive_count, md.indirect_write_index = n, 1
    ref.indirect[first:first + n, 1] = np.arange(n, dtype=np.uint32)
    length = {"all": n, "part": n // 2 + 3, "none": 0}[claimed]
    dev = Device(ref, default_cut(32), 0, claims=(claim(first, 5), claim(first, length)), rng=rng)
    dev.list(1)[first:first + length] = n + rng.integers(0, cap - n, length).astype(np.uint32)
    check(dev, clib, ref, 0, random_frusta(rng, 2, 3))


@pytest.mark.parametrize("size", ["small", "large"])
def test_source_buffer(clib, size):
    """d_src in place of the alive list, shared by every view: a permutation of each instance's live slots (as a depth
    order gives), with some entries past the slice, which are clamped; a claim on column W does not apply to d_src."""
    rng = np.random.default_rng(21)
    tile = clib.semu_cull_tile()
    n = 900 if size == "small" else 2 * tile + 77
    ref = random_world(rng, 8, [n + 50, 300, n], [n, 120, n - 5])
    src = rng.integers(0, 1 << 32, ref.slab_rows, dtype=np.uint64).astype(np.uint32)
    for j, inst in enumerate(ref.instances):
        k = ref.metadata[j].alive_count
        src[inst.slab_offset:inst.slab_offset + k] = rng.permutation(k).astype(np.uint32)
    src[3:n:7] = rng.integers(n + 50, 1 << 32, len(range(3, n, 7)), dtype=np.uint64).astype(np.uint32)
    ref.particles[n + 49, 0:3] = 0  # the slot the clamped entries name: the origin, inside every random frustum
    dev = Device(ref, default_cut(32), 0, claims=(claim(0, n), claim(0, 0)), rng=rng)
    got, _, _ = check(dev, clib, ref, 0, random_frusta(rng, 3, 3), src=src)
    assert all((g[:n + 50] == n + 49).any() for g in got), "a clamped entry is visible in every view"


@pytest.mark.parametrize("size", ["small", "large"])
def test_special_values_and_view_kinds(clib, size):
    """Points exactly on a plane (+0 and -0 results), NaN and infinite positions, NaN and infinite plane words; among eight
    views, one that sees everything, one that sees nothing, and the same frusta twice."""
    rng = np.random.default_rng(9)
    tile = clib.semu_cull_tile()
    n = 700 if size == "small" else tile + 31
    ref = random_world(rng, 8, [n] * 5, [n] * 5)
    specials = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1.0, -1.0, 1e-45, -1e-45], dtype=np.float32).view(np.uint32)
    for j in range(3):
        ref.particles[j * n:(j + 1) * n, 0:3] = rng.choice(specials, (n, 3))
    ones = [[0, 0, 0, 1]] * 6
    special = np.array([
        [[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0], [-1, 0, 0, 0], [0, 0, 0, 0], [0, 0, 0, -0.0]],  # x = +-0, y, z >= 0, finite
        [[1, 0, 0, 0], [0, 0, 0, np.inf]] + ones[:4],                                            # x >= 0 and an infinite d
        [[1, 1, 1, 0], [0, 0, 0, np.nan]] + ones[:4],                                            # a NaN plane: nothing
        ones,                                                                                   # finite positions: everything
        [[0, 0, 0, -1]] + ones[:5],                                                             # nothing
    ], dtype=np.float32)
    everything = np.tile(np.array(ones, dtype=np.float32), (5, 1, 1))
    nothing = np.tile(np.array([[0, 0, 0, -1]] + ones[:5], dtype=np.float32), (5, 1, 1))
    random = random_frusta(rng, 1, 5)[0]
    frusta = np.stack([special, everything, random, nothing, special[::-1], random, special, everything])
    got, args, _ = check(Device(ref, default_cut(32), 0, rng=rng), clib, ref, 0, frusta)
    assert args[0][2, 1] == 0 and args[0][3, 1] == n and args[0][4, 1] == 0 and 0 < args[0][0, 1] < n
    assert (args[1][3:, 1] == n).all() and (args[3][:, 1] == 0).all()  # inf * 0 fails even (0, 0, 0, 1)
    for a, b in ((0, 6), (2, 5), (1, 7)):
        assert got[a].tobytes() == got[b].tobytes() and args[a].tobytes() == args[b].tobytes(), "the same frusta twice"
    for j in (3, 4):  # finite positions
        f = ref.instances[j].slab_offset
        np.testing.assert_array_equal(got[1][f:f + n], ref.indirect[f:f + n, j & 1], "everything visible: the list itself")


def test_unwritten_rows_keep_their_bytes(clib):
    """Only d_visible[first, first + m) of each instance in each view is written: every other row keeps what it held."""
    rng = np.random.default_rng(4)
    tile = clib.semu_cull_tile()
    ref = random_world(rng, 8, [100, tile + 200, 60, 2 * tile], [50, tile + 3, 0, tile + 5])
    before = [rng.integers(0, 1 << 32, ref.slab_rows, dtype=np.uint64).astype(np.uint32) for _ in range(2)]
    frusta = random_frusta(rng, 2, 4)
    dev = Device(ref, default_cut(32), 0, rng=rng)
    got, _, _ = dev.run(clib, 0, frusta, visible=[b.copy() for b in before])
    for v in range(2):
        want, _ = ref_cull(ref, 0, 0, frusta[v], before[v], dev.table())
        np.testing.assert_array_equal(got[v], want)


def test_out_of_range_table_words(clib):
    """List entries, slab offsets, capacities, alive counts, metadata indices, draw-args rows and the batch's own row past
    their tables are clamped as bounds clamps them, and no access leaves the buffers (all between poisoned guards, views
    apart by poisoned gaps). A call over more instances than the device's batch row holds writes args with
    instance_count 0 for the rest, in every view."""
    rng = np.random.default_rng(11)
    ref = random_world(rng, 8, [300, 300, 300, 300, 5000], [200, 250, 100, 300, 50])
    first1 = ref.instances[1].slab_offset
    ref.indirect[first1:first1 + 250:3, 1] = rng.integers(300, 1 << 32, len(range(0, 250, 3)), dtype=np.uint64).astype(np.uint32)
    ref.spawners[2].slab_offset = 0xFFFFFF00            # a slice past the slab: empty
    ref.spawners[3].draw_indirect_index = 0xFFFFFFF0    # clamped to the last draw-args row
    ref.spawners[4].effect_metadata_index = 0x7FFFFFFF  # clamped to the last row: its own
    ref.metadata[4].capacity = 0xFFFFFFFF               # clamped to the rows the slab has from its offset
    ref.metadata[4].alive_count = 0xFFFFFFF0            # n = all of them, through a list of garbage words
    first4 = ref.instances[4].slab_offset
    ref.indirect[first4:, 0] = rng.integers(0, 1 << 32, ref.slab_rows - first4, dtype=np.uint64).astype(np.uint32)
    ref.batch_infos[0].prefix_sum_count = 5
    frusta = random_frusta(rng, 3, 7)
    check(Device(ref, default_cut(32), 0, draw_rows=4, rng=rng), clib, ref, 0, frusta)
    ref.batch_infos[0].prefix_sum_count = 3
    _, args, _ = check(Device(ref, default_cut(32), 0, rng=rng), clib, ref, 0, frusta, count=5)
    assert all((a[3:, 1] == 0).all() for a in args)
