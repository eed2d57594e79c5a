"""hnb_batch_cull's kernels (hnb_static_kernels.cu: k_cull_plan, k_cull_test<FAST>, k_cull_scan, k_cull_write) under the
CPU thread emulation of tests/static_emu.py, bit for bit against the numpy restatement tests/cull_ref.py, with d_visible,
d_args and the scratch between poisoned guards. The host's part (where `position` sits in the slab's columns, the
scratch layout) is restated here."""
import ctypes as C

import numpy as np
import pytest

from tests import static_emu as S
from tests.cull_ref import frustum_planes, ref_cull, visible_mask
from tests.helpers import Instance, RefWorld
from tests.kernel_emu import claim
from tests.static_emu import churned

pytestmark = pytest.mark.timeout(900)

CULL_DRIVER = r"""
extern "C" void semu_batch_cull(const CullArgs* a, int fast, uint32_t grid) {
    CullArgs d = *a;
    emu_run([&] { k_cull_plan(d); }, 1, DO_THREADS);
    if (fast) emu_run([&] { k_cull_test<true>(d); }, grid, DO_THREADS, 4);
    else emu_run([&] { k_cull_test<false>(d); }, grid, DO_THREADS, 4);
    emu_run([&] { k_cull_scan(d); }, d.src.max_instances, DO_THREADS, 8);
    emu_run([&] { k_cull_write(d); }, grid, DO_THREADS, 4);
}
extern "C" uint32_t semu_sizeof_cull_args(void) { return sizeof(CullArgs); }
extern "C" uint32_t semu_cull_tile(void) { return DO_TILE; }
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


MASK_WORDS = 128


@pytest.fixture(scope="module")
def clib():
    lib = S.build(CULL_DRIVER)
    lib.semu_batch_cull.argtypes = [C.c_void_p, C.c_int, C.c_uint32]
    lib.semu_batch_cull.restype = None
    lib.semu_sizeof_cull_args.restype = C.c_uint32
    lib.semu_cull_tile.restype = C.c_uint32
    assert lib.semu_sizeof_cull_args() == C.sizeof(CullArgs)
    assert lib.semu_cull_tile() == 32 * MASK_WORDS
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

GUARD = 64
POISON = np.uint32(0xA5A5A5A5)


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


class Device:
    """A RefWorld's slab in the device's layout under `plan`, a draw-args table, every buffer between poisoned guards,
    and what one hnb_batch_cull call over it enqueues."""

    def __init__(self, ref, plan, pos_word, claims=(0, 0), draw_rows=None, rng=None):
        self.ref, self.plan, self.pos_word = ref, plan, pos_word
        self.planes = [guarded(np.ascontiguousarray(ref.particles[:, off // 4:(off + w) // 4]).reshape(-1), np.uint32(0x7FC00000))
                       for off, w in plan]
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

    def run(self, lib, batch, frusta, src=None, count=None, grid=3, num_spawners=None, num_metadata=None, visible=None):
        """(d_visible after the call, d_args rows, fast); `visible` is d_visible's content before (poison by default)."""
        bi = self.batch_infos[batch]
        count = bi.prefix_sum_count if count is None else count
        rows = self.ref.slab_rows
        where, fast = position_columns(self.plan, self.pos_word)
        max_tiles = rows // lib.semu_cull_tile() + count
        out = guarded(np.full(rows, POISON, dtype=np.uint32) if visible is None else visible, POISON)
        args = guarded(np.full(5 * count, POISON, dtype=np.uint32), POISON)
        frusta_buf = guarded(np.ascontiguousarray(frusta, dtype=np.float32).reshape(-1).view(np.uint32), np.uint32(0x7FC00000))
        src_buf = None if src is None else guarded(np.ascontiguousarray(src, dtype=np.uint32), POISON)
        scratch = guarded(np.full((MASK_WORDS + 1) * max_tiles + 8 * count + 1, 0x5A5A5A5A, dtype=np.uint32), POISON)
        base = scratch[GUARD:]
        a = CullArgs()
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
        a.prefix = base[MASK_WORDS * max_tiles:].ctypes.data
        a.info = base[(MASK_WORDS + 1) * max_tiles:].ctypes.data
        a.total_tiles = base[(MASK_WORDS + 1) * max_tiles + 8 * count:].ctypes.data
        a.max_tiles = max_tiles
        inputs = [frusta_buf] + ([] if src_buf is None else [src_buf])
        state = self.state() + [x.copy() for x in inputs]
        lib.semu_batch_cull(C.byref(a), int(fast), grid)
        for k, (x, y) in enumerate(zip(state, self.state() + inputs)):
            np.testing.assert_array_equal(x, y, err_msg=f"the cull modified buffer {k}")
        for name, buf in (("d_visible", out), ("d_args", args), ("the scratch", scratch)):
            assert (buf[:GUARD] == POISON).all() and (buf[-GUARD:] == POISON).all(), f"stores outside {name}"
        return out[GUARD:-GUARD], args[GUARD:-GUARD].reshape(-1, 5), fast

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


def random_frusta(rng, count, scale=100.0):
    """Six planes of random unit normals, each passing most of a cloud of N(0, scale) points: a few to most visible."""
    f = rng.standard_normal((max(count, 1), 6, 3))
    f /= np.linalg.norm(f, axis=2, keepdims=True)
    d = rng.uniform(0.2, 1.8, (max(count, 1), 6, 1)) * scale
    return np.concatenate([f, d], axis=2).astype(np.float32)


def check(dev, lib, ref, batch, frusta, grid=3, src=None, **kw):
    got, args, fast = dev.run(lib, batch, frusta, src=src, grid=grid, **kw)
    want, want_args = ref_cull(ref, batch, dev.pos_word, frusta, np.full(ref.slab_rows, POISON, dtype=np.uint32),
                               dev.table(), src=src, count=kw.get("count"), num_spawners=kw.get("num_spawners"),
                               num_metadata=kw.get("num_metadata"))
    np.testing.assert_array_equal(got, want, err_msg="visible entries (poison marks rows that must not be written)")
    np.testing.assert_array_equal(args, want_args, err_msg="draw args")
    return got, args, fast


def test_restatement_by_hand():
    """On a plane (+0 and -0) is inside; NaN positions, NaN planes and inf * 0 fail; one ulp outside fails; the six planes
    of a view-projection matrix keep exactly the points of its clip volume; entries keep their order."""
    f32 = np.float32
    half_space = np.array([[1, 0, 0, 0]] + [[0, 0, 0, 1]] * 5, dtype=np.float32)  # x >= 0
    below = -np.nextafter(f32(0), f32(1))
    xs = np.array([0.0, -0.0, below, 1.0, np.nan, np.inf, -np.inf, 5.0], dtype=np.float32)
    words = np.zeros((len(xs), 3), dtype=np.float32)
    words[:, 0] = xs
    # inf * 0 is NaN: the planes (0, 0, 0, 1) fail an infinite x, so +inf is outside too
    assert visible_mask(half_space, words.view(np.uint32)).tolist() == [True, True, False, True, False, False, False, True]
    y_half_space = np.array([[0, 1, 0, 0]] + [[0, 0, 0, 1]] * 5, dtype=np.float32)
    assert visible_mask(y_half_space, words.view(np.uint32)).tolist() == [True, True, True, True, False, False, False, True]
    # a NaN plane fails everything
    nan_plane = half_space.copy()
    nan_plane[3, 3] = np.nan
    assert not visible_mask(nan_plane, words.view(np.uint32)).any()
    # ((a*x + b*y) + c*z) + d, one rounding per step: 1e8 + 1 - 1e8 is 0 in float32 when added in this order
    p = np.array([[f32(1e8), f32(1.0), f32(-1e8)]], dtype=np.float32).view(np.uint32)
    assert visible_mask(np.array([[1, 1, 1, -0.5]] + [[0, 0, 0, 1]] * 5, dtype=np.float32), p).tolist() == [False]
    # an orthographic box [-1, 1]^2 x [0, 1] (the identity view-projection): radius 0.5 widens it by 0.5
    box = frustum_planes(np.eye(4))
    pts = np.array([[0, 0, 0.5], [1, 1, 1], [1.25, 0, 0.5], [0, 0, -0.25], [0, -1.5, 1.5]], dtype=np.float32)
    assert visible_mask(box, pts.view(np.uint32)).tolist() == [True, True, False, False, False]
    assert visible_mask(frustum_planes(np.eye(4), 0.5), pts.view(np.uint32)).tolist() == [True, True, True, True, True]


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_mixed_sizes_in_one_batch(clib, layout):
    """Sizes across the tile boundary in one batch behind a batch of one: 0, 1, tile - 1, tile, tile + 1, several tiles, a
    small one; lists permuted after deaths, in alternating columns. Every position layout, the fast one included."""
    stride_words, plan, pos_word, want_fast = LAYOUTS[layout]
    rng = np.random.default_rng(len(layout) * 17)
    tile = clib.semu_cull_tile()
    caps = [40, 8, 3, tile + 10, tile, tile + 40, 3 * tile + 500, 90]
    alive = [20, 0, 1, tile - 1, tile, tile + 1, 3 * tile + 123, 77]
    ref = random_world(rng, stride_words, caps, alive, pos_word, batches=[[0], list(range(1, 8))])
    _, args, fast = check(Device(ref, plan, pos_word, rng=rng), clib, ref, 1, random_frusta(rng, 7))
    assert fast == want_fast
    assert 0 < args[3:, 1].min() and (args[3:, 1] < np.array(alive[4:])).all(), "some of every large instance is visible, not all"


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
    check(Device(ref, C5_OWN, 0, rng=rng), clib, ref, 0, random_frusta(rng, 300), grid=grid)


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
    check(dev, clib, ref, 0, random_frusta(rng, 3))


@pytest.mark.parametrize("size", ["small", "large"])
def test_source_buffer(clib, size):
    """d_src in place of the alive list: a permutation of each instance's live slots (as a depth order gives), with some
    entries past the slice, which are clamped; a claim on column W does not apply to d_src."""
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
    got, _, _ = check(dev, clib, ref, 0, random_frusta(rng, 3), src=src)
    assert (got[:n + 50] == n + 49).any(), "a clamped entry is visible"


@pytest.mark.parametrize("size", ["small", "large"])
def test_special_values(clib, size):
    """Points exactly on a plane (+0 and -0 results), NaN and infinite positions, NaN and infinite plane words, a frustum
    that keeps everything and one that keeps nothing."""
    rng = np.random.default_rng(9)
    tile = clib.semu_cull_tile()
    n = 700 if size == "small" else tile + 31
    ref = random_world(rng, 8, [n] * 5, [n] * 5)
    specials = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1.0, -1.0, 1e-45, -1e-45], dtype=np.float32).view(np.uint32)
    for j in range(3):
        ref.particles[j * n:(j + 1) * n, 0:3] = rng.choice(specials, (n, 3))
    ones = [[0, 0, 0, 1]] * 6
    frusta = np.array([
        [[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0], [-1, 0, 0, 0], [0, 0, 0, 0], [0, 0, 0, -0.0]],  # x = +-0, y, z >= 0, finite
        [[1, 0, 0, 0], [0, 0, 0, np.inf]] + ones[:4],                                            # x >= 0 and an infinite d
        [[1, 1, 1, 0], [0, 0, 0, np.nan]] + ones[:4],                                            # a NaN plane: nothing
        ones,                                                                                   # finite positions: everything
        [[0, 0, 0, -1]] + ones[:5],                                                             # nothing
    ], dtype=np.float32)
    got, args, _ = check(Device(ref, default_cut(32), 0, rng=rng), clib, ref, 0, frusta)
    assert args[2, 1] == 0 and args[3, 1] == n and args[4, 1] == 0 and 0 < args[0, 1] < n
    f3 = ref.instances[3].slab_offset
    np.testing.assert_array_equal(got[f3:f3 + n], ref.indirect[f3:f3 + n, 1], "everything visible: the list itself")


def test_unwritten_rows_keep_their_bytes(clib):
    """Only d_visible[first, first + m) of each instance is written: every other row keeps what it held."""
    rng = np.random.default_rng(4)
    tile = clib.semu_cull_tile()
    ref = random_world(rng, 8, [100, tile + 200, 60, 2 * tile], [50, tile + 3, 0, tile + 5])
    before = rng.integers(0, 1 << 32, ref.slab_rows, dtype=np.uint64).astype(np.uint32)
    frusta = random_frusta(rng, 4)
    dev = Device(ref, default_cut(32), 0, rng=rng)
    got, _, _ = dev.run(clib, 0, frusta, visible=before.copy())
    want, _ = ref_cull(ref, 0, 0, frusta, before, dev.table())
    np.testing.assert_array_equal(got, want)


def test_out_of_range_table_words(clib):
    """List entries, slab offsets, capacities, alive counts, metadata indices, draw-args rows and the batch's own row past
    their tables are clamped as bounds clamps them, and no access leaves the buffers (all between poisoned guards). A
    call over more instances than the device's batch row holds writes args with instance_count 0 for the rest."""
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
    frusta = random_frusta(rng, 7)
    check(Device(ref, default_cut(32), 0, draw_rows=4, rng=rng), clib, ref, 0, frusta)
    ref.batch_infos[0].prefix_sum_count = 3
    _, args, _ = check(Device(ref, default_cut(32), 0, rng=rng), clib, ref, 0, frusta, count=5)
    assert (args[3:, 1] == 0).all()
