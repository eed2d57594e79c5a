"""hnb_batch_depth_order's kernels (hnb_static_kernels.cu: k_do_plan, k_do_keys<FAST>, k_do_hist, k_do_scan, k_do_scatter)
under the CPU thread emulation of tests/static_emu.py, bit for bit against the numpy restatement tests/depth_order_ref.py.
The host's part (where `position` sits in the slab's columns, the scratch layout) is restated here."""
import ctypes as C

import numpy as np
import pytest

from tests import static_emu as S
from tests.depth_order_ref import depth_permutation, plane_depth, ref_depth_order, sort_keys
from tests.helpers import Instance, RefWorld
from tests.kernel_emu import claim
from tests.static_emu import churned

pytestmark = pytest.mark.timeout(900)

DEPTH_DRIVER = r"""
extern "C" void semu_batch_depth_order(const DepthOrderArgs* a, int fast, uint32_t grid) {
    DepthOrderArgs d = *a;
    const unsigned plan = std::min((d.src.max_instances * 1024u + DO_THREADS * 16u - 1u) / (DO_THREADS * 16u), 1024u);
    const unsigned rows = (d.src.max_instances * 256u + DO_WARPS - 1u) / DO_WARPS;
    emu_run([&] { k_do_plan(d); }, plan, DO_THREADS, 4);
    if (fast) emu_run([&] { k_do_keys<true>(d); }, grid, DO_THREADS, 4);
    else emu_run([&] { k_do_keys<false>(d); }, grid, DO_THREADS, 4);
    for (uint32_t pass = 0; pass < 4u; ++pass) {
        if (pass) emu_run([&] { k_do_hist(d, pass); }, grid, DO_THREADS, 4);
        emu_run([&] { k_do_scan(d, pass); }, rows, DO_THREADS, 16);
        emu_run([&] { k_do_scatter(d, pass); }, grid, DO_THREADS, 4);
    }
}
extern "C" uint32_t semu_sizeof_depth_order_args(void) { return sizeof(DepthOrderArgs); }
extern "C" uint32_t semu_depth_order_tile(void) { return DO_TILE; }
"""


class BoundsArgs(C.Structure):
    """hnb::BoundsArgs (hnb_static_kernels.h)"""
    _fields_ = [("batch_info", C.c_void_p), ("spawners", C.c_void_p), ("metadata", C.c_void_p), ("num_spawners", C.c_uint32),
                ("num_metadata", C.c_uint32), ("ping", C.c_void_p), ("pong", C.c_void_p), ("claim", C.c_void_p),
                ("capacity_rows", C.c_uint32), ("max_instances", C.c_uint32), ("col", C.c_void_p * 3), ("col_words", C.c_uint32 * 3),
                ("col_lane", C.c_uint32 * 3), ("acc", C.c_void_p), ("out", C.c_void_p)]


class DepthOrderArgs(C.Structure):
    """hnb::DepthOrderArgs (hnb_static_kernels.h)"""
    _fields_ = [("src", BoundsArgs), ("planes", C.c_void_p), ("order", C.c_void_p), ("keys", C.c_void_p * 2), ("vals", C.c_void_p * 2),
                ("hist", C.c_void_p), ("totals", C.c_void_p), ("info", C.c_void_p), ("total_tiles", C.c_void_p), ("max_tiles", C.c_uint32)]


@pytest.fixture(scope="module")
def dlib():
    lib = S.build(DEPTH_DRIVER)
    lib.semu_batch_depth_order.argtypes = [C.c_void_p, C.c_int, C.c_uint32]
    lib.semu_batch_depth_order.restype = None
    lib.semu_sizeof_depth_order_args.restype = C.c_uint32
    lib.semu_depth_order_tile.restype = C.c_uint32
    assert lib.semu_sizeof_depth_order_args() == C.sizeof(DepthOrderArgs)
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
    """A RefWorld's slab in the device's layout under `plan`, every buffer between poisoned guards, and what one
    hnb_batch_depth_order call over it enqueues."""

    def __init__(self, ref, plan, pos_word, claims=(0, 0)):
        self.ref, self.plan, self.pos_word = ref, plan, pos_word
        self.planes = [guarded(np.ascontiguousarray(ref.particles[:, off // 4:(off + w) // 4]).reshape(-1), np.uint32(0x7FC00000))
                       for off, w in plan]
        self.lists = [guarded(np.ascontiguousarray(ref.indirect[:, c]), np.uint32(0xFFFFFFF0)) for c in range(2)]
        self.claims = guarded(np.array(claims, dtype=np.uint64), np.uint64(claim(0, 1 << 30)))
        self.spawners = (type(ref.spawners[0]) * len(ref.spawners)).from_buffer_copy(bytes(ref.spawners))
        self.metadata = (type(ref.metadata[0]) * len(ref.metadata)).from_buffer_copy(bytes(ref.metadata))
        self.batch_infos = (type(ref.batch_infos[0]) * len(ref.batch_infos)).from_buffer_copy(bytes(ref.batch_infos))

    def list(self, c):
        return self.lists[c][GUARD:-GUARD]

    def run(self, lib, batch, planes, count=None, grid=3, num_spawners=None, num_metadata=None, order=None):
        """Returns the order buffer (slab rows) after the call; `order` is its content before (poison by default)."""
        bi = self.batch_infos[batch]
        count = bi.prefix_sum_count if count is None else count
        rows = self.ref.slab_rows
        where, fast = position_columns(self.plan, self.pos_word)
        max_tiles = rows // lib.semu_depth_order_tile() + count
        before_order = np.full(rows, POISON, dtype=np.uint32) if order is None else order
        out = guarded(before_order, POISON)
        plane_buf = guarded(np.ascontiguousarray(planes, dtype=np.float32).reshape(-1).view(np.uint32), np.uint32(0x7FC00000))
        scratch = guarded(np.full(4 * rows + 256 * max_tiles + 1032 * count + 1, 0x5A5A5A5A, dtype=np.uint32), POISON)
        base = scratch[GUARD:]
        a = DepthOrderArgs()
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
        a.planes, a.order = plane_buf[GUARD:].ctypes.data, out[GUARD:].ctypes.data
        addr = lambda w: base[w:].ctypes.data  # noqa: E731
        a.keys[0], a.vals[0], a.keys[1], a.vals[1] = addr(0), addr(rows), addr(2 * rows), addr(3 * rows)
        a.hist = addr(4 * rows)
        a.totals = addr(4 * rows + 256 * max_tiles)
        a.info = addr(4 * rows + 256 * max_tiles + 1024 * count)
        a.total_tiles = addr(4 * rows + 256 * max_tiles + 1032 * count)
        a.max_tiles = max_tiles
        state = self.state() + [plane_buf.copy()]
        lib.semu_batch_depth_order(C.byref(a), int(fast), grid)
        for k, (x, y) in enumerate(zip(state, self.state() + [plane_buf])):
            np.testing.assert_array_equal(x, y, err_msg=f"the depth-order pass modified buffer {k}")
        assert (out[:GUARD] == POISON).all() and (out[-GUARD:] == POISON).all(), "stores outside d_order[0, order_rows)"
        assert (scratch[:GUARD] == POISON).all() and (scratch[-GUARD:] == POISON).all(), "stores outside the scratch"
        return out[GUARD:-GUARD], fast

    def state(self):
        tables = [np.frombuffer(bytes(t), dtype=np.uint32).copy() for t in (self.spawners, self.metadata, self.batch_infos)]
        return [p.copy() for p in self.planes] + [l.copy() for l in self.lists] + [self.claims.copy()] + tables


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


def random_planes(rng, count):
    return (rng.standard_normal((max(count, 1), 4))).astype(np.float32)


def check(dev, lib, ref, batch, planes, grid=3, **kw):
    got, fast = dev.run(lib, batch, planes, grid=grid, **kw)
    want = ref_depth_order(ref, batch, dev.pos_word, planes, np.full(ref.slab_rows, POISON, dtype=np.uint32),
                           count=kw.get("count"), num_spawners=kw.get("num_spawners"), num_metadata=kw.get("num_metadata"))
    np.testing.assert_array_equal(got, want, err_msg="depth order (poison marks rows that must not be written)")
    return got, fast


def test_restatement_by_hand():
    """Farthest first; -0 after +0 (smaller); infinities at the ends; NaNs of every pattern last in index order; one ulp
    apart is ordered; ties keep index order."""
    f32 = np.float32
    one_up = np.nextafter(f32(1.0), f32(2.0))
    depth = np.array([1.0, np.nan, -0.0, 0.0, np.inf, -np.inf, one_up, 1.0, -1.0, -np.nan, 0.0], dtype=np.float32)
    bits = depth.view(np.uint32)
    bits[9] = 0xFFFFFFFF
    assert depth_permutation(depth).tolist() == [4, 6, 0, 7, 3, 10, 2, 8, 5, 1, 9]
    assert (np.diff(sort_keys(depth[[4, 6, 0, 3, 2, 8, 5]]).astype(np.int64)) > 0).all()
    # ((a*x + b*y) + c*z) + d, one rounding per step: 1e8 + 1 - 1e8 is 0 in float32 when added in this order
    words = np.array([[f32(1e8), f32(1.0), f32(-1e8)]], dtype=np.float32).view(np.uint32)
    assert plane_depth([1, 1, 1, 0], words)[0] == 0.0
    assert plane_depth([1, 0, 1, 1], words)[0] == 1.0
    assert depth_permutation(np.zeros(5, dtype=np.float32)).tolist() == list(range(5))


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_mixed_sizes_in_one_batch(dlib, layout):
    """Sizes across the one-tile boundary in one batch behind a batch of one: 0, 1, tile - 1, tile, tile + 1, several
    tiles, a small one; lists permuted after deaths, in alternating columns."""
    stride_words, plan, pos_word, want_fast = LAYOUTS[layout]
    rng = np.random.default_rng(len(layout) * 13)
    tile = dlib.semu_depth_order_tile()
    caps = [40, 8, 3, tile + 10, tile, tile + 40, 3 * tile + 500, 90]
    alive = [20, 0, 1, tile - 1, tile, tile + 1, 3 * tile + 123, 77]
    ref = random_world(rng, stride_words, caps, alive, pos_word, batches=[[0], list(range(1, 8))])
    _, fast = check(Device(ref, plan, pos_word), dlib, ref, 1, random_planes(rng, 7))
    assert fast == want_fast


@pytest.mark.parametrize("grid", [1, 2, 5])
def test_any_grid_and_many_instances(dlib, grid):
    """300 instances of uneven sizes (one staging of the plan's scan is 256), two of several tiles, at any grid."""
    rng = np.random.default_rng(grid)
    tile = dlib.semu_depth_order_tile()
    caps = [int(c) for c in rng.integers(1, 30, 300)]
    caps[17], caps[280] = 2 * tile + 9, tile + 1
    alive = [int(rng.integers(0, c + 1)) for c in caps]
    alive[17], alive[280] = 2 * tile + 9, tile + 1
    ref = random_world(rng, 8, caps, alive)
    check(Device(ref, C5_OWN, 0), dlib, ref, 0, random_planes(rng, 300), grid=grid)


@pytest.mark.parametrize("size", ["small", "large"])
@pytest.mark.parametrize("claimed", ["all", "part", "none"])
def test_identity_claims(dlib, size, claimed):
    """Column W is the identity under a claim over all, part or none of the live rows; claimed entries are poisoned with
    dead slots, whose positions would move them."""
    rng = np.random.default_rng(7)
    tile = dlib.semu_depth_order_tile()
    n = 1500 if size == "small" else 2 * tile + 100
    first, cap = 40, n + 300
    ref = random_world(rng, 8, [first, cap, 30], [10, 0, 7])
    md = ref.metadata[1]
    md.alive_count, md.indirect_write_index = n, 1
    ref.indirect[first:first + n, 1] = np.arange(n, dtype=np.uint32)
    length = {"all": n, "part": n // 2 + 3, "none": 0}[claimed]
    dev = Device(ref, default_cut(32), 0, claims=(claim(first, 5), claim(first, length)))
    dev.list(1)[first:first + length] = n + rng.integers(0, cap - n, length).astype(np.uint32)
    check(dev, dlib, ref, 0, random_planes(rng, 3))


@pytest.mark.parametrize("size", ["small", "large"])
def test_equal_and_special_depths(dlib, size):
    """All-equal depths give the identity order (no pass runs for a large instance); a plane of zeros with special d;
    positions with +-0, infinities and NaNs; a large instance whose keys differ only in one byte."""
    rng = np.random.default_rng(9)
    tile = dlib.semu_depth_order_tile()
    n = 700 if size == "small" else 2 * tile + 31
    ref = random_world(rng, 8, [n, n, n, n], [n, n, n, n])
    specials = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1.0, -1.0, 1e-45], dtype=np.float32).view(np.uint32)
    ref.particles[n:2 * n, 0:3] = rng.choice(specials, (n, 3))
    ref.particles[3 * n:4 * n, 0:3] = np.float32(1.0).view(np.uint32)
    ref.particles[3 * n:4 * n, 0] = (np.float32(1.0).view(np.uint32) + rng.integers(0, 200, n)).astype(np.uint32)
    planes = np.array([[0, 0, 0, 2.5], [1, -1, 0.5, 0], [0, 0, 0, np.nan], [1, 0, 0, 0]], dtype=np.float32)
    got, _ = check(Device(ref, default_cut(32), 0), dlib, ref, 0, planes)
    first0 = ref.instances[0].slab_offset
    np.testing.assert_array_equal(got[first0:first0 + n], ref.indirect[first0:first0 + n, 0], "equal depths: identity order")


def test_unwritten_rows_keep_their_bytes(dlib):
    """Only d_order[first, first + n) of each instance is written: every other row keeps what it held."""
    rng = np.random.default_rng(4)
    tile = dlib.semu_depth_order_tile()
    ref = random_world(rng, 8, [100, tile + 200, 60, 2 * tile], [50, tile + 3, 0, tile + 5])
    before = rng.integers(0, 1 << 32, ref.slab_rows, dtype=np.uint64).astype(np.uint32)
    planes = random_planes(rng, 4)
    got, _ = Device(ref, default_cut(32), 0).run(dlib, 0, planes, order=before.copy())
    np.testing.assert_array_equal(got, ref_depth_order(ref, 0, 0, planes, before))


def test_out_of_range_table_words(dlib):
    """List entries, slab offsets, capacities, alive counts, metadata indices and the batch's own row past their tables
    are clamped as bounds clamps them, and no access leaves the buffers (all between poisoned guards)."""
    rng = np.random.default_rng(11)
    ref = random_world(rng, 8, [300, 300, 300, 300, 5000], [200, 250, 100, 300, 50])
    first1 = ref.instances[1].slab_offset
    ref.indirect[first1:first1 + 250:3, 1] = rng.integers(300, 1 << 32, len(range(0, 250, 3)), dtype=np.uint64).astype(np.uint32)
    ref.spawners[2].slab_offset = 0xFFFFFF00            # a slice past the slab: empty
    ref.spawners[4].effect_metadata_index = 0x7FFFFFFF  # clamped to the last row: its own
    ref.metadata[4].capacity = 0xFFFFFFFF               # clamped to the rows the slab has from its offset
    ref.metadata[4].alive_count = 0xFFFFFFF0            # n = all of them, through a list of garbage words
    first4 = ref.instances[4].slab_offset
    ref.indirect[first4:, 0] = rng.integers(0, 1 << 32, ref.slab_rows - first4, dtype=np.uint64).astype(np.uint32)
    ref.batch_infos[0].prefix_sum_count = 5
    planes = random_planes(rng, 5)
    check(Device(ref, default_cut(32), 0), dlib, ref, 0, planes)
