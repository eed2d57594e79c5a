"""hnb_batch_bounds's kernels (hnb_static_kernels.cu: k_bounds_reduce<FAST>, k_bounds_write) under the CPU thread emulation
of tests/static_emu.py, bit for bit against the numpy restatement tests/bounds_ref.py. The host's part (where `position`
sits in the slab's columns, and whether the 16-byte path applies) is restated here by position_columns()."""
import ctypes as C

import numpy as np
import pytest

from tests import static_emu as S
from tests.bounds_ref import BOUNDS_DTYPE, assert_bounds_equal, box_of, ordered_key, ref_bounds
from tests.helpers import Instance, RefWorld
from tests.kernel_emu import claim
from tests.static_emu import churned

pytestmark = pytest.mark.timeout(600)

BOUNDS_DRIVER = r"""
extern "C" void semu_batch_bounds(const BoundsArgs* a, int fast, uint32_t grid) {
    BoundsArgs b = *a;
    if (fast) emu_run([&] { k_bounds_reduce<true>(b); }, grid, BD_THREADS, 4);
    else emu_run([&] { k_bounds_reduce<false>(b); }, grid, BD_THREADS, 4);
    emu_run([&] { k_bounds_write(b); }, (b.max_instances + BD_THREADS - 1) / BD_THREADS, BD_THREADS, 4);
}
extern "C" uint32_t semu_sizeof_bounds_args(void) { return sizeof(BoundsArgs); }
extern "C" uint32_t semu_bounds_tile(void) { return BD_TILE; }
"""


class BoundsArgs(C.Structure):
    """hnb::BoundsArgs (hnb_static_kernels.h)"""
    _fields_ = [("batch_info", C.c_void_p), ("spawners", C.c_void_p), ("metadata", C.c_void_p), ("num_spawners", C.c_uint32),
                ("num_metadata", C.c_uint32), ("ping", C.c_void_p), ("pong", C.c_void_p), ("claim", C.c_void_p),
                ("capacity_rows", C.c_uint32), ("max_instances", C.c_uint32), ("col", C.c_void_p * 3), ("col_words", C.c_uint32 * 3),
                ("col_lane", C.c_uint32 * 3), ("acc", C.c_void_p), ("out", C.c_void_p)]


@pytest.fixture(scope="module")
def blib():
    lib = S.build(BOUNDS_DRIVER)
    lib.semu_batch_bounds.argtypes = [C.c_void_p, C.c_int, C.c_uint32]
    lib.semu_batch_bounds.restype = None
    lib.semu_sizeof_bounds_args.restype = C.c_uint32
    lib.semu_bounds_tile.restype = C.c_uint32
    assert lib.semu_sizeof_bounds_args() == C.sizeof(BoundsArgs)
    return lib


# column plans as (byte offset, byte width) of every physical column
def default_cut(stride, sector=False):
    plan, off = [], 0
    for w in S.physical_widths(stride, sector):
        plan.append((off, w))
        off += w
    return plan


C5_OWN = [(0, 16), (16, 8), (24, 4), (28, 4)]       # C5 with a read-only lifetime
SPLIT = [(0, 8), (8, 4), (12, 4), (16, 16)]         # a read-only fourth word cuts position's run [0, 12) apart

GUARD = 64  # words of poison on both sides of every buffer the kernels get
INF_BITS = np.uint32(0x7F800000)


def guarded(data, poison):
    """A copy of `data` (uint32 or uint64, flat) between two runs of `poison`: an access just outside reads a value that
    would show in the result (and a store there is found by guards_intact)."""
    buf = np.full(len(data) + 2 * GUARD, poison, dtype=data.dtype)
    buf[GUARD:GUARD + len(data)] = data
    return buf


def position_columns(plan, pos_word):
    """What hnb_batch_bounds derives from the slab's plane set: per word of position (column, words per element, word in
    the element), and whether the three share one 16-byte quad of one column."""
    where = []
    for k in range(3):
        byte = 4 * (pos_word + k)
        p = next(i for i, (off, w) in enumerate(plan) if off <= byte < off + w)
        where.append((p, plan[p][1] // 4, (byte - plan[p][0]) // 4))
    fast = where[0][0] == where[2][0] and where[0][2] % 4 == 0 and where[0][1] % 4 == 0
    return where, fast


class Device:
    """A RefWorld's slab in the device's layout under `plan`, every buffer between poisoned guards, and what one
    hnb_batch_bounds call over it enqueues."""

    def __init__(self, ref, plan, pos_word, claims=(0, 0)):
        self.ref, self.plan, self.pos_word = ref, plan, pos_word
        assert sum(w for _, w in plan) == ref.stride_words * 4
        self.planes = [guarded(np.ascontiguousarray(ref.particles[:, off // 4:(off + w) // 4]).reshape(-1), INF_BITS) for off, w in plan]
        self.lists = [guarded(np.ascontiguousarray(ref.indirect[:, c]), np.uint32(0xFFFFFFF0)) for c in range(2)]
        self.claims = guarded(np.array(claims, dtype=np.uint64), np.uint64(claim(0, 1 << 30)))
        self.spawners = (type(ref.spawners[0]) * len(ref.spawners)).from_buffer_copy(bytes(ref.spawners))
        self.metadata = (type(ref.metadata[0]) * len(ref.metadata)).from_buffer_copy(bytes(ref.metadata))
        self.batch_infos = (type(ref.batch_infos[0]) * len(ref.batch_infos)).from_buffer_copy(bytes(ref.batch_infos))

    def list(self, c):
        return self.lists[c][GUARD:-GUARD]

    def run(self, lib, batch, out_rows=None, grid=3, num_spawners=None, num_metadata=None):
        bi = self.batch_infos[batch]
        count = bi.prefix_sum_count if out_rows is None else out_rows
        where, fast = position_columns(self.plan, self.pos_word)
        acc = guarded(np.zeros(count * 8, dtype=np.uint64), np.uint64(0))
        out = guarded(np.full(count * 8, 0xA5A5A5A5, dtype=np.uint32), np.uint32(0xA5A5A5A5))
        a = BoundsArgs()
        a.batch_info = C.addressof(self.batch_infos[batch])
        a.spawners, a.metadata = C.addressof(self.spawners), C.addressof(self.metadata)
        a.num_spawners = len(self.spawners) if num_spawners is None else num_spawners
        a.num_metadata = len(self.metadata) if num_metadata is None else num_metadata
        a.ping, a.pong = self.lists[0][GUARD:].ctypes.data, self.lists[1][GUARD:].ctypes.data
        a.claim = self.claims[GUARD:].ctypes.data
        a.capacity_rows, a.max_instances = self.ref.slab_rows, count
        for k, (p, words, lane) in enumerate(where):
            a.col[k], a.col_words[k], a.col_lane[k] = self.planes[p][GUARD:].ctypes.data, words, lane
        a.acc, a.out = acc[GUARD:].ctypes.data, out[GUARD:].ctypes.data
        before = self.state()
        lib.semu_batch_bounds(C.byref(a), int(fast), grid)
        for k, (x, y) in enumerate(zip(before, self.state())):
            np.testing.assert_array_equal(x, y, err_msg=f"the bounds pass modified buffer {k}")
        assert not acc.any(), "the accumulator is not back to zeroes (or its guards were written)"
        assert (out[:GUARD] == 0xA5A5A5A5).all() and (out[-GUARD:] == 0xA5A5A5A5).all(), "stores outside d_out[0, out_rows)"
        return out[GUARD:-GUARD].view(BOUNDS_DTYPE), fast

    def state(self):
        tables = [np.frombuffer(bytes(t), dtype=np.uint32).copy() for t in (self.spawners, self.metadata, self.batch_infos)]
        return [p.copy() for p in self.planes] + [l.copy() for l in self.lists] + [self.claims.copy()] + tables


def random_world(rng, stride_words, caps, alive, pos_word=0, batches=None, scale=1000.0):
    """Instances back to back, instance j with alive[j] live particles through a permuted list in column j & 1; every
    word random, positions finite floats; the dead rows' positions are infinite (a read of one shows in the box)."""
    insts, off = [], 0
    for c in caps:
        insts.append(Instance(off, c))
        off += c
    ref = RefWorld(max(off, 1), stride_words, insts, batches=batches)
    ref.particles[:] = rng.integers(0, 1 << 32, ref.particles.shape, dtype=np.uint64).astype(np.uint32)
    ref.particles[:, pos_word:pos_word + 3] = (rng.standard_normal((ref.slab_rows, 3)) * scale).astype(np.float32).view(np.uint32)
    for j, n in enumerate(alive):
        churned(rng, ref, j, n, w=j & 1)
        inst = insts[j]
        dead = ref.indirect[inst.slab_offset + n:inst.slab_offset + inst.capacity, 2].astype(np.int64)
        ref.particles[dead, pos_word:pos_word + 3] = np.where(rng.random((len(dead), 3)) < 0.5, INF_BITS, np.uint32(0xFF800000))
    return ref


def test_restatement_by_hand():
    """Keys: -inf < -1 < -0 < +0 < 1 < +inf, NaNs of both signs skipped; a component of NaNs only has no value."""
    f = lambda *v: np.array(v, dtype=np.float32).view(np.uint32)  # noqa: E731
    bits = f(-np.inf, -1.0, -0.0, 0.0, 1.0, np.inf)
    assert (np.diff(ordered_key(bits).astype(np.int64)) > 0).all()
    nan_pos, nan_neg = np.uint32(0x7FC00001), np.uint32(0xFFFFFFFF)
    words = np.stack([np.array([f(0.0)[0], nan_pos, f(-0.0)[0], f(2.5)[0]], dtype=np.uint32),
                      np.array([nan_pos, nan_neg, nan_pos, nan_neg], dtype=np.uint32),
                      np.array([f(np.inf)[0], f(-3.0)[0], nan_neg, f(-np.inf)[0]], dtype=np.uint32)], axis=1)
    lo, hi = box_of(words)
    np.testing.assert_array_equal(lo, [f(-0.0)[0], 0x7F800000, 0xFF800000])
    np.testing.assert_array_equal(hi, [f(2.5)[0], 0xFF800000, 0x7F800000])
    lo, hi = box_of(words[:0])
    assert (lo == 0x7F800000).all() and (hi == 0xFF800000).all()


LAYOUTS = {
    "32-default": (8, default_cut(32), 0, True),
    "32-c5-own": (8, C5_OWN, 0, True),
    "32-split": (8, SPLIT, 0, False),
    "32-unaligned": (8, default_cut(32), 1, False),
    "32-sector": (8, default_cut(32, True), 0, True),
    "32-sector-second-half": (8, default_cut(32, True), 4, True),
    "48-default": (12, default_cut(48), 4, True),
    "48-sector": (12, default_cut(48, True), 8, True),
    "96-default": (24, default_cut(96), 20, True),
    "28-tail": (7, default_cut(28), 4, False),  # 16 + 8 + 4: position in the 8- and the 4-byte tail columns
}


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("grid", [1, 3])
def test_mixed_instances_in_one_batch(blib, layout, grid):
    """Seven instances in the second batch of the slab, behind a batch of one: empty, tiny, one tile exactly, more than
    two tiles, zero capacity. Lists are permutations after deaths, in alternating columns; no claims."""
    stride_words, plan, pos_word, want_fast = LAYOUTS[layout]
    rng = np.random.default_rng(len(layout) * 7 + grid)
    tile = blib.semu_bounds_tile()
    caps = [50, 37, 1100, 64, 0, tile, 2 * tile + 300, 90]
    alive = [20, 0, 1000, 64, 0, tile, 2 * tile + 77, 1]
    ref = random_world(rng, stride_words, caps, alive, pos_word, batches=[[0], list(range(1, 8))])
    dev = Device(ref, plan, pos_word)
    got, fast = dev.run(blib, 1, grid=grid)
    assert fast == want_fast
    want = ref_bounds(ref, 1, pos_word)
    assert want["count"].tolist() == alive[1:]
    assert_bounds_equal(got, want, layout)
    assert np.isinf(got["min"][0]).all() and (got["min"][0] > 0).all() and (got["max"][0] < 0).all(), "an empty instance"
    assert np.isfinite(got["min"][1:][want["count"][1:] > 0]).all(), "a dead row (infinite position) was read"


@pytest.mark.parametrize("fast", [True, False], ids=["fast", "general"])
@pytest.mark.parametrize("claimed", ["all", "more", "part", "none", "other_base"])
def test_identity_claims(blib, fast, claimed):
    """An instance of 1500 live rows whose column W is the identity, at slab row 40, under a claim over all of them, over
    more rows than are alive, over a part, none, and a claim with another instance's base. Rows the claim covers are never
    loaded from the list: their entries are poisoned with the slots of dead rows, whose positions are infinite."""
    rng = np.random.default_rng(5)
    n, first, cap = 1500, 40, 1800
    ref = random_world(rng, 8, [first, cap, 30], [10, 0, 7])
    md = ref.metadata[1]
    md.alive_count, md.indirect_write_index = n, 1
    ref.indirect[first:first + n, 1] = np.arange(n, dtype=np.uint32)
    ref.particles[first:first + n, 0:3] = rng.standard_normal((n, 3)).astype(np.float32).view(np.uint32)
    ref.particles[first + n:first + cap, 0:3] = INF_BITS
    length = {"all": n, "more": cap, "part": 700, "none": 0, "other_base": n}[claimed]
    base = 0 if claimed == "other_base" else first
    dev = Device(ref, default_cut(32) if fast else SPLIT, 0, claims=(claim(first, 5), claim(base, length)))
    covered = 0 if claimed == "other_base" else min(length, n)
    dev.list(1)[first:first + covered] = n + rng.integers(0, cap - n, covered).astype(np.uint32)
    got, _ = dev.run(blib, 0, grid=2)
    assert_bounds_equal(got, ref_bounds(ref, 0, 0), claimed)
    assert np.isfinite(got["max"][1]).all(), "a claimed row's list entry was read"


@pytest.mark.parametrize("fast", [True, False], ids=["fast", "general"])
def test_special_values(blib, fast):
    """Zeroes of both signs, infinities, NaN in one component, NaN in a whole component, NaN everywhere."""
    f = lambda *v: np.array(v, dtype=np.float32).view(np.uint32)  # noqa: E731
    nan = [np.uint32(0x7FC00000), np.uint32(0xFFC00000), np.uint32(0x7F800001), np.uint32(0xFFFFFFFF)]
    ref = RefWorld(40, 8, [Instance(0, 8, alive=4), Instance(8, 8, alive=4), Instance(16, 8, alive=3), Instance(24, 8, alive=2),
                           Instance(32, 8, alive=8)])
    p = ref.particles
    p[0:4, 0], p[0:4, 1], p[0:4, 2] = f(0.0, -0.0, 0.0, -0.0), f(-0.0, -0.0, -0.0, -0.0), f(0.0, 0.0, 0.0, 0.0)
    p[8:12, 0], p[8:12, 1], p[8:12, 2] = f(np.inf, 1, -np.inf, 2), f(3, np.inf, 3, 3), f(-np.inf, -5, -np.inf, -7)
    p[16:19, 0], p[16:19, 1], p[16:19, 2] = [nan[0], f(4.0)[0], f(-4.0)[0]], [f(1e-45)[0], nan[1], f(-1e-45)[0]], [nan[2], nan[3], f(9.0)[0]]
    p[24:26, 0], p[24:26, 1], p[24:26, 2] = f(1.0, 2.0), [nan[0], nan[3]], f(-1.0, -2.0)
    p[32:40, 0:3] = np.array(nan * 6, dtype=np.uint32).reshape(8, 3)
    dev = Device(ref, default_cut(32) if fast else SPLIT, 0)
    got, _ = dev.run(blib, 0, grid=2)
    want = ref_bounds(ref, 0, 0)
    assert_bounds_equal(got, want, "special values")
    w = got.view(np.uint32).reshape(-1, 8)
    assert w[0, 0] == 0x80000000 and w[0, 4] == 0 and w[0, 1] == w[0, 5] == 0x80000000 and w[0, 2] == w[0, 6] == 0, "-0 < +0"
    assert w[1, 0] == 0xFF800000 and w[1, 4] == 0x7F800000, "infinities take part"
    assert w[3, 1] == 0x7F800000 and w[3, 5] == 0xFF800000 and got["count"][3] == 2, "a component of NaNs has no value"
    assert (w[4, 0:3] == 0x7F800000).all() and (w[4, 4:7] == 0xFF800000).all() and got["count"][4] == 8


@pytest.mark.parametrize("fast", [True, False], ids=["fast", "general"])
def test_out_of_range_words_are_clamped(blib, fast):
    """List entries, slab offsets, capacities, alive counts, metadata indices and the batch's own row past their tables:
    every one is clamped, and no access leaves the buffers (all of them sit between poisoned guards)."""
    rng = np.random.default_rng(11)
    ref = random_world(rng, 8, [300, 300, 300, 300, 300], [200, 250, 100, 300, 50])
    first1 = ref.instances[1].slab_offset
    ref.indirect[first1:first1 + 250:3, 1] = rng.integers(300, 1 << 32, len(range(0, 250, 3)), dtype=np.uint64).astype(np.uint32)
    ref.spawners[2].slab_offset = 0xFFFFFF00            # a slice past the slab: empty
    ref.metadata[3].capacity = 0xFFFFFFFF               # clamped to the rows the slab has from its offset
    ref.metadata[3].alive_count = 0xFFFFFFF0
    ref.indirect[ref.instances[3].slab_offset:, 1] = rng.integers(0, 1 << 32, 600, dtype=np.uint64).astype(np.uint32)
    ref.spawners[4].effect_metadata_index = 0x7FFFFFFF  # clamped to the last row: its own
    ref.batch_infos[0].prefix_sum_count = 9             # more instances than spawner rows: the last row repeats
    dev = Device(ref, default_cut(32) if fast else SPLIT, 0)
    got, _ = dev.run(blib, 0, out_rows=7, grid=3)
    want = ref_bounds(ref, 0, 0, out_rows=7)
    assert want["count"].tolist() == [200, 250, 0, 600, 50, 50, 50]
    assert_bounds_equal(got, want, "clamped")
    # fewer records than the device's batch row names: the first out_rows only
    got, _ = dev.run(blib, 0, out_rows=2, grid=3)
    assert_bounds_equal(got, want[:2], "out_rows below the device's count")
    # a batch row naming fewer instances than the call covers: the others get empty records
    dev.batch_infos[0].prefix_sum_count = 1
    got, _ = dev.run(blib, 0, out_rows=3, grid=3)
    assert_bounds_equal(got[:1], want[:1], "device count 1")
    assert (got["count"][1:] == 0).all() and np.isinf(got["min"][1:]).all() and np.isinf(got["max"][1:]).all()


def test_many_instances_and_any_grid(blib):
    """300 instances (more than one staging round of 256) of uneven sizes, some empty, at grids of 1, 5 and 8 CTAs: every
    tile is taken exactly once whatever the grid, and the records do not depend on it."""
    rng = np.random.default_rng(3)
    caps = [int(c) for c in rng.integers(1, 40, 300)]
    caps[17], caps[280] = 1500, 2100
    alive = [int(rng.integers(0, c + 1)) if j % 9 else 0 for j, c in enumerate(caps)]
    alive[280] = 2100
    ref = random_world(rng, 8, caps, alive)
    want = ref_bounds(ref, 0, 0)
    for grid in (1, 5, 8):
        got, _ = Device(ref, C5_OWN, 0).run(blib, 0, grid=grid)
        assert_bounds_equal(got, want, f"grid {grid}")
