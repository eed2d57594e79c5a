"""hnb_instance_append's kernels (hnb_static_kernels.cu: k_append_scatter, then k_append_commit) under the CPU thread
emulation of tests/static_emu.py, against the numpy restatement tests/append_ref.py, which is pinned by a hand-worked
example and tied to tests/snapshot_ref.py's restore. Every buffer the kernels may touch (planes, lists, dead stack, alive
bits, lifetime floors, common ages, claims, metadata) sits between poisoned guard words, and everything but what the
restatement writes must keep its bytes."""
import copy
import ctypes as C

import numpy as np
import pytest

from tests import plan_assets
from tests import static_emu as S
from tests.append_ref import append_count, append_slots, cut_claim, make_snapshot, ref_append
from tests.helpers import Instance, RefWorld
from tests.kernel_emu import assert_same, c5_frame, c5_world, claim, claimed
from tests.snapshot_ref import HEADER_WORDS, ref_restore, ref_snapshot
from tests.static_emu import churned, physical_widths

pytestmark = pytest.mark.timeout(900)

GUARD = 64  # poisoned words before and after every buffer
POISON = 0xDEADBEEF
NONE32 = 0xFFFFFFFF
NONE64 = 0xFFFFFFFFFFFFFFFF

# hnb_instance_append's device work as launch_append issues it
APPEND_DRIVER = r"""
extern "C" void semu_append(const AppendArgs* a, const uint32_t* src) {
    AppendArgs s = *a;
    const uint64_t held = (s.s.src_bytes - HNB_SNAPSHOT_HEADER_WORDS * 4u) / (s.s.stride_words * 4u);
    const uint32_t bound = uint32_t(held < s.s.rows ? held : s.s.rows);
    if (bound == 0u) return;
    emu_run([&] { k_append_scatter(s, src); }, (bound + RP_ROWS_PER_BLOCK - 1) / RP_ROWS_PER_BLOCK, RP_THREADS, 8);
    emu_run([&] { k_append_commit(s, src); }, 1, 1);
}
extern "C" uint32_t semu_sizeof_append_args(void) { return sizeof(AppendArgs); }
"""


class SnapshotArgs(C.Structure):
    """hnb::SnapshotArgs (hnb_static_kernels.h)"""
    _fields_ = [("metadata", C.c_void_p), ("ping", C.c_void_p), ("pong", C.c_void_p), ("planes", S.PlaneSet),
                ("num_planes", C.c_uint32), ("stride_words", C.c_uint32), ("first", C.c_uint32), ("rows", C.c_uint32),
                ("src_bytes", C.c_uint64)]


class AppendArgs(C.Structure):
    """hnb::AppendArgs (hnb_static_kernels.h)"""
    _fields_ = [("s", SnapshotArgs)] + [(f, C.c_void_p) for f in ("ping", "pong", "dead", "alive_bits", "life_floor", "group_age", "claim")]


@pytest.fixture(scope="module")
def alib():
    lib = S.build(APPEND_DRIVER)
    lib.semu_append.argtypes = [C.c_void_p, C.c_void_p]
    lib.semu_append.restype = None
    lib.semu_sizeof_append_args.restype = C.c_uint32
    assert lib.semu_sizeof_append_args() == C.sizeof(AppendArgs)
    return lib


def guarded(values, dtype):
    """`values` between GUARD poisoned words: returns (the whole array, the view of `values`)."""
    values = np.asarray(values, dtype=dtype)
    whole = np.full(len(values) + 2 * GUARD, POISON, dtype=dtype)
    whole[GUARD:GUARD + len(values)] = values
    return whole, whole[GUARD:GUARD + len(values)]


def default_columns(stride_words, sector):
    out, off = [], 0
    for w in physical_widths(stride_words * 4, sector):
        out.append(list(range(off, off + w // 4)))
        off += w // 4
    return out


class Slab:
    """A slab in the device's layout, every buffer guarded: columns holding the record words `columns` (a column plan's
    hnb_effect_column_words), ping / pong / dead, alive bits, lifetime floors, common ages (the groups' words, then the
    count of deferred ones) and the claim words."""

    def __init__(self, ref: RefWorld, columns, rng, claims=None):
        self.ref, self.columns = ref, columns
        rows = ref.slab_rows
        self.planes = []
        for words in columns:
            self.planes.append(guarded(np.ascontiguousarray(ref.particles[:, words]).reshape(-1), np.uint32))
        self.cols = [guarded(ref.indirect[:, c], np.uint32) for c in range(3)]
        rnd = lambda k: rng.integers(0, 1 << 32, k, dtype=np.uint64).astype(np.uint32)  # noqa: E731
        self.bits = guarded(rnd(rows // 32 + 2), np.uint32)
        self.floors = guarded(rnd(rows // 32 + 1), np.uint32)
        ages = rng.integers(0, 1 << 62, rows // 32 + 2, dtype=np.uint64)
        ages[-1] = 0  # no deferred word
        self.ages = guarded(ages, np.uint64)
        self.claims = guarded(claims if claims is not None else [claim(5, 7), claim(9, 11)], np.uint64)
        self.metadata = (S.O.EffectMetadata * len(ref.instances)).from_buffer_copy(bytes(ref.metadata))

    def plane_set(self):
        ps = S.PlaneSet()
        for p, words in enumerate(self.columns):
            ps.ptr[p] = self.planes[p][1].ctypes.data
            ps.words[p] = len(words)
            ps.word_off[p] = words[0] if words == list(range(words[0], words[0] + len(words))) else \
                0x80000000 | sum(w << (6 * l) for l, w in enumerate(words))
            for w in words:
                ps.word_to_plane[w] = p
        return ps

    def append(self, lib, i, src, src_bytes=None, slot_order=True):
        """hnb_instance_append of the words `src` into instance i (its whole capacity). `src` is copied between guards, so
        that a read past src_bytes would read poison (and differ from the restatement)."""
        inst = self.ref.instances[i]
        nbytes = src.nbytes if src_bytes is None else src_bytes
        buf = np.full((nbytes + 3) // 4 + 2 * GUARD, POISON, dtype=np.uint32)
        buf[GUARD:GUARD + (nbytes + 3) // 4] = src[:(nbytes + 3) // 4]
        if nbytes % 4:  # the bytes past src_bytes in the last word are poison too
            b = buf[GUARD:GUARD + (nbytes + 3) // 4].view(np.uint8)
            b[nbytes:] = 0xEF
        sa = SnapshotArgs(C.addressof(self.metadata[i]), self.cols[0][1].ctypes.data, self.cols[1][1].ctypes.data, self.plane_set(),
                          len(self.columns), self.ref.stride_words, inst.slab_offset, inst.capacity, nbytes)
        a = AppendArgs(sa, self.cols[0][1].ctypes.data, self.cols[1][1].ctypes.data, self.cols[2][1].ctypes.data,
                       self.bits[1].ctypes.data if slot_order else None, self.floors[1].ctypes.data, self.ages[1].ctypes.data,
                       self.claims[1].ctypes.data)
        lib.semu_append(C.byref(a), buf[GUARD:].ctypes.data)
        assert (buf[:GUARD] == POISON).all() and (buf[GUARD + (nbytes + 3) // 4:] == POISON).all(), "the source was written"

    def particles(self):
        out = np.zeros_like(self.ref.particles)
        for words, (_, v) in zip(self.columns, self.planes):
            out[:, words] = v.reshape(-1, len(words))
        return out

    def indirect(self):
        return np.stack([v for _, v in self.cols], axis=1)

    def metadata_rows(self):
        return np.frombuffer(bytes(self.metadata), dtype=np.uint32).reshape(len(self.metadata), 15)

    def state(self):
        return [w.copy() for w, _ in self.planes + self.cols + [self.bits, self.floors, self.ages, self.claims]] + [self.metadata_rows().copy()]

    def guards_intact(self):
        for w, v in self.planes + self.cols + [self.bits, self.floors, self.ages, self.claims]:
            assert (w[:GUARD] == w.dtype.type(POISON)).all() and (w[-GUARD:] == w.dtype.type(POISON)).all(), "a guard word was written"


def expect_append(lib, soa: Slab, ref: RefWorld, i, snap, src_bytes=None, slot_order=True):
    """Runs the append on `soa` and the restatement on `ref`, and checks every buffer of the slab: records, lists, dead
    stack and metadata against `ref`; alive bits, floors, common ages and claims against their expected change. Returns m."""
    first, rows = ref.instances[i].slab_offset, ref.instances[i].capacity
    md = ref.metadata[i]
    n, w = min(md.alive_count, rows), md.indirect_write_index
    slots = append_slots(ref, i, snap, src_bytes)
    bits, floors, ages, claims = (soa.bits[1].copy(), soa.floors[1].copy(), soa.ages[1].copy(), soa.claims[1].copy())
    soa.append(lib, i, snap, src_bytes, slot_order)
    m = ref_append(ref, i, snap, src_bytes)
    assert m == len(slots)
    what = f"instance {i}, n {n}, m {m}"
    soa.guards_intact()
    np.testing.assert_array_equal(soa.particles(), ref.particles, err_msg=f"{what}: records")
    np.testing.assert_array_equal(soa.indirect(), ref.indirect, err_msg=f"{what}: ping / pong / dead")
    np.testing.assert_array_equal(soa.metadata_rows(), ref.metadata_rows(), err_msg=f"{what}: metadata")
    rows_written = first + slots.astype(np.int64)
    if slot_order:
        for r in rows_written:
            bits[r >> 5] |= np.uint32(1 << (r & 31))
    np.testing.assert_array_equal(soa.bits[1], bits, err_msg=f"{what}: alive bits")
    groups = np.unique(rows_written >> 5)
    floors[groups] = NONE32
    ages[groups] = np.uint64(NONE64)
    np.testing.assert_array_equal(soa.floors[1], floors, err_msg=f"{what}: lifetime floors")
    np.testing.assert_array_equal(soa.ages[1], ages, err_msg=f"{what}: common ages")
    if m:
        claims[w] = np.uint64(cut_claim(int(claims[w]), first, n))
    np.testing.assert_array_equal(soa.claims[1], claims, err_msg=f"{what}: claims")
    return m


def random_records(rng, k, stride_words):
    return rng.integers(0, 1 << 32, (k, stride_words), dtype=np.uint64).astype(np.uint32)


def world(rng, slab_rows, stride_words, insts, alive, identity_dead=False, first_w=0):
    """Random records; instance j churned with alive[j] live particles, list column (j + first_w) & 1; `identity_dead`: the
    dead stack of each instance holds its free slots in ascending order."""
    ref = RefWorld(slab_rows, stride_words, insts)
    ref.particles[:] = random_records(rng, slab_rows, stride_words)
    for j, k in enumerate(alive):
        churned(rng, ref, j, k, w=(j + first_w) & 1)
        ref.metadata[j].particle_counter = int(rng.integers(0, 1 << 32))
        if identity_dead:
            inst = ref.instances[j]
            d = slice(inst.slab_offset + k, inst.slab_offset + inst.capacity)
            ref.indirect[d, 2] = np.sort(ref.indirect[d, 2])
    return ref


# ---- the restatement by hand --------------------------------------------------------------------------------------------
def test_oracle_restatement_by_hand():
    """An 8-row instance at slab row 3 of an 11-row slab, one-word records 100 + row. 3 alive (W = 0: local slots 5, 0, 2),
    max_spawn 4, dead stack from position 3: slots 7, 1, 6, 3, 4 (global 10, 4, 9, 6, 7). A snapshot of 3 records 900, 901,
    902 goes to slots 7, 1, 6; list_0 rows 3..5 name them; alive_count 6, max_spawn 1, particle_counter 13. A second append
    of 3 records is cut to max_spawn = 1: record 800 goes to slot 3."""
    ref = RefWorld(11, 1, [Instance(0, 3), Instance(3, 8)])
    ref.particles[:, 0] = 100 + np.arange(11)
    ref.indirect[:, 0] = [0, 1, 2, 5, 0, 2, 70, 71, 72, 73, 74]
    ref.indirect[:, 1] = [0, 1, 2, 60, 61, 62, 63, 64, 65, 66, 67]
    ref.indirect[:, 2] = [0, 1, 2, 99, 99, 99, 10, 4, 9, 6, 7]
    md = ref.metadata[1]
    md.alive_count, md.max_spawn, md.indirect_write_index, md.particle_counter = 3, 4, 0, 10
    snap = make_snapshot([900, 901, 902], 1)
    np.testing.assert_array_equal(append_slots(ref, 1, snap), [7, 1, 6])
    assert ref_append(ref, 1, snap) == 3
    np.testing.assert_array_equal(ref.particles[:, 0], [100, 101, 102, 103, 901, 105, 106, 107, 108, 902, 900])
    np.testing.assert_array_equal(ref.indirect[:, 0], [0, 1, 2, 5, 0, 2, 7, 1, 6, 73, 74])
    np.testing.assert_array_equal(ref.indirect[:, 1], [0, 1, 2, 60, 61, 62, 63, 64, 65, 66, 67])
    np.testing.assert_array_equal(ref.indirect[:, 2], [0, 1, 2, 99, 99, 99, 10, 4, 9, 6, 7])
    assert (md.alive_count, md.max_spawn, md.particle_counter, md.indirect_write_index) == (6, 1, 13, 0)
    assert ref_append(ref, 1, make_snapshot([800, 801, 802], 1)) == 1
    np.testing.assert_array_equal(ref.particles[3:, 0], [103, 901, 105, 800, 107, 108, 902, 900])
    assert ref.indirect[3 + 6, 0] == 3 and (md.alive_count, md.max_spawn, md.particle_counter) == (7, 0, 14)
    assert cut_claim((3 << 32) | 8, 3, 6) == (3 << 32) | 6 and cut_claim((3 << 32) | 4, 3, 6) == (3 << 32) | 4
    assert cut_claim((0 << 32) | 8, 3, 6) == 8, "another instance's claim is kept"


def test_hand_example_on_the_kernels(alib):
    """The hand-worked example through the emulated kernels, with both claims on the instance (column 0 over all 8
    rows, column 1 over 2) and slot order."""
    rng = np.random.default_rng(1)
    ref = RefWorld(11, 1, [Instance(0, 3), Instance(3, 8)])
    ref.particles[:, 0] = 100 + np.arange(11)
    ref.indirect[:, 0] = [0, 1, 2, 5, 0, 2, 70, 71, 72, 73, 74]
    ref.indirect[:, 2] = [0, 1, 2, 99, 99, 99, 10, 4, 9, 6, 7]
    md = ref.metadata[1]
    md.alive_count, md.max_spawn, md.indirect_write_index, md.particle_counter = 3, 4, 0, 10
    soa = Slab(ref, [[0]], rng, claims=[claim(3, 8), claim(3, 2)])
    assert expect_append(alib, soa, ref, 1, make_snapshot([900, 901, 902], 1)) == 3
    assert soa.claims[1][0] == claim(3, 3) and soa.claims[1][1] == claim(3, 2)
    assert expect_append(alib, soa, ref, 1, make_snapshot([800, 801, 802], 1)) == 1


# ---- column shapes ------------------------------------------------------------------------------------------------------
# (stride in words, sector planes): default cuts of 4 | 8 | 16 | 16+8+4 | 32 | 32+16 byte columns
LAYOUTS = [(1, False), (2, False), (4, False), (7, False), (8, True), (12, True)]


@pytest.mark.parametrize("stride_words,sector", LAYOUTS, ids=lambda v: str(v))
@pytest.mark.parametrize("dead", ["identity", "permuted"])
@pytest.mark.parametrize("n,k", [(0, 1), (0, 1100), (33, 500), (700, 64), (1099, 5)])
def test_default_cuts_match_the_oracle(alib, stride_words, sector, dead, n, k):
    """k records into an 1100-row instance at slab row 37 with n alive, between two others. The neighbours keep every
    byte, including the bits and group words they share with it."""
    rng = np.random.default_rng(n * 31 + k + stride_words)
    ref = world(rng, 1187, stride_words, [Instance(0, 37), Instance(37, 1100), Instance(1137, 50)], (20, n, 31),
                identity_dead=dead == "identity")
    soa = Slab(ref, default_columns(stride_words, sector), rng, claims=[claim(37, 1100), claim(37, 1100)])
    snap = make_snapshot(random_records(rng, k, stride_words), stride_words)
    assert expect_append(alib, soa, ref, 1, snap) == min(k, 1100 - n)


@pytest.mark.parametrize("seed", plan_assets.SEEDS)
def test_drawn_column_plans(alib, seed):
    """Every drawn asset's own plan (runs plans, word maps, the default-cut fallback) and its sector-plane cut where the
    stride allows one: a permuted dead stack, records from a snapshot of another instance."""
    fx = plan_assets.draw(seed).asset.generate()
    stride_words = fx.particle_stride // 4
    plans = [fx.column_words(), default_columns(stride_words, True)]
    rng = np.random.default_rng(seed)
    for columns in plans:
        ref = world(rng, 1500, stride_words, [Instance(0, 45), Instance(45, 1000), Instance(1045, 455)], (10, 300, 400))
        soa = Slab(ref, columns, rng, claims=[claim(45, 1000), claim(45, 290)])
        snap = ref_snapshot(ref, 2)
        assert expect_append(alib, soa, ref, 1, snap) == 400
        assert expect_append(alib, soa, ref, 1, make_snapshot(random_records(rng, 3, stride_words), stride_words)) == 3


# ---- claims ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["all", "part", "at_n", "none", "other_instance"])
@pytest.mark.parametrize("w", [0, 1])
def test_claims(alib, which, w):
    """Column W's claim over all rows is cut to n, over part of the list (below n) or exactly n is kept, and so is a claim
    of no rows or of another instance; the other column's claim never changes."""
    rng = np.random.default_rng(7 + w)
    n = 300
    ref = world(rng, 1100, 3, [Instance(0, 100), Instance(100, 1000)], (50, n), first_w=w ^ 1)
    assert ref.metadata[1].indirect_write_index == w
    word = {"all": claim(100, 1000), "part": claim(100, 120), "at_n": claim(100, n), "none": claim(100, 0),
            "other_instance": claim(0, 100)}[which]
    claims = [word, claim(100, 1000)] if w == 0 else [claim(100, 1000), word]
    soa = Slab(ref, default_columns(3, False), rng, claims=claims)
    expect_append(alib, soa, ref, 1, make_snapshot(random_records(rng, 40, 3), 3))
    want = {"all": claim(100, n), "part": claim(100, 120), "at_n": claim(100, n), "none": claim(100, 0), "other_instance": claim(0, 100)}[which]
    assert soa.claims[1][w] == want and soa.claims[1][1 - w] == claim(100, 1000)


# ---- the clamps of m --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("clamp", ["count", "max_spawn", "rows", "src_bytes", "src_bytes_odd", "header_only", "zero_count"])
def test_each_clamp_of_m(alib, clamp):
    """m = min(count, max_spawn, rows - n, (src_bytes - 64) / stride), each the smallest in turn. The kernel reads no
    byte past src_bytes (the buffer ends there, followed by poison)."""
    rng = np.random.default_rng(11)
    ref = world(rng, 1300, 5, [Instance(0, 100), Instance(100, 1000), Instance(1100, 200)], (50, 600, 25))
    md = ref.metadata[1]
    records = random_records(rng, 500, 5)
    count, src_bytes = 500, None
    if clamp == "count":
        count = 123
    elif clamp == "max_spawn":
        md.max_spawn = 77
    elif clamp == "rows":
        md.max_spawn = 1000  # above rows - n = 400 (a state the invariant does not allow, but which is never read past)
    elif clamp == "src_bytes":
        src_bytes = 64 + 211 * 20
    elif clamp == "src_bytes_odd":
        src_bytes = 64 + 211 * 20 + 19
    elif clamp == "header_only":
        src_bytes = 64
    elif clamp == "zero_count":
        count = 0
    snap = make_snapshot(records, 5, count=count)
    soa = Slab(ref, default_columns(5, False), rng, claims=[claim(100, 1000)] * 2)
    want = {"count": 123, "max_spawn": 77, "rows": 400, "src_bytes": 211, "src_bytes_odd": 211, "header_only": 0, "zero_count": 0}[clamp]
    assert append_count(ref, 1, snap, src_bytes) == want
    assert expect_append(alib, soa, ref, 1, snap, src_bytes) == want


@pytest.mark.parametrize("corruption", ["magic", "version_2", "stride", "version_0"])
def test_corrupt_headers_append_nothing(alib, corruption):
    """A header that is not a version-1 snapshot of this stride (a version-2 snapshot included) appends nothing at all:
    every byte of every buffer is kept, metadata and claims included."""
    rng = np.random.default_rng(5)
    ref = world(rng, 600, 5, [Instance(0, 100), Instance(100, 450), Instance(550, 50)], (50, 200, 25))
    snap = make_snapshot(random_records(rng, 100, 5), 5)
    if corruption == "magic":
        snap[0] ^= 1
    elif corruption == "version_2":
        snap[1] = 2
    elif corruption == "version_0":
        snap[1] = 0
    else:
        snap[2] = 24
    soa = Slab(ref, default_columns(5, False), rng, claims=[claim(100, 450)] * 2)
    before = soa.state()
    assert append_count(ref, 1, snap) == 0
    soa.append(alib, 1, snap)
    for k, (a, b) in enumerate(zip(before, soa.state())):
        np.testing.assert_array_equal(a, b, err_msg=f"{corruption}: buffer {k} changed")


# ---- slices at group edges ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("first", [0, 31, 32, 45, 63])
@pytest.mark.parametrize("rows", [1, 2, 31, 32, 33, 70])
def test_slices_at_group_edges(alib, first, rows):
    """Instances of 1 to 70 rows starting at, inside and just before a 32-row group, filled from empty to full by appends
    of 1, 2 and 7 records: only the written slots' bits and group words change, neighbours sharing a group included."""
    rng = np.random.default_rng(first * 100 + rows)
    insts = ([Instance(0, first)] if first else []) + [Instance(first, rows), Instance(first + rows, 40)]
    i = 1 if first else 0
    ref = world(rng, first + rows + 40, 3, insts, [x.capacity // 2 for x in insts])
    churned(rng, ref, i, 0, w=1)
    soa = Slab(ref, default_columns(3, False), rng, claims=[claim(first, rows)] * 2)
    total = 0
    for k in (1, 2, 7, 7, 7, 7, 7, 7, 7, 7, 7, 7, 7):
        total += expect_append(alib, soa, ref, i, make_snapshot(random_records(rng, k, 3), 3))
    assert total == rows == ref.metadata[i].alive_count and ref.metadata[i].max_spawn == 0


def test_without_slot_order_the_bits_are_kept(alib):
    rng = np.random.default_rng(2)
    ref = world(rng, 600, 4, [Instance(0, 600)], (100,))
    soa = Slab(ref, default_columns(4, False), rng)
    bits = soa.bits[1].copy()
    expect_append(alib, soa, ref, 0, make_snapshot(random_records(rng, 200, 4), 4), slot_order=False)
    np.testing.assert_array_equal(soa.bits[1], bits)


def test_corrupt_dead_stack_stays_in_the_slice(alib):
    """Dead-stack entries that name rows outside the slice (a state the invariant does not allow) are clamped to its last
    row: nothing outside the slice is written."""
    rng = np.random.default_rng(4)
    ref = world(rng, 300, 2, [Instance(0, 100), Instance(100, 100), Instance(200, 100)], (10, 20, 30))
    ref.indirect[100 + 20:100 + 40, 2] = rng.integers(0, 1 << 32, 20, dtype=np.uint64).astype(np.uint32)
    soa = Slab(ref, default_columns(2, False), rng)
    outside = [soa.particles()[:100].copy(), soa.particles()[200:].copy()]
    snap = make_snapshot(random_records(rng, 20, 2), 2)
    soa.append(alib, 1, snap)
    soa.guards_intact()
    np.testing.assert_array_equal(soa.particles()[:100], outside[0])
    np.testing.assert_array_equal(soa.particles()[200:], outside[1])


# ---- against restore ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stride_words,sector", LAYOUTS, ids=lambda v: str(v))
@pytest.mark.parametrize("n", [0, 1, 33, 1000])
def test_append_into_a_fresh_instance_writes_what_restore_writes(alib, stride_words, sector, n):
    """snapshot(A) appended into an empty, fresh instance (dead stack the identity, max_spawn = rows) writes the records
    and list entries that restore(snapshot(A)) writes: the same records at rows [0, m), list_W = 0, 1, ..."""
    rng = np.random.default_rng(n + 3 * stride_words)
    src = world(rng, 1187, stride_words, [Instance(0, 37), Instance(37, 1100), Instance(1137, 50)], (20, n, 31))
    snap = ref_snapshot(src, 1)
    dst = RefWorld(45 + 1100 + 40, stride_words, [Instance(0, 45), Instance(45, 1100), Instance(1145, 40)])
    dst.particles[:] = random_records(rng, dst.slab_rows, stride_words)
    dst.metadata[1].indirect_write_index = 1
    restored = copy.deepcopy(dst)
    soa = Slab(dst, default_columns(stride_words, sector), rng, claims=[claim(45, 1100)] * 2)
    assert expect_append(alib, soa, dst, 1, snap) == n
    assert ref_restore(restored, 1, snap) == n
    np.testing.assert_array_equal(dst.particles, restored.particles)
    np.testing.assert_array_equal(dst.indirect[:, [1, 2]], restored.indirect[:, [1, 2]])
    md, rmd = dst.metadata[1], restored.metadata[1]
    assert (md.alive_count, md.max_spawn) == (rmd.alive_count, rmd.max_spawn)


# ---- frames after appends ----------------------------------------------------------------------------------------------------
def test_appends_between_emulated_frames(orc, alib):
    """C5 through the emulated init and update kernels: frames with deaths and bursts into recycled slots, and an append of
    a snapshot of another world after every other frame, under the claims the kernels keep. Every buffer equals the
    oracle after every frame."""
    rng = np.random.default_rng(3)
    other = c5_world(rng, [Instance(0, 800, alive=600, seed=7)])
    snap = ref_snapshot(other, 0)
    ref = c5_world(rng, [Instance(0, 3000, alive=1500, seed=42)])
    ref.indirect[1500:, 2] = rng.permutation(np.arange(1500, 3000)).astype(np.uint32)
    emu, claims = claimed(ref, 2, 1500)
    bits = np.zeros(3000 // 32 + 2, dtype=np.uint32)
    floors = np.full(3000 // 32 + 1, NONE32, dtype=np.uint32)
    ages = np.full(3000 // 32 + 2, np.uint64(NONE64), dtype=np.uint64)
    for f, spawn in enumerate([0, 400, 0, 300, 0, 0, 250, 0]):
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        c5_frame(orc, ref, emu, spawn)
        assert_same(ref, emu.pull(), f"frame {f}")
        if f % 2:
            continue
        md = ref.metadata[0]
        sa = SnapshotArgs(C.addressof(emu.metadata[0]), emu.cols[0].ctypes.data, emu.cols[1].ctypes.data, S.PlaneSet(), 2, 8, 0, 3000,
                          snap.nbytes)
        for p in range(2):
            sa.planes.ptr[p], sa.planes.words[p], sa.planes.word_off[p] = emu.planes[p].ctypes.data, 4, 4 * p
        for w in range(8):
            sa.planes.word_to_plane[w] = w // 4
        a = AppendArgs(sa, emu.cols[0].ctypes.data, emu.cols[1].ctypes.data, emu.cols[2].ctypes.data, None, floors.ctypes.data,
                       ages.ctypes.data, claims.ctypes.data)
        want = append_count(ref, 0, snap)
        n = md.alive_count
        alib.semu_append(C.byref(a), snap.ctypes.data)
        assert ref_append(ref, 0, snap) == want and md.alive_count == n + want
        assert_same(ref, emu.pull(), f"append after frame {f}")
    assert ref.metadata[0].alive_count > 1500
