"""hnb_instance_snapshot / hnb_instance_restore's kernels (hnb_static_kernels.cu: k_snapshot_gather, k_restore_scatter,
then k_repack_lists) under the CPU thread emulation of tests/static_emu.py, against the numpy restatement
tests/snapshot_ref.py, which is itself pinned by a hand-written example and tied to tests/repack_ref.py."""
import copy
import ctypes as C

import numpy as np
import pytest

from tests import static_emu as S
from tests.helpers import Instance, RefWorld
from tests.repack_ref import ref_repack
from tests.snapshot_ref import HEADER_WORDS, SNAPSHOT_MAGIC, ref_restore, ref_snapshot, restore_count, snapshot_bytes
from tests.test_identity_claim_emu_cpu import _claim, _claimed, _frame, claimed_driver  # noqa: F401
from tests.test_kernel_emu_cpu import _assert_same, _c5_world
from tests.test_repack_emu_cpu import REPACK_DRIVER, RepackArgs, SoaSlab, churned, expected_bits

pytestmark = pytest.mark.timeout(600)

# Entry points of the snapshot kernels, appended (with the repack ones) to the static emulation's driver for this module
SNAPSHOT_DRIVER = r"""
extern "C" void semu_snapshot_gather(const SnapshotArgs* a, uint32_t* dst) {
    SnapshotArgs s = *a;
    emu_run([&] { k_snapshot_gather(s, dst); }, (s.rows + RP_ROWS_PER_BLOCK - 1) / RP_ROWS_PER_BLOCK, RP_THREADS, 8);
}
extern "C" void semu_restore_scatter(const SnapshotArgs* a, const uint32_t* src) {
    SnapshotArgs s = *a;
    emu_run([&] { k_restore_scatter(s, src); }, (s.rows + RP_ROWS_PER_BLOCK - 1) / RP_ROWS_PER_BLOCK, RP_THREADS, 8);
}
extern "C" uint32_t semu_sizeof_snapshot_args(void) { return sizeof(SnapshotArgs); }
"""


class SnapshotArgs(C.Structure):
    """hnb::SnapshotArgs (hnb_static_kernels.h)"""
    _fields_ = [("metadata", C.c_void_p), ("ping", C.c_void_p), ("pong", C.c_void_p), ("planes", S.PlaneSet),
                ("num_planes", C.c_uint32), ("stride_words", C.c_uint32), ("first", C.c_uint32), ("rows", C.c_uint32),
                ("src_bytes", C.c_uint64)]


@pytest.fixture(scope="module")
def slib():
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(S, "DRIVER", S.DRIVER + REPACK_DRIVER + SNAPSHOT_DRIVER)
        lib = S.build()
    lib.semu_snapshot_gather.argtypes = [C.c_void_p, C.c_void_p]
    lib.semu_restore_scatter.argtypes = [C.c_void_p, C.c_void_p]
    lib.semu_repack_lists.argtypes = [C.c_void_p]
    for f in (lib.semu_snapshot_gather, lib.semu_restore_scatter, lib.semu_repack_lists):
        f.restype = None
    lib.semu_sizeof_snapshot_args.restype = C.c_uint32
    assert lib.semu_sizeof_snapshot_args() == C.sizeof(SnapshotArgs)
    return lib


def _args(planes, widths, cols, metadata, i, first, rows, stride_words, src_bytes=0):
    ps = S.PlaneSet()
    off = 0
    for p, (plane, w) in enumerate(zip(planes, widths)):
        ps.ptr[p], ps.words[p], ps.word_off[p] = plane.ctypes.data, w // 4, off
        off += w // 4
    return SnapshotArgs(C.addressof(metadata[i]), cols[0].ctypes.data, cols[1].ctypes.data, ps, len(widths), stride_words,
                        first, rows, src_bytes)


def emulate_snapshot(lib, planes, widths, cols, metadata, i, first, rows, stride_words, dst):
    """hnb_instance_snapshot's device work."""
    a = _args(planes, widths, cols, metadata, i, first, rows, stride_words)
    lib.semu_snapshot_gather(C.byref(a), dst.ctypes.data)


def emulate_restore(lib, planes, widths, cols, bits, claims, metadata, i, first, rows, stride_words, src, src_bytes=None):
    """hnb_instance_restore's device work, in its order."""
    a = _args(planes, widths, cols, metadata, i, first, rows, stride_words, src.nbytes if src_bytes is None else src_bytes)
    lib.semu_restore_scatter(C.byref(a), src.ctypes.data)
    r = RepackArgs(C.addressof(metadata[i]), cols[0].ctypes.data, cols[1].ctypes.data, cols[2].ctypes.data, bits.ctypes.data,
                   claims.ctypes.data, first, rows)
    lib.semu_repack_lists(C.byref(r))


def soa_snapshot(lib, soa, ref, i, sentinel=0xA5A5A5A5):
    """Snapshot instance i of `soa` into a buffer of hnb_instance_snapshot_bytes filled with `sentinel`."""
    inst = ref.instances[i]
    dst = np.full(snapshot_bytes(ref.stride_words * 4, inst.capacity) // 4, sentinel, dtype=np.uint32)
    emulate_snapshot(lib, soa.planes, soa.widths, soa.cols, soa.metadata, i, inst.slab_offset, inst.capacity, ref.stride_words, dst)
    return dst


def soa_restore(lib, soa, ref, i, src, src_bytes=None):
    inst = ref.instances[i]
    emulate_restore(lib, soa.planes, soa.widths, soa.cols, soa.bits, soa.claims, soa.metadata, i, inst.slab_offset, inst.capacity,
                    ref.stride_words, src, src_bytes)


def _state(soa):
    return [p.copy() for p in soa.planes] + [c.copy() for c in soa.cols] + [soa.bits.copy(), soa.claims.copy(),
                                                                            np.frombuffer(bytes(soa.metadata), dtype=np.uint32).copy()]


def _metadata(soa):
    return np.frombuffer(bytes(soa.metadata), dtype=np.uint32).reshape(len(soa.metadata), 15)


def _assert_soa(soa, ref, what):
    np.testing.assert_array_equal(soa.particles(), ref.particles, err_msg=f"{what}: records")
    np.testing.assert_array_equal(soa.indirect(), ref.indirect, err_msg=f"{what}: ping / pong / dead")
    np.testing.assert_array_equal(_metadata(soa), ref.metadata_rows(), err_msg=f"{what}: metadata")


def _random_world(rng, slab_rows, stride_words, insts, alive, first_w=0):
    ref = RefWorld(slab_rows, stride_words, insts)
    ref.particles[:] = rng.integers(0, 1 << 32, ref.particles.shape, dtype=np.uint64).astype(np.uint32)
    for j, k in enumerate(alive):
        churned(rng, ref, j, k, w=(j + first_w) & 1)
        ref.metadata[j].particle_counter = int(rng.integers(0, 1 << 32))
    return ref


def test_oracle_restatement_by_hand():
    """A 6-row instance at slab row 3 (after a 3-row one), 4 alive, W = 1, particle_counter 9. Records are one word,
    100 + row. Restored into a 3-row instance at slab row 2 of another slab, then back into its own slice."""
    ref = RefWorld(9, 1, [Instance(0, 3), Instance(3, 6)])
    ref.particles[:, 0] = 100 + np.arange(9)
    ref.indirect[:, 0] = [0, 1, 2, 50, 51, 52, 53, 54, 55]  # ping: a stale list
    ref.indirect[:, 1] = [0, 1, 2, 4, 1, 5, 2, 77, 77]      # pong (W = 1): local slots 4, 1, 5, 2 alive in this order
    ref.indirect[:, 2] = [0, 1, 2, 99, 99, 99, 99, 6, 3]    # dead stack from row 3 + 4
    ref.metadata[1].alive_count, ref.metadata[1].indirect_write_index, ref.metadata[1].particle_counter = 4, 1, 9
    before = (ref.particles.copy(), ref.indirect.copy(), ref.metadata_rows())
    snap = ref_snapshot(ref, 1)
    np.testing.assert_array_equal(snap, [SNAPSHOT_MAGIC, 1, 4, 4, 9, 6] + [0] * 10 + [107, 104, 108, 105])
    for a, b in zip(before, (ref.particles, ref.indirect, ref.metadata_rows())):
        np.testing.assert_array_equal(a, b, err_msg="a snapshot modifies nothing")

    dst = RefWorld(6, 1, [Instance(0, 2), Instance(2, 3)])
    dst.particles[:, 0] = 200 + np.arange(6)
    dst.metadata[1].alive_count, dst.metadata[1].max_spawn, dst.metadata[1].indirect_write_index = 1, 2, 1
    assert ref_restore(dst, 1, snap) == 3, "the first `rows` particles in alive-list order are kept"
    np.testing.assert_array_equal(dst.particles[:, 0], [200, 201, 107, 104, 108, 205])
    np.testing.assert_array_equal(dst.indirect[:, 0], [0, 0, 0, 1, 2, 0])
    np.testing.assert_array_equal(dst.indirect[:, 1], [0, 0, 0, 1, 2, 0])
    np.testing.assert_array_equal(dst.indirect[:, 2], [0, 1, 2, 3, 4, 5])
    md = dst.metadata[1]
    assert (md.alive_count, md.max_spawn, md.particle_counter, md.indirect_write_index) == (3, 0, 9, 1)

    assert ref_restore(ref, 1, snap) == 4
    np.testing.assert_array_equal(ref.particles[:, 0], [100, 101, 102, 107, 104, 108, 105, 107, 108])
    np.testing.assert_array_equal(ref.indirect[:, 0], [0, 1, 2, 0, 1, 2, 3, 54, 55])
    np.testing.assert_array_equal(ref.indirect[:, 1], [0, 1, 2, 0, 1, 2, 3, 77, 77])
    np.testing.assert_array_equal(ref.indirect[:, 2], [0, 1, 2, 99, 99, 99, 99, 7, 8])
    assert ref.metadata[1].max_spawn == 2


# (stride in words, sector planes): physical column widths 4 | 8 | 16 | 16+8+4 | 32 | 32+16
LAYOUTS = [(1, False), (2, False), (4, False), (7, False), (8, True), (12, True)]


@pytest.mark.parametrize("stride_words,sector", LAYOUTS, ids=lambda v: str(v))
@pytest.mark.parametrize("n", [0, 1, 33, 1000, 1100])
def test_snapshot_matches_the_oracle(slib, stride_words, sector, n):
    """One instance of 1100 rows at slab row 37, between two others. The buffer holds the header and n records; bytes
    past them keep their sentinel; the slab (records, lists, bits, claims, metadata) keeps every byte."""
    rng = np.random.default_rng(n * 31 + stride_words)
    ref = _random_world(rng, 1187, stride_words, [Instance(0, 37), Instance(37, 1100), Instance(1137, 50)], (20, n, 31), n)
    soa = SoaSlab(ref, sector, rng)
    before = _state(soa)
    got = soa_snapshot(slib, soa, ref, 1)
    want = ref_snapshot(ref, 1)
    np.testing.assert_array_equal(got[:len(want)], want, err_msg="header and records")
    assert (got[len(want):] == 0xA5A5A5A5).all(), "bytes past 64 + n * stride were written"
    for k, (a, b) in enumerate(zip(before, _state(soa))):
        np.testing.assert_array_equal(a, b, err_msg=f"a snapshot modified buffer {k}")


@pytest.mark.parametrize("stride_words,sector", LAYOUTS, ids=lambda v: str(v))
@pytest.mark.parametrize("n", [0, 1, 33, 1000, 1100])
@pytest.mark.parametrize("target", ["same", "moved", "smaller"])
def test_restore_matches_the_oracle(slib, stride_words, sector, n, target):
    """A snapshot of an 1100-row instance restored into its own slice, into a 1300-row instance at slab row 45 of another
    slab, or into a 700-row one at slab row 45. The neighbours keep every byte, including the alive bits they share
    words with; the claims become {first, m}."""
    rng = np.random.default_rng(n * 17 + stride_words)
    src_ref = _random_world(rng, 1187, stride_words, [Instance(0, 37), Instance(37, 1100), Instance(1137, 50)], (20, n, 31), n)
    src = SoaSlab(src_ref, sector, rng)
    snap = soa_snapshot(slib, src, src_ref, 1)
    if target == "same":
        ref, soa, first = src_ref, src, 37
    else:
        cap = 1300 if target == "moved" else 700
        ref = _random_world(rng, 45 + cap + 40, stride_words, [Instance(0, 45), Instance(45, cap), Instance(45 + cap, 40)], (10, 300, 17))
        soa, first = SoaSlab(ref, sector, rng), 45
    bits0 = soa.bits.copy()
    soa_restore(slib, soa, ref, 1, snap)
    m = ref_restore(ref, 1, snap)
    assert m == min(n, ref.instances[1].capacity)
    _assert_soa(soa, ref, target)
    np.testing.assert_array_equal(soa.bits, expected_bits(bits0, first, ref.instances[1].capacity, m), err_msg="alive bitmap")
    assert soa.claims[0] == soa.claims[1] == _claim(first, m), "claim words"


@pytest.mark.parametrize("first", [0, 32, 45])
def test_small_slices_and_word_edges(slib, first):
    """Snapshots of 70-row instances restored into instances of 1 to 70 rows starting inside, at and past a bitmap word."""
    rng = np.random.default_rng(first)
    src_ref = _random_world(rng, 70, 3, [Instance(0, 70)], (0,))
    for n in (0, 1, 35, 70):
        churned(rng, src_ref, 0, n, w=n & 1)
        src = SoaSlab(src_ref, False, rng)
        snap = soa_snapshot(slib, src, src_ref, 0)
        for rows in (1, 2, 31, 32, 33, 70):
            insts = [Instance(0, first), Instance(first, rows), Instance(first + rows, 40)] if first else [Instance(0, rows), Instance(rows, 40)]
            i = 1 if first else 0
            ref = _random_world(rng, first + rows + 40, 3, [x for x in insts if x.capacity], [x.capacity // 2 for x in insts if x.capacity])
            soa = SoaSlab(ref, False, rng)
            bits0 = soa.bits.copy()
            soa_restore(slib, soa, ref, i, snap)
            m = ref_restore(ref, i, snap)
            what = f"first {first}, rows {rows}, n {n}"
            _assert_soa(soa, ref, what)
            np.testing.assert_array_equal(soa.bits, expected_bits(bits0, first, rows, m), err_msg=what)
            assert soa.claims[0] == soa.claims[1] == _claim(first, m), what


@pytest.mark.parametrize("corruption", ["magic", "version", "stride", "short", "very_short", "header_only"])
def test_corrupt_or_short_snapshots(slib, corruption):
    """A header that is not a version-1 snapshot of this stride restores an empty instance and leaves particle_counter;
    a short `src_bytes` restores the records it holds in full, and the kernel reads nothing past it."""
    rng = np.random.default_rng(9)
    src_ref = _random_world(rng, 500, 5, [Instance(0, 500)], (400,))
    src = SoaSlab(src_ref, False, rng)
    snap = soa_snapshot(slib, src, src_ref, 0)[:HEADER_WORDS + 400 * 5].copy()
    src_bytes = snap.nbytes
    if corruption == "magic":
        snap[0] ^= 1
    elif corruption == "version":
        snap[1] = 2
    elif corruption == "stride":
        snap[2] = 24
    else:
        src_bytes = {"short": 64 + 123 * 20 + 19, "very_short": 64 + 19, "header_only": 64}[corruption]
        snap = snap[:(src_bytes + 3) // 4].copy()  # the kernel must not read past src_bytes: the array ends there
    ref = _random_world(rng, 600, 5, [Instance(0, 100), Instance(100, 450), Instance(550, 50)], (50, 200, 25))
    soa = SoaSlab(ref, False, rng)
    counter = ref.metadata[1].particle_counter
    soa_restore(slib, soa, ref, 1, snap, src_bytes)
    m = ref_restore(ref, 1, snap, src_bytes)
    assert m == {"short": 123, "very_short": 0, "header_only": 0}.get(corruption, 0)
    assert restore_count(ref, 1, snap, src_bytes) == m
    _assert_soa(soa, ref, corruption)
    if corruption in ("magic", "version", "stride"):
        assert ref.metadata[1].particle_counter == counter
    assert soa.claims[0] == soa.claims[1] == _claim(100, m)


def test_round_trip_equals_repack(slib):
    """restore(snapshot(X)) into X's own slice leaves the lists, claims, bits, metadata and live records of
    hnb_slab_repack(X); the repack also permutes the dead rows' records, the restore leaves them."""
    rng = np.random.default_rng(21)
    ref = _random_world(rng, 1187, 7, [Instance(0, 37), Instance(37, 1100), Instance(1137, 50)], (20, 777, 31))
    soa = SoaSlab(ref, False, rng)
    repacked = copy.deepcopy(ref)
    n = ref_repack(repacked, 1)
    snap = soa_snapshot(slib, soa, ref, 1)
    soa_restore(slib, soa, ref, 1, snap)
    assert ref_restore(ref, 1, snap) == n
    _assert_soa(soa, ref, "restored")
    np.testing.assert_array_equal(ref.indirect, repacked.indirect)
    np.testing.assert_array_equal(ref.metadata_rows(), repacked.metadata_rows())
    np.testing.assert_array_equal(ref.particles[37:37 + n], repacked.particles[37:37 + n])
    assert soa.claims[0] == soa.claims[1] == _claim(37, n)


def test_restore_between_emulated_frames(orc, slib, claimed_driver):  # noqa: F811
    """C5 through the emulated init and update kernels: frames with deaths and bursts into recycled slots, a snapshot,
    then a restore into a fresh 1200-row world (fewer rows than are alive) and more frames there. Every buffer equals
    the oracle after every frame; the frames after the restore run under the claims the restore wrote."""
    rng = np.random.default_rng(3)
    ref = _c5_world(rng, [Instance(0, 3000, alive=2500, seed=42)])
    emu, _ = _claimed(ref, 2, 0)
    for f, spawn in enumerate([0, 400, 0, 300, 0, 0, 250]):
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        _frame(orc, ref, emu, spawn)
        _assert_same(ref, emu.pull(), f"frame {f}")
    assert ref.metadata[0].alive_count > 1200
    snap = np.full(snapshot_bytes(32, 3000) // 4, 0xA5A5A5A5, dtype=np.uint32)
    emulate_snapshot(slib, emu.planes, [16, 16], emu.cols, emu.metadata, 0, 0, 3000, 8, snap)
    np.testing.assert_array_equal(snap[:HEADER_WORDS + 8 * ref.metadata[0].alive_count], ref_snapshot(ref, 0))

    dst = _c5_world(rng, [Instance(0, 1200, alive=0, seed=42)])
    dst.indirect[:, 2] = rng.permutation(1200).astype(np.uint32)
    demu, claims = _claimed(dst, 2, 0)
    bits = np.zeros(1200 // 32 + 2, dtype=np.uint32)
    emulate_restore(slib, demu.planes, [16, 16], demu.cols, bits, claims, demu.metadata, 0, 0, 1200, 8, snap)
    m = ref_restore(dst, 0, snap)
    assert m == 1200
    _assert_same(dst, demu.pull(), "after the restore")
    assert claims[0] == claims[1] == _claim(0, m)
    for f, spawn in enumerate([0, 0, 200, 0, 0], start=7):
        dst.sim.time = np.float32(f) * dst.sim.delta_time
        _frame(orc, dst, demu, spawn)
        _assert_same(dst, demu.pull(), f"frame {f}, after the restore")
    assert dst.metadata[0].alive_count < 1200
