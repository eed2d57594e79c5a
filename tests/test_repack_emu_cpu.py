"""hnb_slab_repack's kernels (hnb_static_kernels.cu: k_repack_gather, k_repack_lists) under the CPU thread emulation of
tests/static_emu.py, against the numpy restatement tests/repack_ref.py, which is itself pinned by a hand-written example.
The host sequence is mirrored here: one gather per physical column into a scratch, the scratch copied back over the slice,
then the lists, claims and alive bits."""
import ctypes as C

import numpy as np
import pytest

from tests import static_emu as S
from tests.helpers import Instance, RefWorld
from tests.kernel_emu import assert_same, c5_frame, c5_world, claim, claimed
from tests.repack_ref import ref_repack
from tests.static_emu import REPACK_DRIVER, RepackArgs, SoaSlab, churned, emulate_repack, expected_bits

pytestmark = pytest.mark.timeout(600)

@pytest.fixture(scope="module")
def slib():
    lib = S.build(REPACK_DRIVER)
    lib.semu_repack_gather.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]
    lib.semu_repack_gather.restype = None
    lib.semu_repack_lists.argtypes = [C.c_void_p]
    lib.semu_repack_lists.restype = None
    lib.semu_sizeof_repack_args.restype = C.c_uint32
    assert lib.semu_sizeof_repack_args() == C.sizeof(RepackArgs)
    return lib


def test_oracle_restatement_by_hand():
    """A 6-row instance at slab row 3 (after a 3-row one), 4 alive, W = 1. Records are one word, 100 + row."""
    ref = RefWorld(9, 1, [Instance(0, 3), Instance(3, 6)])
    ref.particles[:, 0] = 100 + np.arange(9)
    ref.indirect[:, 0] = [0, 1, 2, 50, 51, 52, 53, 54, 55]  # ping: a stale list
    ref.indirect[:, 1] = [0, 1, 2, 4, 1, 5, 2, 77, 77]      # pong (W = 1): local slots 4, 1, 5, 2 alive in this order
    ref.indirect[:, 2] = [0, 1, 2, 99, 99, 99, 99, 6, 3]    # dead stack from row 3 + 4: global slots 6 (local 3), 3 (local 0)
    ref.metadata[1].alive_count, ref.metadata[1].indirect_write_index = 4, 1
    assert ref_repack(ref, 1) == 4
    # src = [4, 1, 5, 2, 3, 0]
    np.testing.assert_array_equal(ref.particles[:, 0], [100, 101, 102, 107, 104, 108, 105, 106, 103])
    np.testing.assert_array_equal(ref.indirect[:, 0], [0, 1, 2, 0, 1, 2, 3, 54, 55])
    np.testing.assert_array_equal(ref.indirect[:, 1], [0, 1, 2, 0, 1, 2, 3, 77, 77])
    np.testing.assert_array_equal(ref.indirect[:, 2], [0, 1, 2, 99, 99, 99, 99, 7, 8])
    assert ref.metadata[1].alive_count == 4 and ref.metadata[1].indirect_write_index == 1, "metadata is not changed"


# (stride in words, sector planes): physical column widths 4 | 8 | 16 | 16+8+4 | 32 | 32+16
LAYOUTS = [(1, False), (2, False), (4, False), (7, False), (8, True), (12, True)]


@pytest.mark.parametrize("stride_words,sector", LAYOUTS, ids=lambda v: str(v))
@pytest.mark.parametrize("n", [0, 1, 33, 1000, 1100])
def test_repack_matches_the_oracle(slib, stride_words, sector, n):
    """One instance of 1100 rows at slab row 37 (neither bitmap words nor blocks aligned), between two others that must
    keep every byte: records, index columns and the alive bits they share words with."""
    rng = np.random.default_rng(n * 31 + stride_words)
    insts = [Instance(0, 37), Instance(37, 1100), Instance(1137, 50)]
    ref = RefWorld(1187, stride_words, insts)
    ref.particles[:] = rng.integers(0, 1 << 32, ref.particles.shape, dtype=np.uint64).astype(np.uint32)
    for i, k in enumerate((20, n, 31)):
        churned(rng, ref, i, k, w=(i + n) & 1)
    soa = SoaSlab(ref, sector, rng)
    bits0 = soa.bits.copy()
    soa.repack(slib, 1, 37, 1100)
    assert ref_repack(ref, 1) == n
    np.testing.assert_array_equal(soa.particles(), ref.particles, err_msg="records")
    np.testing.assert_array_equal(soa.indirect(), ref.indirect, err_msg="ping / pong / dead")
    np.testing.assert_array_equal(soa.bits, expected_bits(bits0, 37, 1100, n), err_msg="alive bitmap")
    assert soa.claims[0] == soa.claims[1] == claim(37, n), "claim words"


@pytest.mark.parametrize("first", [0, 32, 45])
def test_small_slices_and_word_edges(slib, first):
    """Instances of 1 to 70 rows starting inside, at and past a bitmap word; the rest of the slab is another instance's."""
    rng = np.random.default_rng(first)
    for rows in (1, 2, 31, 32, 33, 70):
        for n in sorted({0, 1, rows // 2, rows}):
            insts = [Instance(0, first), Instance(first, rows), Instance(first + rows, 40)] if first else [Instance(0, rows), Instance(rows, 40)]
            i = 1 if first else 0
            ref = RefWorld(first + rows + 40, 3, [x for x in insts if x.capacity])
            ref.particles[:] = rng.integers(0, 1 << 32, ref.particles.shape, dtype=np.uint64).astype(np.uint32)
            for j, inst in enumerate(ref.instances):
                churned(rng, ref, j, n if j == i else inst.capacity // 2, w=rows & 1)
            soa = SoaSlab(ref, False, rng)
            bits0 = soa.bits.copy()
            soa.repack(slib, i, first, rows)
            ref_repack(ref, i)
            what = f"first {first}, rows {rows}, n {n}"
            np.testing.assert_array_equal(soa.particles(), ref.particles, err_msg=what)
            np.testing.assert_array_equal(soa.indirect(), ref.indirect, err_msg=what)
            np.testing.assert_array_equal(soa.bits, expected_bits(bits0, first, rows, n), err_msg=what)
            assert soa.claims[0] == soa.claims[1] == claim(first, n), what


def test_corrupt_state_stays_in_the_slice(slib):
    """Index words that break the invariant (out-of-slice list entries, dead values below `first`) are clamped: the kernels
    touch nothing outside the slice, and the result equals the restatement's."""
    rng = np.random.default_rng(5)
    ref = RefWorld(300, 4, [Instance(0, 100), Instance(100, 150), Instance(250, 50)])
    ref.particles[:] = rng.integers(0, 1 << 32, ref.particles.shape, dtype=np.uint64).astype(np.uint32)
    ref.indirect[:] = rng.integers(0, 1 << 32, ref.indirect.shape, dtype=np.uint64).astype(np.uint32)
    ref.indirect[100:250, 2] = rng.integers(0, 400, 150).astype(np.uint32)
    ref.metadata[1].alive_count, ref.metadata[1].indirect_write_index = 90, 0
    soa = SoaSlab(ref, False, rng)
    soa.repack(slib, 1, 100, 150)
    ref_repack(ref, 1)
    np.testing.assert_array_equal(soa.particles(), ref.particles)
    np.testing.assert_array_equal(soa.indirect(), ref.indirect)


def test_repack_between_emulated_frames(orc, slib):
    """C5 through the emulated init and update kernels: frames with deaths and bursts into recycled slots, a repack, then
    more frames. Every buffer equals the oracle (with ref_repack at the same point) after every frame. The update
    after the repack runs under the claims the repack wrote."""
    rng = np.random.default_rng(3)
    ref = c5_world(rng, [Instance(0, 3000, alive=2500, seed=42)])
    emu, claims = claimed(ref, 2, 0)
    for f, spawn in enumerate([0, 400, 0, 300, 0, 0, 250]):
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        c5_frame(orc, ref, emu, spawn)
        assert_same(ref, emu.pull(), f"frame {f}")
    list_w = ref.indirect[:ref.metadata[0].alive_count, ref.metadata[0].indirect_write_index]
    assert (list_w != np.arange(len(list_w))).any(), "the list is not the identity before the repack"
    bits = np.zeros(3000 // 32 + 2, dtype=np.uint32)
    emulate_repack(slib, emu.planes, [16, 16], emu.cols, bits, claims, emu.metadata, 0, 0, 3000)
    n = ref_repack(ref, 0)
    assert_same(ref, emu.pull(), "after the repack")
    assert claims[0] == claims[1] == claim(0, n)
    for f, spawn in enumerate([0, 0, 200, 0, 0], start=7):
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        c5_frame(orc, ref, emu, spawn)
        assert_same(ref, emu.pull(), f"frame {f}, after the repack")
