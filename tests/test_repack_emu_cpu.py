"""hnb_slab_repack's kernels (hnb_static_kernels.cu: k_repack_gather, k_repack_lists) under the CPU thread emulation of
tests/static_emu.py, against the numpy restatement tests/repack_ref.py, which is itself pinned by a hand-written example.
The host sequence is mirrored here: one gather per physical column into a scratch, the scratch copied back over the slice,
then the lists, claims and alive bits."""
import ctypes as C

import numpy as np
import pytest

from oracle import c_oracle as O
from tests import static_emu as S
from tests.helpers import Instance, RefWorld
from tests.repack_ref import ref_repack
from tests.test_identity_claim_emu_cpu import _claim, _claimed, _frame, claimed_driver  # noqa: F401
from tests.test_kernel_emu_cpu import _assert_same, _c5_world

pytestmark = pytest.mark.timeout(600)

# Entry points of the repack kernels, appended to the static emulation's driver for the build of this module
REPACK_DRIVER = r"""
extern "C" void semu_repack_gather(const RepackArgs* a, const void* col, void* scratch, uint32_t width) {
    RepackArgs r = *a;
    const unsigned blocks = (r.rows + RP_ROWS_PER_BLOCK - 1) / RP_ROWS_PER_BLOCK;
    switch (width) {
    case 4: emu_run([&] { k_repack_gather<1>(r, (const RepackPiece<1>*)col, (RepackPiece<1>*)scratch); }, blocks, RP_THREADS, 8); break;
    case 8: emu_run([&] { k_repack_gather<2>(r, (const RepackPiece<2>*)col, (RepackPiece<2>*)scratch); }, blocks, RP_THREADS, 8); break;
    case 16: emu_run([&] { k_repack_gather<4>(r, (const RepackPiece<4>*)col, (RepackPiece<4>*)scratch); }, blocks, RP_THREADS, 8); break;
    case 32: emu_run([&] { k_repack_gather<8>(r, (const RepackPiece<8>*)col, (RepackPiece<8>*)scratch); }, blocks, RP_THREADS, 8); break;
    }
}
extern "C" void semu_repack_lists(const RepackArgs* a) { RepackArgs r = *a; emu_run([&] { k_repack_lists(r); }, (r.rows + RP_THREADS - 1) / RP_THREADS, RP_THREADS, 8); }
extern "C" uint32_t semu_sizeof_repack_args(void) { return sizeof(RepackArgs); }
"""


class RepackArgs(C.Structure):
    """hnb::RepackArgs (hnb_static_kernels.h)"""
    _fields_ = [("metadata", C.c_void_p), ("ping", C.c_void_p), ("pong", C.c_void_p), ("dead", C.c_void_p), ("alive_bits", C.c_void_p),
                ("claim", C.c_void_p), ("first", C.c_uint32), ("rows", C.c_uint32)]


@pytest.fixture(scope="module")
def slib():
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(S, "DRIVER", S.DRIVER + REPACK_DRIVER)
        lib = S.build()
    lib.semu_repack_gather.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]
    lib.semu_repack_gather.restype = None
    lib.semu_repack_lists.argtypes = [C.c_void_p]
    lib.semu_repack_lists.restype = None
    lib.semu_sizeof_repack_args.restype = C.c_uint32
    assert lib.semu_sizeof_repack_args() == C.sizeof(RepackArgs)
    return lib


def physical_widths(stride: int, sector: bool):
    """Byte widths of a slab's physical columns (effect_source.cpp physical_planes)."""
    pieces, off = [], 0
    while off < stride:
        w = 16 if stride - off >= 16 else (8 if stride - off >= 8 else 4)
        pieces.append(w)
        off += w
    if not sector:
        return pieces
    out, p = [], 0
    while p < len(pieces):
        if p + 1 < len(pieces) and pieces[p] == pieces[p + 1] == 16:
            out.append(32)
            p += 2
        else:
            out.append(pieces[p])
            p += 1
    return out


class SoaSlab:
    """A slab in the device's layout (one array per physical column, ping / pong / dead, alive bitmap, claim words),
    made from and read back into a RefWorld's reference layouts."""

    def __init__(self, ref: RefWorld, sector: bool, rng):
        self.widths = physical_widths(ref.stride_words * 4, sector)
        self.planes, off = [], 0
        for w in self.widths:
            self.planes.append(np.ascontiguousarray(ref.particles[:, off:off + w // 4]).reshape(-1).copy())
            off += w // 4
        self.cols = [np.ascontiguousarray(ref.indirect[:, c]).copy() for c in range(3)]
        self.bits = rng.integers(0, 1 << 32, ref.slab_rows // 32 + 2, dtype=np.uint64).astype(np.uint32)
        self.claims = np.array([_claim(5, 7), _claim(9, 11)], dtype=np.uint64)
        self.metadata = (O.EffectMetadata * len(ref.instances)).from_buffer_copy(bytes(ref.metadata))

    def repack(self, lib, i: int, first: int, rows: int):
        emulate_repack(lib, self.planes, self.widths, self.cols, self.bits, self.claims, self.metadata, i, first, rows)

    def particles(self):
        return np.concatenate([p.reshape(-1, w // 4) for p, w in zip(self.planes, self.widths)], axis=1)

    def indirect(self):
        return np.stack(self.cols, axis=1)


def emulate_repack(lib, planes, widths, cols, bits, claims, metadata, i, first, rows):
    """hnb_slab_repack's device work, in its order."""
    a = RepackArgs(C.addressof(metadata[i]), cols[0].ctypes.data, cols[1].ctypes.data, cols[2].ctypes.data, bits.ctypes.data,
                   claims.ctypes.data, first, rows)
    scratch = np.zeros(rows * 8 + 8, dtype=np.uint32)
    for plane, w in zip(planes, widths):
        k = w // 4
        lib.semu_repack_gather(C.byref(a), plane.ctypes.data, scratch.ctypes.data, w)
        plane[first * k:(first + rows) * k] = scratch[:rows * k]
    lib.semu_repack_lists(C.byref(a))


def expected_bits(bits, first, rows, n):
    b = np.unpackbits(bits.view(np.uint8), bitorder="little").copy()
    b[first:first + n] = 1
    b[first + n:first + rows] = 0
    return np.packbits(b, bitorder="little").view(np.uint32)


def churned(rng, ref, i, n, w):
    """Instance `i` in a state the update invariant allows: column `w` lists n distinct local slots, the dead stack holds
    the other slots (global values) in a shuffled order from row n up; every other index word is garbage."""
    inst = ref.instances[i]
    first, rows = inst.slab_offset, inst.capacity
    perm = rng.permutation(rows).astype(np.uint32)
    garbage = lambda k: rng.integers(0, 1 << 32, k, dtype=np.uint64).astype(np.uint32)  # noqa: E731
    ref.indirect[first:first + rows, w] = np.concatenate([perm[:n], garbage(rows - n)])
    ref.indirect[first:first + rows, 1 - w] = garbage(rows)
    ref.indirect[first:first + rows, 2] = np.concatenate([garbage(n), perm[n:] + np.uint32(first)])
    md = ref.metadata[i]
    md.alive_count, md.max_spawn, md.indirect_write_index = n, rows - n, w


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
    assert soa.claims[0] == soa.claims[1] == _claim(37, n), "claim words"


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
            assert soa.claims[0] == soa.claims[1] == _claim(first, n), what


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


def test_repack_between_emulated_frames(orc, slib, claimed_driver):  # noqa: F811
    """C5 through the emulated init and update kernels: frames with deaths and bursts into recycled slots, a repack, then
    more frames. Every buffer equals the oracle (with ref_repack at the same point) after every frame. The update
    after the repack runs under the claims the repack wrote."""
    rng = np.random.default_rng(3)
    ref = _c5_world(rng, [Instance(0, 3000, alive=2500, seed=42)])
    emu, claims = _claimed(ref, 2, 0)
    for f, spawn in enumerate([0, 400, 0, 300, 0, 0, 250]):
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        _frame(orc, ref, emu, spawn)
        _assert_same(ref, emu.pull(), f"frame {f}")
    list_w = ref.indirect[:ref.metadata[0].alive_count, ref.metadata[0].indirect_write_index]
    assert (list_w != np.arange(len(list_w))).any(), "the list is not the identity before the repack"
    bits = np.zeros(3000 // 32 + 2, dtype=np.uint32)
    emulate_repack(slib, emu.planes, [16, 16], emu.cols, bits, claims, emu.metadata, 0, 0, 3000)
    n = ref_repack(ref, 0)
    _assert_same(ref, emu.pull(), "after the repack")
    assert claims[0] == claims[1] == _claim(0, n)
    for f, spawn in enumerate([0, 0, 200, 0, 0], start=7):
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        _frame(orc, ref, emu, spawn)
        _assert_same(ref, emu.pull(), f"frame {f}, after the repack")
