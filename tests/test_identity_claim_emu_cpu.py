"""Identity claims of the alive-list columns (SlabView::ident_claim, DESIGN.md §3) on the real hnb_update kernel under the
CPU thread emulation: rows a claim covers are neither loaded nor stored again, the claim is carried over frames without
deaths and dropped by a frame with deaths, and every result stays bit-identical to the oracle."""
import ctypes as C

import numpy as np
import pytest

from bevy_hanabi_b200 import recipes
from tests import kernel_emu
from tests.helpers import Instance
from tests.kernel_emu import EmuWorld
from tests.test_kernel_emu_cpu import _assert_same, _c5_world

pytestmark = pytest.mark.timeout(600)

# The emulator's update launcher, given the slab's claim words (the plain harness passes none: SlabView::ident_claim = NULL)
_PLAIN_UPDATE = 'extern "C" void emu_update(const EmuBatch* b, uint32_t blocks, uint32_t smem) { emu_launch(hnb::hnb_update, make_params(b), blocks, smem); }'
_CLAIMED_UPDATE = r"""static unsigned long long* g_ident_claim = nullptr;  // [2]: identity claims of ping / pong
extern "C" void emu_set_ident_claim(unsigned long long* claim) { g_ident_claim = claim; }
extern "C" void emu_update(const EmuBatch* b, uint32_t blocks, uint32_t smem) {
    hnb::BatchParams P = make_params(b);
    P.slab.ident_claim = g_ident_claim;
    emu_launch(hnb::hnb_update, P, blocks, smem);
}"""


@pytest.fixture
def claimed_driver(monkeypatch):
    assert kernel_emu.DRIVER.count(_PLAIN_UPDATE) == 1, "tests/kernel_emu.py changed its update launcher"
    monkeypatch.setattr(kernel_emu, "DRIVER", kernel_emu.DRIVER.replace(_PLAIN_UPDATE, _CLAIMED_UPDATE))


ACCEL_DRAG = (C.c_float * 4)(0.0, -9.8, 0.0, 0.5)
POISON = np.uint32(0xDEADBEEF)


def _claim(base, length):
    return np.uint64((base << 32) | length)


def _claimed_world(orc, n, cap, immortal, claim_len):
    rng = np.random.default_rng(n)
    ref = _c5_world(rng, [Instance(0, cap, alive=n, seed=42)])
    if immortal:
        ref.particles[:n, 7] = np.float32(1e9).view(np.uint32)
    emu = EmuWorld(ref, recipes.c5_lowered(), chunks=2, update_ctas=2)
    claims = np.array([_claim(0, claim_len)] * 2, dtype=np.uint64)  # both lists start as the identity (RefWorld)
    emu.lib.emu_set_ident_claim.argtypes = [C.c_void_p]
    emu.lib.emu_set_ident_claim.restype = None
    emu.lib.emu_set_ident_claim(claims.ctypes.data)
    return ref, emu, claims


def _frame(orc, ref, emu):
    ref.oracle_frame(orc, orc.orc_body_update_c5(), ACCEL_DRAG)
    emu.frame_step(orc, ref.sim, [0], [42])


def test_claimed_rows_are_neither_loaded_nor_stored(orc, claimed_driver):
    n = 3000  # not a multiple of the 256-row tile: the last tile is only partly covered
    ref, emu, claims = _claimed_world(orc, n, 3500, immortal=True, claim_len=n)
    _frame(orc, ref, emu)
    _assert_same(ref, emu.pull(), "frame 0")
    written = ref.metadata[0].indirect_write_index
    assert claims[written] == _claim(0, n), "a frame without deaths keeps the claim on the list it wrote"
    # The next frame reads column `written` and writes the other one. Poison both without touching the claims.
    read_col, write_col = emu.cols[written], emu.cols[1 - written]
    read_col[:n] = POISON
    write_col[:n] = POISON
    _frame(orc, ref, emu)
    got = emu.pull()
    assert (read_col[:n] == POISON).all() and (write_col[:n] == POISON).all(), "claimed stores were not skipped"
    got["indirect"][:n, :2] = ref.indirect[:n, :2]  # the poison stands where the oracle has the identity
    _assert_same(ref, got, "frame 1: claimed entries were loaded")


def test_partial_claim_then_deaths_match_the_oracle(orc, claimed_driver):
    """A claim shorter than the list (rows past it are loaded), then frames with deaths: the claim is dropped and
    the lists, dead stack and counters stay those of the oracle."""
    n = 2900
    ref, emu, claims = _claimed_world(orc, n, 3200, immortal=False, claim_len=1700)
    for step in range(6):
        _frame(orc, ref, emu)
        _assert_same(ref, emu.pull(), f"step {step}")
        assert claims[ref.metadata[0].indirect_write_index] == 0, "a frame with a partial claim or deaths drops the claim"
    assert 0 < ref.metadata[0].alive_count < n
