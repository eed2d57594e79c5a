"""Identity claims of the alive-list columns (SlabView::ident_claim, DESIGN.md §3) on the real hnb_update kernel under the
CPU thread emulation: rows a claim covers are neither loaded nor stored again, the claim is carried over frames without
deaths and dropped by a frame with deaths, and every result stays bit-identical to the oracle."""
import numpy as np
import pytest

from tests.helpers import CLAIM_EDGE_SPAWNS, CLAIM_ENDS, Instance, claim_edge_world, claim_end
from tests.kernel_emu import assert_same, c5_frame, c5_world, claim, claimed

pytestmark = pytest.mark.timeout(600)

SUB_TILES = pytest.mark.parametrize("chunks", [1, 2, 3, 4], ids=lambda n: f"{n}sub")
POISON = np.uint32(0xDEADBEEF)


def _claimed_world(orc, n, cap, immortal, claim_len, chunks):
    rng = np.random.default_rng(n)
    ref = c5_world(rng, [Instance(0, cap, alive=n, seed=42)])
    if immortal:
        ref.particles[:n, 7] = np.float32(1e9).view(np.uint32)
    emu, claims = claimed(ref, chunks, claim_len)  # both lists start as the identity over [0, n) (RefWorld)
    return ref, emu, claims


def test_claimed_rows_are_neither_loaded_nor_stored(orc, chunks=2):
    n = 3000  # not a multiple of any tile size: the last tile is only partly covered
    ref, emu, claims = _claimed_world(orc, n, 3500, immortal=True, claim_len=n, chunks=chunks)
    c5_frame(orc, ref, emu)
    assert_same(ref, emu.pull(), "frame 0")
    written = ref.metadata[0].indirect_write_index
    assert claims[written] == claim(0, n), "a frame without deaths keeps the claim on the list it wrote"
    # The next frame reads column `written` and writes the other one. Poison both without touching the claims.
    read_col, write_col = emu.cols[written], emu.cols[1 - written]
    read_col[:n] = POISON
    write_col[:n] = POISON
    c5_frame(orc, ref, emu)
    got = emu.pull()
    assert (read_col[:n] == POISON).all() and (write_col[:n] == POISON).all(), "claimed stores were not skipped"
    got["indirect"][:n, :2] = ref.indirect[:n, :2]  # the poison stands where the oracle has the identity
    assert_same(ref, got, "frame 1: claimed entries were loaded")


def test_partial_claim_then_deaths_match_the_oracle(orc, chunks=2, claim_len=1700):
    """A claim shorter than the list (rows past it are loaded), then frames with deaths: the claim is dropped and
    the lists, dead stack and counters stay those of the oracle. With `claim_len` = the list, the first frame with a
    death drops the claim instead."""
    n = 2900
    ref, emu, claims = _claimed_world(orc, n, 3200, immortal=False, claim_len=claim_len, chunks=chunks)
    for step in range(6):
        alive = ref.metadata[0].alive_count
        c5_frame(orc, ref, emu)
        assert_same(ref, emu.pull(), f"step {step}")
        kept = claim_len == n and ref.metadata[0].alive_count == alive == n
        assert claims[ref.metadata[0].indirect_write_index] == (claim(0, n) if kept else 0), f"step {step}: claim on the list it wrote"
    assert 0 < ref.metadata[0].alive_count < n


@pytest.mark.parametrize("chunks", [1, 3, 4], ids=lambda n: f"{n}sub")
@pytest.mark.parametrize("test", [test_claimed_rows_are_neither_loaded_nor_stored, test_partial_claim_then_deaths_match_the_oracle],
                         ids=lambda t: t.__name__[len("test_"):])
def test_at_other_tile_sizes(orc, test, chunks):
    """The two tests above (2 sub-tiles per tile) at 1, 3 and 4 sub-tiles."""
    test(orc, chunks=chunks)


@SUB_TILES
def test_full_claim_then_deaths_match_the_oracle(orc, chunks):
    """A claim covering the whole list is kept by frames without deaths and dropped by the first frame with one."""
    test_partial_claim_then_deaths_match_the_oracle(orc, chunks=chunks, claim_len=2900)


@SUB_TILES
@pytest.mark.parametrize("end", CLAIM_ENDS)
def test_claim_ending_at_tile_edges(orc, chunks, end):
    """The GPU scenario of the same name, with the claim words asserted after every frame: kept by the frame without
    deaths, shrunk to the first appended row by the burst, then dropped: the burst's update reads a list longer than
    its claim, and the next update reads a list without one."""
    L = claim_end(end, 128 * chunks)
    cap = L + 1100  # room for both bursts
    ref = claim_edge_world(L, cap)
    emu, claims = claimed(ref, chunks, cap)  # as hnb_slab_fill_c5 over the whole capacity
    for f, spawn in enumerate(CLAIM_EDGE_SPAWNS):
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        c5_frame(orc, ref, emu, spawn)
        assert_same(ref, emu.pull(), f"claim ending at row {L}, frame {f}")
        written = ref.metadata[0].indirect_write_index
        want = {0: (claim(0, cap), claim(0, cap)), 1: (0, claim(0, L))}.get(f, (0, 0))  # (written column, read column)
        assert (claims[written], claims[1 - written]) == want, f"claim ending at row {L}, frame {f}: claim words"
    assert ref.metadata[0].alive_count == 1000
