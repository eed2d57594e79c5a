"""GPU parity of the update pass on slabs filled by hnb_slab_fill_c5, whose alive lists carry an identity claim
(DESIGN.md §3): every buffer is compared bit for bit with the C oracle after every frame while the claim is used,
shrunk by spawns, dropped by deaths, and invalidated by other writers of the index columns. Every scenario also runs at 2,
3 and 4 sub-tiles per update tile: a claim that covers the first sub-tile of a tile but not the rest, and the prefetch of
the next sub-tile under a claim, only exist from 2 up."""
import numpy as np
import pytest

from tests.helpers import (CLAIM_ENDS, CLAIM_EDGE_SPAWNS, FORCED_SUB_TILES, SUB_TILE_C5, Instance, assert_claims_trusted,  # noqa: F401
                           at_tile_sizes, claim_edge_lockstep, claim_end, filled_c5, tiled_ctx)

pytestmark = pytest.mark.gpu


def test_no_death_frames_then_deaths_then_spawns_into_recycled_slots(ctx, orc):
    """Lifetimes >= 0.1 s: five frames without deaths on the claimed lists (the fill covers more rows than are alive), then
    deaths, then bursts into the freed slots."""
    lock = filled_c5(ctx, orc, [Instance(0, 8192, alive=6000, seed=42)], [(0, 8192, 77, 0.1, 0.5)])
    lock.run([[0]] * 5, what="no deaths")
    assert lock.ref.metadata[0].alive_count == 6000
    lock.run([[0]] * 8, what="deaths")
    assert lock.ref.metadata[0].alive_count < 6000
    lock.run([[700], [0], [0], [1500], [0], [0]], what="spawns")
    assert lock.ref.metadata[0].particle_counter == 2200


def test_spawn_shrinks_the_claim(ctx, orc):
    """A claim longer than the alive count, then a burst whose dead slots are not in row order: the spawned rows must be
    read through the list."""
    lock = filled_c5(ctx, orc, [Instance(0, 8192, alive=5000, seed=3)], [(0, 8192, 5, 1e9, 1e9)], dead_perm_seed=11)
    lock.run([[0], [0], [900], [0], [0], [300], [0]], what="spawn under a claim")


def test_upload_indirect_drops_the_claim(ctx, orc):
    """After the fill, different permutations are uploaded into ping and pong: a stale claim would read the identity and
    skip the stores."""
    n = 6000
    lock = filled_c5(ctx, orc, [Instance(0, n, alive=n, seed=8)], [(0, n, 9, 0.05, 0.4)])
    rng = np.random.default_rng(12)
    lock.ref.indirect[:, 0] = rng.permutation(n)
    lock.ref.indirect[:, 1] = rng.permutation(n)
    ctx.slab_upload_indirect(lock.gpu.slab, 0, lock.ref.indirect)
    lock.run([[0]] * 12, what="after upload")
    assert lock.ref.metadata[0].alive_count < n


@at_tile_sizes("batches,parities", [(None, (0, 0)), ([[0], [1]], (0, 0)), (None, (1, 0)), ([[0], [1]], (1, 0))],
               ids=["one_batch", "two_batches", "one_batch_mixed_parity", "two_batches_mixed_parity"])
def test_two_instances_one_claim(tiled_ctx, orc, batches, parities):
    """Two instances in one slab: the second fill takes the claim, the first instance runs through its lists. As two
    batches, the two updates run concurrently on side streams and both read the claim words. With mixed parity, the
    unclaimed instance writes the column the claimed one reads, in the same frame."""
    insts = [Instance(0, 4096, alive=4096, seed=1), Instance(4096, 5000, alive=5000, seed=2)]
    lock = filled_c5(tiled_ctx, orc, insts, [(0, 4096, 21, 0.15, 0.6), (4096, 5000, 22, 0.15, 0.6)], batches=batches, parities=parities)
    lock.run([[0, 0]] * 14, what="two instances")
    assert lock.ref.metadata[0].alive_count < 4096 and lock.ref.metadata[1].alive_count < 5000


@pytest.mark.parametrize("tiled_ctx", FORCED_SUB_TILES, ids=lambda n: f"{n}sub", indirect=True)
@pytest.mark.parametrize("test", [test_no_death_frames_then_deaths_then_spawns_into_recycled_slots, test_spawn_shrinks_the_claim,
                                  test_upload_indirect_drops_the_claim], ids=lambda t: t.__name__[len("test_"):])
def test_at_forced_tile_sizes(test, tiled_ctx, orc):
    """The tests above at 2, 3 and 4 sub-tiles per update tile (the slab-size rule picks 1 at their sizes)."""
    test(tiled_ctx, orc)


# ---- claims that end at and around tile edges ------------------------------------------------------------------------
@pytest.mark.parametrize("end", CLAIM_ENDS)
def test_claim_ending_at_tile_edges(tiled_ctx, orc, end):
    ctx = tiled_ctx
    L, cap = claim_end(end, SUB_TILE_C5 * ctx.tile_chunks), 4096
    lock = claim_edge_lockstep(ctx, orc, L, cap)
    lock.run([[s] for s in CLAIM_EDGE_SPAWNS], what=f"claim ending at row {L}")
    assert lock.ref.metadata[0].alive_count == 1000, "every filled particle died, both bursts live"


# ---- claims the device trusts ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("tiled_ctx", [1, 4], ids=["1sub", "4sub"], indirect=True)
def test_claimed_entries_are_neither_loaded_nor_stored(tiled_ctx, orc):
    """While both columns are claimed, their claimed rows are overwritten through the device view with two different
    permutations (in range: a load of them stays in bounds and shows up as a mismatch). The next frame must read rows as
    their own index and skip the stores: both permutations survive, and with the identity put back where they stand, every
    buffer equals the oracle. This guards the update's 64 B per particle-step."""
    ctx = tiled_ctx
    n, cap = 3000, 3500  # no multiple of a sub-tile or tile: the last tile is only partly claimed
    lock = filled_c5(ctx, orc, [Instance(0, cap, alive=n, seed=42)], [(0, cap, 13, 1e9, 1e9)])
    lock.run([[0]], what="before the poison")
    assert_claims_trusted(lock, n, 1)


# ---- parked tiles under a claim ---------------------------------------------------------------------------------------
def test_parked_tiles_at_4_mi_rows(native, orc, monkeypatch):
    """4 Mi rows in one batch of three instances, with the slab-size rule: 4 sub-tiles, about 8 K tiles for 3168 resident
    warps, so tiles are parked behind a warp's next tile and compacted after the instance's last tile has rewritten the
    claim. Only the first instance holds the claim; the second appends to the other column. A frame that keeps the claim, a
    burst that shrinks it, a frame without deaths, then two frames with deaths, each compared row by row."""
    monkeypatch.delenv("HNB_TILE_CHUNKS", raising=False)
    c = native.Context(0)
    try:
        caps = [1_500_000, 1_400_000, 1_294_304]
        insts = [Instance(0, caps[0], alive=1_450_000, seed=1), Instance(caps[0], caps[1], alive=1_400_000, seed=2),
                 Instance(caps[0] + caps[1], caps[2], alive=1_000_000, seed=3)]
        fills = [(caps[0], caps[1], 22, 0.06, 0.5), (caps[0] + caps[1], caps[2], 23, 0.06, 0.5), (0, caps[0], 21, 0.06, 0.5)]
        lock = filled_c5(c, orc, insts, fills, dead_perm_seed=4, parities=[0, 1, 0])
        assert lock.ref.slab_rows == 4 << 20
        lock.run([[0, 0, 0], [40_000, 10_000, 0], [0, 0, 0], [0, 0, 0], [0, 0, 0]], what="4 Mi rows")
        assert c.read_tile_size(0) == 4 * SUB_TILE_C5
        assert lock.ref.metadata[0].alive_count < 1_490_000 and lock.ref.metadata[2].alive_count < 1_000_000, "the last frames had deaths"
    finally:
        c.close()
