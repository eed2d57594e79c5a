"""GPU parity of the update pass on slabs filled by hnb_slab_fill_c5, whose alive lists carry an identity claim
(DESIGN.md §3): every buffer is compared bit for bit with the C oracle after every frame while the claim is used,
shrunk by spawns, dropped by deaths, and invalidated by other writers of the index columns. Every scenario also runs at 2,
3 and 4 sub-tiles per update tile: a claim that covers the first sub-tile of a tile but not the rest, and the prefetch of
the next sub-tile under a claim, only exist from 2 up."""
import ctypes as C

import numpy as np
import pytest

from bevy_hanabi_b200 import recipes
from oracle import c_oracle as O
from tests.helpers import (FORCED_SUB_TILES, SUB_TILE_C5, GpuWorld, Instance, RefWorld, assert_world_equal, at_tile_sizes,  # noqa: F401
                           tiled_ctx)

pytestmark = pytest.mark.gpu

ACCEL_DRAG = (C.c_float * 4)(0.0, -9.8, 0.0, 0.5)


def _c5_init():
    """The C5 effect's init: position = velocity = 0, age 0, lifetime 1."""
    ci = O.ConstInit()
    ci.stride_words = 8
    ci.words[7] = int(np.float32(1.0).view(np.uint32))
    return ci


def _filled(ctx, orc, insts, fills, batches=None, dead_perm_seed=None, parities=None):
    """`fills`: (first, count, seed, lifetime_lo, lifetime_hi) ranges filled by hnb_slab_fill_c5 on the device and
    orc_fill_c5 in the oracle, after the world was uploaded; the last fill holds the claim. `parities`: the alive-list
    column each instance's first frame appends to (metadata indirect_write_index)."""
    ref = RefWorld(sum(i.capacity for i in insts), 8, insts, batches=batches)
    for i, parity in enumerate(parities or []):
        ref.metadata[i].indirect_write_index = parity
    if dead_perm_seed is not None:  # a dead stack whose slots are not in row order: spawns then append non-identity entries
        rng = np.random.default_rng(dead_perm_seed)
        for inst in insts:
            rows = slice(inst.slab_offset + inst.alive, inst.slab_offset + inst.capacity)
            ref.indirect[rows, 2] = rng.permutation(ref.indirect[rows, 2])
    gpu = GpuWorld(ctx, ref, recipes.c5_lowered())
    for first, count, seed, lo, hi in fills:
        orc.orc_fill_c5(O.ptr(ref.particles), O.ptr(ref.indirect), first, count, seed, lo, hi)
        ctx.slab_fill_c5(gpu.slab, first, count, seed, lo, hi)
    return ref, gpu


def _frames(orc, ref, gpu, spawns_per_frame, what):
    init = _c5_init()
    for f, spawns in enumerate(spawns_per_frame):
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        ref.set_spawns(spawns)
        ref.oracle_frame(orc, orc.orc_body_update_c5(), ACCEL_DRAG, orc.orc_body_init_const(), C.byref(init))
        gpu.frame()
        assert_world_equal(ref, gpu.pull(), what=f"{what}, frame {f}")


def test_no_death_frames_then_deaths_then_spawns_into_recycled_slots(ctx, orc):
    """Lifetimes >= 0.1 s: five frames without deaths on the claimed lists (the fill covers more rows than are alive), then
    deaths, then bursts into the freed slots."""
    ref, gpu = _filled(ctx, orc, [Instance(0, 8192, alive=6000, seed=42)], [(0, 8192, 77, 0.1, 0.5)])
    _frames(orc, ref, gpu, [[0]] * 5, "no deaths")
    assert ref.metadata[0].alive_count == 6000
    _frames(orc, ref, gpu, [[0]] * 8, "deaths")
    assert ref.metadata[0].alive_count < 6000
    _frames(orc, ref, gpu, [[700], [0], [0], [1500], [0], [0]], "spawns")
    assert ref.metadata[0].particle_counter == 2200


def test_spawn_shrinks_the_claim(ctx, orc):
    """A claim longer than the alive count, then a burst whose dead slots are not in row order: the spawned rows must be
    read through the list."""
    ref, gpu = _filled(ctx, orc, [Instance(0, 8192, alive=5000, seed=3)], [(0, 8192, 5, 1e9, 1e9)], dead_perm_seed=11)
    _frames(orc, ref, gpu, [[0], [0], [900], [0], [0], [300], [0]], "spawn under a claim")


def test_upload_indirect_drops_the_claim(ctx, orc):
    """After the fill, different permutations are uploaded into ping and pong: a stale claim would read the identity and
    skip the stores."""
    n = 6000
    ref, gpu = _filled(ctx, orc, [Instance(0, n, alive=n, seed=8)], [(0, n, 9, 0.05, 0.4)])
    rng = np.random.default_rng(12)
    ref.indirect[:, 0] = rng.permutation(n)
    ref.indirect[:, 1] = rng.permutation(n)
    ctx.slab_upload_indirect(gpu.slab, 0, ref.indirect)
    _frames(orc, ref, gpu, [[0]] * 12, "after upload")
    assert ref.metadata[0].alive_count < n


@at_tile_sizes("batches,parities", [(None, (0, 0)), ([[0], [1]], (0, 0)), (None, (1, 0)), ([[0], [1]], (1, 0))],
               ids=["one_batch", "two_batches", "one_batch_mixed_parity", "two_batches_mixed_parity"])
def test_two_instances_one_claim(tiled_ctx, orc, batches, parities):
    """Two instances in one slab: the second fill takes the claim, the first instance runs through its lists. As two
    batches, the two updates run concurrently on side streams and both read the claim words. With mixed parity, the
    unclaimed instance writes the column the claimed one reads, in the same frame."""
    insts = [Instance(0, 4096, alive=4096, seed=1), Instance(4096, 5000, alive=5000, seed=2)]
    ref, gpu = _filled(tiled_ctx, orc, insts, [(0, 4096, 21, 0.15, 0.6), (4096, 5000, 22, 0.15, 0.6)], batches=batches, parities=parities)
    _frames(orc, ref, gpu, [[0, 0]] * 14, "two instances")
    assert ref.metadata[0].alive_count < 4096 and ref.metadata[1].alive_count < 5000


@pytest.mark.parametrize("tiled_ctx", FORCED_SUB_TILES, ids=lambda n: f"{n}sub", indirect=True)
@pytest.mark.parametrize("test", [test_no_death_frames_then_deaths_then_spawns_into_recycled_slots, test_spawn_shrinks_the_claim,
                                  test_upload_indirect_drops_the_claim], ids=lambda t: t.__name__[len("test_"):])
def test_at_forced_tile_sizes(test, tiled_ctx, orc):
    """The tests above at 2, 3 and 4 sub-tiles per update tile (the slab-size rule picks 1 at their sizes)."""
    test(tiled_ctx, orc)


# ---- claims that end at and around tile edges ------------------------------------------------------------------------
# Where the claim ends, with S = rows per tile: inside or at the end of a warp's 32 rows, of a 128-row sub-tile, of a tile.
CLAIM_ENDS = [0, 1, 31, 32, 33, 127, 128, 129, "S-1", "S", "S+1", "3S+17"]
# Spawns per frame: a frame that keeps the claim, a burst that shrinks it to the alive count L, the frame whose write
# column is claimed only up to L (particle L-1 dies in it), two frames without deaths, four frames in which every other
# filled particle dies, and a burst into the freed slots.
CLAIM_EDGE_SPAWNS = [0, 600, 0, 0, 0, 0, 0, 0, 0, 400, 0]


def claim_end(end, S):
    return {"S-1": S - 1, "S": S, "S+1": S + 1, "3S+17": 3 * S + 17}.get(end, end)


def claim_edge_world(L, cap):
    """One C5 instance of `cap` rows, L of them alive, with both alive lists the identity over the whole capacity (as
    hnb_slab_fill_c5 leaves them, with a claim on all `cap` rows). The dead stack hands out slot L+1 first and slot L
    second, the rest shuffled: after the burst, list rows L and L+1 hold slots L+1 and L. Particle L-1 dies in the frame
    after the burst, so the survivor at rank L is slot L while the write column's claim ends at L and its row L still holds
    L+1; every other filled particle dies in frames 5-8 (dt = 1/60)."""
    rng = np.random.default_rng(L)
    ref = RefWorld(cap, 8, [Instance(0, cap, alive=L, seed=31)])
    dt = float(ref.sim.delta_time)
    ref.indirect[:, 0] = ref.indirect[:, 1] = np.arange(cap, dtype=np.uint32)
    ref.indirect[L:, 2] = np.concatenate([[L + 1, L], rng.permutation(np.arange(L + 2, cap))]).astype(np.uint32)
    p = np.zeros((cap, 8), dtype=np.float32)
    p[:, 0:3] = rng.uniform(-1, 1, (cap, 3))
    p[:, 4:7] = rng.uniform(-1, 1, (cap, 3))
    p[:, 7] = rng.uniform(5.5 * dt, 9.0 * dt, cap)
    if L:
        p[L - 1, 7] = 2.5 * dt
    ref.particles[:] = p.view(np.uint32)
    return ref


@pytest.mark.parametrize("end", CLAIM_ENDS)
def test_claim_ending_at_tile_edges(tiled_ctx, orc, end):
    ctx = tiled_ctx
    L, cap = claim_end(end, SUB_TILE_C5 * ctx.tile_chunks), 4096
    ref = claim_edge_world(L, cap)
    gpu = GpuWorld(ctx, ref, recipes.c5_lowered())
    ctx.slab_fill_c5(gpu.slab, 0, cap, 1, 1e9, 1e9)  # identity lists with a claim on all rows ...
    ctx.slab_upload_aos(gpu.slab, 0, ref.particles)  # ... under the scenario's records (writing records keeps the claim)
    _frames(orc, ref, gpu, [[s] for s in CLAIM_EDGE_SPAWNS], f"claim ending at row {L}")
    assert ref.metadata[0].alive_count == 1000, "every filled particle died, both bursts live"


# ---- claims the device trusts ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("tiled_ctx", [1, 4], ids=["1sub", "4sub"], indirect=True)
def test_claimed_entries_are_neither_loaded_nor_stored(tiled_ctx, orc):
    """While both columns are claimed, their claimed rows are overwritten through the device view with two different
    permutations (in range: a load of them stays in bounds and shows up as a mismatch). The next frame must read rows as
    their own index and skip the stores: both permutations survive, and with the identity put back where they stand, every
    buffer equals the oracle. This guards the update's 64 B per particle-step."""
    ctx = tiled_ctx
    n, cap = 3000, 3500  # no multiple of a sub-tile or tile: the last tile is only partly claimed
    ref, gpu = _filled(ctx, orc, [Instance(0, cap, alive=n, seed=42)], [(0, cap, 13, 1e9, 1e9)])
    _frames(orc, ref, gpu, [[0]], "before the poison")
    rng = np.random.default_rng(77)
    poison = [rng.permutation(n).astype(np.uint32) for _ in range(2)]
    view = ctx.slab_device_view(gpu.slab)
    ctx.sync()
    for col, ptr in enumerate((view.ping, view.pong)):
        ctx.device_upload(ptr, poison[col])  # not supported for users: done here to observe the claim
    read = ref.metadata[0].indirect_write_index  # the column the next frame reads
    ref.sim.time = ref.sim.delta_time
    ref.set_spawns([0])
    ref.oracle_frame(orc, orc.orc_body_update_c5(), ACCEL_DRAG, orc.orc_body_init_const(), C.byref(_c5_init()))
    gpu.frame()
    got = gpu.pull()
    np.testing.assert_array_equal(got["indirect"][:n, 1 - read], poison[1 - read], err_msg="claimed stores were not skipped")
    np.testing.assert_array_equal(got["indirect"][:n, read], poison[read], err_msg="the read column was written")
    got["indirect"][:n, :2] = ref.indirect[:n, :2]
    assert_world_equal(ref, got, what="claimed entries were loaded")


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
        ref, gpu = _filled(c, orc, insts, fills, dead_perm_seed=4, parities=[0, 1, 0])
        assert ref.slab_rows == 4 << 20
        _frames(orc, ref, gpu, [[0, 0, 0], [40_000, 10_000, 0], [0, 0, 0], [0, 0, 0], [0, 0, 0]], "4 Mi rows")
        assert c.read_tile_size(0) == 4 * SUB_TILE_C5
        assert ref.metadata[0].alive_count < 1_490_000 and ref.metadata[2].alive_count < 1_000_000, "the last frames had deaths"
    finally:
        c.close()
