"""GPU parity of the update pass on config C5 (Accel + LinearDrag + Euler, age/lifetime kill) against
the C oracle: every buffer bit-exact after every frame — particle words, alive lists (ping/pong), dead
stack, metadata counters, draw-indirect instance counts, prefix sums, dispatch args.

All arithmetic on this path is add/mul/max/compare, compiled without FMA contraction on both sides, so
the tolerance is zero (north_star: "bit-exact for dead-list indices and indirect counts, fp32 attributes
within 1e-5 relative" — met with 0).
"""
import ctypes as C

import numpy as np
import pytest

from tests.helpers import FORCED_SUB_TILES, SUB_TILE_C5, GpuWorld, Instance, RefWorld, assert_world_equal, at_tile_sizes, tiled_ctx  # noqa: F401

pytestmark = pytest.mark.gpu

ACCEL_DRAG = (C.c_float * 4)(0.0, -9.8, 0.0, 0.5)


def _fill(ref: RefWorld, rng, life_lo, life_hi):
    for inst in ref.instances:
        n = inst.alive
        rows = slice(inst.slab_offset, inst.slab_offset + n)
        p = np.zeros((n, 8), dtype=np.float32)
        p[:, 0:3] = rng.uniform(-1, 1, (n, 3))
        p[:, 3] = 0.0
        p[:, 4:7] = rng.uniform(-1, 1, (n, 3))
        p[:, 7] = rng.uniform(life_lo, life_hi, n)
        ref.particles[rows] = p.view(np.uint32)


def _run(ctx, orc, ref, steps, check_every=1):
    from bevy_hanabi_b200 import recipes
    gpu = GpuWorld(ctx, ref, recipes.c5_lowered())
    body = orc.orc_body_update_c5()
    for step in range(steps):
        ref.sim.time = np.float32(step) * ref.sim.delta_time
        ref.oracle_frame(orc, body, ACCEL_DRAG)
        gpu.frame()
        if step % check_every == 0 or step == steps - 1:
            assert_world_equal(ref, gpu.pull(), what=f"step {step}")
    return gpu


def test_single_instance_with_deaths(ctx, orc):
    rng = np.random.default_rng(42)
    ref = RefWorld(8192, 8, [Instance(0, 8192, alive=5000, seed=42)])
    _fill(ref, rng, 0.05, 0.6)
    _run(ctx, orc, ref, 40)
    assert ref.metadata[0].alive_count == 0  # everything died, dead stack fully rebuilt


# Alive counts at the edges of a 128-row sub-tile and of larger powers of two; with forced sub-tiles also at the edges of
# the tile S = 128 x sub-tiles.
_TILE_EDGES = {"S-1": lambda S: S - 1, "S": lambda S: S, "S+1": lambda S: S + 1, "2S+1": lambda S: 2 * S + 1}


@at_tile_sizes("alive", [1, 63, 64, 127, 128, 129, 1023, 1024, 1025, 2048, 4097], forced_values=list(_TILE_EDGES))
def test_tile_boundaries(tiled_ctx, orc, alive):
    ctx = tiled_ctx
    if isinstance(alive, str):
        alive = _TILE_EDGES[alive](SUB_TILE_C5 * ctx.tile_chunks)
    rng = np.random.default_rng(alive)
    ref = RefWorld(8192, 8, [Instance(0, 8192, alive=alive, seed=7)])
    _fill(ref, rng, 0.02, 0.2)
    _run(ctx, orc, ref, 14)


def test_many_instances_one_batch(ctx, orc):
    rng = np.random.default_rng(3)
    caps = [3000, 1, 1024, 5000, 64, 2500, 7]
    alive = [3000, 1, 1024, 4321, 0, 2049, 3]
    insts, off = [], 0
    for c, a in zip(caps, alive):
        insts.append(Instance(off, c, alive=a, seed=1000 + off))
        off += c
    ref = RefWorld(off, 8, insts)
    _fill(ref, rng, 0.03, 0.4)
    _run(ctx, orc, ref, 26)


def test_two_batches(ctx, orc):
    rng = np.random.default_rng(5)
    insts = [Instance(0, 2000, alive=1500, seed=1), Instance(2000, 2000, alive=2000, seed=2), Instance(4000, 3000, alive=2999, seed=3)]
    ref = RefWorld(7000, 8, insts, batches=[[0, 1], [2]])
    _fill(ref, rng, 0.03, 0.3)
    _run(ctx, orc, ref, 20)


def test_no_deaths_identity_list(ctx, orc):
    """The benchmark's steady state: nothing dies, the alive list stays the identity."""
    rng = np.random.default_rng(9)
    ref = RefWorld(20000, 8, [Instance(0, 20000, alive=20000, seed=42)])
    _fill(ref, rng, 1e9, 1e9)
    gpu = _run(ctx, orc, ref, 5)
    got = gpu.pull()
    assert got["draw"][1] == 20000
    np.testing.assert_array_equal(got["indirect"][:, 0], np.arange(20000))
    np.testing.assert_array_equal(got["indirect"][:, 1], np.arange(20000))


@pytest.mark.parametrize("tiled_ctx", FORCED_SUB_TILES, ids=lambda n: f"{n}sub", indirect=True)
@pytest.mark.parametrize("test", [test_single_instance_with_deaths, test_many_instances_one_batch, test_two_batches, test_no_deaths_identity_list],
                         ids=lambda t: t.__name__[len("test_"):])
def test_at_forced_tile_sizes(test, tiled_ctx, orc):
    """The tests above at 2, 3 and 4 sub-tiles per update tile (the slab-size rule picks 1 at their sizes): the prefetch of
    the next sub-tile's alive-list entries and the stash and ballot slots of sub-tiles after the first."""
    test(tiled_ctx, orc)
