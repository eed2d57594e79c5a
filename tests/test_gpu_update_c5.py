"""GPU parity of the update pass on config C5 (Accel + LinearDrag + Euler, age/lifetime kill) against
the C oracle: every buffer bit-exact after every frame — particle words, alive lists (ping/pong), dead
stack, metadata counters, draw-indirect instance counts, prefix sums, dispatch args.

All arithmetic on this path is add/mul/max/compare, compiled without FMA contraction on both sides, so
the tolerance is zero (north_star: "bit-exact for dead-list indices and indirect counts, fp32 attributes
within 1e-5 relative" — met with 0).
"""
import numpy as np
import pytest

from tests.effects import fill_c5
from tests.helpers import FORCED_SUB_TILES, SUB_TILE_C5, Instance, Lockstep, RefWorld, at_tile_sizes, tiled_ctx  # noqa: F401

pytestmark = pytest.mark.gpu

def test_single_instance_with_deaths(ctx, orc):
    rng = np.random.default_rng(42)
    ref = RefWorld(8192, 8, [Instance(0, 8192, alive=5000, seed=42)])
    fill_c5(ref, rng, 0.05, 0.6)
    Lockstep(ctx, orc, ref).run(40)
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
    fill_c5(ref, rng, 0.02, 0.2)
    Lockstep(ctx, orc, ref).run(14)


def test_many_instances_one_batch(ctx, orc):
    rng = np.random.default_rng(3)
    caps = [3000, 1, 1024, 5000, 64, 2500, 7]
    alive = [3000, 1, 1024, 4321, 0, 2049, 3]
    insts, off = [], 0
    for c, a in zip(caps, alive):
        insts.append(Instance(off, c, alive=a, seed=1000 + off))
        off += c
    ref = RefWorld(off, 8, insts)
    fill_c5(ref, rng, 0.03, 0.4)
    Lockstep(ctx, orc, ref).run(26)


def test_two_batches(ctx, orc):
    rng = np.random.default_rng(5)
    insts = [Instance(0, 2000, alive=1500, seed=1), Instance(2000, 2000, alive=2000, seed=2), Instance(4000, 3000, alive=2999, seed=3)]
    ref = RefWorld(7000, 8, insts, batches=[[0, 1], [2]])
    fill_c5(ref, rng, 0.03, 0.3)
    Lockstep(ctx, orc, ref).run(20)


def test_no_deaths_identity_list(ctx, orc):
    """The benchmark's steady state: nothing dies, the alive list stays the identity."""
    rng = np.random.default_rng(9)
    ref = RefWorld(20000, 8, [Instance(0, 20000, alive=20000, seed=42)])
    fill_c5(ref, rng, 1e9, 1e9)
    got = Lockstep(ctx, orc, ref).run(5)
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
