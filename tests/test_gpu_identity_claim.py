"""GPU parity of the update pass on slabs filled by hnb_slab_fill_c5, whose alive lists carry an identity claim
(DESIGN.md §3): every buffer is compared bit for bit with the C oracle after every frame while the claim is used,
shrunk by spawns, dropped by deaths, and invalidated by other writers of the index columns."""
import ctypes as C

import numpy as np
import pytest

from oracle import c_oracle as O
from tests.helpers import GpuWorld, Instance, RefWorld, assert_world_equal

pytestmark = pytest.mark.gpu

ACCEL_DRAG = (C.c_float * 4)(0.0, -9.8, 0.0, 0.5)


def _c5_init():
    """The C5 effect's init: position = velocity = 0, age 0, lifetime 1."""
    ci = O.ConstInit()
    ci.stride_words = 8
    ci.words[7] = int(np.float32(1.0).view(np.uint32))
    return ci


def _filled(ctx, orc, insts, fills, batches=None, dead_perm_seed=None):
    """`fills`: (first, count, seed, lifetime_lo, lifetime_hi) ranges filled by hnb_slab_fill_c5 on the device and
    orc_fill_c5 in the oracle, after the world was uploaded."""
    from bevy_hanabi_b200 import recipes
    ref = RefWorld(sum(i.capacity for i in insts), 8, insts, batches=batches)
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


@pytest.mark.parametrize("batches", [None, [[0], [1]]], ids=["one_batch", "two_batches"])
def test_two_instances_one_claim(ctx, orc, batches):
    """Two instances in one slab: the second fill takes the claim, the first instance runs through its lists. As two
    batches, the two updates run concurrently on side streams and both read the claim words."""
    insts = [Instance(0, 4096, alive=4096, seed=1), Instance(4096, 5000, alive=5000, seed=2)]
    ref, gpu = _filled(ctx, orc, insts, [(0, 4096, 21, 0.15, 0.6), (4096, 5000, 22, 0.15, 0.6)], batches=batches)
    _frames(orc, ref, gpu, [[0, 0]] * 14, "two instances")
    assert ref.metadata[0].alive_count < 4096 and ref.metadata[1].alive_count < 5000
