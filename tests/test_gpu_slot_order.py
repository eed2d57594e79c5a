"""HNB_EFFECT_SLOT_ORDER on the device: the update pass walks each instance's SLOTS in ascending order, guided by the
slab's alive bitmap, instead of walking the alive list. That is the reference's update (vfx_update.wgsl:106-167) for an alive
list that happens to be sorted by particle index — an order the reference's own scheduling-dependent atomics may produce —
so the oracle is the same oracle, reading each list through a sorted copy. Every buffer is compared bit for bit after every
frame, exactly like the default (alive-list order) tests."""
import numpy as np
import pytest

from bevy_hanabi_b200 import _native as N, recipes
from tests.effects import drifting_sparks, fill_c5
from tests.helpers import GpuWorld, Instance, Lockstep, RefWorld, at_tile_sizes, tiled_ctx  # noqa: F401

pytestmark = pytest.mark.gpu


@at_tile_sizes("capacity,alive", [(8192, 5000), (8192, 8192), (8192, 1), (70, 70), (33, 0), (400_000, 380_000), (2_200_000, 2_000_001)])
def test_c5_with_deaths(tiled_ctx, orc, capacity, alive):
    """The sub-tile counts tile_chunks picks (1 up to 8192 rows, more at 400 K and 2.2 M), then 2, 3 and 4 forced at every size
    (the bitmap words a warp owns: chunks x K of them), capacities that are no multiple of 32 or of the tile."""
    rng = np.random.default_rng(capacity + alive)
    ref = RefWorld(capacity, 8, [Instance(0, capacity, alive=alive, seed=42)])
    fill_c5(ref, rng, 0.02, 0.3)
    Lockstep(tiled_ctx, orc, ref, slot=True).run(8 if capacity > 100_000 else 24)
    assert ref.metadata[0].alive_count < max(alive, 1)


def test_many_instances_one_batch(ctx, orc):
    rng = np.random.default_rng(3)
    caps = [3008, 32, 1024, 5024, 64, 2528, 7]
    alive = [3000, 1, 1024, 4321, 0, 2049, 3]
    insts, off = [], 0
    for c, a in zip(caps, alive):
        insts.append(Instance(off, c, alive=a, seed=1000 + off))
        off += (c + 31) // 32 * 32
    ref = RefWorld(off, 8, insts)
    fill_c5(ref, rng, 0.03, 0.4)
    Lockstep(ctx, orc, ref, slot=True).run(26)


def test_instances_must_start_on_word_boundaries(ctx):
    ref = RefWorld(200, 8, [Instance(0, 100, alive=10, seed=1), Instance(100, 100, alive=10, seed=2)])
    gpu = GpuWorld(ctx, ref, recipes.c5_lowered())      # default order: fine
    gpu.frame()
    ctx.sync()
    fx = ctx.effect_compile(recipes.c5_lowered(slot_order=True))
    with pytest.raises(N.HanabiError) as e:
        ctx.simulate([N.BatchLaunch.make(fx, gpu.slab, 0, 0)])
    assert e.value.code == N.HNB_ERR_LAYOUT and "multiple of 32" in e.value.message


def test_flag_combinations_are_refused():
    for other in (N.EFFECT_RELAXED_ORDER, N.EFFECT_SECTOR_PLANES):
        fx = recipes.c5_lowered(slot_order=True)
        fx.flags |= other
        with pytest.raises(N.HanabiError):
            fx.generate_source()


@pytest.mark.parametrize("caps", [[4096], [3008, 64, 9024, 33]])
def test_spawning_into_recycled_slots(ctx, orc, caps):
    """Churn: constant spawning into whatever slots died. In alive-list order the list turns into a permutation of the slab;
    here every frame's list comes out sorted, new particles included, and the dead stack is pushed in slot order."""
    asset = drifting_sparks(max(caps), name="sparks_slot_order", lifetime=(0.05, 0.4))
    _, size, _ = asset.particle_layout()
    insts, off = [], 0
    for i, c in enumerate(caps):
        insts.append(Instance(off, c, alive=0, seed=77 + i))
        off += (c + 31) // 32 * 32
    ref = RefWorld(off, size // 4, insts, dt=1.0 / 30.0)
    lock = Lockstep(ctx, orc, ref, asset, slot=True, seeds=lambda n, f: [1000 + 17 * f + i for i in range(n)])
    for f in range(40):
        got = lock.run([[c // 6 if f % 2 == 0 else c // 11 for c in caps]], start=f)
        for i, inst in enumerate(insts):
            md = ref.metadata[i]
            lst = got["indirect"][inst.slab_offset:inst.slab_offset + md.alive_count, md.indirect_write_index]
            assert np.all(np.diff(lst.astype(np.int64)) > 0), "the written alive list is in ascending slot order"
    assert sum(ref.metadata[i].particle_counter for i in range(len(caps))) > 3 * sum(caps), "slots were recycled several times"


def test_same_population_as_alive_list_order(ctx, orc, native):
    """Slot order changes the ORDER of the lists, never who lives: for an effect whose per-particle results do not depend on
    the order (no per-thread counters), both modes hold the same particle records and the same alive SET after every frame
    once spawning stops (while spawning, the dead stack order decides which slot a new particle gets)."""
    rng = np.random.default_rng(11)
    worlds = []
    ctx2 = native.Context(0)  # one context per world: both use metadata / draw / spawner row 0 of their context
    for slot, c in ((False, ctx), (True, ctx2)):
        ref = RefWorld(6016, 8, [Instance(0, 6016, alive=6000, seed=5)])
        fill_c5(ref, np.random.default_rng(11), 0.02, 0.5)
        worlds.append((ref, GpuWorld(c, ref, recipes.c5_lowered(slot_order=slot))))
    # scramble the alive list of both worlds identically (a permutation, as after long churn)
    perm = rng.permutation(6000).astype(np.uint32)
    for ref, gpu in worlds:
        ref.indirect[:6000, 0] = perm
        ref.indirect[:6000, 1] = perm
        gpu.ctx.slab_upload_indirect(gpu.slab, 0, ref.indirect)
    for step in range(12):
        states = []
        for ref, gpu in worlds:
            gpu.frame()
            got = gpu.pull()
            n = int(got["metadata"][0][1])
            states.append((got["particles"], n, np.sort(got["indirect"][:n, got["metadata"][0][4]])))
        np.testing.assert_array_equal(states[0][0], states[1][0])
        assert states[0][1] == states[1][1]
        np.testing.assert_array_equal(states[0][2], states[1][2])
    ctx2.close()
