"""hnb_slab_repack on the device: every buffer is compared bit for bit with the oracle, with ref_repack applied at the
same point, before and after every frame that follows. Also: the identity claims the repack writes are trusted by the next
update (authored effects reach the 64 B per particle-step path), a 4 Mi-row repack only relabels slots, and refusals leave
the state untouched."""
import numpy as np
import pytest

from bevy_hanabi_b200 import _native as N
from bevy_hanabi_b200 import recipes
from bevy_hanabi_b200 import runtime as R
from tests.effects import EFFECTS, event_assets, ribbon_asset, table_asset, table_props
from tests.helpers import (Instance, Lockstep, RefWorld, assert_claims_trusted, assert_world_equal, is_identity, seeds,  # noqa: F401
                           sparks_world, table_world, tiled_ctx)
from tests.repack_ref import ref_repack

pytestmark = pytest.mark.gpu


def _run(ctx, orc, asset, ref, schedule, repack_at, repack=(0,), *, churned=True, **mode):
    """Frames of `schedule` (spawns per instance), with the instances of `repack` repacked before frame `repack_at`."""
    lock = Lockstep(ctx, orc, ref, asset, seeds=seeds, **mode)
    lock.run(schedule[:repack_at])
    if repack_at is not None:
        for i in repack:
            if churned:
                assert not is_identity(ref, i), f"instance {i}: the alive list must be a permutation before the repack"
            inst = ref.instances[i]
            ctx.slab_repack(lock.gpu.slab, lock.gpu.effect, i, inst.slab_offset, inst.capacity)
            ref_repack(ref, i)
            assert is_identity(ref, i)
        lock.compare("after the repack")
        lock.run(schedule[repack_at:], start=repack_at)
    return lock.gpu


# 24 frames at 300 spawns per frame (lifetimes of 4 to 18 frames): the alive list is a permutation of the slice
CHURN = [[300]] * 24 + [[300]] * 10


@pytest.mark.parametrize("mode", ["default", "sector", "slot", "relaxed"])
def test_churned_sparks(ctx, orc, mode):
    asset, ref = sparks_world([4096])
    _run(ctx, orc, asset, ref, CHURN, 24, sector=mode == "sector", slot=mode == "slot", relaxed=mode == "relaxed")
    assert ref.metadata[0].alive_count > 2000


def test_churned_ribbons(ctx, orc):
    """After the sort the repack makes the sorted order the slot order; the next sort drops the claims again."""
    asset = ribbon_asset(4096)
    fields, size, _ = asset.particle_layout()
    ref = RefWorld(4096, size // 4, [Instance(0, 4096, alive=0, seed=3)], dt=1 / 30)
    ref.set_sort_keys(fields)
    schedule = [[900 if f % 4 == 0 else 23] for f in range(26)]
    _run(ctx, orc, asset, ref, schedule, 16)


@pytest.mark.parametrize("name", list(EFFECTS))
def test_churned_wide_records(ctx, orc, name):
    """48 and 64-byte records (K = 2), 96 and 144 bytes (K = 1), with per-instance properties where the effect has them."""
    ref = table_world(name, [3000])
    schedule = [[500]] * 12 + [[300]] * 8
    _run(ctx, orc, table_asset(name, 3000), ref, schedule, 12, props=table_props(name, 1))


@pytest.mark.parametrize("batches", [None, [[0], [1]]], ids=["one_batch", "two_batches"])
def test_two_instances_one_repacked(ctx, orc, batches):
    """The other instance of the slab keeps every byte; as two batches its update runs concurrently on a side stream."""
    asset, ref = sparks_world([3000, 2500], batches=batches)
    _run(ctx, orc, asset, ref, [[250, 200]] * 24 + [[250, 200]] * 8, 24, repack=(1,))


def test_empty_full_and_off_grid_instances(ctx, orc):
    """One batch: an instance that never spawned, a full one, and one of 1037 rows, all repacked; then more frames."""
    asset, ref = sparks_world([500, 700, 1037])
    schedule = [[0, 700, 900], [0, 0, 0]] + [[40, 0, 100]] * 5
    _run(ctx, orc, asset, ref, schedule, 2, repack=(0, 1, 2), churned=False)
    assert ref.metadata[1].alive_count < 700


# ---- the claims a repack writes are trusted --------------------------------------------------------------------------
@pytest.mark.parametrize("tiled_ctx", [1, 4], ids=["1sub", "4sub"], indirect=True)
def test_repack_claim_engages(tiled_ctx, orc):
    """C5 filled through hnb_init only (dt = 0.25 s, lifetime 1 s): a burst, a second burst, both die off, a burst into
    the recycled slots. After the repack both columns are overwritten through the device view with two different in-range
    permutations; a frame without spawns or deaths must neither load nor store the claimed rows: the poison survives, and
    with the identity put back every buffer equals the oracle."""
    ctx = tiled_ctx
    cap = 3500
    ref = RefWorld(cap, 8, [Instance(0, cap, alive=0, seed=42)], dt=0.25)
    ref.indirect[:, 2] = np.random.default_rng(4).permutation(cap).astype(np.uint32)
    lock = Lockstep(ctx, orc, ref, init=True)
    lock.run([[2000], [600], [0], [0], [0], [1500], [0]], what="init only")
    n = ref.metadata[0].alive_count
    assert n == 1500 and not is_identity(ref, 0)
    ctx.slab_repack(lock.gpu.slab, lock.gpu.effect, 0, 0, cap)
    ref_repack(ref, 0)
    assert_world_equal(ref, lock.gpu.pull(), what="after the repack")
    assert_claims_trusted(lock, n, 7)
    assert ref.metadata[0].alive_count == n, "the frame after the repack has no deaths"


# ---- a large repack only relabels slots -------------------------------------------------------------------------------
def _row_hashes(records):
    h = np.full(len(records), 0xcbf29ce484222325, dtype=np.uint64)
    for w in range(records.shape[1]):
        h = (h ^ records[:, w].astype(np.uint64)) * np.uint64(0x100000001b3)
    return np.sort(h)


def test_relabelling_at_4_mi_rows(native):
    """Two C5 slabs in one context from the same fill, lifetimes of 0.5 to 20.5 frames (5 % of the fill dies per frame,
    6 to 13 % of the living); one of them is repacked after three frames. Over the 10 update-only frames that follow, the
    alive records in list order, the counts and the multiset of records on the dead stack stay identical between the two
    (compared after the frames 2, 3, 7 and 12: a comparison downloads both slabs)."""
    P, dt = 4 << 20, 1 / 60
    c = native.Context(0)
    try:
        effect = c.effect_compile(recipes.c5_lowered())
        slabs = [c.slab_create(P, 32) for _ in range(2)]
        sp, bis = [], []
        for i, s in enumerate(slabs):
            c.slab_fill_c5(s, 0, P, 99, 0.5 * dt, 20.5 * dt)
            md = R.initial_metadata(P, i, 8)
            md.alive_count, md.max_spawn = P, 0
            c.metadata_insert(i, md)
            c.draw_args_insert(i)
            sp.append(R.make_spawner(seed=5, effect_metadata_index=i, draw_indirect_index=i, slab_offset=0))
            bis.append(N.BatchInfo(0, 0, i, 0, i, 1))
        c.upload_spawners(sp)
        c.upload_batches(bis, [0, 0])
        la = [N.BatchLaunch.make(effect, s, i, 0) for i, s in enumerate(slabs)]

        def state(i):
            md = c.read_metadata(i)
            n, w = md.alive_count, md.indirect_write_index
            rec = c.slab_download_aos(slabs[i], 0, P, 32)
            ind = c.slab_download_indirect(slabs[i], 0, P)
            return (n, c.read_draw_args(i).instance_count, rec[ind[:n, w].astype(np.int64)], _row_hashes(rec[ind[n:, 2].astype(np.int64)]))

        for f in range(13):
            c.set_sim_params(dt, f * dt, 2)
            c.simulate(la)
            if f == 2:
                c.slab_repack(slabs[1], effect, 1, 0, P)
            if f in (2, 3, 7, 12):
                a, b = state(0), state(1)
                assert a[0] == b[0] and a[1] == b[1] == a[0], f"frame {f}: alive_count / instance_count"
                np.testing.assert_array_equal(a[2], b[2], err_msg=f"frame {f}: alive records in list order")
                np.testing.assert_array_equal(a[3], b[3], err_msg=f"frame {f}: records on the dead stack")
        assert 0.2 * P < a[0] < 0.5 * P, "about 10 % died per frame"
    finally:
        c.close()


# ---- refusals ---------------------------------------------------------------------------------------------------------
def test_refusals_leave_the_state_untouched(ctx, orc):
    asset, ref = sparks_world([2000])
    gpu = _run(ctx, orc, asset, ref, [[300]] * 6, None, churned=False)
    before = gpu.pull()
    other_stride = ctx.effect_compile(table_asset("vec4x2_64", 2000).generate())
    sector = ctx.effect_compile(asset.generate(sector_planes=True))
    parent = event_assets()[0]
    emitting = ctx.effect_compile(parent.generate(num_event_bindings=1))
    assert parent.particle_layout()[1] == 32, "the emitting effect differs from the slab in its flag only"
    cases = [("rows outside the slab", gpu.effect, 0, 1, 2000), ("rows outside the slab", gpu.effect, 0, 0, 2001),
             ("metadata row out of range", gpu.effect, 1 << 20, 0, 2000), ("stride does not match", other_stride, 0, 0, 2000),
             ("SECTOR_PLANES", sector, 0, 0, 2000), ("GPU spawn events", emitting, 0, 0, 2000)]
    for why, effect, row, first, rows in cases:
        with pytest.raises(N.HanabiError) as e:
            ctx.slab_repack(gpu.slab, effect, row, first, rows)
        assert e.value.code == N.HNB_ERR_INVALID_ARG and why in e.value.message, e.value.message
        got = gpu.pull()
        for k in before:
            np.testing.assert_array_equal(got[k], before[k], err_msg=f"{why}: {k}")
