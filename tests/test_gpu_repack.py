"""hnb_slab_repack on the device: every buffer is compared bit for bit with the oracle, with ref_repack applied at the
same point, before and after every frame that follows. Also: the identity claims the repack writes are trusted by the next
update (authored effects reach the 64 B per particle-step path), a 4 Mi-row repack only relabels slots, and refusals leave
the state untouched."""
import ctypes as C

import numpy as np
import pytest

from bevy_hanabi_b200 import _native as N
from bevy_hanabi_b200 import recipes
from bevy_hanabi_b200 import runtime as R
from oracle.hanabi_oracle import EffectOracle, pcg_hash
from tests.helpers import GpuWorld, Instance, RefWorld, assert_world_equal, tiled_ctx  # noqa: F401
from tests.repack_ref import ref_repack
from tests.test_gpu_effects import _assert_relaxed_equal
from tests.test_gpu_events import _assets as _event_assets
from tests.test_gpu_identity_claim import ACCEL_DRAG, _c5_init, _frames
from tests.test_gpu_ribbons import _ribbon_asset
from tests.test_gpu_scene import _drifting_sparks
from tests.test_gpu_tile_shapes import EFFECTS, _asset, _world

pytestmark = pytest.mark.gpu


def _seeds(n, f):
    return [int(s) for s in pcg_hash(np.arange(n, dtype=np.uint32) + np.uint32(100 * f + 7))]


def _is_identity(ref, i):
    md, base = ref.metadata[i], ref.instances[i].slab_offset
    lst = ref.indirect[base:base + md.alive_count, md.indirect_write_index]
    return bool((lst == np.arange(len(lst))).all())


def _run(ctx, orc, asset, ref, schedule, repack_at, repack=(0,), *, props=None, sector=False, slot=False, relaxed=False,
         churned=True):
    """Frames of `schedule` (spawns per instance), with the instances of `repack` repacked before frame `repack_at`."""
    blobs = None
    if props is not None:
        blobs = [asset.serialize_properties(props(i)) for i in range(len(ref.instances))]
        for i in range(len(ref.instances)):
            ref.metadata[i].properties_array_index = i
    ref.slot_order = slot
    eo = EffectOracle(asset, {i: props(i) for i in range(len(ref.instances))} if props else None)
    gpu = GpuWorld(ctx, ref, asset.generate(sector_planes=sector, slot_order=slot, relaxed_order=relaxed), property_blobs=blobs,
                   sector_planes=sector)

    def compare(what):
        got = gpu.pull()
        if relaxed:
            _assert_relaxed_equal(ref, got, None, 0.0)
            ref.indirect[:, :] = got["indirect"]  # the next frame reads the lists in the order the device wrote them
        else:
            assert_world_equal(ref, got, what=what)

    for f, spawns in enumerate(schedule):
        if f == repack_at:
            for i in repack:
                if churned:
                    assert not _is_identity(ref, i), f"instance {i}: the alive list must be a permutation before the repack"
                inst = ref.instances[i]
                ctx.slab_repack(gpu.slab, gpu.effect, i, inst.slab_offset, inst.capacity)
                ref_repack(ref, i)
                assert _is_identity(ref, i)
            compare("after the repack")
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        ref.set_spawns(spawns, _seeds(len(spawns), f))
        eo.frame(ref, orc)
        gpu.frame()
        compare(f"frame {f}")
    if slot:
        assert ctx.read_debug(False)[15] == 0, "alive bitmap and counters disagree"
    return ref, gpu


def _sparks_world(caps, dt=0.05, batches=None, seed=1):
    asset = _drifting_sparks(max(caps))
    fields, size, _ = asset.particle_layout()
    insts, off = [], 0
    for i, c in enumerate(caps):
        insts.append(Instance(off, c, alive=0, seed=11 + 7 * i))
        off += c
    ref = RefWorld(off, size // 4, insts, batches=batches, dt=dt)
    rng = np.random.default_rng(seed)
    for inst in insts:
        rows = slice(inst.slab_offset, inst.slab_offset + inst.capacity)
        ref.indirect[rows, 2] = rng.permutation(ref.indirect[rows, 2])
    return asset, ref


# 24 frames at 300 spawns per frame (lifetimes of 4 to 18 frames): the alive list is a permutation of the slice
CHURN = [[300]] * 24 + [[300]] * 10


@pytest.mark.parametrize("mode", ["default", "sector", "slot", "relaxed"])
def test_churned_sparks(ctx, orc, mode):
    asset, ref = _sparks_world([4096])
    _run(ctx, orc, asset, ref, CHURN, 24, sector=mode == "sector", slot=mode == "slot", relaxed=mode == "relaxed")
    assert ref.metadata[0].alive_count > 2000


def test_churned_ribbons(ctx, orc):
    """After the sort the repack makes the sorted order the slot order; the next sort drops the claims again."""
    asset = _ribbon_asset(4096)
    fields, size, _ = asset.particle_layout()
    ref = RefWorld(4096, size // 4, [Instance(0, 4096, alive=0, seed=3)], dt=1 / 30)
    ref.set_sort_keys(fields)
    schedule = [[900 if f % 4 == 0 else 23] for f in range(26)]
    _run(ctx, orc, asset, ref, schedule, 16)


@pytest.mark.parametrize("name", list(EFFECTS))
def test_churned_wide_records(ctx, orc, name):
    """48 and 64-byte records (K = 2), 96 and 144 bytes (K = 1), with per-instance properties where the effect has them."""
    ref = _world(name, [3000])
    schedule = [[500]] * 12 + [[300]] * 8
    _run(ctx, orc, _asset(name, 3000), ref, schedule, 12, props=EFFECTS[name][3])


@pytest.mark.parametrize("batches", [None, [[0], [1]]], ids=["one_batch", "two_batches"])
def test_two_instances_one_repacked(ctx, orc, batches):
    """The other instance of the slab keeps every byte; as two batches its update runs concurrently on a side stream."""
    asset, ref = _sparks_world([3000, 2500], batches=batches)
    _run(ctx, orc, asset, ref, [[250, 200]] * 24 + [[250, 200]] * 8, 24, repack=(1,))


def test_empty_full_and_off_grid_instances(ctx, orc):
    """One batch: an instance that never spawned, a full one, and one of 1037 rows, all repacked; then more frames."""
    asset, ref = _sparks_world([500, 700, 1037])
    schedule = [[0, 700, 900], [0, 0, 0]] + [[40, 0, 100]] * 5
    ref, gpu = _run(ctx, orc, asset, ref, schedule, 2, repack=(0, 1, 2), churned=False)
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
    gpu = GpuWorld(ctx, ref, recipes.c5_lowered())
    _frames(orc, ref, gpu, [[2000], [600], [0], [0], [0], [1500], [0]], "init only")
    n = ref.metadata[0].alive_count
    assert n == 1500 and not _is_identity(ref, 0)
    ctx.slab_repack(gpu.slab, gpu.effect, 0, 0, cap)
    ref_repack(ref, 0)
    assert_world_equal(ref, gpu.pull(), what="after the repack")
    rng = np.random.default_rng(77)
    poison = [rng.permutation(n).astype(np.uint32) for _ in range(2)]
    view = ctx.slab_device_view(gpu.slab)
    ctx.sync()
    for col, ptr in enumerate((view.ping, view.pong)):
        ctx.device_upload(ptr, poison[col])  # not supported for users: done here to observe the claim
    read = ref.metadata[0].indirect_write_index  # the column the next frame reads
    ref.sim.time = np.float32(7) * ref.sim.delta_time
    ref.set_spawns([0])
    ref.oracle_frame(orc, orc.orc_body_update_c5(), ACCEL_DRAG, orc.orc_body_init_const(), C.byref(_c5_init()))
    gpu.frame()
    assert ref.metadata[0].alive_count == n, "the frame after the repack has no deaths"
    got = gpu.pull()
    np.testing.assert_array_equal(got["indirect"][:n, 1 - read], poison[1 - read], err_msg="claimed stores were not skipped")
    np.testing.assert_array_equal(got["indirect"][:n, read], poison[read], err_msg="the read column was written")
    got["indirect"][:n, :2] = ref.indirect[:n, :2]
    assert_world_equal(ref, got, what="claimed entries were loaded")


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
    asset, ref = _sparks_world([2000])
    ref, gpu = _run(ctx, orc, asset, ref, [[300]] * 6, None, churned=False)
    before = gpu.pull()
    other_stride = ctx.effect_compile(_asset("vec4x2_64", 2000).generate())
    sector = ctx.effect_compile(asset.generate(sector_planes=True))
    parent = _event_assets()[0]
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
