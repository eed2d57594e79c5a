"""hnb_batch_bounds on the device: after every frame of a lock-step run, the records of every batch equal the numpy
restatement (tests/bounds_ref.py) applied to the oracle world, bit for bit. Worlds: filled C5 whose claim goes as particles
die, the 48-byte C2 with bursts into recycled slots, the force field under its kill box, a local-space effect, 1024
instances in one batch, sector planes, slot order, a plan that splits position, output into pinned host memory. Also:
every refusal enqueues nothing, the call changes no byte of the slab or the tables, and a 64 Mi-row instance against an
independent reduction of the same column."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from bevy_hanabi_b200 import _native as N
from bevy_hanabi_b200 import graph as G
from bevy_hanabi_b200 import recipes
from bevy_hanabi_b200 import runtime as R
from tests.bounds_ref import BOUNDS_DTYPE, assert_bounds_equal, ref_bounds
from tests.effects import event_assets, firework_trails, force_field, table_asset
from tests.helpers import Instance, Lockstep, RefWorld, filled_c5, is_identity, seeds, sparks_world

pytestmark = pytest.mark.gpu
A = G.Attribute
SENTINEL = np.uint32(0xA5A5A5A5)


def position_word(asset):
    return next(f.offset for f in asset.particle_layout()[0] if f.name == "position") // 4


class Boxes:
    """A device buffer of bounds records, reused for every call of a test."""

    def __init__(self, ctx, rows):
        self.ctx, self.rows = ctx, rows
        self.ptr = ctx.device_alloc(32 * rows)

    def of(self, launch, count):
        """The `count` records of one call; the rest of the buffer keeps a sentinel."""
        ctx = self.ctx
        ctx.device_upload(self.ptr, np.full(8 * self.rows, SENTINEL, dtype=np.uint32))
        before = ctx.launch_count
        ctx.batch_bounds(launch, self.ptr, self.rows)
        assert ctx.launch_count == before + 2, "two launches per call"
        words = ctx.device_download(self.ptr, 32 * self.rows)
        assert (words[8 * count:] == SENTINEL).all(), "records past the batch's instances were written"
        return words[:8 * count].view(BOUNDS_DTYPE)

    def free(self):
        self.ctx.device_free(self.ptr)


@pytest.fixture()
def boxes(ctx):
    made = []

    def make(rows):
        made.append(Boxes(ctx, rows))
        return made[-1]
    yield make
    for b in made:
        b.free()


def check(lock, box, pos_word, what):
    """Every batch of the lock-step world against the restatement on the oracle world. Returns the records per batch."""
    out = []
    for b, launch in enumerate(lock.gpu.launches()):
        want = ref_bounds(lock.ref, b, pos_word)
        got = box.of(launch, len(want))
        assert_bounds_equal(got, want, f"{what}, batch {b}")
        out.append(got)
    return out


def run(lock, box, pos_word, schedule, what, start=0):
    """Frames of `schedule` (per-instance spawns), each compared with the oracle (which, for effects held to a tolerance,
    also restarts the device from the oracle's records), then the bounds."""
    for k, spawns in enumerate(schedule):
        lock.step(start + k, spawns)
        lock.compare(f"{what} frame {start + k}")
        last = check(lock, box, pos_word, f"{what} frame {start + k}")
    return last


@pytest.mark.parametrize("module", ["hand_lowered", "authored"])
def test_c5_filled_then_dying(ctx, orc, boxes, module):
    """hnb_slab_fill_c5 leaves a claim over every row: the first frames read no list. Lifetimes of 3 to 24 frames: the
    particles die, the claim shrinks and goes, bursts land in recycled slots. The authored C5 runs in its own column plan."""
    n = 6000
    effect = ctx.effect_compile(recipes.c5_asset(n).generate()) if module == "authored" else None
    lock = filled_c5(ctx, orc, [Instance(0, n, alive=n, seed=8)], [(0, n, 9, 0.05, 0.4)], effect=effect)
    box = boxes(4)
    run(lock, box, 0, [[0]] * 14 + [[900], [0], [0], [1500]] + [[0]] * 12, module)
    md = lock.ref.metadata[0]
    assert 0 < md.alive_count < n and not is_identity(lock.ref, 0)
    plan = ctx.slab_device_view(lock.gpu.slab)
    assert plan.num_planes == (4 if module == "authored" else 2)


def test_c2_trails_with_bursts_into_recycled_slots(ctx, orc, boxes):
    asset = firework_trails(4096)
    ref = RefWorld(4096, 12, [Instance(0, 4096, alive=0)], dt=1.0 / 20.0)
    lock = Lockstep(ctx, orc, ref, asset, seeds=seeds)
    run(lock, boxes(1), position_word(asset), [[1200 if f % 10 == 0 else 40] for f in range(40)], "C2")
    assert ref.metadata[0].particle_counter > 4096 and not is_identity(ref, 0)


def test_force_field_stays_inside_its_kill_box(ctx, orc, boxes):
    half = (0.8, 0.6, 0.8)
    asset = force_field(8192, aabb_half=half, kill_center=(0.6, -0.2, 0.), kill_r2=0.0025)
    ref = RefWorld(8192, asset.particle_layout()[1] // 4, [Instance(0, 8192, alive=0, seed=77)])
    props = [{"attraction_accel": 18.0, "repulsor_position": G.Vec3(0.25, 0.5, 0.1)}]
    lock = Lockstep(ctx, orc, ref, asset, rtol=1e-5, props=props)
    box = boxes(1)
    for f in range(25):
        lock.step(f, [5000 if f == 0 else (30 if f % 5 == 0 else 0)])
        lock.compare(f"force field frame {f}")
        got = check(lock, box, position_word(asset), f"force field frame {f}")[0]
        # the kill test sees the position before the frame's integration step: a survivor is outside by at most one step
        reach = np.array(half) + 0.25
        assert (np.abs(got["min"][0]) <= reach).all() and (np.abs(got["max"][0]) <= reach).all(), "a survivor far outside the kill box"
    assert 0 < ref.metadata[0].alive_count < 5000


def test_local_space_effect_gives_a_local_box(ctx, orc, boxes):
    """Simulation space LOCAL under a rotated, scaled and translated emitter: the box is the stored (local) one."""
    w = G.ExprWriter()
    axis, center = w.lit(G.Vec3(0., 0., 1.)), w.lit(G.Vec3(0.5, -0.25, 0.))
    asset = (G.EffectAsset(3000, w.module, name="shapes", simulation_space=G.LOCAL)
             .init(G.SetPositionCircleModifier(center, axis, w.lit(2.), G.VOLUME))
             .init(G.SetVelocityTangentModifier(center, axis, w.lit(1.5)))
             .init(G.SetAttributeModifier(A.AGE, w.lit(0.)))
             .init(G.SetAttributeModifier(A.LIFETIME, w.lit(5.)))
             .update(G.RadialAccelModifier(center, w.lit(-0.5))))
    ref = RefWorld(3000, asset.particle_layout()[1] // 4, [Instance(0, 3000, alive=0, seed=31337)])
    c, s = np.float32(np.cos(0.7)), np.float32(np.sin(0.7))
    for k, v in enumerate([1.5 * c, -1.5 * s, 0., 40.,   1.5 * s, 1.5 * c, 0., -10.,   0., 0., 0.5, 20.]):
        ref.spawners[0].transform[k] = v
    lock = Lockstep(ctx, orc, ref, asset, rtol=1e-5)
    got = run(lock, boxes(1), position_word(asset), [[2000 if f == 0 else 100] for f in range(6)], "local space")[0]
    assert (got["max"][0] < 5.0).all() and (got["min"][0] > -5.0).all(), "the emitter's translation is not in a local box"


def test_1024_instances_in_one_batch(ctx, orc, boxes):
    """C4's topology: one batch of 1024 instances, uneven alive counts, every ninth instance empty, one call."""
    n_inst, cap = 1024, 192
    asset, ref = sparks_world([cap] * n_inst)
    lock = Lockstep(ctx, orc, ref, asset, seeds=seeds)
    box = boxes(n_inst)
    rng = np.random.default_rng(6)
    for f in range(4):
        lock.step(f, [0 if i % 9 == 0 else int(x) for i, x in enumerate(rng.integers(0, 70, n_inst))])
        got = check(lock, box, position_word(asset), f"1024 instances frame {f}")[0]
    lock.compare("1024 instances")
    assert (got["count"][::9] == 0).all() and np.isinf(got["min"][::9]).all() and len(set(got["count"].tolist())) > 50


@pytest.mark.parametrize("mode", ["sector", "slot", "two_batches"])
def test_churned_sparks(ctx, orc, boxes, mode):
    """Sector planes (position in one half of a 32-byte column), slot order, and two batches of two instances each."""
    caps = [4096, 1000, 2048, 512] if mode == "two_batches" else [4096]
    batches = [[0, 1], [2, 3]] if mode == "two_batches" else None
    asset, ref = sparks_world(caps, batches=batches)
    lock = Lockstep(ctx, orc, ref, asset, seeds=seeds, sector=mode == "sector", slot=mode == "slot")
    sched = [[300 if j % 2 == 0 else 35 for j in range(len(caps))]] * 16 + [[0] * len(caps)] * 4
    run(lock, boxes(2), position_word(asset), sched, mode)
    assert not is_identity(ref, 0)


def split_position_asset(capacity):
    """position's fourth word is a size no update writes: the effect's plan cuts position into [0, 8) and [8, 12)."""
    w = G.ExprWriter()
    return (G.EffectAsset(capacity, w.module, name="split_position")
            .init(G.SetAttributeModifier(A.POSITION, w.rand(G.VEC3) - w.lit(0.5)))
            .init(G.SetAttributeModifier(A.VELOCITY, (w.rand(G.VEC3) - w.lit(0.5)) * w.lit(3.)))
            .init(G.SetAttributeModifier(A.SIZE, w.rand(G.FLOAT)))
            .update(G.KillAabbModifier(w.lit(G.Vec3(0., 0., 0.)), w.lit(G.Vec3(1.5, 1.0, 1.25)))))


def test_plan_that_splits_position(ctx, orc, boxes):
    asset = split_position_asset(3000)
    assert asset.generate().column_plan()[:3] == [(0, 8), (8, 4), (12, 4)]
    ref = RefWorld(3500, 8, [Instance(0, 500, alive=0, seed=5), Instance(500, 3000, alive=0, seed=6)], dt=0.05)
    lock = Lockstep(ctx, orc, ref, asset, seeds=seeds)
    run(lock, boxes(2), 0, [[60, 400]] * 20, "split position")
    view = ctx.slab_device_view(lock.gpu.slab)
    assert [view.plane_width[p] for p in range(3)] == [8, 4, 4]
    assert 0 < ref.metadata[1].alive_count < ref.metadata[1].particle_counter


def test_output_into_pinned_host_memory(ctx, orc):
    asset, ref = sparks_world([2048, 700])
    lock = Lockstep(ctx, orc, ref, asset, seeds=seeds)
    lock.run([[200, 90]] * 6, what="pinned")
    host = N.lib.hnb_host_alloc(64)
    assert host
    try:
        C.memset(host, 0xA5, 64)
        ctx.batch_bounds(lock.gpu.launches()[0], host, 2)
        ctx.sync()
        got = np.frombuffer(C.string_at(host, 64), dtype=BOUNDS_DTYPE)
        assert_bounds_equal(got, ref_bounds(ref, 0, position_word(asset)), "pinned host output")
    finally:
        N.lib.hnb_host_free(host)


def _state(ctx, lock):
    ctx.sync()
    rows = lock.ref.slab_rows
    return (ctx.slab_checksum(lock.gpu.slab, 0, rows), ctx.slab_checksum_indirect(lock.gpu.slab, 0, rows), lock.gpu.pull())


def test_nothing_changes_and_refusals_enqueue_nothing(ctx, orc, boxes):
    asset, ref = sparks_world([2000, 600])
    lock = Lockstep(ctx, orc, ref, asset, seeds=seeds)
    lock.run([[300, 80]] * 10, what="churn")
    launch = lock.gpu.launches()[0]
    box = boxes(3)
    sum0, ind0, pull0 = _state(ctx, lock)
    check(lock, box, position_word(asset), "before the refusals")
    sum1, ind1, pull1 = _state(ctx, lock)
    assert (sum0, ind0) == (sum1, ind1), "slab or list checksums changed"
    for k in pull0:
        np.testing.assert_array_equal(pull0[k], pull1[k], err_msg=f"the bounds pass modified {k}")

    other_stride = ctx.effect_compile(table_asset("vec4x2_64", 2000).generate())
    sector = ctx.effect_compile(asset.generate(sector_planes=True))
    no_position = ctx.effect_compile(R.LoweredEffect(name="no_position", particle_stride=32, attrs=[
        R.AttrField("f32x4_0", N.VEC4, 0), R.AttrField("f32x4_1", N.VEC4, 16)]))
    emitting = ctx.effect_compile(event_assets()[0].generate(num_event_bindings=1))
    make = N.BatchLaunch.make
    e, s = lock.gpu.effect, lock.gpu.slab
    cases = [("invalid effect", make(1 << 20, s), box.ptr, 3), ("invalid slab", make(e, 1 << 20), box.ptr, 3),
             ("batch_info_index", make(e, s, 7), box.ptr, 3), ("stride does not match", make(other_stride, s), box.ptr, 3),
             ("SECTOR_PLANES", make(sector, s), box.ptr, 3), ("no `position` attribute", make(no_position, s), box.ptr, 3),
             ("NULL or not 16-byte aligned", launch, 0, 3), ("NULL or not 16-byte aligned", launch, box.ptr + 8, 3),
             ("out_rows", launch, box.ptr, 1)]
    ctx.device_upload(box.ptr, np.full(24, SENTINEL, dtype=np.uint32))
    for why, bl, ptr, rows in cases:
        before = ctx.launch_count
        with pytest.raises(N.HanabiError) as err:
            ctx.batch_bounds(bl, ptr, rows)
        assert err.value.code == N.HNB_ERR_INVALID_ARG and why in err.value.message, (why, err.value.message)
        assert ctx.launch_count == before, f"{why}: something was enqueued"
    assert (ctx.device_download(box.ptr, 96) == SENTINEL).all()
    with pytest.raises(N.HanabiError):
        N.check(N.lib.hnb_batch_bounds(ctx._h, None, box.ptr, 3))
    # an emitting effect of the slab's stride is accepted: nothing moves, so pending events are not a concern
    assert event_assets()[0].particle_layout()[1] == 32
    ctx.batch_bounds(make(emitting, s), box.ptr, 3)
    assert_bounds_equal(ctx.download_bounds(box.ptr, 2), ref_bounds(ref, 0, 0), "through an emitting effect's descriptor")
    # ... and the world still steps in lock-step afterwards
    lock.run([[100, 100]] * 3, start=10, what="after the calls")


class _DeviceArray:
    """A device column as torch sees it through __cuda_array_interface__."""

    def __init__(self, ptr, shape):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": "<f4", "data": (ptr, False), "version": 2}


def test_c5_64_mi_rows_against_a_torch_reduction(ctx):
    """The benchmarked size: 64 Mi rows of hnb_slab_fill_c5 under its claim, against torch's min / max over the slab's
    own position column."""
    import torch
    P = 64 << 20
    effect = ctx.effect_compile(recipes.c5_lowered())
    slab = ctx.slab_create(P, 32)
    ctx.slab_fill_c5(slab, 0, P, 99, 0.5, 2.0)
    md = R.initial_metadata(P, 0, 8)
    md.alive_count, md.max_spawn = P, 0
    ctx.metadata_insert(0, md)
    ctx.draw_args_insert(0)
    ctx.upload_spawners([R.make_spawner(seed=42)])
    ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, 1)], [0])
    ctx.set_sim_params(1.0 / 60.0, 0.0, 1)
    launch = N.BatchLaunch.make(effect, slab, 0, 0)
    ctx.simulate([launch])
    out = ctx.device_alloc(32)
    try:
        ctx.batch_bounds(launch, out, 1)
        got = ctx.download_bounds(out, 1)[0]
        view = ctx.slab_device_view(slab)
        assert view.plane_width[0] == 16
        col = torch.as_tensor(_DeviceArray(view.planes[0], (P, 4)), device="cuda")
        want_min, want_max = col.amin(dim=0).cpu().numpy(), col.amax(dim=0).cpu().numpy()
        assert got["count"] == P and ctx.read_metadata(0).alive_count == P
        np.testing.assert_array_equal(got["min"].view(np.uint32), want_min[:3].view(np.uint32))
        np.testing.assert_array_equal(got["max"].view(np.uint32), want_max[:3].view(np.uint32))
        assert (got["min"] < -0.999).all() and (got["max"] > 0.999).all()
    finally:
        ctx.device_free(out)
        ctx.slab_destroy(slab)
