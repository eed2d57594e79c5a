"""hnb_batch_depth_order on the device: after every frame of a lock-step run, the order of every batch equals the numpy
restatement (tests/depth_order_ref.py) applied to the oracle world, bit for bit, and the world itself still equals the
oracle (which never sees the calls). Worlds: filled C5 whose claim goes as particles die, the 48-byte C2 with bursts into
recycled slots, the force field, a local-space effect, 1024 instances in one batch, sector planes, slot order, a plan that
splits position, planes and order in pinned host memory. Also: every refusal enqueues nothing, the call changes no byte
of the slab or the tables, and a 64 Mi-row instance against torch's stable argsort of independently computed keys."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from bevy_hanabi_b200 import _native as N
from bevy_hanabi_b200 import graph as G
from bevy_hanabi_b200 import recipes
from bevy_hanabi_b200 import runtime as R
from tests.depth_order_ref import ref_depth_order
from tests.effects import event_assets, firework_trails, force_field, ribbon_asset, table_asset
from tests.helpers import Instance, Lockstep, RefWorld, filled_c5, is_identity, seeds, sparks_world

pytestmark = pytest.mark.gpu
A = G.Attribute
SENTINEL = np.uint32(0xA5A5A5A5)
LAUNCHES = 13


def position_word(asset):
    return next(f.offset for f in asset.particle_layout()[0] if f.name == "position") // 4


def camera_planes(rng, count):
    """Unit forward axes and offsets, as a camera gives them: (f, -f.p)."""
    f = rng.standard_normal((count, 3))
    f /= np.linalg.norm(f, axis=1, keepdims=True)
    p = rng.standard_normal((count, 3)) * 2.0
    return np.concatenate([f, -(f * p).sum(axis=1, keepdims=True)], axis=1).astype(np.float32)


class Orders:
    """A device order buffer of the slab's rows and a device plane buffer, reused for every call of a test."""

    def __init__(self, ctx, rows, instances):
        self.ctx, self.rows, self.instances = ctx, rows, instances
        self.order = ctx.device_alloc(4 * rows)
        self.planes = ctx.device_alloc(16 * instances)

    def of(self, launch, planes):
        """The order buffer after one call over a buffer of sentinels."""
        ctx = self.ctx
        ctx.device_upload(self.order, np.full(self.rows, SENTINEL, dtype=np.uint32))
        ctx.device_upload(self.planes, np.ascontiguousarray(planes, dtype=np.float32).reshape(-1).view(np.uint32))
        before = ctx.launch_count
        ctx.batch_depth_order(launch, self.planes, self.instances, self.order, self.rows)
        assert ctx.launch_count == before + LAUNCHES, "a fixed number of launches per call"
        return ctx.device_download(self.order, 4 * self.rows).view(np.uint32)

    def free(self):
        self.ctx.device_free(self.order)
        self.ctx.device_free(self.planes)


@pytest.fixture()
def orders(ctx):
    made = []

    def make(rows, instances):
        made.append(Orders(ctx, rows, instances))
        return made[-1]
    yield make
    for o in made:
        o.free()


def check(lock, buf, pos_word, what, rng):
    """Every batch of the lock-step world against the restatement on the oracle world."""
    for b, launch in enumerate(lock.gpu.launches()):
        count = lock.ref.batch_infos[b].prefix_sum_count
        planes = camera_planes(rng, max(count, 1))
        got = buf.of(launch, planes)
        want = ref_depth_order(lock.ref, b, pos_word, planes, np.full(buf.rows, SENTINEL, dtype=np.uint32))
        np.testing.assert_array_equal(got, want, err_msg=f"{what}, batch {b}: depth order")


def run(lock, buf, pos_word, schedule, what, start=0):
    rng = np.random.default_rng(len(what))
    for k, spawns in enumerate(schedule):
        lock.step(start + k, spawns)
        lock.compare(f"{what} frame {start + k}")
        check(lock, buf, pos_word, f"{what} frame {start + k}", rng)


@pytest.mark.parametrize("module", ["hand_lowered", "authored"])
def test_c5_filled_then_dying(ctx, orc, orders, module):
    """Filled C5 under a claim over every row, then deaths and bursts into recycled slots. The authored C5 runs in its
    own column plan, which the calls leave as the frames made it."""
    n = 6000
    effect = ctx.effect_compile(recipes.c5_asset(n).generate()) if module == "authored" else None
    lock = filled_c5(ctx, orc, [Instance(0, n, alive=n, seed=8)], [(0, n, 9, 0.05, 0.4)], effect=effect)
    run(lock, orders(n, 1), 0, [[0]] * 14 + [[900], [0], [0], [1500]] + [[0]] * 8, module)
    assert 0 < lock.ref.metadata[0].alive_count < n and not is_identity(lock.ref, 0)
    assert ctx.slab_device_view(lock.gpu.slab).num_planes == (4 if module == "authored" else 2)


def test_c2_trails_with_bursts_into_recycled_slots(ctx, orc, orders):
    asset = firework_trails(4096)
    ref = RefWorld(4096, 12, [Instance(0, 4096, alive=0)], dt=1.0 / 20.0)
    lock = Lockstep(ctx, orc, ref, asset, seeds=seeds)
    run(lock, orders(4096, 1), position_word(asset), [[1200 if f % 10 == 0 else 40] for f in range(30)], "C2")
    assert ref.metadata[0].particle_counter > 4096 and not is_identity(ref, 0)


def test_force_field(ctx, orc, orders):
    asset = force_field(8192, aabb_half=(0.8, 0.6, 0.8), kill_center=(0.6, -0.2, 0.), kill_r2=0.0025)
    ref = RefWorld(8192, asset.particle_layout()[1] // 4, [Instance(0, 8192, alive=0, seed=77)])
    props = [{"attraction_accel": 18.0, "repulsor_position": G.Vec3(0.25, 0.5, 0.1)}]
    lock = Lockstep(ctx, orc, ref, asset, rtol=1e-5, props=props)
    run(lock, orders(8192, 1), position_word(asset), [[5000 if f == 0 else (30 if f % 5 == 0 else 0)] for f in range(15)], "force field")


def test_local_space_effect(ctx, orc, orders):
    """Simulation space LOCAL under a rotated, scaled and translated emitter: depths of the stored (local) positions."""
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
    run(lock, orders(3000, 1), position_word(asset), [[2000 if f == 0 else 100] for f in range(6)], "local space")


def test_1024_instances_in_one_batch(ctx, orc, orders):
    """C4's topology: one batch of 1024 instances, uneven alive counts, every ninth instance empty, one call."""
    n_inst, cap = 1024, 192
    asset, ref = sparks_world([cap] * n_inst)
    lock = Lockstep(ctx, orc, ref, asset, seeds=seeds)
    buf = orders(ref.slab_rows, n_inst)
    rng = np.random.default_rng(6)
    for f in range(4):
        lock.step(f, [0 if i % 9 == 0 else int(x) for i, x in enumerate(rng.integers(0, 70, n_inst))])
        check(lock, buf, position_word(asset), f"1024 instances frame {f}", rng)
    lock.compare("1024 instances")


@pytest.mark.parametrize("mode", ["sector", "slot", "two_batches"])
def test_churned_sparks(ctx, orc, orders, mode):
    """Sector planes (position in one half of a 32-byte column), slot order, and two batches of two instances each, the
    larger instances more than one 4096-row tile."""
    caps = [9000, 1000, 4097, 512] if mode == "two_batches" else [9000]
    batches = [[0, 1], [2, 3]] if mode == "two_batches" else None
    asset, ref = sparks_world(caps, batches=batches)
    lock = Lockstep(ctx, orc, ref, asset, seeds=seeds, sector=mode == "sector", slot=mode == "slot")
    sched = [[900 if j % 2 == 0 else 35 for j in range(len(caps))]] * 14 + [[0] * len(caps)] * 3
    run(lock, orders(ref.slab_rows, 2), position_word(asset), sched, mode)
    assert not is_identity(ref, 0)


def split_position_asset(capacity):
    """position's fourth word is a size no update writes: the effect's plan cuts position into [0, 8) and [8, 12)."""
    w = G.ExprWriter()
    return (G.EffectAsset(capacity, w.module, name="split_position")
            .init(G.SetAttributeModifier(A.POSITION, w.rand(G.VEC3) - w.lit(0.5)))
            .init(G.SetAttributeModifier(A.VELOCITY, (w.rand(G.VEC3) - w.lit(0.5)) * w.lit(3.)))
            .init(G.SetAttributeModifier(A.SIZE, w.rand(G.FLOAT)))
            .update(G.KillAabbModifier(w.lit(G.Vec3(0., 0., 0.)), w.lit(G.Vec3(1.5, 1.0, 1.25)))))


def test_plan_that_splits_position(ctx, orc, orders):
    asset = split_position_asset(9000)
    assert asset.generate().column_plan()[:3] == [(0, 8), (8, 4), (12, 4)]
    ref = RefWorld(9500, 8, [Instance(0, 500, alive=0, seed=5), Instance(500, 9000, alive=0, seed=6)], dt=0.05)
    lock = Lockstep(ctx, orc, ref, asset, seeds=seeds)
    run(lock, orders(9500, 2), 0, [[60, 1200]] * 15, "split position")
    view = ctx.slab_device_view(lock.gpu.slab)
    assert [view.plane_width[p] for p in range(3)] == [8, 4, 4]


def test_planes_and_order_in_pinned_host_memory(ctx, orc):
    asset, ref = sparks_world([5000, 700])
    lock = Lockstep(ctx, orc, ref, asset, seeds=seeds)
    lock.run([[900, 90]] * 6, what="pinned")
    rows = ref.slab_rows
    planes = camera_planes(np.random.default_rng(1), 2)
    h_planes, h_order = N.lib.hnb_host_alloc(32), N.lib.hnb_host_alloc(4 * rows)
    assert h_planes and h_order
    try:
        C.memmove(h_planes, planes.tobytes(), 32)
        C.memset(h_order, 0xA5, 4 * rows)
        ctx.batch_depth_order(lock.gpu.launches()[0], h_planes, 2, h_order, rows)
        ctx.sync()
        got = np.frombuffer(C.string_at(h_order, 4 * rows), dtype=np.uint32)
        want = ref_depth_order(ref, 0, position_word(asset), planes, np.full(rows, SENTINEL, dtype=np.uint32))
        np.testing.assert_array_equal(got, want, err_msg="pinned host planes and order")
    finally:
        N.lib.hnb_host_free(h_planes)
        N.lib.hnb_host_free(h_order)


def _state(ctx, lock):
    ctx.sync()
    rows = lock.ref.slab_rows
    return (ctx.slab_checksum(lock.gpu.slab, 0, rows), ctx.slab_checksum_indirect(lock.gpu.slab, 0, rows), lock.gpu.pull())


def test_nothing_changes_and_refusals_enqueue_nothing(ctx, orc, orders):
    asset, ref = sparks_world([5000, 600])
    lock = Lockstep(ctx, orc, ref, asset, seeds=seeds)
    lock.run([[900, 80]] * 10, what="churn")
    launch = lock.gpu.launches()[0]
    rows = ref.slab_rows
    buf = orders(rows, 3)
    sum0, ind0, pull0 = _state(ctx, lock)
    check(lock, buf, position_word(asset), "before the refusals", np.random.default_rng(2))
    sum1, ind1, pull1 = _state(ctx, lock)
    assert (sum0, ind0) == (sum1, ind1), "slab or list checksums changed"
    for k in pull0:
        np.testing.assert_array_equal(pull0[k], pull1[k], err_msg=f"the depth-order pass modified {k}")

    other_stride = ctx.effect_compile(table_asset("vec4x2_64", 2000).generate())
    sector = ctx.effect_compile(asset.generate(sector_planes=True))
    no_position = ctx.effect_compile(R.LoweredEffect(name="no_position", particle_stride=32, attrs=[
        R.AttrField("f32x4_0", N.VEC4, 0), R.AttrField("f32x4_1", N.VEC4, 16)]))
    ribbon = ctx.effect_compile(ribbon_asset(2000).generate())  # refused before its stride is compared with the slab's
    emitting = ctx.effect_compile(event_assets()[0].generate(num_event_bindings=1))
    make = N.BatchLaunch.make
    e, s = lock.gpu.effect, lock.gpu.slab
    P, O = buf.planes, buf.order
    cases = [("invalid effect", make(1 << 20, s), P, 3, O, rows), ("invalid slab", make(e, 1 << 20), P, 3, O, rows),
             ("batch_info_index", make(e, s, 7), P, 3, O, rows), ("stride does not match", make(other_stride, s), P, 3, O, rows),
             ("SECTOR_PLANES", make(sector, s), P, 3, O, rows), ("no `position` attribute", make(no_position, s), P, 3, O, rows),
             ("ribbon", make(ribbon, s), P, 3, O, rows),
             ("d_planes is NULL", launch, 0, 3, O, rows), ("d_planes is NULL or not 16-byte aligned", launch, P + 8, 3, O, rows),
             ("plane_rows", launch, P, 1, O, rows), ("d_order is NULL", launch, P, 3, 0, rows), ("order_rows", launch, P, 3, O, rows - 1)]
    ctx.device_upload(O, np.full(rows, SENTINEL, dtype=np.uint32))
    for why, bl, planes, prow, order, orow in cases:
        before = ctx.launch_count
        with pytest.raises(N.HanabiError) as err:
            ctx.batch_depth_order(bl, planes, prow, order, orow)
        assert err.value.code == N.HNB_ERR_INVALID_ARG and why in err.value.message, (why, err.value.message)
        assert ctx.launch_count == before, f"{why}: something was enqueued"
    assert (ctx.device_download(O, 4 * rows) == SENTINEL).all()
    with pytest.raises(N.HanabiError):
        N.check(N.lib.hnb_batch_depth_order(ctx._h, None, P, 3, O, rows))
    # an emitting effect of the slab's stride is accepted
    planes = camera_planes(np.random.default_rng(3), 3)
    ctx.device_upload(P, planes.reshape(-1).view(np.uint32))
    ctx.batch_depth_order(make(emitting, s), P, 3, O, rows)
    ctx.sync()
    want = ref_depth_order(ref, 0, 0, planes, np.full(rows, SENTINEL, dtype=np.uint32))
    np.testing.assert_array_equal(ctx.device_download(O, 4 * rows).view(np.uint32), want, "through an emitting effect's descriptor")
    # ... and the world still steps in lock-step afterwards
    lock.run([[100, 100]] * 3, start=10, what="after the calls")


class _DeviceArray:
    """A device column as torch sees it through __cuda_array_interface__."""

    def __init__(self, ptr, shape):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": "<f4", "data": (ptr, False), "version": 2}


def test_c5_64_mi_rows_against_torch_argsort(ctx):
    """The benchmarked size: 64 Mi rows of hnb_slab_fill_c5 under its claim (the list is the identity), against torch's
    stable argsort of keys computed from the slab's own position column."""
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
    plane = np.array([0.48, -0.6, 0.64, 0.25], dtype=np.float32)
    order = torch.empty(P, dtype=torch.int32, device="cuda")
    planes = torch.as_tensor(plane, device="cuda")
    try:
        ctx.batch_depth_order(launch, planes.data_ptr(), 1, order.data_ptr(), P)
        ctx.sync()
        view = ctx.slab_device_view(slab)
        assert view.plane_width[0] == 16
        col = torch.as_tensor(_DeviceArray(view.planes[0], (P, 4)), device="cuda")
        a, b, c, d = (float(v) for v in plane)
        depth = ((col[:, 0] * a + col[:, 1] * b) + col[:, 2] * c) + d  # one rounding per elementwise op
        bits = depth.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
        key = torch.where(bits >= 0x80000000, bits ^ 0xFFFFFFFF, bits ^ 0x80000000)
        key = torch.where(torch.isnan(depth), torch.full_like(key, 0xFFFFFFFF), 0xFFFFFFFF - key)
        want = torch.argsort(key, stable=True).to(torch.int32)
        assert ctx.read_metadata(0).alive_count == P
        assert torch.equal(order, want)
        assert not torch.equal(want[:1024], torch.arange(1024, device="cuda", dtype=torch.int32))
    finally:
        ctx.slab_destroy(slab)
