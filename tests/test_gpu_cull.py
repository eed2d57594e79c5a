"""hnb_batch_cull on the device: after every frame of a lock-step run, the visible entries and draw arguments of every
batch equal the numpy restatement (tests/cull_ref.py) applied to the oracle world, bit for bit, and the world itself
still equals the oracle (which never sees the calls). Worlds: those of the depth-order tests (filled C5 whose claim goes
as particles die, the 48-byte C2 with bursts into recycled slots, the force field, a local-space effect, 1024 instances
in one batch, sector planes, slot order, a plan that splits position). Also: culling hnb_batch_depth_order's output,
pinned host buffers, every refusal enqueuing nothing, the launch count, no byte of the slab or the tables changing, and
a 64 Mi-row instance against an independent torch evaluation."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from bevy_hanabi_b200 import _native as N
from bevy_hanabi_b200 import graph as G
from bevy_hanabi_b200 import recipes
from bevy_hanabi_b200 import runtime as R
from tests.cull_ref import frustum_planes, ref_cull
from tests.depth_order_ref import ref_depth_order
from tests.effects import event_assets, firework_trails, force_field, ribbon_asset, table_asset
from tests.helpers import Instance, Lockstep, RefWorld, filled_c5, is_identity, seeds, sparks_world

pytestmark = pytest.mark.gpu
A = G.Attribute
SENTINEL = np.uint32(0xA5A5A5A5)
LAUNCHES = 4


def position_word(asset):
    return next(f.offset for f in asset.particle_layout()[0] if f.name == "position") // 4


def camera_frusta(rng, count, distance=3.0, fov=None):
    """Perspective cameras (z in [0, 1] clip space) at `distance` from the origin looking near it, with a field of view of
    `fov` degrees or a random one of 30-70: each sees part of a cloud around the origin. (count, 6, 4) float32, radius
    0.01 added."""
    out = []
    for _ in range(max(count, 1)):
        eye = rng.standard_normal(3)
        eye *= distance / np.linalg.norm(eye)
        f = rng.standard_normal(3) * 0.4 - eye
        f /= np.linalg.norm(f)
        s = np.cross(f, [0.0, 1.0, 0.0])
        s /= np.linalg.norm(s)
        u = np.cross(s, f)
        view = np.array([[*s, -s @ eye], [*u, -u @ eye], [*-f, f @ eye], [0, 0, 0, 1]])
        t = 1.0 / np.tan(np.radians(rng.uniform(30, 70) if fov is None else fov) / 2)
        near, far = 0.1, 2 * distance
        proj = np.array([[t, 0, 0, 0], [0, t, 0, 0], [0, 0, far / (near - far), near * far / (near - far)], [0, 0, -1, 0]])
        out.append(frustum_planes(proj @ view, 0.01))
    return np.stack(out)


class Culls:
    """Device buffers for one hnb_batch_cull call (frusta, visible entries, draw args), reused for every call of a test."""

    def __init__(self, ctx, rows, instances):
        self.ctx, self.rows, self.instances = ctx, rows, instances
        self.visible = ctx.device_alloc(4 * rows)
        self.frusta = ctx.device_alloc(96 * instances)
        self.args = ctx.device_alloc(20 * instances)

    def of(self, launch, frusta, src=0, count=None):
        """(visible buffer, args rows) after one call over buffers of sentinels."""
        ctx = self.ctx
        count = self.instances if count is None else count
        ctx.device_upload(self.visible, np.full(self.rows, SENTINEL, dtype=np.uint32))
        ctx.device_upload(self.args, np.full(5 * self.instances, SENTINEL, dtype=np.uint32))
        ctx.device_upload(self.frusta, np.ascontiguousarray(frusta, dtype=np.float32).reshape(-1).view(np.uint32))
        before = ctx.launch_count
        ctx.batch_cull(launch, self.frusta, self.instances, src, self.rows if src else 0, self.visible, self.rows, self.args, self.instances)
        assert ctx.launch_count == before + LAUNCHES, "a fixed number of launches per call"
        args = ctx.device_download(self.args, 20 * self.instances).view(np.uint32).reshape(-1, 5)
        assert (args[count:] == SENTINEL).all(), "args rows past the batch's instances were written"
        return ctx.device_download(self.visible, 4 * self.rows).view(np.uint32), args[:count]

    def free(self):
        for p in (self.visible, self.frusta, self.args):
            self.ctx.device_free(p)


@pytest.fixture()
def culls(ctx):
    made = []

    def make(rows, instances):
        made.append(Culls(ctx, rows, instances))
        return made[-1]
    yield make
    for c in made:
        c.free()


def check(lock, buf, pos_word, what, rng):
    """Every batch of the lock-step world against the restatement on the oracle world."""
    seen = 0
    for b, launch in enumerate(lock.gpu.launches()):
        count = lock.ref.batch_infos[b].prefix_sum_count
        frusta = camera_frusta(rng, count)
        got, args = buf.of(launch, frusta, count=count)
        want, want_args = ref_cull(lock.ref, b, pos_word, frusta, np.full(buf.rows, SENTINEL, dtype=np.uint32), lock.ref.draw)
        np.testing.assert_array_equal(got, want, err_msg=f"{what}, batch {b}: visible entries")
        np.testing.assert_array_equal(args, want_args, err_msg=f"{what}, batch {b}: draw args")
        seen += int(args[:, 1].sum())
    return seen


def run(lock, buf, pos_word, schedule, what, start=0):
    rng = np.random.default_rng(len(what))
    seen = 0
    for k, spawns in enumerate(schedule):
        lock.step(start + k, spawns)
        lock.compare(f"{what} frame {start + k}")
        seen += check(lock, buf, pos_word, f"{what} frame {start + k}", rng)
    assert seen > 0, f"{what}: no particle was ever visible"


@pytest.mark.parametrize("module", ["hand_lowered", "authored"])
def test_c5_filled_then_dying(ctx, orc, culls, module):
    """Filled C5 under a claim over every row, then deaths and bursts into recycled slots. The authored C5 runs in its
    own column plan, which the calls leave as the frames made it."""
    n = 6000
    effect = ctx.effect_compile(recipes.c5_asset(n).generate()) if module == "authored" else None
    lock = filled_c5(ctx, orc, [Instance(0, n, alive=n, seed=8)], [(0, n, 9, 0.05, 0.4)], effect=effect)
    run(lock, culls(n, 1), 0, [[0]] * 14 + [[900], [0], [0], [1500]] + [[0]] * 8, module)
    assert 0 < lock.ref.metadata[0].alive_count < n and not is_identity(lock.ref, 0)
    assert ctx.slab_device_view(lock.gpu.slab).num_planes == (4 if module == "authored" else 2)


def test_c2_trails_with_bursts_into_recycled_slots(ctx, orc, culls):
    asset = firework_trails(4096)
    ref = RefWorld(4096, 12, [Instance(0, 4096, alive=0)], dt=1.0 / 20.0)
    lock = Lockstep(ctx, orc, ref, asset, seeds=seeds)
    run(lock, culls(4096, 1), position_word(asset), [[1200 if f % 10 == 0 else 40] for f in range(30)], "C2")
    assert ref.metadata[0].particle_counter > 4096 and not is_identity(ref, 0)


def test_force_field(ctx, orc, culls):
    asset = force_field(8192, aabb_half=(0.8, 0.6, 0.8), kill_center=(0.6, -0.2, 0.), kill_r2=0.0025)
    ref = RefWorld(8192, asset.particle_layout()[1] // 4, [Instance(0, 8192, alive=0, seed=77)])
    props = [{"attraction_accel": 18.0, "repulsor_position": G.Vec3(0.25, 0.5, 0.1)}]
    lock = Lockstep(ctx, orc, ref, asset, rtol=1e-5, props=props)
    run(lock, culls(8192, 1), position_word(asset), [[5000 if f == 0 else (30 if f % 5 == 0 else 0)] for f in range(15)], "force field")


def test_local_space_effect(ctx, orc, culls):
    """Simulation space LOCAL under a rotated, scaled and translated emitter: the stored (local) positions are tested."""
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
    run(lock, culls(3000, 1), position_word(asset), [[2000 if f == 0 else 100] for f in range(6)], "local space")


def test_1024_instances_in_one_batch(ctx, orc, culls):
    """C4's topology: one batch of 1024 instances, uneven alive counts, every ninth instance empty, one call."""
    n_inst, cap = 1024, 192
    asset, ref = sparks_world([cap] * n_inst)
    lock = Lockstep(ctx, orc, ref, asset, seeds=seeds)
    buf = culls(ref.slab_rows, n_inst)
    rng = np.random.default_rng(6)
    seen = 0
    for f in range(4):
        lock.step(f, [0 if i % 9 == 0 else int(x) for i, x in enumerate(rng.integers(0, 70, n_inst))])
        seen += check(lock, buf, position_word(asset), f"1024 instances frame {f}", rng)
    lock.compare("1024 instances")
    assert seen > 0


@pytest.mark.parametrize("mode", ["sector", "slot", "two_batches"])
def test_churned_sparks(ctx, orc, culls, mode):
    """Sector planes (position in one half of a 32-byte column), slot order, and two batches of two instances each, the
    larger instances more than one 4096-row tile."""
    caps = [9000, 1000, 4097, 512] if mode == "two_batches" else [9000]
    batches = [[0, 1], [2, 3]] if mode == "two_batches" else None
    asset, ref = sparks_world(caps, batches=batches)
    lock = Lockstep(ctx, orc, ref, asset, seeds=seeds, sector=mode == "sector", slot=mode == "slot")
    sched = [[900 if j % 2 == 0 else 35 for j in range(len(caps))]] * 14 + [[0] * len(caps)] * 3
    run(lock, culls(ref.slab_rows, 2 if mode == "two_batches" else 1), position_word(asset), sched, mode)
    assert not is_identity(ref, 0)


def split_position_asset(capacity):
    """position's fourth word is a size no update writes: the effect's plan cuts position into [0, 8) and [8, 12)."""
    w = G.ExprWriter()
    return (G.EffectAsset(capacity, w.module, name="split_position")
            .init(G.SetAttributeModifier(A.POSITION, w.rand(G.VEC3) - w.lit(0.5)))
            .init(G.SetAttributeModifier(A.VELOCITY, (w.rand(G.VEC3) - w.lit(0.5)) * w.lit(3.)))
            .init(G.SetAttributeModifier(A.SIZE, w.rand(G.FLOAT)))
            .update(G.KillAabbModifier(w.lit(G.Vec3(0., 0., 0.)), w.lit(G.Vec3(1.5, 1.0, 1.25)))))


def test_plan_that_splits_position(ctx, orc, culls):
    asset = split_position_asset(9000)
    assert asset.generate().column_plan()[:3] == [(0, 8), (8, 4), (12, 4)]
    ref = RefWorld(9500, 8, [Instance(0, 500, alive=0, seed=5), Instance(500, 9000, alive=0, seed=6)], dt=0.05)
    lock = Lockstep(ctx, orc, ref, asset, seeds=seeds)
    run(lock, culls(9500, 2), 0, [[60, 1200]] * 15, "split position")
    view = ctx.slab_device_view(lock.gpu.slab)
    assert [view.plane_width[p] for p in range(3)] == [8, 4, 4]


def test_cull_of_depth_order(ctx, orc, culls):
    """d_src = hnb_batch_depth_order's d_order: the culled list is the reference back-to-front order, filtered."""
    asset, ref = sparks_world([9000, 700])
    lock = Lockstep(ctx, orc, ref, asset, seeds=seeds)
    lock.run([[900, 90]] * 12, what="churn")
    rows, pos = ref.slab_rows, position_word(asset)
    buf = culls(rows, 2)
    order, planes = ctx.device_alloc(4 * rows), ctx.device_alloc(32)
    rng = np.random.default_rng(12)
    try:
        for k in range(3):
            plane = np.concatenate([rng.standard_normal((2, 3)), np.zeros((2, 1))], axis=1).astype(np.float32)
            ctx.device_upload(order, np.full(rows, SENTINEL, dtype=np.uint32))
            ctx.device_upload(planes, plane.reshape(-1).view(np.uint32))
            launch = lock.gpu.launches()[0]
            ctx.batch_depth_order(launch, planes, 2, order, rows)
            frusta = camera_frusta(rng, 2)
            got, args = buf.of(launch, frusta, src=order)
            want_order = ref_depth_order(ref, 0, pos, plane, np.full(rows, SENTINEL, dtype=np.uint32))
            want, want_args = ref_cull(ref, 0, pos, frusta, np.full(rows, SENTINEL, dtype=np.uint32), ref.draw, src=want_order)
            np.testing.assert_array_equal(got, want, err_msg=f"call {k}: culled depth order")
            np.testing.assert_array_equal(args, want_args, err_msg=f"call {k}: draw args")
            assert 0 < args[0, 1] < ref.metadata[0].alive_count
    finally:
        ctx.device_free(order)
        ctx.device_free(planes)


def test_pinned_host_buffers(ctx, orc):
    asset, ref = sparks_world([5000, 700])
    lock = Lockstep(ctx, orc, ref, asset, seeds=seeds)
    lock.run([[900, 90]] * 6, what="pinned")
    rows, pos = ref.slab_rows, position_word(asset)
    frusta = camera_frusta(np.random.default_rng(1), 2)
    src = np.random.default_rng(2).permutation(rows).astype(np.uint32)
    h = [N.lib.hnb_host_alloc(n) for n in (192, 4 * rows, 4 * rows, 40)]
    assert all(h)
    h_frusta, h_src, h_visible, h_args = h
    try:
        C.memmove(h_frusta, frusta.tobytes(), 192)
        C.memmove(h_src, src.tobytes(), 4 * rows)
        for s, ref_src in ((0, None), (h_src, src)):
            C.memset(h_visible, 0xA5, 4 * rows)
            C.memset(h_args, 0xA5, 40)
            ctx.batch_cull(lock.gpu.launches()[0], h_frusta, 2, s, rows if s else 0, h_visible, rows, h_args, 2)
            ctx.sync()
            got = np.frombuffer(C.string_at(h_visible, 4 * rows), dtype=np.uint32)
            args = np.frombuffer(C.string_at(h_args, 40), dtype=np.uint32).reshape(2, 5)
            want, want_args = ref_cull(ref, 0, pos, frusta, np.full(rows, SENTINEL, dtype=np.uint32), ref.draw, src=ref_src)
            np.testing.assert_array_equal(got, want, err_msg="pinned host buffers: visible entries")
            np.testing.assert_array_equal(args, want_args, err_msg="pinned host buffers: draw args")
    finally:
        for p in h:
            N.lib.hnb_host_free(p)


def _state(ctx, lock):
    ctx.sync()
    rows = lock.ref.slab_rows
    return (ctx.slab_checksum(lock.gpu.slab, 0, rows), ctx.slab_checksum_indirect(lock.gpu.slab, 0, rows), lock.gpu.pull())


def test_nothing_changes_and_refusals_enqueue_nothing(ctx, orc, culls):
    asset, ref = sparks_world([5000, 600])
    lock = Lockstep(ctx, orc, ref, asset, seeds=seeds)
    lock.run([[900, 80]] * 10, what="churn")
    launch = lock.gpu.launches()[0]
    rows = ref.slab_rows
    buf = culls(rows, 3)
    sum0, ind0, pull0 = _state(ctx, lock)
    check(lock, buf, position_word(asset), "before the refusals", np.random.default_rng(2))
    sum1, ind1, pull1 = _state(ctx, lock)
    assert (sum0, ind0) == (sum1, ind1), "slab or list checksums changed"
    for k in pull0:
        np.testing.assert_array_equal(pull0[k], pull1[k], err_msg=f"the cull modified {k}")

    other_stride = ctx.effect_compile(table_asset("vec4x2_64", 2000).generate())
    sector = ctx.effect_compile(asset.generate(sector_planes=True))
    no_position = ctx.effect_compile(R.LoweredEffect(name="no_position", particle_stride=32, attrs=[
        R.AttrField("f32x4_0", N.VEC4, 0), R.AttrField("f32x4_1", N.VEC4, 16)]))
    ribbon = ctx.effect_compile(ribbon_asset(2000).generate())  # refused before its stride is compared with the slab's
    emitting = ctx.effect_compile(event_assets()[0].generate(num_event_bindings=1))
    make = N.BatchLaunch.make
    e, s = lock.gpu.effect, lock.gpu.slab
    F, V, D = buf.frusta, buf.visible, buf.args
    src = ctx.device_alloc(8 * rows)  # room for a source and a visible buffer side by side
    try:
        ok = (F, 3, 0, 0, V, rows, D, 3)
        cases = [("invalid effect", make(1 << 20, s), ok), ("invalid slab", make(e, 1 << 20), ok),
                 ("batch_info_index", make(e, s, 7), ok), ("stride does not match", make(other_stride, s), ok),
                 ("SECTOR_PLANES", make(sector, s), ok), ("no `position` attribute", make(no_position, s), ok),
                 ("ribbon", make(ribbon, s), ok),
                 ("d_frusta is NULL", launch, (0, 3, 0, 0, V, rows, D, 3)),
                 ("d_frusta is NULL or not 16-byte aligned", launch, (F + 8, 3, 0, 0, V, rows, D, 3)),
                 ("frustum_rows", launch, (F, 1, 0, 0, V, rows, D, 3)),
                 ("src_rows", launch, (F, 3, src, rows - 1, V, rows, D, 3)),
                 ("d_visible is NULL", launch, (F, 3, 0, 0, 0, rows, D, 3)),
                 ("visible_rows", launch, (F, 3, 0, 0, V, rows - 1, D, 3)),
                 ("overlap", launch, (F, 3, V, rows, V, rows, D, 3)),
                 ("overlap", launch, (F, 3, V + 4 * (rows - 1), rows, V, rows, D, 3)),
                 ("overlap", launch, (F, 3, src + 64, rows, src, rows, D, 3)),
                 ("d_args is NULL", launch, (F, 3, 0, 0, V, rows, 0, 3)),
                 ("d_args is NULL or not 4-byte aligned", launch, (F, 3, 0, 0, V, rows, D + 2, 3)),
                 ("args_rows", launch, (F, 3, 0, 0, V, rows, D, 1))]
        ctx.device_upload(V, np.full(rows, SENTINEL, dtype=np.uint32))
        ctx.device_upload(D, np.full(15, SENTINEL, dtype=np.uint32))
        for why, bl, call in cases:
            before = ctx.launch_count
            with pytest.raises(N.HanabiError) as err:
                ctx.batch_cull(bl, *call)
            assert err.value.code == N.HNB_ERR_INVALID_ARG and why in err.value.message, (why, err.value.message)
            assert ctx.launch_count == before, f"{why}: something was enqueued"
        assert (ctx.device_download(V, 4 * rows) == SENTINEL).all()
        assert (ctx.device_download(D, 60) == SENTINEL).all()
        with pytest.raises(N.HanabiError):
            N.check(N.lib.hnb_batch_cull(ctx._h, None, F, 3, None, 0, V, rows, D, 3))
        # an emitting effect of the slab's stride is accepted, and so are a source and a visible buffer side by side
        frusta = camera_frusta(np.random.default_rng(3), 3)
        ctx.device_upload(F, frusta.reshape(-1).view(np.uint32))
        ctx.batch_cull(make(emitting, s), F, 3, 0, 0, V, rows, D, 3)
        ctx.sync()
        want, want_args = ref_cull(ref, 0, 0, frusta, np.full(rows, SENTINEL, dtype=np.uint32), ref.draw)
        np.testing.assert_array_equal(ctx.device_download(V, 4 * rows).view(np.uint32), want, "through an emitting effect's descriptor")
        np.testing.assert_array_equal(ctx.device_download(D, 40).view(np.uint32).reshape(-1, 5), want_args)
        source = np.random.default_rng(4).permutation(rows).astype(np.uint32)
        ctx.device_upload(src, np.concatenate([source, np.full(rows, SENTINEL, dtype=np.uint32)]))
        ctx.batch_cull(launch, F, 3, src, rows, src + 4 * rows, rows, D, 3)
        want, _ = ref_cull(ref, 0, 0, frusta, np.full(rows, SENTINEL, dtype=np.uint32), ref.draw, src=source)
        np.testing.assert_array_equal(ctx.device_download(src + 4 * rows, 4 * rows).view(np.uint32), want, "adjacent buffers")
    finally:
        ctx.device_free(src)
    # ... and the world still steps in lock-step afterwards
    lock.run([[100, 100]] * 3, start=10, what="after the calls")


class _DeviceArray:
    """A device column as torch sees it through __cuda_array_interface__."""

    def __init__(self, ptr, shape):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": "<f4", "data": (ptr, False), "version": 2}


def test_c5_64_mi_rows_against_torch(ctx):
    """The benchmarked size: 64 Mi rows of hnb_slab_fill_c5 under its claim (the list is the identity), against a torch
    evaluation of the six planes on the slab's own position column, then `nonzero`."""
    import torch
    P = 64 << 20
    effect = ctx.effect_compile(recipes.c5_lowered())
    slab = ctx.slab_create(P, 32)
    ctx.slab_fill_c5(slab, 0, P, 99, 0.5, 2.0)
    md = R.initial_metadata(P, 0, 8)
    md.alive_count, md.max_spawn = P, 0
    ctx.metadata_insert(0, md)
    ctx.draw_args_insert(0, N.DrawIndexedIndirectArgs(6, 0, 3, -2, 7))
    ctx.upload_spawners([R.make_spawner(seed=42)])
    ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, 1)], [0])
    ctx.set_sim_params(1.0 / 60.0, 0.0, 1)
    launch = N.BatchLaunch.make(effect, slab, 0, 0)
    ctx.simulate([launch])
    frustum = camera_frusta(np.random.default_rng(64), 1, distance=4.0, fov=20.0)[0]  # a part of the [-1, 1]^3 cloud
    visible = torch.full((P,), -1, dtype=torch.int32, device="cuda")
    args = torch.zeros(5, dtype=torch.int32, device="cuda")
    frusta = torch.as_tensor(frustum.reshape(-1), device="cuda")
    try:
        ctx.batch_cull(launch, frusta.data_ptr(), 1, 0, 0, visible.data_ptr(), P, args.data_ptr(), 1)
        ctx.sync()
        view = ctx.slab_device_view(slab)
        assert view.plane_width[0] == 16
        col = torch.as_tensor(_DeviceArray(view.planes[0], (P, 4)), device="cuda")
        inside = torch.ones(P, dtype=torch.bool, device="cuda")
        for a, b, c, d in frustum.tolist():
            inside &= (((col[:, 0] * a + col[:, 1] * b) + col[:, 2] * c) + d) >= 0  # one rounding per elementwise op
        want = torch.nonzero(inside).flatten().to(torch.int32)
        m = want.numel()
        assert ctx.read_metadata(0).alive_count == P and 0 < m < P
        draw = ctx.read_draw_args(0)
        assert args.tolist() == [draw.index_count, m, draw.first_index, draw.base_vertex, draw.first_instance]
        assert torch.equal(visible[:m], want)
        assert bool((visible[m:] == -1).all())
    finally:
        ctx.slab_destroy(slab)
