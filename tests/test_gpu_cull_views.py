"""hnb_batch_cull_views on the device: after every frame of a lock-step run, every view's visible entries and draw
arguments equal the numpy restatement (tests/cull_ref.py) for that view's frusta, applied to the oracle world, bit for
bit, and the world itself still equals the oracle. Also: culling of a depth order, pinned host buffers, every refusal
enqueuing nothing and writing nothing, four launches for every view count, no byte of the slab or the tables changing,
one view equal to hnb_batch_cull byte for byte, and a 64 Mi-row instance in four views against torch."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from bevy_hanabi_b200 import _native as N
from bevy_hanabi_b200 import recipes
from bevy_hanabi_b200 import runtime as R
from tests.cull_ref import frustum_planes, ref_cull
from tests.depth_order_ref import ref_depth_order
from tests.effects import ribbon_asset
from tests.helpers import Instance, Lockstep, filled_c5, is_identity, seeds, sparks_world

pytestmark = pytest.mark.gpu
SENTINEL = np.uint32(0xA5A5A5A5)
LAUNCHES = 4
MAX_VIEWS = 8


def position_word(asset):
    return next(f.offset for f in asset.particle_layout()[0] if f.name == "position") // 4


def camera_frusta(rng, count, distance=3.0, fov=None):
    """Perspective cameras at `distance` from the origin, looking near it from random directions, each seeing part of a
    cloud around the origin. (count, 6, 4) float32, radius 0.01 added."""
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


class Views:
    """Device buffers for hnb_batch_cull_views calls of up to MAX_VIEWS views: frusta, visible entries and args rows,
    stacked view-major, each view's visible slice 256-byte aligned and followed by a gap of sentinels."""

    def __init__(self, ctx, rows, instances):
        self.ctx, self.rows, self.instances = ctx, rows, instances
        self.visible_rows = (rows + 64 + 63) // 64 * 64
        self.visible = ctx.device_alloc(4 * MAX_VIEWS * self.visible_rows)
        self.frusta = ctx.device_alloc(96 * MAX_VIEWS * instances)
        self.args = ctx.device_alloc(20 * MAX_VIEWS * instances)

    def of(self, launch, frusta, src=0, count=None):
        """([visible entries of each view], [args rows of each view]) after one call over buffers of sentinels; `frusta`
        is (views, instances, 6, 4)."""
        ctx, views, vr, inst = self.ctx, len(frusta), self.visible_rows, self.instances
        count = inst if count is None else count
        ctx.device_upload(self.visible, np.full(MAX_VIEWS * vr, SENTINEL, dtype=np.uint32))
        ctx.device_upload(self.args, np.full(5 * MAX_VIEWS * inst, SENTINEL, dtype=np.uint32))
        ctx.device_upload(self.frusta, np.ascontiguousarray(frusta, dtype=np.float32).reshape(-1).view(np.uint32))
        before = ctx.launch_count
        ctx.batch_cull_views(launch, views, self.frusta, inst, src, self.rows if src else 0, self.visible, vr, self.args, inst)
        assert ctx.launch_count == before + LAUNCHES, "a fixed number of launches per call"
        vis = ctx.device_download(self.visible, 4 * MAX_VIEWS * vr).view(np.uint32).reshape(MAX_VIEWS, vr)
        args = ctx.device_download(self.args, 20 * MAX_VIEWS * inst).view(np.uint32).reshape(MAX_VIEWS, inst, 5)
        assert (vis[:, self.rows:] == SENTINEL).all() and (vis[views:] == SENTINEL).all(), "stores past a view's slice"
        assert (args[:, count:] == SENTINEL).all() and (args[views:] == SENTINEL).all(), "stores past a view's args rows"
        return list(vis[:views, :self.rows]), list(args[:views, :count])

    def free(self):
        for p in (self.visible, self.frusta, self.args):
            self.ctx.device_free(p)


@pytest.fixture()
def views_bufs(ctx):
    made = []

    def make(rows, instances):
        made.append(Views(ctx, rows, instances))
        return made[-1]
    yield make
    for c in made:
        c.free()


def check(lock, buf, pos_word, what, rng, views):
    """Every batch of the lock-step world, in `views` views, against the restatement on the oracle world."""
    seen = 0
    for b, launch in enumerate(lock.gpu.launches()):
        count = lock.ref.batch_infos[b].prefix_sum_count
        frusta = np.stack([camera_frusta(rng, buf.instances) for _ in range(views)])
        got, args = buf.of(launch, frusta, count=count)
        for v in range(views):
            want, want_args = ref_cull(lock.ref, b, pos_word, frusta[v], np.full(buf.rows, SENTINEL, dtype=np.uint32), lock.ref.draw)
            np.testing.assert_array_equal(got[v], want, err_msg=f"{what}, batch {b}, view {v}: visible entries")
            np.testing.assert_array_equal(args[v], want_args, err_msg=f"{what}, batch {b}, view {v}: draw args")
            seen += int(args[v][:, 1].sum())
    return seen


def run(lock, buf, pos_word, schedule, what):
    rng = np.random.default_rng(len(what))
    seen = 0
    for k, spawns in enumerate(schedule):
        lock.step(k, spawns)
        lock.compare(f"{what} frame {k}")
        seen += check(lock, buf, pos_word, f"{what} frame {k}", rng, views=1 + k % MAX_VIEWS)
    assert seen > 0, f"{what}: no particle was ever visible"


def test_c5_filled_then_dying(ctx, orc, views_bufs):
    """Filled C5 under a claim over every row, then deaths and bursts into recycled slots; 1 to 8 views."""
    n = 6000
    lock = filled_c5(ctx, orc, [Instance(0, n, alive=n, seed=8)], [(0, n, 9, 0.05, 0.4)])
    run(lock, views_bufs(n, 1), 0, [[0]] * 10 + [[900], [0], [0], [1500]] + [[0]] * 4, "C5")
    assert 0 < lock.ref.metadata[0].alive_count < n and not is_identity(lock.ref, 0)


@pytest.mark.parametrize("mode", ["sector", "two_batches"])
def test_churned_sparks(ctx, orc, views_bufs, mode):
    """Sector planes, and two batches of two instances each, the larger instances more than one 4096-row tile."""
    caps = [9000, 1000, 4097, 512] if mode == "two_batches" else [9000]
    batches = [[0, 1], [2, 3]] if mode == "two_batches" else None
    asset, ref = sparks_world(caps, batches=batches)
    lock = Lockstep(ctx, orc, ref, asset, seeds=seeds, sector=mode == "sector")
    sched = [[900 if j % 2 == 0 else 35 for j in range(len(caps))]] * 12 + [[0] * len(caps)] * 4
    run(lock, views_bufs(ref.slab_rows, 2 if mode == "two_batches" else 1), position_word(asset), sched, mode)


def test_1024_instances_in_one_batch(ctx, orc, views_bufs):
    n_inst, cap = 1024, 192
    asset, ref = sparks_world([cap] * n_inst)
    lock = Lockstep(ctx, orc, ref, asset, seeds=seeds)
    buf = views_bufs(ref.slab_rows, n_inst)
    rng = np.random.default_rng(6)
    seen = 0
    for f, views in enumerate([2, 8, 5]):
        lock.step(f, [0 if i % 9 == 0 else int(x) for i, x in enumerate(rng.integers(0, 70, n_inst))])
        seen += check(lock, buf, position_word(asset), f"1024 instances frame {f}", rng, views)
    lock.compare("1024 instances")
    assert seen > 0


def test_cull_of_depth_order(ctx, orc, views_bufs):
    """d_src = hnb_batch_depth_order's d_order, shared by three views: each view's list is the order, filtered."""
    asset, ref = sparks_world([9000, 700])
    lock = Lockstep(ctx, orc, ref, asset, seeds=seeds)
    lock.run([[900, 90]] * 12, what="churn")
    rows, pos = ref.slab_rows, position_word(asset)
    buf = views_bufs(rows, 2)
    order, planes = ctx.device_alloc(4 * rows), ctx.device_alloc(32)
    rng = np.random.default_rng(12)
    try:
        plane = np.concatenate([rng.standard_normal((2, 3)), np.zeros((2, 1))], axis=1).astype(np.float32)
        ctx.device_upload(order, np.full(rows, SENTINEL, dtype=np.uint32))
        ctx.device_upload(planes, plane.reshape(-1).view(np.uint32))
        launch = lock.gpu.launches()[0]
        ctx.batch_depth_order(launch, planes, 2, order, rows)
        frusta = np.stack([camera_frusta(rng, 2) for _ in range(3)])
        got, args = buf.of(launch, frusta, src=order)
        want_order = ref_depth_order(ref, 0, pos, plane, np.full(rows, SENTINEL, dtype=np.uint32))
        for v in range(3):
            want, want_args = ref_cull(ref, 0, pos, frusta[v], np.full(rows, SENTINEL, dtype=np.uint32), ref.draw, src=want_order)
            np.testing.assert_array_equal(got[v], want, err_msg=f"view {v}: culled depth order")
            np.testing.assert_array_equal(args[v], want_args, err_msg=f"view {v}: draw args")
            assert 0 < args[v][0, 1] < ref.metadata[0].alive_count
    finally:
        ctx.device_free(order)
        ctx.device_free(planes)


def test_pinned_host_buffers(ctx, orc):
    asset, ref = sparks_world([5000, 700])
    lock = Lockstep(ctx, orc, ref, asset, seeds=seeds)
    lock.run([[900, 90]] * 6, what="pinned")
    rows, pos, views = ref.slab_rows, position_word(asset), 3
    rng = np.random.default_rng(1)
    frusta = np.stack([camera_frusta(rng, 2) for _ in range(views)])
    src = np.random.default_rng(2).permutation(rows).astype(np.uint32)
    h = [N.lib.hnb_host_alloc(n) for n in (192 * views, 4 * rows, 4 * rows * views, 40 * views)]
    assert all(h)
    h_frusta, h_src, h_visible, h_args = h
    try:
        C.memmove(h_frusta, frusta.tobytes(), 192 * views)
        C.memmove(h_src, src.tobytes(), 4 * rows)
        for s, ref_src in ((0, None), (h_src, src)):
            C.memset(h_visible, 0xA5, 4 * rows * views)
            C.memset(h_args, 0xA5, 40 * views)
            ctx.batch_cull_views(lock.gpu.launches()[0], views, h_frusta, 2, s, rows if s else 0, h_visible, rows, h_args, 2)
            ctx.sync()
            got = np.frombuffer(C.string_at(h_visible, 4 * rows * views), dtype=np.uint32).reshape(views, rows)
            args = np.frombuffer(C.string_at(h_args, 40 * views), dtype=np.uint32).reshape(views, 2, 5)
            for v in range(views):
                want, want_args = ref_cull(ref, 0, pos, frusta[v], np.full(rows, SENTINEL, dtype=np.uint32), ref.draw, src=ref_src)
                np.testing.assert_array_equal(got[v], want, err_msg=f"pinned host buffers, view {v}: visible entries")
                np.testing.assert_array_equal(args[v], want_args, err_msg=f"pinned host buffers, view {v}: draw args")
    finally:
        for p in h:
            N.lib.hnb_host_free(p)


def _state(ctx, lock):
    ctx.sync()
    rows = lock.ref.slab_rows
    return (ctx.slab_checksum(lock.gpu.slab, 0, rows), ctx.slab_checksum_indirect(lock.gpu.slab, 0, rows), lock.gpu.pull())


def test_every_view_count_and_nothing_changes(ctx, orc, views_bufs):
    """Four launches for every view count from 1 to 8, and no byte of the slab, its lists or the tables changes."""
    asset, ref = sparks_world([5000, 600])
    lock = Lockstep(ctx, orc, ref, asset, seeds=seeds)
    lock.run([[900, 80]] * 10, what="churn")
    buf = views_bufs(ref.slab_rows, 2)
    before = _state(ctx, lock)
    rng = np.random.default_rng(2)
    for views in range(1, MAX_VIEWS + 1):
        check(lock, buf, position_word(asset), f"{views} views", rng, views)
    after = _state(ctx, lock)
    assert before[:2] == after[:2], "slab or list checksums changed"
    for k in before[2]:
        np.testing.assert_array_equal(before[2][k], after[2][k], err_msg=f"the cull modified {k}")
    lock.run([[100, 100]] * 3, start=10, what="after the calls")


def test_one_view_is_batch_cull(ctx, orc):
    """views = 1 writes byte for byte what hnb_batch_cull writes, over buffers of random words, from the alive list and
    from a source buffer."""
    asset, ref = sparks_world([9000, 700])
    lock = Lockstep(ctx, orc, ref, asset, seeds=seeds)
    lock.run([[900, 90]] * 8, what="churn")
    rows, launch = ref.slab_rows, lock.gpu.launches()[0]
    rng = np.random.default_rng(5)
    frusta = camera_frusta(rng, 2)
    junk = rng.integers(0, 1 << 32, rows + 10, dtype=np.uint64).astype(np.uint32)
    F, S, V, D = (ctx.device_alloc(n) for n in (192, 4 * rows, 4 * rows, 40))
    try:
        ctx.device_upload(F, frusta.reshape(-1).view(np.uint32))
        ctx.device_upload(S, rng.permutation(rows).astype(np.uint32))
        for src in (0, S):
            outs = []
            for call in (ctx.batch_cull, lambda *a: ctx.batch_cull_views(a[0], 1, *a[1:])):
                ctx.device_upload(V, junk[:rows])
                ctx.device_upload(D, junk[:10])
                call(launch, F, 2, src, rows if src else 0, V, rows, D, 2)
                outs.append((ctx.device_download(V, 4 * rows).tobytes(), ctx.device_download(D, 40).tobytes()))
            assert outs[0] == outs[1], f"src={'buffer' if src else 'alive list'}"
    finally:
        for p in (F, S, V, D):
            ctx.device_free(p)


def test_refusals_enqueue_nothing(ctx, orc, views_bufs):
    """Every refusal of hnb_batch_cull, checked over the stacked ranges, and the multi-view ones: no launch, and the
    sentinel-filled buffers keep every byte."""
    asset, ref = sparks_world([5000, 600])
    lock = Lockstep(ctx, orc, ref, asset, seeds=seeds)
    lock.run([[900, 80]] * 4, what="churn")
    launch = lock.gpu.launches()[0]
    rows = ref.slab_rows
    buf = views_bufs(rows, 3)
    ribbon = ctx.effect_compile(ribbon_asset(2000).generate())
    make = N.BatchLaunch.make
    e, s = lock.gpu.effect, lock.gpu.slab
    F, V, D, vr = buf.frusta, buf.visible, buf.args, buf.visible_rows
    src = ctx.device_alloc(4 * rows)
    try:
        ok = (3, F, 3, 0, 0, V, vr, D, 3)
        cases = [("invalid effect", make(1 << 20, s), ok), ("invalid slab", make(e, 1 << 20), ok),
                 ("batch_info_index", make(e, s, 7), ok), ("ribbon", make(ribbon, s), ok),
                 ("views is 0", launch, (0, F, 3, 0, 0, V, vr, D, 3)),
                 ("above HNB_CULL_MAX_VIEWS", launch, (9, F, 3, 0, 0, V, vr, D, 3)),
                 ("d_frusta is NULL", launch, (3, 0, 3, 0, 0, V, vr, D, 3)),
                 ("not 16-byte aligned", launch, (3, F + 8, 3, 0, 0, V, vr, D, 3)),
                 ("frustum_rows", launch, (3, F, 1, 0, 0, V, vr, D, 3)),
                 ("src_rows", launch, (3, F, 3, src, rows - 1, V, vr, D, 3)),
                 ("d_visible is NULL", launch, (3, F, 3, 0, 0, 0, vr, D, 3)),
                 ("visible_rows", launch, (3, F, 3, 0, 0, V, rows - 1, D, 3)),
                 ("overlap", launch, (3, F, 3, V, rows, V, vr, D, 3)),
                 ("overlap", launch, (3, F, 3, V + 4 * 2 * vr, rows, V, vr, D, 3)),           # inside view 2's slice
                 ("overlap", launch, (3, F, 3, V + 4 * (3 * vr - 1), rows, V, vr, D, 3)),     # its last word
                 ("d_args is NULL", launch, (3, F, 3, 0, 0, V, vr, 0, 3)),
                 ("not 4-byte aligned", launch, (3, F, 3, 0, 0, V, vr, D + 2, 3)),
                 ("args_rows", launch, (3, F, 3, 0, 0, V, vr, D, 1))]
        ctx.device_upload(V, np.full(MAX_VIEWS * vr, SENTINEL, dtype=np.uint32))
        ctx.device_upload(D, np.full(5 * MAX_VIEWS * 3, SENTINEL, dtype=np.uint32))
        for why, bl, call in cases:
            before = ctx.launch_count
            with pytest.raises(N.HanabiError) as err:
                ctx.batch_cull_views(bl, *call)
            assert err.value.code == N.HNB_ERR_INVALID_ARG and why in err.value.message, (why, err.value.message)
            assert why.startswith("invalid") or "hnb_batch_cull_views" in err.value.message, err.value.message
            assert ctx.launch_count == before, f"{why}: something was enqueued"
        assert (ctx.device_download(V, 4 * MAX_VIEWS * vr) == SENTINEL).all()
        assert (ctx.device_download(D, 60 * MAX_VIEWS) == SENTINEL).all()
        with pytest.raises(N.HanabiError):
            N.check(N.lib.hnb_batch_cull_views(ctx._h, None, 3, F, 3, None, 0, V, vr, D, 3))
        # a source right after the last view's slice is accepted
        ctx.batch_cull_views(launch, 2, F, 3, V + 4 * 2 * vr, rows, V, vr, D, 3)
        ctx.sync()
    finally:
        ctx.device_free(src)


class _DeviceArray:
    """A device column as torch sees it through __cuda_array_interface__."""

    def __init__(self, ptr, shape):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": "<f4", "data": (ptr, False), "version": 2}


def test_c5_64_mi_rows_four_views_against_torch(ctx):
    """64 Mi rows of hnb_slab_fill_c5 under its claim, four cameras from different directions, against a torch evaluation
    of each view's six planes on the slab's own position column, then `nonzero`."""
    import torch
    P, views = 64 << 20, 4
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
    frusta_np = camera_frusta(np.random.default_rng(64), views, distance=4.0, fov=20.0)
    visible = torch.full((views, P), -1, dtype=torch.int32, device="cuda")
    args = torch.zeros(views, 5, dtype=torch.int32, device="cuda")
    frusta = torch.as_tensor(frusta_np.reshape(-1), device="cuda")
    try:
        ctx.batch_cull_views(launch, views, frusta.data_ptr(), 1, 0, 0, visible.data_ptr(), P, args.data_ptr(), 1)
        ctx.sync()
        view = ctx.slab_device_view(slab)
        assert view.plane_width[0] == 16
        col = torch.as_tensor(_DeviceArray(view.planes[0], (P, 4)), device="cuda")
        draw = ctx.read_draw_args(0)
        counts = []
        for v in range(views):
            inside = torch.ones(P, dtype=torch.bool, device="cuda")
            for a, b, c, d in frusta_np[v].tolist():
                inside &= (((col[:, 0] * a + col[:, 1] * b) + col[:, 2] * c) + d) >= 0  # one rounding per elementwise op
            want = torch.nonzero(inside).flatten().to(torch.int32)
            m = want.numel()
            assert 0 < m < P
            assert args[v].tolist() == [draw.index_count, m, draw.first_index, draw.base_vertex, draw.first_instance]
            assert torch.equal(visible[v, :m], want), f"view {v}"
            assert bool((visible[v, m:] == -1).all()), f"view {v}"
            counts.append(m)
        assert len(set(counts)) > 1, "the cameras see different parts"
    finally:
        ctx.slab_destroy(slab)
