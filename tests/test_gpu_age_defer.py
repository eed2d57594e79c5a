"""Deferred common ages on the device (DESIGN.md §3): the authored C5 leaves the age column of every floor group whose 32
rows all survive a frame unwritten and keeps the group's age in its word. The rows take it back when an update meets them
outside a floor tile, and every other reader or writer of records writes it back first. As in test_gpu_group_age.py, a
second slab runs the hand-lowered C5 (default cut, no floors, no common ages) and both slabs must hold the same records,
lists and counters; here the slabs are compared rarely, so groups stay deferred over many frames between the reads."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

STRIDE = 32


class Pair:
    """Slab 0: the authored C5; slab 1: the hand-lowered C5; one instance of `cap` rows each, lifetimes U(lo, hi), age 0."""

    def __init__(self, ctx, cap, lo, hi, seed=91):
        from bevy_hanabi_b200 import _native as N, recipes, runtime as R
        self.N, self.R, self.ctx, self.cap = N, R, ctx, cap
        authored = recipes.c5_asset(cap).generate()
        assert "#define HNB_GROUP_AGE_WORD 3" in authored.generate_source()
        self.effects = [ctx.effect_compile(authored), ctx.effect_compile(recipes.c5_lowered())]
        self.slabs = [ctx.slab_create(cap, STRIDE) for _ in range(2)]
        for i in range(2):
            ctx.slab_fill_c5(self.slabs[i], 0, cap, seed, lo, hi)
            md = R.initial_metadata(cap, i, STRIDE // 4)
            md.alive_count, md.max_spawn = cap, 0
            ctx.metadata_insert(i, md)
            ctx.draw_args_insert(i, N.DrawIndexedIndirectArgs(0, 0, 0, 0, 0))
        self.spawn(0)
        self.frame = 0

    def spawn(self, n, seed=5):
        R, N = self.R, self.N
        self.ctx.upload_spawners([R.make_spawner(spawn=n, seed=seed, effect_metadata_index=i, draw_indirect_index=i) for i in range(2)])
        self.ctx.upload_batches([N.BatchInfo(0, 0, i, 0, i, 1) for i in range(2)], [0, 0])
        self.launches = [N.BatchLaunch.make(self.effects[i], self.slabs[i], i, n) for i in range(2)]

    def step(self, frames=1, dt=1.0 / 60.0):
        for _ in range(frames):
            self.ctx.set_sim_params(dt, self.frame * dt, 2)
            self.ctx.simulate(self.launches)
            self.frame += 1

    def sit_out(self, frames):
        """Frames without any batch: the epoch moves on, nothing is updated."""
        for _ in range(frames):
            self.ctx.upload_batches([], [])
            self.ctx.set_sim_params(1.0 / 60.0, 0.0, 0)
            self.ctx.simulate([])
        self.spawn(0)

    def same(self, what):
        ctx = self.ctx
        assert ctx.slab_checksum(self.slabs[0], 0, self.cap) == ctx.slab_checksum(self.slabs[1], 0, self.cap), f"{what}: records"
        assert ctx.slab_checksum_indirect(self.slabs[0], 0, self.cap) == ctx.slab_checksum_indirect(self.slabs[1], 0, self.cap), f"{what}: lists"
        a, b = ctx.read_metadata(0), ctx.read_metadata(1)
        assert (a.alive_count, a.max_spawn, a.max_update) == (b.alive_count, b.max_spawn, b.max_update), what

    def alive(self):
        return self.ctx.read_metadata(1).alive_count


SHAPES = [(k, c) for k in (1, 2, 4, 8) for c in sorted({1, 2, 16 // k})]


@pytest.mark.parametrize("k,chunks", SHAPES, ids=[f"K{k}-{c}sub" for k, c in SHAPES])
def test_deferred_over_many_frames_at_every_tile_shape(native, monkeypatch, k, chunks):
    """Long stretches without a read: groups stay deferred, then deaths turn the list into a gather (deferred groups are
    consumed outside floor tiles), spawns refill the freed slots, and a repack claims the list again."""
    monkeypatch.setenv("HNB_TILE_K", str(k))
    monkeypatch.setenv("HNB_TILE_CHUNKS", str(chunks))
    ctx = native.Context(0)
    try:
        cap = 1 << 16
        p = Pair(ctx, cap, 0.5, 3.0)
        p.step(25)
        p.same("before deaths")
        p.step(30)
        p.same("deaths")
        assert p.alive() < cap
        for f in range(3):
            p.spawn(400, seed=600 + f)
            p.step(5)
            p.spawn(0)
            p.step(10)
            p.same(f"spawns {f}")
        for i in range(2):
            ctx.slab_repack(p.slabs[i], p.effects[i], i, 0, cap)
        p.step(12)
        p.same("after the repack")
    finally:
        ctx.close()


def test_batch_sits_out_while_deferred(ctx):
    """Frames without any batch between frames that defer: the deferred words need no epoch test."""
    cap = 1 << 16
    p = Pair(ctx, cap, 20.0, 30.0)
    for gap in (1, 5, 64):
        p.step(4)
        p.sit_out(gap)
        p.step(3)
        p.same(f"after sitting out {gap} frames")


def test_readers_in_the_middle_of_a_run(ctx):
    """AoS download, device export, snapshot and checksum of part of the slab while groups are deferred: each sees the
    records, and the run goes on alike (the words they leave are read as known by the next update)."""
    cap = 1 << 16
    p = Pair(ctx, cap, 20.0, 30.0)
    p.step(6)
    a, b = (ctx.slab_download_aos(s, 40, 5000, STRIDE) for s in p.slabs)
    np.testing.assert_array_equal(a, b)
    assert (a[:, 3].view(np.float32) == np.float32(a[0, 3].view(np.float32))).all() and a[0, 3] != 0
    p.step(5)
    assert ctx.slab_checksum(p.slabs[0], 100, 7000) == ctx.slab_checksum(p.slabs[1], 100, 7000)
    p.step(5)
    nbytes = ctx.instance_snapshot_bytes(STRIDE, cap)
    bufs = [ctx.device_alloc(nbytes) for _ in range(2)]
    try:
        for i in range(2):
            ctx.instance_snapshot(p.slabs[i], p.effects[i], i, 0, cap, bufs[i], nbytes)
        ctx.sync()
        np.testing.assert_array_equal(ctx.device_download(bufs[0], nbytes), ctx.device_download(bufs[1], nbytes))
        p.step(5)
        for i in range(2):
            ctx.slab_export_aos_device(p.slabs[i], 0, cap, bufs[i])
        ctx.sync()
        np.testing.assert_array_equal(ctx.device_download(bufs[0], cap * STRIDE), ctx.device_download(bufs[1], cap * STRIDE))
        p.step(5)
        ctx.instance_snapshot(p.slabs[1], p.effects[1], 1, 0, cap, bufs[0], nbytes)  # restored into both slabs
        ctx.sync()
        for i in range(2):
            ctx.instance_restore(p.slabs[i], p.effects[i], i, 0, cap, bufs[0], nbytes)
        p.step(8)
        p.same("after the restore")
    finally:
        for d in bufs:
            ctx.device_free(d)


def test_upload_into_deferred_groups(ctx):
    """An AoS upload of rows starting and ending inside groups: the rest of each group gets its deferred age back."""
    cap = 1 << 16
    p = Pair(ctx, cap, 20.0, 30.0)
    p.step(5)
    recs = ctx.slab_download_aos(p.slabs[1], 70, 1000, STRIDE)
    recs[:, 3] = np.full(1000, 0.75, dtype=np.float32).view(np.uint32)
    p.step(3)
    for s in p.slabs:
        ctx.slab_upload_aos(s, 70, recs)
    p.step(6)
    p.same("after the upload")


def test_device_view_then_module_without_group_ages(ctx):
    """A device view mid-run writes every deferred age back (the slab keeps no words from then on); on a second pair, the
    hand-lowered C5 takes over the authored C5's slab."""
    cap = 1 << 16
    p = Pair(ctx, cap, 20.0, 30.0)
    p.step(7)
    ctx.slab_device_view(p.slabs[0])
    p.same("after the view")
    p.step(6)
    p.same("updates after the view")
    q = Pair(ctx, cap, 20.0, 30.0)
    q.step(7)
    q.launches[0] = q.N.BatchLaunch.make(q.effects[1], q.slabs[0], 0, 0)
    q.step(6)
    q.same("lowered C5 on the authored slab")


def test_start_near_the_epoch_wrap(native, monkeypatch):
    """The 30-bit epoch wraps during the run: the wrap writes every deferred age back before it clears the words."""
    monkeypatch.setenv("HNB_EPOCH_START", str((1 << 30) - 6))
    ctx = native.Context(0)
    try:
        cap = 1 << 16
        p = Pair(ctx, cap, 20.0, 30.0)
        for f in range(4):
            p.step(4)
            p.same(f"across the wrap, round {f}")
    finally:
        ctx.close()
