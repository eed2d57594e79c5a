"""Lifetime floors on the device (DESIGN.md §3): the authored C5 (recipes.c5_asset, lifetime HNB_ATTR_REAP_ONLY) keeps a
floor per 32 slab rows and skips the lifetime loads it proves unnecessary. Every test runs the same instances on a second
slab with the hand-lowered C5, which keeps no floors, and asserts that both slabs hold the same records, lists and counters
frame after frame, also after each writer that must clear the floors has put short-lived particles where long-lived ones
had stored a high floor."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

STRIDE = 32


class Pair:
    """Slab 0: the authored C5 (floors); slab 1: the hand-lowered C5 (no floors). `insts`: (first row, rows) of each instance
    of the slab, all in one batch per slab, each filled with lifetimes U(lo, hi)."""

    def __init__(self, ctx, cap, insts, lo, hi, seed=77):
        from bevy_hanabi_b200 import _native as N, recipes, runtime as R
        self.ctx, self.cap, self.insts, self.n = ctx, cap, insts, len(insts)
        flagged = recipes.c5_asset(cap).generate()
        assert "#define HNB_LIFE_FLOOR 1" in flagged.generate_source()
        self.effects = [ctx.effect_compile(flagged), ctx.effect_compile(recipes.c5_lowered())]
        self.slabs = [ctx.slab_create(cap, STRIDE) for _ in range(2)]
        spawners, batches = [], []
        for i in range(2):
            for j, (first, rows) in reversed(list(enumerate(insts))):  # the last fill's claim is instance 0's
                ctx.slab_fill_c5(self.slabs[i], first, rows, seed, lo, hi, logical_first=first)
            for j, (first, rows) in enumerate(insts):
                row = self.row(i, j)
                md = R.initial_metadata(rows, row, STRIDE // 4)
                md.alive_count, md.max_spawn = rows, 0
                ctx.metadata_insert(row, md)
                ctx.draw_args_insert(row, N.DrawIndexedIndirectArgs(0, 0, 0, 0, 0))
                spawners.append(R.make_spawner(seed=42, effect_metadata_index=row, draw_indirect_index=row, slab_offset=first))
            batches.append(N.BatchInfo(0, 0, i * self.n, 0, i * self.n, self.n))
        ctx.upload_spawners(spawners)
        ctx.upload_batches(batches, [0] * (2 * self.n))
        self.launches = [N.BatchLaunch.make(self.effects[i], self.slabs[i], i, 0) for i in range(2)]
        self.frame = 0

    def row(self, i, j):
        return i * self.n + j

    def step(self, frames=1, dt=1.0 / 60.0):
        for _ in range(frames):
            self.ctx.set_sim_params(dt, self.frame * dt, 2 * self.n)
            self.ctx.simulate(self.launches)
            self.frame += 1

    def same(self, what):
        ctx = self.ctx
        assert ctx.slab_checksum(self.slabs[0], 0, self.cap) == ctx.slab_checksum(self.slabs[1], 0, self.cap), f"{what}: records"
        assert ctx.slab_checksum_indirect(self.slabs[0], 0, self.cap) == ctx.slab_checksum_indirect(self.slabs[1], 0, self.cap), f"{what}: lists"
        for j in range(self.n):
            a, b = ctx.read_metadata(self.row(0, j)), ctx.read_metadata(self.row(1, j))
            assert (a.alive_count, a.max_spawn, a.max_update, a.indirect_write_index) == (b.alive_count, b.max_spawn, b.max_update, b.indirect_write_index), f"{what}: instance {j}"

    def alive(self, j=0):
        return self.ctx.read_metadata(self.row(1, j)).alive_count

    def run_checked(self, frames, what, every=1):
        for f in range(frames):
            self.step()
            if f % every == every - 1 or f == frames - 1:
                self.same(f"{what}, frame {self.frame}")


@pytest.fixture(params=[1, 2, 4], ids=lambda n: f"{n}sub")
def chunk_ctx(request, native, monkeypatch):
    """A context with HNB_TILE_CHUNKS forced."""
    monkeypatch.setenv("HNB_TILE_CHUNKS", str(request.param))
    c = native.Context(0)
    yield c
    c.close()


def test_c5_variant_b_with_deaths_inside_groups(chunk_ctx):
    """C5 variant B (lifetimes U(1, 3)) over 2.5 s: floors are stored on the first frame and prove rows alive until the
    first deaths, which fall in the middle of groups and end the identity claim."""
    p = Pair(chunk_ctx, 1 << 18, [(0, 1 << 18)], 1.0, 3.0)
    p.run_checked(150, "variant B", every=15)
    assert 0 < p.alive() < (1 << 18)


def test_init_spawns_into_groups_with_floors(ctx):
    """Short-lived particles die in every group and spawns land in the freed slots of groups whose floors long-lived
    particles set; a repack every 10 frames makes the lists identities again, so floors come back into use."""
    from bevy_hanabi_b200 import runtime as R
    cap = 1 << 16
    p = Pair(ctx, cap, [(0, cap)], 0.05, 30.0)
    p.run_checked(20, "before the spawns", every=5)
    assert p.alive() < cap
    for f in range(30):
        spawners = [R.make_spawner(spawn=500, seed=900 + f, effect_metadata_index=r, draw_indirect_index=r) for r in range(2)]
        ctx.upload_spawners(spawners)
        from bevy_hanabi_b200 import _native as N
        p.launches = [N.BatchLaunch.make(p.effects[i], p.slabs[i], i, 500) for i in range(2)]
        p.run_checked(1, "spawning")
        if f % 10 == 9:
            for i in range(2):
                ctx.slab_repack(p.slabs[i], p.effects[i], p.row(i, 0), 0, cap)


def test_special_values_and_zero_dt(ctx):
    """NaN, infinite and negative lifetimes and negative ages, uploaded into both slabs, then frames with dt = 0 and 1/60."""
    cap = 1 << 14
    p = Pair(ctx, cap, [(0, cap)], 5.0, 9.0)
    p.run_checked(2, "filled")
    recs = ctx.slab_download_aos(p.slabs[1], 0, cap, STRIDE)
    rng = np.random.default_rng(4)
    life, age = recs[:, 7].view(np.float32), recs[:, 3].view(np.float32)
    life[rng.choice(cap, 64, replace=False)] = np.nan
    life[rng.choice(cap, 64, replace=False)] = np.inf
    life[rng.choice(cap, 64, replace=False)] = rng.uniform(-1, 0.02, 64)
    life[32:64] = np.nan
    age[rng.choice(cap, 256, replace=False)] = rng.uniform(-2, 0, 256)
    for s in p.slabs:
        ctx.slab_upload_aos(s, 0, recs)
    for f in range(8):
        p.step(dt=0.0 if f in (2, 3) else 1.0 / 60.0)
        p.same(f"special values, frame {f}")


def _short_records(ctx, p, rows):
    recs = ctx.slab_download_aos(p.slabs[1], 0, rows, STRIDE)
    recs[:, 7] = np.full(rows, 0.1, dtype=np.float32).view(np.uint32)  # far below the floors the fill's lifetimes set
    recs[:, 3] = np.zeros(rows, dtype=np.float32).view(np.uint32)
    return recs


@pytest.mark.parametrize("writer", ["fill", "upload_aos", "import_aos_device", "reset_rows", "repack", "restore", "device_view"])
def test_each_clearing_writer(ctx, writer):
    """Long lifetimes first (floors of about 20 s are stored), then the writer puts 0.1 s particles into those groups: they
    must die on time on the floor slab too."""
    cap = 1 << 16
    p = Pair(ctx, cap, [(0, cap)], 20.0, 40.0)
    p.run_checked(3, "long-lived")
    if writer == "fill":
        for s in p.slabs:
            ctx.slab_fill_c5(s, 0, cap, 5, 0.1, 0.1)
    elif writer == "upload_aos":
        recs = _short_records(ctx, p, 4096)
        for s in p.slabs:
            ctx.slab_upload_aos(s, 0, recs)
    elif writer == "import_aos_device":
        recs = _short_records(ctx, p, 4096)
        d = ctx.device_alloc(recs.nbytes)
        try:
            ctx.device_upload(d, recs)
            for s in p.slabs:
                ctx.slab_import_aos_device(s, 0, 4096, d)
            ctx.sync()
        finally:
            ctx.device_free(d)
    elif writer == "reset_rows":
        for s in p.slabs:  # the lists start again from the identity; a fill writes short-lived records behind the reset
            ctx.slab_reset_rows(s, 0, cap)
            ctx.slab_fill_c5(s, 0, cap, 6, 0.1, 0.5)
    elif writer == "repack":
        # rows 0..31 die soon; a repack then moves every later row 32 places down, so 0.1 s particles (rows 96..127)
        # land in group 2, whose floor rows 64..95 set at 20 s or more
        recs = ctx.slab_download_aos(p.slabs[1], 0, cap, STRIDE)
        recs[:32, 7] = recs[:32, 3]  # age == lifetime: dies on the next frame
        recs[96:128, 7] = (recs[96:128, 3].view(np.float32) + np.float32(0.3)).view(np.uint32)
        for s in p.slabs:
            ctx.slab_upload_aos(s, 0, recs)
        p.run_checked(3, "long-lived again")  # floors stored again after the upload cleared them
        assert p.alive() == cap - 32
        for i in range(2):
            ctx.slab_repack(p.slabs[i], p.effects[i], p.row(i, 0), 0, cap)
    elif writer == "restore":
        # a snapshot of the instance itself, its records turned into 0.1 s particles, restored into both slices
        nbytes = ctx.instance_snapshot_bytes(STRIDE, cap)
        d = ctx.device_alloc(nbytes)
        try:
            ctx.instance_snapshot(p.slabs[1], p.effects[1], p.row(1, 0), 0, cap, d, nbytes)
            snap = ctx.device_download(d, nbytes).view(np.uint32)
            recs = snap[16:].reshape(-1, STRIDE // 4)
            recs[:, 7] = (recs[:, 3].view(np.float32) + np.float32(0.1)).view(np.uint32)
            ctx.device_upload(d, snap)
            for i in range(2):
                ctx.instance_restore(p.slabs[i], p.effects[i], p.row(i, 0), 0, cap, d, nbytes)
            ctx.sync()
        finally:
            ctx.device_free(d)
    elif writer == "device_view":
        # a view stops the floors; short lifetimes are then written straight into the lifetime column
        v = ctx.slab_device_view(p.slabs[0])
        assert (v.plane_offset[3], v.plane_width[3]) == (28, 4)
        ctx.device_upload(v.planes[3], np.full(4096, 0.1, dtype=np.float32))
        recs = ctx.slab_download_aos(p.slabs[1], 0, 4096, STRIDE)
        recs[:, 7] = np.full(4096, 0.1, dtype=np.float32).view(np.uint32)
        ctx.slab_upload_aos(p.slabs[1], 0, recs)
    before = p.alive()
    p.run_checked(40, writer, every=4)
    assert p.alive() < before, "the short-lived particles must have died"


@pytest.mark.parametrize("second", [1000, 1024], ids=["sharing", "aligned"])
def test_two_instances_around_a_shared_group(ctx, second):
    """Two instances of one batch, the first ending inside a 32-row group: the second starts in that group or on the next
    one. Long lifetimes and repacks of both every 20 frames keep their lists claimed; short ones kill along the way."""
    insts = [(0, 1000), (second, 5120 - second)]
    p = Pair(ctx, 5120, insts, 0.3, 40.0)
    for r in range(4):
        p.run_checked(20, f"two instances, round {r}", every=5)
        for i in range(2):
            for j, (first, rows) in enumerate(insts):
                ctx.slab_repack(p.slabs[i], p.effects[i], p.row(i, j), first, rows)
