"""Common ages on the device (DESIGN.md §3): the authored C5 (recipes.c5_asset, a word map with the age in a column of its
own) keeps the age bits of each 32-row group beside its lifetime floor and skips the age column where the previous frame's
update stored them. Every test runs the same instances on a second slab with the hand-lowered C5 (default cut, neither
floors nor common ages, held to the C oracle by the rest of the suite) and asserts that both slabs hold the same records,
lists and counters frame after frame: at every tile shape, when the tile size changes between frames with the batch, after
each writer that must clear the words has put rows of another age into known groups, and across AoS and snapshot round
trips between the two plans."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

STRIDE = 32


class Pair:
    """Slab 0: the authored C5; slab 1: the hand-lowered C5. `insts`: (first row, rows) of each instance of the slab, each
    filled with lifetimes U(lo, hi) and age 0."""

    def __init__(self, ctx, cap, insts, lo, hi, seed=77):
        from bevy_hanabi_b200 import _native as N, recipes, runtime as R
        self.N, self.R = N, R
        self.ctx, self.cap, self.insts, self.n = ctx, cap, insts, len(insts)
        authored = recipes.c5_asset(cap).generate()
        assert "#define HNB_GROUP_AGE 1" in authored.generate_source()
        self.effects = [ctx.effect_compile(authored), ctx.effect_compile(recipes.c5_lowered())]
        self.slabs = [ctx.slab_create(cap, STRIDE) for _ in range(2)]
        spawners = []
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
        ctx.upload_spawners(spawners)
        self.set_batch()
        self.frame = 0

    def row(self, i, j):
        return i * self.n + j

    def set_batch(self, split=False, spawn=0):
        """One batch per slab holding all its instances, or (`split`) one batch per instance."""
        N, n = self.N, self.n
        if split:
            infos = [N.BatchInfo(0, 0, r, 0, r, 1) for r in range(2 * n)]
            slab_of = [r // n for r in range(2 * n)]
        else:
            infos = [N.BatchInfo(0, 0, i * n, 0, i * n, n) for i in range(2)]
            slab_of = [0, 1]
        self.ctx.upload_batches(infos, [0] * (2 * n))
        self.launches = [N.BatchLaunch.make(self.effects[i], self.slabs[i], b, spawn) for b, i in enumerate(slab_of)]

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


SHAPES = [(k, c) for k in (1, 2, 4, 8) for c in sorted({1, 2, 16 // k})]


@pytest.mark.parametrize("k,chunks", SHAPES, ids=[f"K{k}-{c}sub" for k, c in SHAPES])
def test_variant_b_spawns_and_repacks_at_every_tile_shape(native, monkeypatch, k, chunks):
    """Lifetimes U(1, 3) filled with age 0: the common ages are known from the second frame until the first deaths; then
    bursts spawn into the freed slots and a repack every 15 frames claims the lists again (and clears the words)."""
    monkeypatch.setenv("HNB_TILE_K", str(k))
    monkeypatch.setenv("HNB_TILE_CHUNKS", str(chunks))
    ctx = native.Context(0)
    try:
        cap = 1 << 16
        p = Pair(ctx, cap, [(0, cap)], 1.0, 3.0)
        p.run_checked(70, "variant B", every=10)
        assert p.alive() < cap
        for f in range(45):
            from bevy_hanabi_b200 import runtime as R
            ctx.upload_spawners([R.make_spawner(spawn=300, seed=500 + f, effect_metadata_index=r, draw_indirect_index=r) for r in range(2)])
            p.set_batch(spawn=300)
            p.run_checked(1, "spawning")
            if f % 15 == 14:
                for i in range(2):
                    ctx.slab_repack(p.slabs[i], p.effects[i], p.row(i, 0), 0, cap)
    finally:
        ctx.close()


def test_tile_size_changes_with_the_batch(ctx):
    """A 1.2 Mi-row slab is under eight waves, so the tile size follows the batch's instance count: instance 0 in a batch of
    its own gets other tiles than in one batch with instance 1, and the rows of instance 0 that lie in floor tiles change
    from frame to frame while its claim stays."""
    cap = 1_200_000
    p = Pair(ctx, cap, [(0, 1000), (1024, 200_000)], 30.0, 40.0)
    for f in range(24):
        p.set_batch(split=f % 3 != 1)
        p.run_checked(1, f"split {f % 3 != 1}")


def _aged(recs, age):
    recs[:, 3] = np.full(len(recs), age, dtype=np.float32).view(np.uint32)
    return recs


@pytest.mark.parametrize("writer", ["fill", "upload_aos", "import_aos_device", "reset_rows", "repack", "restore"])
def test_each_clearing_writer_with_another_age(ctx, writer):
    """Every group's common age is known (long lifetimes, age 0 plus some frames); then the writer puts rows of another age
    into those groups. A stale common age would give them the old one."""
    cap = 1 << 16
    p = Pair(ctx, cap, [(0, cap)], 20.0, 40.0)
    p.run_checked(3, "known ages")
    if writer == "fill":
        for s in p.slabs:
            ctx.slab_fill_c5(s, 0, cap, 5, 20.0, 40.0)  # age 0 again, three frames younger than the groups' words
    elif writer in ("upload_aos", "import_aos_device"):
        recs = _aged(ctx.slab_download_aos(p.slabs[1], 0, 4096, STRIDE), 0.5)
        recs[7, 3] = np.float32(0.25).view(np.uint32)  # and one row of group 0 differs from the rest
        if writer == "upload_aos":
            for s in p.slabs:
                ctx.slab_upload_aos(s, 0, recs)
        else:
            d = ctx.device_alloc(recs.nbytes)
            try:
                ctx.device_upload(d, recs)
                for s in p.slabs:
                    ctx.slab_import_aos_device(s, 0, 4096, d)
                ctx.sync()
            finally:
                ctx.device_free(d)
    elif writer == "reset_rows":
        for s in p.slabs:
            ctx.slab_reset_rows(s, 0, cap)
            ctx.slab_fill_c5(s, 0, cap, 6, 20.0, 40.0)
    elif writer == "repack":
        # rows 0..31 die on the next frame; the repack then moves every later row 32 places down, so rows of another age
        # (rows 96..127, age 0.5) land in group 2, whose word the update stored
        recs = ctx.slab_download_aos(p.slabs[1], 0, cap, STRIDE)
        recs[:32, 7] = recs[:32, 3]
        recs[96:128] = _aged(recs[96:128], 0.5)
        for s in p.slabs:
            ctx.slab_upload_aos(s, 0, recs)
        p.run_checked(3, "known ages again")
        assert p.alive() == cap - 32
        for i in range(2):
            ctx.slab_repack(p.slabs[i], p.effects[i], p.row(i, 0), 0, cap)
    elif writer == "restore":
        nbytes = ctx.instance_snapshot_bytes(STRIDE, cap)
        d = ctx.device_alloc(nbytes)
        try:
            ctx.instance_snapshot(p.slabs[1], p.effects[1], p.row(1, 0), 0, cap, d, nbytes)
            snap = ctx.device_download(d, nbytes).view(np.uint32)
            recs = snap[16:].reshape(-1, STRIDE // 4)
            recs[:, 3] = (recs[:, 3].view(np.float32) + np.float32(0.5)).view(np.uint32)
            ctx.device_upload(d, snap)
            for i in range(2):
                ctx.instance_restore(p.slabs[i], p.effects[i], p.row(i, 0), 0, cap, d, nbytes)
            ctx.sync()
        finally:
            ctx.device_free(d)
    p.run_checked(12, writer, every=3)


def test_aos_and_snapshot_round_trips_between_plans(ctx):
    """AoS download of both slabs, upload of each into the other, and snapshots of both restored crosswise: the word-map
    slab and the default-cut slab hold the same records, bit for bit, and keep stepping alike."""
    cap = 1 << 16
    p = Pair(ctx, cap, [(0, cap)], 0.05, 2.0)
    p.run_checked(10, "before")
    a, b = (ctx.slab_download_aos(s, 0, cap, STRIDE) for s in p.slabs)
    np.testing.assert_array_equal(a, b)
    rng = np.random.default_rng(3)
    recs = a.copy()
    recs[:, :7] = rng.standard_normal((cap, 7)).astype(np.float32).view(np.uint32)
    ctx.slab_upload_aos(p.slabs[0], 0, recs)
    np.testing.assert_array_equal(ctx.slab_download_aos(p.slabs[0], 0, cap, STRIDE), recs)
    ctx.slab_upload_aos(p.slabs[1], 0, ctx.slab_download_aos(p.slabs[0], 0, cap, STRIDE))
    p.same("after the AoS round trip")
    p.run_checked(5, "after the AoS round trip")
    nbytes = ctx.instance_snapshot_bytes(STRIDE, cap)
    bufs = [ctx.device_alloc(nbytes) for _ in range(2)]
    try:
        for i in range(2):
            ctx.instance_snapshot(p.slabs[i], p.effects[i], p.row(i, 0), 0, cap, bufs[i], nbytes)
        ctx.sync()
        np.testing.assert_array_equal(ctx.device_download(bufs[0], nbytes), ctx.device_download(bufs[1], nbytes))
        ctx.instance_restore(p.slabs[0], p.effects[0], p.row(0, 0), 0, cap, bufs[1], nbytes)
        ctx.instance_restore(p.slabs[1], p.effects[1], p.row(1, 0), 0, cap, bufs[0], nbytes)
        ctx.sync()
        p.same("after the crossed restores")
        p.run_checked(10, "after the crossed restores", every=2)
    finally:
        for d in bufs:
            ctx.device_free(d)
