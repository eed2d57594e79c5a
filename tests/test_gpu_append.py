"""hnb_instance_append on the device. Each case runs a lock-step world (the device and the oracle, tests/append_ref.py
applied at the same point) and compares every buffer bit for bit after the append and after every following frame:
churned sparks in default, sector and slot modes; appends every frame while the spawner spawns; two appends in one window;
a snapshot handed to another slice, slab and context; bounds, cull and snapshot in the same window; the benchmarked C5
module with lifetime floors and deferred ages; a 64 Mi-row C5 instance taking 1 Mi records; refusals."""
from __future__ import annotations

import numpy as np
import pytest

from bevy_hanabi_b200 import _native as N
from bevy_hanabi_b200 import recipes
from bevy_hanabi_b200 import runtime as R
from oracle import c_oracle as O
from tests.append_ref import append_count, make_snapshot, ref_append
from tests.bounds_ref import BOUNDS_DTYPE, assert_bounds_equal, ref_bounds
from tests.cull_ref import ref_cull
from tests.effects import event_assets, table_asset
from tests.helpers import Instance, Lockstep, filled_c5, is_identity, seeds, sparks_world
from tests.snapshot_ref import HEADER_WORDS, ref_snapshot

pytestmark = pytest.mark.gpu

SENTINEL = np.uint32(0xA5A5A5A5)


@pytest.fixture()
def bufs(ctx):
    live = []

    def upload(c, words):
        """A device buffer of `c` holding `words`; returns (ptr, bytes)."""
        p = c.device_alloc(max(words.nbytes, 16))
        live.append((c, p))
        c.device_upload(p, words)
        return p, words.nbytes

    def alloc(c, nbytes):
        p = c.device_alloc(nbytes)
        live.append((c, p))
        return p
    upload.alloc = alloc
    yield upload
    for c, p in live:
        c.device_free(p)


def clones(ref, i, k):
    """A snapshot of the first k live records of instance i of `ref` (a clone of its current particles)."""
    words = ref_snapshot(ref, i)
    k = min(k, int(words[3]))
    words = words[:HEADER_WORDS + k * ref.stride_words].copy()
    words[3] = k
    return words


def append(side, i, ptr, nbytes, words, what=""):
    """The append on the device and in the oracle, then a comparison of every buffer. Returns m."""
    want = append_count(side.ref, i, words, nbytes)
    side.ctx.instance_append(side.gpu.slab, side.gpu.effect, i, *side.span(i), ptr, nbytes)
    m = ref_append(side.ref, i, words, nbytes)
    assert m == want
    side.compare(f"{what}: after the append into instance {i}")
    return m


def _churned_sparks(ctx, orc, caps=(4096,), **kw):
    asset, ref = sparks_world(list(caps))
    side = Lockstep(ctx, orc, ref, asset, seeds=seeds, **kw)
    side.run([[300] + [0] * (len(caps) - 1)] * 24, what="churn")
    assert not is_identity(side.ref, 0) and side.ref.metadata[0].alive_count > min(2000, caps[0] // 2)
    return asset, side


@pytest.mark.parametrize("mode", ["default", "sector", "slot"])
def test_churned_sparks(ctx, orc, bufs, mode):
    """500 clones of the instance's own particles go to 500 slots of its permuted dead stack, then 10 frames."""
    _, side = _churned_sparks(ctx, orc, sector=mode == "sector", slot=mode == "slot")
    words = clones(side.ref, 0, 500)
    assert append(side, 0, *bufs(ctx, words), words, mode) == 500
    side.run([[300]] * 10, start=24, what=f"{mode}, after the append")


def test_appends_every_frame(ctx, orc, bufs):
    """For 30 frames, the spawner spawns 150 and 7 + 13 f clones are appended after the frame (cut to max_spawn when the
    instance fills up)."""
    _, side = _churned_sparks(ctx, orc)
    total = 0
    for f in range(24, 54):
        side.step(f, [150])
        side.compare(f"frame {f}")
        words = clones(side.ref, 0, 7 + 13 * (f - 24))
        total += append(side, 0, *bufs(ctx, words), words, f"frame {f}")
    assert total > 2000
    side.run([[150]] * 3, start=54, what="after the appends")


def test_two_appends_in_one_window(ctx, orc, bufs):
    """Two appends between two frames compose: the second takes the slots after the first's."""
    _, side = _churned_sparks(ctx, orc)
    a = clones(side.ref, 0, 200)
    assert append(side, 0, *bufs(ctx, a), a, "first") == 200
    b = clones(side.ref, 0, 250)
    assert append(side, 0, *bufs(ctx, b), b, "second") == 250
    side.run([[300]] * 8, start=24, what="after two appends")


@pytest.mark.parametrize("target", ["other_slice", "other_slab", "other_context"])
def test_orphan_hand_off(ctx, orc, bufs, native, target):
    """The particles of a dying instance outlive it: a device snapshot of instance 0 is appended to a live instance of the
    same effect in the same slab, another slab, or a slab of a second context, which runs on."""
    caps = (4096, 4096) if target == "other_slice" else (4096,)
    asset, src = _churned_sparks(ctx, orc, caps)
    nbytes = ctx.instance_snapshot_bytes(src.gpu.stride, 4096)
    ptr = bufs.alloc(ctx, nbytes)
    ctx.instance_snapshot(src.gpu.slab, src.gpu.effect, 0, 0, 4096, ptr, nbytes)
    words = ref_snapshot(src.ref, 0)
    np.testing.assert_array_equal(ctx.device_download(ptr, words.nbytes), words)
    ctx2 = native.Context(0) if target == "other_context" else ctx
    try:
        if target == "other_slice":
            dst, i = src, 1
            src.run([[0, 400]] * 3, start=24, what="the target spawns")
        else:
            dst, i = Lockstep(ctx2, orc, sparks_world([777, 6000, 500], seed=2)[1], asset, seeds=seeds), 1
            dst.run([[50, 400, 40]] * 3, what="the target spawns")
        m = append(dst, i, ptr, nbytes, words, target)
        assert m == min(int(words[3]), dst.ref.metadata[i].max_spawn + m) and m > 1000
        if target == "other_slice":  # the emitter is removed: its instance spawns no more
            dst.run([[0, 300]] * 10, start=27, what="after the hand-off")
        else:
            dst.run([[50, 300, 40]] * 10, start=3, what="after the hand-off")
    finally:
        if ctx2 is not ctx:
            ctx2.close()


def test_readers_in_the_same_window_see_the_appended(ctx, orc, bufs):
    """Bounds, cull (every position passes) and a snapshot between the append and the next frame include the appended
    particles."""
    asset, side = _churned_sparks(ctx, orc)
    pos = {f.name: f.offset // 4 for f in asset.particle_layout()[0]}["position"]
    far_words = clones(side.ref, 0, 64)
    recs = far_words[HEADER_WORDS:].reshape(64, -1)
    recs[:, pos:pos + 3] = np.float32(1000.0 + np.arange(64 * 3).reshape(64, 3)).view(np.uint32)  # outside every box so far
    assert append(side, 0, *bufs(ctx, far_words), far_words, "far records") == 64
    launch = side.gpu.launches()[0]
    box = bufs.alloc(ctx, 32)
    ctx.batch_bounds(launch, box, 1)
    got = ctx.device_download(box, 32).view(BOUNDS_DTYPE)
    want = ref_bounds(side.ref, 0, pos)
    assert_bounds_equal(got, want, "bounds")
    assert got["count"][0] == side.ref.metadata[0].alive_count and got["max"][0][0] >= 1000.0
    rows = side.ref.slab_rows
    frusta = np.tile(np.array([0, 0, 0, 1], dtype=np.float32), (1, 6, 1))
    fptr, _ = bufs(ctx, frusta.reshape(-1).view(np.uint32))
    vis = bufs.alloc(ctx, 4 * rows)
    args = bufs.alloc(ctx, 20)
    ctx.device_upload(vis, np.full(rows, SENTINEL, dtype=np.uint32))
    ctx.batch_cull(launch, fptr, 1, 0, 0, vis, rows, args, 1)
    want_vis, want_args = ref_cull(side.ref, 0, pos, frusta, np.full(rows, SENTINEL, dtype=np.uint32), side.ref.draw)
    np.testing.assert_array_equal(ctx.device_download(vis, 4 * rows), want_vis, err_msg="cull: visible entries")
    np.testing.assert_array_equal(ctx.device_download(args, 20).reshape(1, 5), want_args, err_msg="cull: args")
    assert want_args[0, 1] == side.ref.metadata[0].alive_count
    nbytes = ctx.instance_snapshot_bytes(side.gpu.stride, 4096)
    snap = bufs.alloc(ctx, nbytes)
    ctx.instance_snapshot(side.gpu.slab, side.gpu.effect, 0, 0, 4096, snap, nbytes)
    words = ref_snapshot(side.ref, 0)
    np.testing.assert_array_equal(ctx.device_download(snap, words.nbytes), words, err_msg="snapshot")
    side.run([[300]] * 4, start=24, what="after the readers")


# ---- the benchmarked C5 module: lifetime floors and deferred ages ---------------------------------------------------------
CAP_A, ALIVE_A = 4173, 4128
B0, CAP_B, ALIVE_B = 4173, 3000, 2900
C0, CAP_C, ALIVE_C = 7173, 2000, 1500
ROWS = C0 + CAP_C
DT = 1.0 / 60.0


def f32(x):
    return np.float32(x).view(np.uint32)


def deferring_c5(ctx, orc):
    """The authored C5 on one slab: instance 0 (4128 of 4173 rows alive, lifetimes 20-30 s, the identity claim) defers
    its floor groups; rows 5 and 1000 die in the last deferring frame; instance 1 shares its last group and dies from the
    third frame on; instance 2 runs in a batch of its own. Returns (lock, next frame)."""
    authored = recipes.c5_asset(ROWS).generate()
    assert "#define HNB_GROUP_AGE 1" in authored.generate_source()
    insts = [Instance(0, CAP_A, alive=ALIVE_A, seed=3), Instance(B0, CAP_B, alive=ALIVE_B, seed=4),
             Instance(C0, CAP_C, alive=ALIVE_C, seed=5)]
    fills = [(ALIVE_A, CAP_A - ALIVE_A, 31, 20.0, 30.0), (B0, ALIVE_B, 32, 0.55, 0.8), (C0, ALIVE_C, 33, 20.0, 30.0),
             (0, ALIVE_A, 34, 20.0, 30.0)]
    lock = filled_c5(ctx, orc, insts, fills, batches=[[0, 1], [2]], effect=ctx.effect_compile(authored))
    ref, slab = lock.ref, lock.gpu.slab
    ref.particles[B0:B0 + ALIVE_B, 3] = f32(0.5)
    ctx.slab_upload_aos(slab, B0, ref.particles[B0:B0 + ALIVE_B])
    for r in (5, 1000):
        ref.particles[r, 7] = f32(4.5 * DT)
        ctx.slab_upload_aos(slab, r, ref.particles[r:r + 1])
    f = 0
    while ref.metadata[0].alive_count == ALIVE_A:
        lock.step(f)
        f += 1
        assert f <= 8
    return lock, f


@pytest.mark.parametrize("k", [2, 40])
def test_c5_floors_and_deferred_ages(native, orc, monkeypatch, k):
    """k records go to the first k slots of instance 0's dead stack (the rows that just died, then the tail of the slice
    and the group instance 1 shares) while its floor groups are deferred: hnb_slab_deferred_groups does not change, and
    the next updates equal the oracle."""
    monkeypatch.delenv("HNB_DEFER_AGES", raising=False)
    ctx = native.Context(0)
    ptr = None
    try:
        lock, f = deferring_c5(ctx, orc)
        before = ctx.slab_deferred_groups(lock.gpu.slab)
        assert before > 0, "no group is deferred, so the case proves nothing"
        words = make_snapshot(ref_snapshot(lock.ref, 2)[HEADER_WORDS:HEADER_WORDS + 8 * k], 8)
        ptr = ctx.device_alloc(words.nbytes)
        ctx.device_upload(ptr, words)
        ctx.instance_append(lock.gpu.slab, lock.gpu.effect, 0, 0, CAP_A, ptr, words.nbytes)
        assert ctx.slab_deferred_groups(lock.gpu.slab) == before, "the append changed the deferred words"
        assert ref_append(lock.ref, 0, words) == k
        for j in range(8):
            lock.step(f + j)
            if j in (0, 1, 7):
                lock.compare(f"k {k}, frame {f + j}")
    finally:
        if ptr:
            ctx.device_free(ptr)
        ctx.close()


def test_c5_64_mi_takes_1_mi(native, orc):
    """A filled 64 Mi-row C5 instance with its last 1 Mi slots free in a permuted dead stack takes 1 Mi records: the
    rows it kept hash as before, the 1 Mi written rows hash as the oracle's, and list rows [P - F, P) name the slots."""
    P, F = 64 << 20, 1 << 20
    rng = np.random.default_rng(64)
    c = native.Context(0)
    ptr = None
    try:
        effect = c.effect_compile(recipes.c5_lowered())
        slab = c.slab_create(P, 32)
        c.slab_fill_c5(slab, 0, P, 99, 0.5, 2.0)
        perm = (rng.permutation(F) + (P - F)).astype(np.uint32)
        rows3 = c.slab_download_indirect(slab, P - F, F)
        rows3[:, 2] = perm
        c.slab_upload_indirect(slab, P - F, rows3)
        md = R.initial_metadata(P, 0, 8)
        md.alive_count, md.max_spawn, md.particle_counter = P - F, F, 777
        c.metadata_insert(0, md)
        kept = c.slab_checksum(slab, 0, P - F)
        recs = rng.uniform(-1, 1, (F, 8)).astype(np.float32)
        recs[:, 7] = rng.uniform(0.5, 2.0, F)
        words = make_snapshot(recs.view(np.uint32), 8)
        ptr = c.device_alloc(words.nbytes)
        c.device_upload(ptr, words)
        c.instance_append(slab, effect, 0, 0, P, ptr, words.nbytes)
        c.sync()
        md = c.read_metadata(0)
        assert (md.alive_count, md.max_spawn, md.particle_counter) == (P, 0, 777 + F)
        assert c.slab_checksum(slab, 0, P - F) == kept
        want = np.zeros((F, 8), dtype=np.uint32)
        want[perm.astype(np.int64) - (P - F)] = recs.view(np.uint32)
        assert c.slab_checksum(slab, P - F, F) == orc.orc_checksum(O.ptr(want), 0, F, 8)
        np.testing.assert_array_equal(c.slab_download_indirect(slab, P - F, F)[:, 0], perm, err_msg="list entries")
    finally:
        if ptr:
            c.device_free(ptr)
        c.close()


def test_refusals_leave_the_state_untouched(ctx, orc, bufs):
    asset, side = _churned_sparks(ctx, orc, caps=(2000,))
    gpu = side.gpu
    before = gpu.pull()
    words = clones(side.ref, 0, 100)
    ptr = bufs.alloc(ctx, words.nbytes + 16)
    ctx.device_upload(ptr, np.concatenate([words, np.full(4, SENTINEL, dtype=np.uint32)]))
    nbytes = words.nbytes
    other_stride = ctx.effect_compile(table_asset("vec4x2_64", 2000).generate())
    sector = ctx.effect_compile(asset.generate(sector_planes=True))
    parent = event_assets()[0]
    emitting = ctx.effect_compile(parent.generate(num_event_bindings=1))
    cases = [("rows outside the slab", gpu.effect, 0, 1, 2000, ptr, nbytes), ("rows outside the slab", gpu.effect, 0, 0, 2001, ptr, nbytes),
             ("metadata row out of range", gpu.effect, 1 << 20, 0, 2000, ptr, nbytes),
             ("stride does not match", other_stride, 0, 0, 2000, ptr, nbytes), ("SECTOR_PLANES", sector, 0, 0, 2000, ptr, nbytes),
             ("cannot be appended to without its event buffers", emitting, 0, 0, 2000, ptr, nbytes),
             ("src_bytes", gpu.effect, 0, 0, 2000, ptr, 63)]
    cases += [("NULL or not 16-byte aligned", gpu.effect, 0, 0, 2000, p, nbytes) for p in (0, ptr + 4, ptr + 8)]
    for why, effect, row, first, rows, p, size in cases:
        with pytest.raises(N.HanabiError) as e:
            ctx.instance_append(gpu.slab, effect, row, first, rows, p, size)
        assert e.value.code == N.HNB_ERR_INVALID_ARG and why in e.value.message, (why, e.value.message)
        for k, v in before.items():
            np.testing.assert_array_equal(v, gpu.pull()[k], err_msg=f"{why}: {k}")
    # rows == 0, a header-only buffer and a version-2 header append nothing
    ctx.instance_append(gpu.slab, gpu.effect, 0, 0, 0, ptr, nbytes)
    ctx.instance_append(gpu.slab, gpu.effect, 0, 0, 2000, ptr, 64)
    v2 = words.copy()
    v2[1] = 2
    ctx.device_upload(ptr, v2)
    ctx.instance_append(gpu.slab, gpu.effect, 0, 0, 2000, ptr, nbytes)
    after = gpu.pull()
    for k, v in before.items():
        np.testing.assert_array_equal(v, after[k], err_msg=f"no-op appends: {k}")
    side.run([[300]] * 3, start=24, what="after the refusals")
