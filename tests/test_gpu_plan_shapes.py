"""Every reader and writer of slab records on drawn column plans (tests/plan_assets.py), held to the oracle's AoS bytes.

A slab stores records as SoA columns whose cut depends on the effect (DESIGN.md §3): runs plans, word maps whose columns
hold record words that are not consecutive, and the default cut. Each device path maps record words to columns through
`PlaneSet` or through generated code, with separate branches per column width, alignment and word list. One case per
drawn asset runs, on two contexts:
- A: the asset's own module on a slab in its plan; B: the same module with its read-only flags cleared (the default cut)
  on a slab of its own. Both run 12 lock-step frames of the numpy interpreter with bursts into recycled slots and deaths,
  compared in full after every frame (ribbon assets sort every frame by both keys, wherever the plan put them);
- the readers (AoS download over ranges off tile and group edges, device export to an address that is not 16-byte
  aligned, checksum, instance snapshot) against the oracle's bytes;
- the writers (AoS upload and device import of odd ranges, repack, snapshots restored across the two plans) against
  their restatements, then a frame;
- for word-map assets, deferred common ages: every reader runs while groups are deferred, so k_flush_group_ages writes
  the age into the lane and column the plan gave it;
- cross-plan modules: each context's effect is swapped for the other's, so that each slab runs a module generated for
  its plan, one compile per (effect, plan) pair;
- bounds, depth order and cull of the `position` against their restatements;
- at the end, the slab's device view: the plan is `column_plan()`, and each column holds the words
  `hnb_effect_column_words` names."""
import dataclasses

import numpy as np
import pytest

from oracle import c_oracle as O
from tests.bounds_ref import assert_bounds_equal, live_rows, ref_bounds
from tests.cull_ref import ref_cull
from tests.depth_order_ref import ref_depth_order
from tests.effects import tile_k
from tests.helpers import Instance, Lockstep, RefWorld, seeds
from tests.plan_assets import DT, SEEDS, default_cut, draw, is_word_map
from tests.repack_ref import ref_repack
from tests.snapshot_ref import ref_restore, ref_snapshot

pytestmark = pytest.mark.gpu

ROWS = 3000
INSTANCES = [(0, 1600, 11), (1611, 1300, 23)]  # (first row, capacity, seed): the second starts inside a 32-row group
SPAWNS = [[700, 500], [0, 0], [300, 200], [0, 150], [400, 0], [0, 0], [250, 300], [0, 0], [500, 100], [0, 0], [100, 400], [0, 0]]
# (first, count) of the AoS readers: whole slab, then ranges starting and ending off 32-row groups and off tiles, one over
# the end of instance 0 and the gap before instance 1
RANGES = [(0, ROWS), (37, 1234), (1599, 15), (2901, 99), (1, 1)]
SENTINEL = 0xDEADBEEF


def f32(x):
    return np.float32(x).view(np.uint32)


def world(asset, fields):
    _, size, _ = asset.particle_layout()
    ref = RefWorld(ROWS, size // 4, [Instance(first, cap, seed=s) for first, cap, s in INSTANCES], dt=DT)
    rng = np.random.default_rng(5)
    for inst in ref.instances:
        rows = slice(inst.slab_offset, inst.slab_offset + inst.capacity)
        ref.indirect[rows, 2] = rng.permutation(ref.indirect[rows, 2])
    if "ribbon_id" in fields:
        ref.set_sort_keys([f for f in asset.particle_layout()[0]])
    return ref


def cleared(fx):
    """The module of `fx` with every attribute writable: its plan is the default cut."""
    return dataclasses.replace(fx, attrs=[dataclasses.replace(a, flags=0) for a in fx.attrs])


def device_snapshot(ctx, lock, i):
    first, rows = lock.span(i)
    nbytes = ctx.instance_snapshot_bytes(lock.gpu.stride, rows)
    d = ctx.device_alloc(nbytes)
    try:
        ctx.instance_snapshot(lock.gpu.slab, lock.gpu.effect, i, first, rows, d, nbytes)
        return ctx.device_download(d, nbytes)
    finally:
        ctx.device_free(d)


def restore(ctx, lock, i, snap):
    d = ctx.device_alloc(snap.nbytes)
    try:
        ctx.device_upload(d, snap)
        first, rows = lock.span(i)
        ctx.instance_restore(lock.gpu.slab, lock.gpu.effect, i, first, rows, d, snap.nbytes)
        ctx.sync()
    finally:
        ctx.device_free(d)
    ref_restore(lock.ref, i, snap)


# ---- readers -----------------------------------------------------------------------------------------------------------
def read_download(lock, what):
    ctx, ref, g = lock.ctx, lock.ref, lock.gpu
    for first, count in RANGES:
        np.testing.assert_array_equal(ctx.slab_download_aos(g.slab, first, count, g.stride), ref.particles[first:first + count],
                                      err_msg=f"{what}: download of rows [{first}, {first + count})")


def read_export(lock, what):
    ctx, ref, g = lock.ctx, lock.ref, lock.gpu
    d = ctx.device_alloc(ROWS * g.stride + 64)
    try:
        for (first, count), skew in zip(RANGES, (4, 12, 8, 0, 4)):
            ctx.slab_export_aos_device(g.slab, first, count, d + skew)
            got = ctx.device_download(d + skew, count * g.stride).reshape(count, -1)
            np.testing.assert_array_equal(got, ref.particles[first:first + count],
                                          err_msg=f"{what}: export of rows [{first}, {first + count}) to +{skew} bytes")
    finally:
        ctx.device_free(d)


def read_checksum(lock, what):
    ctx, ref, g = lock.ctx, lock.ref, lock.gpu
    for first, count in RANGES:
        want = lock.orc.orc_checksum(O.ptr(ref.particles), first, count, ref.stride_words)
        assert ctx.slab_checksum(g.slab, first, count) == want, f"{what}: checksum of rows [{first}, {first + count})"


def assert_snapshot(got, want, what):
    """The header and the records of the live particles; the rest of the buffer is not written."""
    np.testing.assert_array_equal(got[:want.size], want, err_msg=what)


def read_snapshot(lock, what):
    for i in range(len(lock.ref.instances)):
        assert_snapshot(device_snapshot(lock.ctx, lock, i), ref_snapshot(lock.ref, i), f"{what}: snapshot of instance {i}")


READERS = [read_download, read_export, read_checksum, read_snapshot]


# ---- writers -----------------------------------------------------------------------------------------------------------
def write_upload(lock):
    """Rows [41, 818) of instance 0 take their records in reverse order, through a host upload."""
    first, end = 41, 818
    lock.ref.particles[first:end] = lock.ref.particles[first:end][::-1].copy()
    lock.ctx.slab_upload_aos(lock.gpu.slab, first, lock.ref.particles[first:end])


def write_import(lock):
    """Rows [1650, 2173) of instance 1 (off its groups) take their records in reverse order, through a device import."""
    ctx, ref, first, end = lock.ctx, lock.ref, 1650, 2173
    ref.particles[first:end] = ref.particles[first:end][::-1].copy()
    d = ctx.device_alloc((end - first) * lock.gpu.stride)
    try:
        ctx.device_upload(d, ref.particles[first:end])
        ctx.slab_import_aos_device(lock.gpu.slab, first, end - first, d)
        ctx.sync()
    finally:
        ctx.device_free(d)


def repack(lock, i):
    first, rows = lock.span(i)
    lock.ctx.slab_repack(lock.gpu.slab, lock.gpu.effect, i, first, rows)
    ref_repack(lock.ref, i)


# ---- batch passes ------------------------------------------------------------------------------------------------------
FRUSTUM = np.array([[1, 0, 0, 0], [-1, 0, 0, 1e30], [0, 1, 0, 1e30], [0, -1, 0, 1e30], [0, 0, 1, 1e30], [0, 0, -1, 1e30]],
                   dtype=np.float32)  # x >= -d of the first plane, set to the median x of the live particles
PLANES = np.array([[0.6, 0.8, 0, 0.25], [0, 0, -1, 0]], dtype=np.float32)


def batch_passes(lock, pos, ribbons, what):
    """Bounds, then depth order and cull of batch 0 (not for ribbons, which are drawn in ribbon order, whole)."""
    ctx, ref = lock.ctx, lock.ref
    launch = lock.gpu.launches()[0]
    n = len(ref.instances)
    frusta = np.stack([FRUSTUM] * n)
    live = np.concatenate([live_rows(ref, i) for i in range(n)])
    frusta[:, 0, 3] = -np.median(ref.particles[live, pos].view(np.float32))
    bufs = {k: ctx.device_alloc(b) for k, b in (("bounds", 32 * n), ("planes", PLANES.nbytes), ("order", 4 * ROWS),
                                                 ("frusta", frusta.nbytes), ("visible", 4 * ROWS), ("args", 20 * n))}
    try:
        ctx.batch_bounds(launch, bufs["bounds"], n)
        assert_bounds_equal(ctx.download_bounds(bufs["bounds"], n), ref_bounds(ref, 0, pos), what)
        if ribbons:
            return
        ctx.device_upload(bufs["planes"], PLANES.view(np.uint32))
        ctx.device_upload(bufs["order"], np.full(ROWS, SENTINEL, dtype=np.uint32))
        ctx.batch_depth_order(launch, bufs["planes"], n, bufs["order"], ROWS)
        want = ref_depth_order(ref, 0, pos, PLANES, np.full(ROWS, SENTINEL, dtype=np.uint32))
        np.testing.assert_array_equal(ctx.device_download(bufs["order"], 4 * ROWS), want, err_msg=f"{what}: depth order")
        ctx.device_upload(bufs["frusta"], frusta.view(np.uint32))
        ctx.device_upload(bufs["visible"], np.full(ROWS, SENTINEL, dtype=np.uint32))
        ctx.batch_cull(launch, bufs["frusta"], n, 0, 0, bufs["visible"], ROWS, bufs["args"], n)
        want, want_args = ref_cull(ref, 0, pos, frusta, np.full(ROWS, SENTINEL, dtype=np.uint32), ref.draw)
        np.testing.assert_array_equal(ctx.device_download(bufs["visible"], 4 * ROWS), want, err_msg=f"{what}: visible lists")
        np.testing.assert_array_equal(ctx.device_download(bufs["args"], 20 * n).reshape(n, 5), want_args, err_msg=f"{what}: cull args")
        assert 0 < want_args[:, 1].sum() < sum(ref.metadata[i].alive_count for i in range(n)), f"{what}: the frustum must cut"
    finally:
        for d in bufs.values():
            ctx.device_free(d)


def assert_view_is_the_plan(ctx, lock, plan, words, what):
    """The slab's device view shows `plan`, and column p holds record words words[p] of every row, in lane order."""
    v = ctx.slab_device_view(lock.gpu.slab)
    assert [(v.plane_offset[p], v.plane_width[p]) for p in range(v.num_planes)] == plan, what
    ctx.sync()
    for p, ws in enumerate(words):
        col = ctx.device_download(v.planes[p], ROWS * 4 * len(ws)).reshape(ROWS, len(ws))
        np.testing.assert_array_equal(col, lock.ref.particles[:, ws], err_msg=f"{what}: column {p} (words {ws})")


def both(locks, f, spawns, what):
    for lock in locks:
        lock.step(f, spawns)
        lock.compare(f"{what}, frame {f}")


@pytest.mark.parametrize("seed", SEEDS, ids=lambda s: f"seed{s}")
def test_drawn_plan(native, orc, seed):
    d = draw(seed)
    asset, fields = d.asset, {f.name: f.offset // 4 for f in d.asset.particle_layout()[0]}
    fx = asset.generate()
    plan, words = fx.column_plan(), fx.column_words()
    dc_fx = cleared(fx)
    assert dc_fx.column_plan() == default_cut(fx.particle_stride)
    pos = fields["position"]
    mapped = is_word_map(words)
    defers = mapped and "ribbon_id" not in fields  # a ribbon sort clears the claims a floor tile needs
    if mapped:
        assert "#define HNB_GROUP_AGE 1" in fx.generate_source(), "a word map keeps common ages"
    with native.Context(0) as ca, native.Context(0) as cb:
        a = Lockstep(ca, orc, world(asset, fields), asset, seeds=seeds, effect=ca.effect_compile(fx))
        b = Lockstep(cb, orc, world(asset, fields), asset, seeds=seeds, effect=cb.effect_compile(dc_fx))
        locks = (a, b)

        # 1. frames
        for f, spawns in enumerate(SPAWNS):
            both(locks, f, spawns, "frames")
        alive = [a.ref.metadata[i].alive_count for i in range(2)]
        assert all(alive), f"every instance must have live particles: {alive}"
        if "lifetime" in fields:
            assert a.ref.metadata[0].particle_counter > alive[0], "the frames must kill particles"
        assert ca.read_tile_size(0) == 32 * tile_k(fx.particle_stride)
        f = len(SPAWNS)

        # 2. readers, on both plans
        for lock in locks:
            for reader in READERS:
                reader(lock, f"{reader.__name__} ({'drawn' if lock is a else 'default cut'})")

        # 3. writers, then a frame
        for lock in locks:
            write_upload(lock)
            write_import(lock)
        both(locks, f, [60, 40], "upload + import")
        for lock in locks:
            repack(lock, 0)
            repack(lock, 1)
        both(locks, f + 1, [90, 0], "repack")
        snap_a, snap_b = device_snapshot(ca, a, 0), device_snapshot(cb, b, 1)
        assert_snapshot(snap_a, ref_snapshot(a.ref, 0), "snapshot, drawn plan")
        assert_snapshot(snap_b, ref_snapshot(b.ref, 1), "snapshot, default cut")
        restore(cb, b, 0, snap_a)  # drawn plan -> default cut
        restore(ca, a, 1, snap_b)  # default cut -> drawn plan
        restore(ca, a, 0, snap_a)  # drawn plan -> drawn plan, a round trip
        both(locks, f + 2, [0, 70], "crossed restores")
        f += 3

        # 4. deferred common ages: every record lives long with one age, instance 0 holds the claim after a repack
        if defers:
            for lock in locks:
                lock.ref.particles[:, fields["lifetime"]] = f32(1000.0)
                lock.ref.particles[:, fields["age"]] = f32(0.25)
                lock.ctx.slab_upload_aos(lock.gpu.slab, 0, lock.ref.particles)
                repack(lock, 0)
            for reader in READERS:
                for _ in range(3):
                    for lock in locks:
                        lock.step(f, [0, 0])
                    f += 1
                assert ca.slab_deferred_groups(a.gpu.slab) > 0, f"{reader.__name__}: no group is deferred, so the case proves nothing"
                reader(a, f"{reader.__name__} with deferred groups")
                a.compare(f"after {reader.__name__} with deferred groups")

        # 5. cross-plan modules: each slab runs the other context's effect, compiled for the slab's plan
        compiles = [ca.plan_compiles(), cb.plan_compiles()]
        a.gpu.effect, b.gpu.effect = ca.effect_compile(dc_fx), cb.effect_compile(fx)
        for k in range(3):
            both(locks, f + k, [120, 80] if k == 0 else [0, 0], "cross-plan modules")
        f += 3
        rise = int(plan != default_cut(fx.particle_stride))
        assert [ca.plan_compiles() - compiles[0], cb.plan_compiles() - compiles[1]] == [rise, rise]

        # 6. batch passes
        batch_passes(a, pos, "ribbon_id" in fields, "drawn plan")
        batch_passes(b, pos, "ribbon_id" in fields, "default cut")

        assert_view_is_the_plan(ca, a, plan, words, "drawn plan")
        assert_view_is_the_plan(cb, b, default_cut(fx.particle_stride), [list(range(o // 4, (o + w) // 4)) for o, w in default_cut(fx.particle_stride)],
                                "default cut")
