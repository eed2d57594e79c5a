"""Deferred common ages (DESIGN.md §3) against the oracle, through every host call that reads or writes a slab's records or
lists. A deferring update leaves a 32-row group's age only in its group word: the age column of its rows is stale until the
next update of the group takes the word, or a flush writes it back. Every other reader or writer must flush first, and
must flush every group its effect reaches, not only the groups of the rows it is given.

Each case runs frames that defer groups, calls nothing that reads records, checks with hnb_slab_deferred_groups (which
flushes nothing) that groups are deferred right then, runs one operation on the device and its restatement on the oracle,
then two frames, a full comparison (records, both lists, dead stack, metadata, draw args), six more frames (ages a stale
word froze would now differ) and a second comparison. The control runs every case again on a context with
HNB_DEFER_AGES=0: nothing is ever deferred there, and the results equal the same oracle.

C5 world (the authored recipes.c5_asset against the C oracle), one slab of 9173 rows:
- instance 0 at row 0, 4173 rows (ends inside a group), 4128 alive with lifetimes U(20, 30) s and the identity claim, so
  the floor tiles over its first 128 groups defer them. Its 45 dead rows hold filled records. Rows 5 and 1000 die in the
  last deferring frame, so the list the next update reads is a gather that names row r at position r - 1 or r - 2;
- instance 1 at row 4173 (inside instance 0's last group), 3000 rows, 2900 alive of age 0.5 dying from the third frame on:
  it gets no floor tiles and shares a group with instance 0;
- instance 2 at row 7173, 2000 rows, 1500 alive, in a batch of its own.
The sparks world runs tests.effects.drifting_sparks against the numpy oracle: shuffled dead stacks, capacities that are
not multiples of 32, a repack that gives instance 0 the claim, and spawns into instance 1 while instance 0 defers."""
import numpy as np
import pytest

from oracle import c_oracle as O
from tests.helpers import Instance, Lockstep, filled_c5, seeds, sparks_world
from tests.repack_ref import ref_repack
from tests.snapshot_ref import ref_restore, ref_snapshot

pytestmark = pytest.mark.gpu

STRIDE = 32
CAP_A, ALIVE_A = 4173, 4128
B0, CAP_B, ALIVE_B = 4173, 3000, 2900
C0, CAP_C, ALIVE_C = 7173, 2000, 1500
ROWS = C0 + CAP_C
DIE = (5, 1000)        # rows of instance 0 that die in the last deferring frame
RANGE = (70, 1070)     # inside instance 0, starting and ending inside a group
DT = 1.0 / 60.0


@pytest.fixture(params=[True, False], ids=["deferred", "control"])
def dctx(request, native, monkeypatch):
    """A fresh context; `control`: HNB_DEFER_AGES=0, so its updates never leave a group deferred."""
    if request.param:
        monkeypatch.delenv("HNB_DEFER_AGES", raising=False)
    else:
        monkeypatch.setenv("HNB_DEFER_AGES", "0")
    c = native.Context(0)
    c.defers = request.param
    try:
        yield c
    finally:
        c.close()


def deferred_now(ctx, slab, what):
    """The slab's deferred-group count right before `what`: non-zero, or 0 in the control."""
    n = ctx.slab_deferred_groups(slab)
    if ctx.defers:
        assert n > 0, f"{what}: no group is deferred, so the case proves nothing"
    else:
        assert n == 0, f"{what}: a group is deferred with HNB_DEFER_AGES=0"
    return n


def f32(x):
    return np.float32(x).view(np.uint32)


def c5_world(ctx, orc):
    """The C5 world of the module docstring after its deferring frames; returns (lock, next frame)."""
    from bevy_hanabi_b200 import recipes
    authored = recipes.c5_asset(ROWS).generate()
    assert "#define HNB_GROUP_AGE 1" in authored.generate_source()
    insts = [Instance(0, CAP_A, alive=ALIVE_A, seed=3), Instance(B0, CAP_B, alive=ALIVE_B, seed=4),
             Instance(C0, CAP_C, alive=ALIVE_C, seed=5)]
    fills = [(ALIVE_A, CAP_A - ALIVE_A, 31, 20.0, 30.0), (B0, ALIVE_B, 32, 0.55, 0.8), (C0, ALIVE_C, 33, 20.0, 30.0),
             (0, ALIVE_A, 34, 20.0, 30.0)]  # the last fill holds the claim
    lock = filled_c5(ctx, orc, insts, fills, batches=[[0, 1], [2]], effect=ctx.effect_compile(authored))
    ref, slab = lock.ref, lock.gpu.slab
    ref.particles[B0:B0 + ALIVE_B, 3] = f32(0.5)
    ctx.slab_upload_aos(slab, B0, ref.particles[B0:B0 + ALIVE_B])
    for r in DIE:
        ref.particles[r, 7] = f32(4.5 * DT)
        ctx.slab_upload_aos(slab, r, ref.particles[r:r + 1])
    f = 0
    while ref.metadata[0].alive_count == ALIVE_A:
        lock.step(f)
        f += 1
        assert f <= 8
    assert ref.metadata[0].alive_count == ALIVE_A - len(DIE) and f >= 4
    return lock, f


def device_buffer(ctx, words):
    d = ctx.device_alloc(max(words.nbytes, 16))
    ctx.device_upload(d, words)
    return d


def read_column(ref, i):
    """(column the next update reads, alive count) of instance i."""
    return ref.metadata[i].indirect_write_index, ref.metadata[i].alive_count


# ---- operations: each changes the device and the oracle alike ---------------------------------------------------------
def op_fill(lock, ctx, orc):
    """hnb_slab_fill_c5 over RANGE; its identity lists are put back by an upload (a fill lists the rows from its first)."""
    ref, slab, (first, end) = lock.ref, lock.gpu.slab, RANGE
    lists = ref.indirect[first:end].copy()
    scratch = ref.indirect.copy()  # the oracle's fill lists the rows too: only its records are kept
    orc.orc_fill_c5(O.ptr(ref.particles), O.ptr(scratch), first, end - first, 77, 20.0, 30.0)
    ctx.slab_fill_c5(slab, first, end - first, 77, 20.0, 30.0)
    ctx.slab_upload_indirect(slab, first, lists)


def _aged_range(ref, first, end, age):
    ref.particles[first:end, 3] = f32(age)
    return ref.particles[first:end].copy()


def op_upload_aos(lock, ctx, orc):
    lock.ctx.slab_upload_aos(lock.gpu.slab, RANGE[0], _aged_range(lock.ref, *RANGE, 0.75))


def op_import_aos_device(lock, ctx, orc):
    recs = _aged_range(lock.ref, *RANGE, 0.75)
    d = device_buffer(ctx, recs)
    try:
        ctx.slab_import_aos_device(lock.gpu.slab, RANGE[0], len(recs), d)
        ctx.sync()
    finally:
        ctx.device_free(d)


def op_reset_fill(lock, ctx, orc):
    """Instance 0's rows reset (lists and dead stack as a new slab's), then filled afresh."""
    ref, slab = lock.ref, lock.gpu.slab
    ctx.slab_reset_rows(slab, 0, CAP_A)
    ctx.slab_fill_c5(slab, 0, ALIVE_A, 78, 20.0, 30.0)
    orc.orc_indirect_reset(O.ptr(ref.indirect), 0, CAP_A)
    orc.orc_fill_c5(O.ptr(ref.particles), O.ptr(ref.indirect), 0, ALIVE_A, 78, 20.0, 30.0)


def _repack(i):
    def op(lock, ctx, orc):
        first, rows = lock.span(i)
        ctx.slab_repack(lock.gpu.slab, lock.gpu.effect, i, first, rows)
        ref_repack(lock.ref, i)
    return op


def _restore(i, age):
    """Instance i restored from the oracle's snapshot of it, every record given age `age`."""
    def op(lock, ctx, orc):
        snap = ref_snapshot(lock.ref, i)
        snap[16:].reshape(-1, STRIDE // 4)[:, 3] = f32(age)
        d = device_buffer(ctx, snap)
        try:
            first, rows = lock.span(i)
            ctx.instance_restore(lock.gpu.slab, lock.gpu.effect, i, first, rows, d, snap.nbytes)
            ctx.sync()
        finally:
            ctx.device_free(d)
        ref_restore(lock.ref, i, snap)
    return op


def _reversed_lists(ref):
    """Instance 0's indirect rows with the alive list the next update reads in reverse order."""
    read, alive = read_column(ref, 0)
    ref.indirect[:alive, read] = ref.indirect[:alive, read][::-1].copy()
    return ref.indirect[:CAP_A].copy()


def op_upload_indirect(lock, ctx, orc):
    ctx.slab_upload_indirect(lock.gpu.slab, 0, _reversed_lists(lock.ref))


def op_import_indirect_device(lock, ctx, orc):
    rows = _reversed_lists(lock.ref)
    d = device_buffer(ctx, rows)
    try:
        ctx.slab_import_indirect_device(lock.gpu.slab, 0, len(rows), d)
        ctx.sync()
    finally:
        ctx.device_free(d)


def _swap(device):
    """Live row 64 (of a deferred group) and dead row ALIVE_A + 3 trade places: list position 63 (deferred group 1) names
    the dead row, and the dead stack's entry of the dead row names row 64. Two one-row uploads, neither at a position of
    row 64's group: row 64's group then has a dead row, and the next update walks only 31 of its rows."""
    def op(lock, ctx, orc):
        ref, slab = lock.ref, lock.gpu.slab
        read, alive = read_column(ref, 0)
        r1, r2 = 64, ALIVE_A + 3
        p1 = int(np.flatnonzero(ref.indirect[:alive, read] == r1)[0])
        p2 = alive + int(np.flatnonzero(ref.indirect[alive:CAP_A, 2] == r2)[0])
        assert p1 // 32 != r1 // 32 and p2 // 32 != r1 // 32
        ref.indirect[p1, read] = r2
        ref.indirect[p2, 2] = r1
        for p in (p1, p2):
            if device:
                d = device_buffer(ctx, ref.indirect[p:p + 1].copy())
                try:
                    ctx.slab_import_indirect_device(slab, p, 1, d)
                    ctx.sync()
                finally:
                    ctx.device_free(d)
            else:
                ctx.slab_upload_indirect(slab, p, ref.indirect[p:p + 1])
    return op


def _insert_metadata(lock, **fields):
    N = lock.gpu.N
    md = lock.ref.metadata[0]
    for k, v in fields.items():
        setattr(md, k, v)
    lock.ctx.metadata_insert(0, N.EffectMetadata.from_buffer_copy(bytes(md)))


def op_shrink(lock, ctx, orc):
    """Instance 0 shrinks to its first 3000 rows and its first 2990 live particles; the rest are dropped. The group of rows
    2976-3007 keeps 16 walked rows."""
    read, _ = read_column(lock.ref, 0)
    assert lock.ref.indirect[:2990, read].max() < 3000
    _insert_metadata(lock, capacity=3000, alive_count=2990, max_spawn=10)


def op_end(lock, ctx, orc):
    """Instance 0 ends: a new instance takes its slice with no particle alive and spawns into it (below)."""
    _insert_metadata(lock, alive_count=0, max_spawn=CAP_A, particle_counter=0)


def op_download_aos(lock, ctx, orc):
    first, end = RANGE
    np.testing.assert_array_equal(ctx.slab_download_aos(lock.gpu.slab, first, end - first, STRIDE), lock.ref.particles[first:end])


def op_export_aos_device(lock, ctx, orc):
    first, end = 1500, 2700
    d = ctx.device_alloc((end - first) * STRIDE)
    try:
        ctx.slab_export_aos_device(lock.gpu.slab, first, end - first, d)
        got = ctx.device_download(d, (end - first) * STRIDE).reshape(-1, STRIDE // 4)
    finally:
        ctx.device_free(d)
    np.testing.assert_array_equal(got, lock.ref.particles[first:end])


def op_instance_snapshot(lock, ctx, orc):
    want = ref_snapshot(lock.ref, 0)
    nbytes = ctx.instance_snapshot_bytes(STRIDE, CAP_A)
    d = ctx.device_alloc(nbytes)
    try:
        ctx.instance_snapshot(lock.gpu.slab, lock.gpu.effect, 0, 0, CAP_A, d, nbytes)
        got = ctx.device_download(d, want.nbytes)
    finally:
        ctx.device_free(d)
    np.testing.assert_array_equal(got, want)


def op_slab_checksum(lock, ctx, orc):
    """Rows 2100-3599 hash as the oracle's records do in a slab that never deferred."""
    first, count = 2100, 1500
    got = ctx.slab_checksum(lock.gpu.slab, first, count)
    plain = ctx.slab_create(ROWS, STRIDE)
    ctx.slab_upload_aos(plain, 0, lock.ref.particles)
    assert got == ctx.slab_checksum(plain, first, count)
    ctx.slab_destroy(plain)


def op_position_readers(lock, ctx, orc):
    """Bounds, depth order, cull and cull for two views of batch 0: they read positions only, so the count stays."""
    slab, launch = lock.gpu.slab, lock.gpu.launches()[0]
    before = ctx.slab_deferred_groups(slab)
    everything = np.tile(np.array([0, 0, 0, 1], dtype=np.float32), 6)  # six planes every position passes
    bufs = {k: ctx.device_alloc(n) for k, n in (("out", 64), ("planes", 32), ("order", 4 * ROWS), ("frusta", 2 * 2 * 96),
                                                ("visible", 2 * 4 * ROWS), ("args", 2 * 2 * 20))}
    try:
        ctx.device_upload(bufs["planes"], np.tile(np.array([0, 0, 1, 0], dtype=np.float32), 2).view(np.uint32))
        ctx.device_upload(bufs["frusta"], np.tile(everything, 4).view(np.uint32))
        calls = [("bounds", lambda: ctx.batch_bounds(launch, bufs["out"], 2)),
                 ("depth order", lambda: ctx.batch_depth_order(launch, bufs["planes"], 2, bufs["order"], ROWS)),
                 ("cull", lambda: ctx.batch_cull(launch, bufs["frusta"], 2, 0, 0, bufs["visible"], ROWS, bufs["args"], 2)),
                 ("cull views", lambda: ctx.batch_cull_views(launch, 2, bufs["frusta"], 2, 0, 0, bufs["visible"], ROWS,
                                                             bufs["args"], 2))]
        for name, call in calls:
            call()
            assert ctx.slab_deferred_groups(slab) == before, f"{name} changed the deferred words"
        visible = ctx.device_download(bufs["args"], 2 * 2 * 20).reshape(2, 2, 5)[:, :, 1]
        assert (visible == [[lock.ref.metadata[0].alive_count, lock.ref.metadata[1].alive_count]] * 2).all()
    finally:
        for d in bufs.values():
            ctx.device_free(d)


CASES = {
    "fill": op_fill,
    "upload_aos": op_upload_aos,
    "import_aos_device": op_import_aos_device,
    "reset_rows_and_fill": op_reset_fill,
    "repack": _repack(0),
    "repack_neighbour": _repack(1),
    "restore": _restore(0, 0.25),
    "restore_neighbour": _restore(1, 0.5),
    "upload_indirect": op_upload_indirect,
    "import_indirect_device": op_import_indirect_device,
    "swap_alive_dead_upload": _swap(device=False),
    "swap_alive_dead_import": _swap(device=True),
    "metadata_shrinks": op_shrink,
    "metadata_ends": op_end,
    "download_aos": op_download_aos,
    "export_aos_device": op_export_aos_device,
    "instance_snapshot": op_instance_snapshot,
    "slab_checksum": op_slab_checksum,
    "position_readers": op_position_readers,
}


@pytest.mark.parametrize("case", list(CASES))
def test_c5_operation_with_groups_deferred(dctx, orc, case):
    lock, f = c5_world(dctx, orc)
    deferred_now(dctx, lock.gpu.slab, case)
    CASES[case](lock, dctx, orc)
    spawns = [300, 0, 0] if case == "metadata_ends" else None
    for k in range(8):
        lock.step(f + k, spawns)
        if k in (1, 7):
            lock.compare(f"{case}, frame {f + k}")
    if case == "metadata_ends":
        assert lock.ref.metadata[0].alive_count == 8 * 300
    if not dctx.defers:
        assert dctx.slab_deferred_groups(lock.gpu.slab) == 0


@pytest.mark.parametrize("writer", ["upload_aos", "upload_indirect"])
def test_sparks_spawn_beside_deferred_groups(dctx, orc, writer):
    """drifting_sparks: instance 0 spawns one burst and is repacked (the claim), then defers while instance 1 spawns from
    its shuffled dead stack; then `writer` rewrites part of instance 0's records (ages), or instance 1's whole alive list
    (reversed)."""
    asset, ref = sparks_world([2500, 1700], dt=0.005)
    fields = {fl.name: fl.offset // 4 for fl in asset.particle_layout()[0]}
    lock = Lockstep(dctx, orc, ref, asset, seeds=seeds)
    assert "#define HNB_GROUP_AGE 1" in asset.generate().generate_source()
    ctx, slab = dctx, lock.gpu.slab
    lock.step(0, [2000, 0])
    lock.step(1, [0, 0])
    ctx.slab_repack(slab, lock.gpu.effect, 0, 0, 2500)
    ref_repack(ref, 0)
    for f in range(2, 7):
        lock.step(f, [0, 90])
    deferred_now(ctx, slab, writer)
    if writer == "upload_aos":
        first, end = RANGE
        ref.particles[first:end, fields["age"]] = f32(0.02)
        ctx.slab_upload_aos(slab, first, ref.particles[first:end])
    else:
        first, rows = lock.span(1)
        read, alive = read_column(ref, 1)
        ref.indirect[first:first + alive, read] = ref.indirect[first:first + alive, read][::-1].copy()
        ctx.slab_upload_indirect(slab, first, ref.indirect[first:first + rows])
    for k in range(8):
        lock.step(7 + k, [0, 90])
        if k in (1, 7):
            lock.compare(f"sparks {writer}, frame {7 + k}")
    assert ref.metadata[0].alive_count == 2000
