"""hnb_instance_snapshot / hnb_instance_restore on the device. Every buffer is compared bit for bit with the oracle
(tests/snapshot_ref.py applied at the same point) before and after every frame, on churned worlds restored into the same
slice, another offset, another slab, a larger and a smaller capacity, and a second context. Also: the snapshot bytes
themselves, the source left untouched, a host round trip of the prefix, two restores that stay identical for 30 frames,
a 64 Mi-row C5 round trip, and refusals that leave the state untouched."""
from __future__ import annotations

import numpy as np
import pytest

from bevy_hanabi_b200 import _native as N
from bevy_hanabi_b200 import recipes
from bevy_hanabi_b200 import runtime as R
from oracle.hanabi_oracle import EffectOracle, pcg_hash
from tests.helpers import GpuWorld, Instance, RefWorld, assert_world_equal
from tests.snapshot_ref import HEADER_WORDS, SNAPSHOT_MAGIC, ref_restore, ref_snapshot
from tests.test_gpu_events import _assets as _event_assets
from tests.test_gpu_ribbons import _ribbon_asset
from tests.test_gpu_scene import _drifting_sparks
from tests.test_gpu_tile_shapes import EFFECTS, _asset, _world

pytestmark = pytest.mark.gpu

SENTINEL = np.uint32(0xA5A5A5A5)


def _seeds(n, f):
    return [int(s) for s in pcg_hash(np.arange(n, dtype=np.uint32) + np.uint32(100 * f + 7))]


class Side:
    """A GpuWorld and the oracle world it must equal."""

    def __init__(self, ctx, asset, ref, *, props=None, sector=False, slot=False):
        blobs = None
        if props is not None:
            blobs = [asset.serialize_properties(props(i)) for i in range(len(ref.instances))]
            for i in range(len(ref.instances)):
                ref.metadata[i].properties_array_index = i
        ref.slot_order = slot
        self.ctx, self.ref, self.slot, self.fresh = ctx, ref, slot, True
        self.eo = EffectOracle(asset, {i: props(i) for i in range(len(ref.instances))} if props else None)
        self.gpu = GpuWorld(ctx, ref, asset.generate(sector_planes=sector, slot_order=slot), property_blobs=blobs, sector_planes=sector)

    def compare(self, what):
        if self.fresh:  # no frame ran yet: the context has no per-frame tables of this world to read back
            ctx, ref, n = self.ctx, self.ref, len(self.ref.instances)
            ctx.sync()
            got = {"particles": ctx.slab_download_aos(self.gpu.slab, 0, ref.slab_rows, self.gpu.stride),
                   "indirect": ctx.slab_download_indirect(self.gpu.slab, 0, ref.slab_rows),
                   "metadata": np.stack([np.frombuffer(bytes(ctx.read_metadata(i)), dtype=np.uint32) for i in range(n)]),
                   "draw": np.concatenate([np.frombuffer(bytes(ctx.read_draw_args(i)), dtype=np.uint32) for i in range(n)])}
            for k, want in (("particles", ref.particles), ("indirect", ref.indirect), ("metadata", ref.metadata_rows()), ("draw", ref.draw)):
                np.testing.assert_array_equal(got[k], want, err_msg=f"{what}: {k}")
        else:
            assert_world_equal(self.ref, self.gpu.pull(), what=what)
        if self.slot:
            assert self.ctx.read_debug(False)[15] == 0, f"{what}: alive bitmap and counters disagree"

    def frames(self, orc, schedule, start=0, what=""):
        for f, spawns in enumerate(schedule, start=start):
            self.ref.sim.time = np.float32(f) * self.ref.sim.delta_time
            self.ref.set_spawns(spawns, _seeds(len(spawns), f))
            self.eo.frame(self.ref, orc)
            self.gpu.frame()
            self.fresh = False
            self.compare(f"{what} frame {f}")

    def span(self, i):
        inst = self.ref.instances[i]
        return inst.slab_offset, inst.capacity


class Buffers:
    """Device buffers of one test, freed at its end."""

    def __init__(self):
        self.live = []

    def alloc(self, ctx, nbytes):
        p = ctx.device_alloc(nbytes)
        self.live.append((ctx, p))
        return p

    def free(self):
        for ctx, p in self.live:
            ctx.device_free(p)
        self.live = []


@pytest.fixture()
def bufs():
    b = Buffers()
    yield b
    b.free()


def _pull_equal(a, b, what):
    for k in a:
        np.testing.assert_array_equal(a[k], b[k], err_msg=f"{what}: {k}")


def snapshot(side, i, bufs):
    """Snapshot instance i into a fresh buffer of instance_snapshot_bytes filled with a sentinel; checks the bytes against
    ref_snapshot, that nothing past them was written and that the source kept every byte. Returns (ptr, bytes, words)."""
    ctx, first_rows = side.ctx, side.span(i)
    nbytes = ctx.instance_snapshot_bytes(side.gpu.stride, first_rows[1])
    assert nbytes == 64 + first_rows[1] * side.gpu.stride
    buf = bufs.alloc(ctx, nbytes)
    ctx.device_upload(buf, np.full(nbytes // 4, SENTINEL, dtype=np.uint32))
    before = side.gpu.pull()
    ctx.instance_snapshot(side.gpu.slab, side.gpu.effect, i, *first_rows, buf, nbytes)
    got = ctx.device_download(buf, nbytes)
    want = ref_snapshot(side.ref, i)
    np.testing.assert_array_equal(got[:len(want)], want, err_msg="snapshot header and records")
    assert (got[len(want):] == SENTINEL).all(), "bytes past 64 + n * stride were written"
    _pull_equal(before, side.gpu.pull(), "the snapshot modified its source")
    return buf, nbytes, want


def restore(side, i, buf, nbytes, words):
    side.ctx.instance_restore(side.gpu.slab, side.gpu.effect, i, *side.span(i), buf, nbytes)
    m = ref_restore(side.ref, i, words, nbytes)
    side.compare(f"after the restore into instance {i}")
    return m


def _sparks_ref(caps, dt=0.05, seed=1):
    _, size, _ = _drifting_sparks(max(caps)).particle_layout()
    insts, off = [], 0
    for i, c in enumerate(caps):
        insts.append(Instance(off, c, alive=0, seed=11 + 7 * i))
        off += c
    ref = RefWorld(off, size // 4, insts, dt=dt)
    rng = np.random.default_rng(seed)
    for inst in insts:
        rows = slice(inst.slab_offset, inst.slab_offset + inst.capacity)
        ref.indirect[rows, 2] = rng.permutation(ref.indirect[rows, 2])
    return ref


def _is_identity(ref, i):
    md, base = ref.metadata[i], ref.instances[i].slab_offset
    lst = ref.indirect[base:base + md.alive_count, md.indirect_write_index]
    return bool((lst == np.arange(len(lst))).all())


# frames after a restore; _churned_sparks runs 24 frames at 300 spawns (lifetimes of 4 to 18 frames) before a snapshot
AFTER = [[300]] * 8


def _churned_sparks(ctx, orc, caps=(4096,), **kw):
    asset = _drifting_sparks(max(caps))
    side = Side(ctx, asset, _sparks_ref(list(caps)), **kw)
    side.frames(orc, [[300] + [0] * (len(caps) - 1)] * 24, what="churn")
    assert not _is_identity(side.ref, 0) and side.ref.metadata[0].alive_count > min(2000, caps[0] // 2)
    return asset, side


@pytest.mark.parametrize("mode", ["default", "sector", "slot"])
def test_churned_sparks_into_their_own_slice(ctx, orc, bufs, mode):
    kw = dict(sector=mode == "sector", slot=mode == "slot")
    asset, side = _churned_sparks(ctx, orc, **kw)
    buf, nbytes, words = snapshot(side, 0, bufs)
    assert restore(side, 0, buf, nbytes, words) == side.ref.metadata[0].alive_count
    assert _is_identity(side.ref, 0)
    side.frames(orc, AFTER, start=24, what="after the restore")


@pytest.mark.parametrize("target", ["other_offset", "other_slab", "larger", "smaller", "other_context"])
def test_churned_sparks_moved(ctx, orc, bufs, native, target):
    """Into instance 1 of the same slab; into the middle instance of another slab; into 6000 and 1500 rows (fewer than are
    alive: the first 1500 in alive-list order are kept); into a slab of a second context on the same device."""
    caps = (4096, 4096) if target == "other_offset" else (4096,)
    asset, src = _churned_sparks(ctx, orc, caps)
    buf, nbytes, words = snapshot(src, 0, bufs)
    n = int(words[3])
    ctx2 = native.Context(0) if target == "other_context" else ctx
    try:
        if target == "other_offset":
            dst, i = src, 1
        else:
            cap = {"larger": 6000, "smaller": 1500}.get(target, 4096)
            dst, i = Side(ctx2, asset, _sparks_ref([777, cap, 500], seed=2)), 1
        assert restore(dst, i, buf, nbytes, words) == min(n, dst.span(i)[1])
        spawns = [[300, 300]] * 8 if target == "other_offset" else [[50, 300, 40]] * 8
        dst.frames(orc, spawns, start=24, what=f"{target}, after the restore")
    finally:
        if ctx2 is not ctx:
            ctx2.close()


def test_churned_ribbons(ctx, orc, bufs):
    """Snapshot in sorted order, restored into another slab; the next frames sort again."""
    asset = _ribbon_asset(4096)
    fields, size, _ = asset.particle_layout()

    def world(caps, seed):
        insts, off = [], 0
        for i, c in enumerate(caps):
            insts.append(Instance(off, c, alive=0, seed=seed + i))
            off += c
        ref = RefWorld(off, size // 4, insts, dt=1 / 30)
        ref.set_sort_keys(fields)
        return ref

    src = Side(ctx, asset, world([4096], 3))
    src.frames(orc, [[900 if f % 4 == 0 else 23] for f in range(16)], what="churn")
    buf, nbytes, words = snapshot(src, 0, bufs)
    dst = Side(ctx, asset, world([300, 4096], 9))
    restore(dst, 1, buf, nbytes, words)
    dst.frames(orc, [[0, 900 if f % 4 == 0 else 23] for f in range(16, 26)], start=16, what="ribbons, after the restore")


@pytest.mark.parametrize("name", list(EFFECTS))
def test_churned_wide_records(ctx, orc, bufs, name):
    """48 and 64-byte records (K = 2), 96 and 144 bytes (K = 1), with per-instance properties where the effect has them:
    instance 0 churns, its snapshot goes to instance 1 of the same slab."""
    ref = _world(name, [3000, 3000])
    side = Side(ctx, _asset(name, 3000), ref, props=EFFECTS[name][3])
    side.frames(orc, [[500, 0]] * 12, what="churn")
    buf, nbytes, words = snapshot(side, 0, bufs)
    restore(side, 1, buf, nbytes, words)
    side.frames(orc, [[300, 300]] * 8, start=12, what="after the restore")


def test_host_round_trip_of_the_prefix(ctx, orc, bufs):
    """Read the header, download the 64 + n * stride prefix, upload it into a buffer of exactly that size in a fresh
    context's slab, restore from there."""
    asset, src = _churned_sparks(ctx, orc)
    buf, nbytes, _ = snapshot(src, 0, bufs)
    header = np.frombuffer(ctx.device_download(buf, 64).tobytes(), dtype=np.uint32)
    assert header[0] == SNAPSHOT_MAGIC and header[1] == 1 and header[2] == src.gpu.stride and header[5] == 4096
    assert not header[6:].any(), "reserved words are zero"
    prefix_bytes = 64 + int(header[3]) * int(header[2])
    host = ctx.device_download(buf, prefix_bytes)
    dst = Side(ctx, asset, _sparks_ref([4096], seed=5))
    copy = bufs.alloc(ctx, prefix_bytes)
    ctx.device_upload(copy, host)
    assert restore(dst, 0, copy, prefix_bytes, host) == header[3]
    dst.frames(orc, AFTER, start=24, what="after the host round trip")


def test_two_restores_stay_identical(ctx, orc, bufs, native):
    """One snapshot restored into two identical fresh slabs, each in a context of its own (a context's metadata rows and
    tables are shared by its slabs), then 30 frames with the same tables: every buffer of the two stays identical (and
    equal to the oracle at the end)."""
    asset, src = _churned_sparks(ctx, orc)
    buf, nbytes, words = snapshot(src, 0, bufs)
    ctxs = [native.Context(0) for _ in range(2)]
    try:
        sides = [Side(c, asset, _sparks_ref([4096], seed=7)) for c in ctxs]
        for side in sides:
            restore(side, 0, buf, nbytes, words)
        for f in range(24, 54):
            pulled = []
            for side in sides:
                side.ref.sim.time = np.float32(f) * side.ref.sim.delta_time
                side.ref.set_spawns([300], _seeds(1, f))
                side.eo.frame(side.ref, orc)
                side.gpu.frame()
                pulled.append(side.gpu.pull())
            _pull_equal(pulled[0], pulled[1], f"frame {f}: the two restored instances")
        for side in sides:
            side.fresh = False
            side.compare("after 30 frames")
    finally:
        for c in ctxs:
            c.close()


def test_c5_64_mi_round_trip(native):
    """A filled 64 Mi-row C5 instance (2 GiB of records): snapshot, restore into a second slab; both slabs have the same
    hnb_slab_checksum over every row and the same index columns, and the restored metadata row carries the count."""
    P = 64 << 20
    c = native.Context(0)
    buf = None
    try:
        effect = c.effect_compile(recipes.c5_lowered())
        slabs = [c.slab_create(P, 32) for _ in range(2)]
        c.slab_fill_c5(slabs[0], 0, P, 99, 0.5, 2.0)
        for i in range(2):
            md = R.initial_metadata(P, i, 8)
            if i == 0:
                md.alive_count, md.max_spawn, md.particle_counter = P, 0, 12345
            c.metadata_insert(i, md)
        nbytes = c.instance_snapshot_bytes(32, P)
        buf = c.device_alloc(nbytes)
        c.instance_snapshot(slabs[0], effect, 0, 0, P, buf, nbytes)
        c.instance_restore(slabs[1], effect, 1, 0, P, buf, nbytes)
        c.sync()
        assert c.slab_checksum(slabs[1], 0, P) == c.slab_checksum(slabs[0], 0, P)
        assert c.slab_checksum_indirect(slabs[1], 0, P) == c.slab_checksum_indirect(slabs[0], 0, P)
        md = c.read_metadata(1)
        assert (md.alive_count, md.max_spawn, md.particle_counter) == (P, 0, 12345)
    finally:
        if buf:
            c.device_free(buf)
        c.close()


def test_refusals_leave_the_state_untouched(ctx, orc, bufs):
    asset, side = _churned_sparks(ctx, orc, caps=(2000,))
    gpu = side.gpu
    before = gpu.pull()
    nbytes = ctx.instance_snapshot_bytes(gpu.stride, 2000)
    buf = bufs.alloc(ctx, nbytes + 16)
    ctx.device_upload(buf, np.full((nbytes + 16) // 4, SENTINEL, dtype=np.uint32))
    ctx.instance_snapshot(gpu.slab, gpu.effect, 0, 0, 2000, buf, nbytes)
    ctx.sync()
    snap = ctx.device_download(buf, nbytes + 16)
    other_stride = ctx.effect_compile(_asset("vec4x2_64", 2000).generate())
    sector = ctx.effect_compile(asset.generate(sector_planes=True))
    parent = _event_assets()[0]
    emitting = ctx.effect_compile(parent.generate(num_event_bindings=1))
    assert parent.particle_layout()[1] == 32, "the emitting effect differs from the slab in its flag only"
    common = [("rows outside the slab", gpu.effect, 0, 1, 2000), ("rows outside the slab", gpu.effect, 0, 0, 2001),
              ("metadata row out of range", gpu.effect, 1 << 20, 0, 2000), ("stride does not match", other_stride, 0, 0, 2000),
              ("SECTOR_PLANES", sector, 0, 0, 2000), ("GPU spawn events", emitting, 0, 0, 2000)]
    cases = [(call, why, effect, row, first, rows, buf, nbytes) for call in ("snapshot", "restore") for why, effect, row, first, rows in common]
    cases += [(call, "NULL or not 16-byte aligned", gpu.effect, 0, 0, 2000, p, nbytes) for call in ("snapshot", "restore") for p in (0, buf + 4, buf + 8)]
    cases += [("snapshot", "dst_bytes", gpu.effect, 0, 0, 2000, buf, nbytes - 1), ("restore", "src_bytes", gpu.effect, 0, 0, 2000, buf, 63)]
    for call, why, effect, row, first, rows, p, size in cases:
        fn = ctx.instance_snapshot if call == "snapshot" else ctx.instance_restore
        with pytest.raises(N.HanabiError) as e:
            fn(gpu.slab, effect, row, first, rows, p, size)
        assert e.value.code == N.HNB_ERR_INVALID_ARG and why in e.value.message, (call, e.value.message)
        _pull_equal(before, gpu.pull(), f"{call}: {why}")
        np.testing.assert_array_equal(ctx.device_download(buf, nbytes + 16), snap, err_msg=f"{call}: {why}: the buffer")
    # rows == 0 is a no-op for both
    ctx.instance_snapshot(gpu.slab, gpu.effect, 0, 0, 0, buf, 64)
    ctx.instance_restore(gpu.slab, gpu.effect, 0, 0, 0, buf, nbytes)
    _pull_equal(before, gpu.pull(), "rows == 0")
    np.testing.assert_array_equal(ctx.device_download(buf, nbytes + 16), snap, err_msg="rows == 0: the buffer")
    assert snap[HEADER_WORDS - 1] == 0 and snap[3] == side.ref.metadata[0].alive_count
