"""hnb_slab_repack_events, hnb_instance_snapshot_events and hnb_instance_restore_events on the device, in the two-channel
emitter scene of tests.effects.emitter_assets (channel 0: Always; channel 1: OnDie x 4, which overflows its 256-entry
buffer), with and without HNB_EFFECT_ORDERED_EVENTS, at the slab-size tile rule and at 3 forced sub-tiles. The oracle runs
the same frames and applies tests/emitter_relocation_ref.py where the device relocates the parent. Every buffer is
compared after every frame: event buffers exactly in ordered mode, as multisets otherwise (as tests.helpers.emitter_scene
does); everything else exactly."""
from __future__ import annotations

from collections import Counter

import numpy as np
import pytest

from bevy_hanabi_b200 import _native as N
from bevy_hanabi_b200 import runtime as R
from tests.effects import EVENT_CAP, emitter_assets
from tests.emitter_relocation_ref import dead_count, inverse, ref_repack_events, ref_restore_events, ref_snapshot_events
from tests.helpers import Instance, RefWorld, oracle_append_events, oracle_child_init, pcg_hash, tiled_ctx  # noqa: F401
from tests.snapshot_ref import ref_restore, ref_snapshot

pytestmark = pytest.mark.gpu

PCAP, CCAP = 1024, 4096
SPAWNS = [700, 0, 0, 150, 0, 0, 0, 800, 0, 0, 0, 0, 100, 0, 0, 0, 0, 0, 0, 0, 300, 0, 0, 0, 0]
DT = 1.0 / 30.0


class Scene:
    """The emitter scene on one context: metadata rows 0, 1 = the children, 2 = the parent; child-info rows 0, 1 = its
    channels. The parent's instance sits at slab row `p_first` of its slab; the oracle keeps it at row 0 of its own world
    (the lists hold instance-local values, the dead stack slab-global ones)."""

    def __init__(self, ctx, orc, ordered):
        from oracle.hanabi_oracle import EffectOracle
        self.ctx, self.orc, self.ordered = ctx, orc, ordered
        self.parent, self.children = emitter_assets(PCAP)
        p_fx = self.parent.generate(num_event_bindings=2, ordered_events=ordered)
        c_fx = [c.generate(parent=self.parent) for c in self.children]
        self.p_stride, self.c_stride = p_fx.particle_stride, c_fx[0].particle_stride
        self.p_fx, self.c_fx = p_fx, c_fx
        self.pw = RefWorld(PCAP, self.p_stride // 4, [Instance(0, PCAP, alive=0, seed=1)], dt=DT)
        self.cw = [RefWorld(CCAP, self.c_stride // 4, [Instance(0, CCAP, alive=0, seed=2 + k)], dt=DT) for k in (0, 1)]
        self.po, self.co = EffectOracle(self.parent), [EffectOracle(c) for c in self.children]
        self.events = [np.zeros(EVENT_CAP, dtype=np.uint32) for _ in (0, 1)]
        self.event_count = [0, 0]
        self.all_emitted = [[], []]
        self.overflowed = False
        self.p_first = 0
        self.p_slab = ctx.slab_create(PCAP, self.p_stride)
        self.c_slab = [ctx.slab_create(CCAP, self.c_stride) for _ in (0, 1)]
        self.p_eff = ctx.effect_compile(p_fx)
        self.c_eff = [ctx.effect_compile(fx) for fx in c_fx]
        self.evbuf = [ctx.event_buffer_create(EVENT_CAP) for _ in (0, 1)]
        for k in (0, 1):
            ctx.child_info_insert(k, 0, 0)
            md_c = R.initial_metadata(CCAP, k, self.c_stride // 4)
            md_c.global_child_index, md_c.local_child_index = k, k
            ctx.metadata_insert(k, md_c)
            ctx.draw_args_insert(k)
        md_p = R.initial_metadata(PCAP, 2, self.p_stride // 4)
        md_p.base_child_index = 0
        ctx.metadata_insert(2, md_p)
        ctx.draw_args_insert(2)

    def check_events(self, what):
        """What the last update left in the two buffers: exact in ordered mode, else the same multiset (on overflow, a
        sub-multiset of what was emitted); the oracle then consumes the device's order."""
        ctx = self.ctx
        n_valid = []
        for k in (0, 1):
            assert ctx.read_child_info(k).event_count == self.event_count[k], f"{what}: channel {k} event_count"
            nv = min(self.event_count[k], EVENT_CAP)
            self.overflowed |= self.event_count[k] > EVENT_CAP
            got = ctx.event_buffer_download(self.evbuf[k], 0, EVENT_CAP)
            if self.ordered:
                np.testing.assert_array_equal(got[:nv], self.events[k][:nv], err_msg=f"{what}: channel {k} events")
            elif self.event_count[k] <= EVENT_CAP:
                assert sorted(got[:nv].tolist()) == sorted(self.events[k][:nv].tolist()), f"{what}: channel {k} events"
            else:
                emitted, kept = Counter(self.all_emitted[k]), Counter(got[:nv].tolist())
                assert all(kept[p] <= emitted[p] for p in kept), f"{what}: channel {k}: an event nobody emitted"
            self.events[k][:nv] = got[:nv]
            n_valid.append(nv)
        return n_valid

    def step(self, f):
        ctx, spawn = self.ctx, SPAWNS[f]
        seed_p = int(pcg_hash(np.array([5000 + f], dtype=np.uint32))[0])
        seed_c = [int(pcg_hash(np.array([6000 + 10 * f + k], dtype=np.uint32))[0]) for k in (0, 1)]
        ctx.upload_spawners([R.make_spawner(spawn=0, seed=seed_c[k], effect_metadata_index=k, draw_indirect_index=k, slab_offset=0,
                                            parent_slab_offset=self.p_first) for k in (0, 1)]
                            + [R.make_spawner(spawn=spawn, seed=seed_p, effect_metadata_index=2, draw_indirect_index=2, slab_offset=self.p_first)])
        ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, 1), N.BatchInfo(0, 0, 1, 0, 1, 1), N.BatchInfo(0, 0, 2, 0, 2, 1)], [0, 0, 0])
        ctx.set_sim_params(DT, f * DT, 3)
        n_valid = self.check_events(f"frame {f}")
        ctx.simulate([N.BatchLaunch.make(self.c_eff[0], self.c_slab[0], 0, 0, parent_slab=self.p_slab, consume_events=self.evbuf[0]),
                      N.BatchLaunch.make(self.c_eff[1], self.c_slab[1], 1, 0, parent_slab=self.p_slab, consume_events=self.evbuf[1]),
                      N.BatchLaunch.make(self.p_eff, self.p_slab, 2, spawn, emit_events=self.evbuf)])
        pw, cw = self.pw, self.cw
        t = np.float32(f * DT)
        pw.sim.time = t
        for k in (0, 1):
            cw[k].sim.time = t
            cw[k].set_spawns([0], [seed_c[k]])
            oracle_child_init(self.children[k], self.co[k], cw[k], self.po, pw, self.events[k], n_valid[k], seed_c[k])
        pw.set_spawns([spawn], [seed_p])
        self.po.init_pass(pw)
        self.event_count = [0, 0]
        for w in (cw[0], cw[1], pw):
            w.oracle_indirect(self.orc)
            w.oracle_prefix_sum(self.orc)
        for k in (0, 1):
            self.co[k].update_pass(cw[k])
        self.po.update_pass(pw)
        for channel, counts in self.po.last_emitted:
            self.event_count[channel] = oracle_append_events(pw, counts, self.events[channel], self.event_count[channel])
            rows_read = pw.indirect[:pw.metadata[0].max_update, 1 - pw.metadata[0].indirect_write_index]
            self.all_emitted[channel] = np.repeat(rows_read, counts[:len(rows_read)]).tolist()
        self.compare(f"frame {f}")

    def pulled(self):
        ctx = self.ctx
        ctx.sync()
        out = []
        for world, slab, row, stride, first, rows in ((self.cw[0], self.c_slab[0], 0, self.c_stride, 0, CCAP),
                                                      (self.cw[1], self.c_slab[1], 1, self.c_stride, 0, CCAP),
                                                      (self.pw, self.p_slab, 2, self.p_stride, self.p_first, PCAP)):
            ind = ctx.slab_download_indirect(slab, first, rows).copy()
            ind[:, 2] -= np.uint32(first)
            out.append((world, row, np.frombuffer(bytes(ctx.read_metadata(row)), dtype=np.uint32), ind,
                        ctx.slab_download_aos(slab, first, rows, stride)))
        return out

    def compare(self, what, draw=True):
        for world, row, m_gpu, ind, particles in self.pulled():
            m_ref = world.metadata_rows()[0].copy()
            m_ref[5] = row
            for fld in (7, 8, 9, 10):
                m_ref[fld] = m_gpu[fld]
            np.testing.assert_array_equal(m_gpu, m_ref, err_msg=f"{what}: metadata row {row}")
            if draw:
                assert self.ctx.read_draw_args(row).instance_count == world.draw[1], f"{what}: draw args {row}"
            np.testing.assert_array_equal(ind, world.indirect, err_msg=f"{what}: row {row}: lists")
            np.testing.assert_array_equal(particles, world.particles, err_msg=f"{what}: row {row}: particles")

    def adopt(self, world, slab, first, rows, stride, records, m):
        """After a restore into a fresh slab: the world takes the device's records from row `records` on, its dead-stack
        entries below m and its alive-list entries from m on. No pass reads them before writing them (a restore leaves
        them as they were)."""
        ind = self.ctx.slab_download_indirect(slab, first, rows).copy()
        ind[:, 2] -= np.uint32(first)
        world.indirect[:m, 2] = ind[:m, 2]
        world.indirect[m:, :2] = ind[m:, :2]
        world.particles[records:] = self.ctx.slab_download_aos(slab, first, rows, stride)[records:]

    def pending(self):
        """Both channels have events, and their buffers are the device's."""
        assert self.event_count[0] > 0 and self.event_count[1] > 0, self.event_count
        self.ctx.sync()
        return [self.ctx.event_buffer_download(self.evbuf[k], 0, EVENT_CAP) for k in (0, 1)]

    def translate_emitted(self, inv):
        self.all_emitted = [inv[np.array(e, dtype=np.int64)].tolist() for e in self.all_emitted]


@pytest.fixture()
def bufs():
    live = []

    def alloc(ctx, nbytes):
        p = ctx.device_alloc(nbytes)
        live.append((ctx, p))
        return p
    yield alloc
    for ctx, p in live:
        ctx.device_free(p)


TILES = pytest.mark.parametrize("tiled_ctx", [None, 3], ids=["rule", "3sub"], indirect=True)
MODES = pytest.mark.parametrize("ordered", [False, True], ids=["default", "ordered"])
RELOCATE_AT = 9  # after frame 8: the 800-particle burst of frame 7 is dying, channel 1 is full and overflowing


def _scene(tiled_ctx, orc, ordered, frames=RELOCATE_AT):
    tiled_ctx.tile_batch = 2  # the parent: 32-byte records, 128-row sub-tiles
    scene = Scene(tiled_ctx, orc, ordered)
    for f in range(frames):
        scene.step(f)
    return scene


def _sync_events(scene, what):
    """The oracle consumes the device's buffer order (default mode), as the next frame would."""
    scene.check_events(what)


@TILES
@MODES
def test_repack_mid_run(tiled_ctx, orc, ordered):
    """1. The parent repacked between frames 8 and 9 with events pending on both channels, then ten more frames against
    the oracle repacked the same way."""
    scene = _scene(tiled_ctx, orc, ordered)
    scene.pending()
    _sync_events(scene, "before the repack")
    md = scene.pw.metadata[0]
    assert dead_count(md, md.alive_count, PCAP) > 0, "the last update freed slots"
    inv = inverse(scene.pw, 0)
    scene.ctx.slab_repack_events(scene.p_slab, scene.p_eff, 2, 0, PCAP, scene.evbuf)
    ref_repack_events(scene.pw, 0, scene.events, scene.event_count)
    scene.translate_emitted(inv)
    scene.compare("after the repack", draw=False)
    for f in range(RELOCATE_AT, RELOCATE_AT + 10):
        scene.step(f)
    assert scene.overflowed


@TILES
@MODES
def test_snapshot_into_its_own_slice_equals_the_repack(tiled_ctx, orc, ordered, bufs):
    """2. A version-2 snapshot restored into the parent's own slice leaves every buffer the repack leaves (records up to
    n + D); ten more frames follow."""
    scene = _scene(tiled_ctx, orc, ordered)
    scene.pending()
    _sync_events(scene, "before the snapshot")
    ctx = scene.ctx
    nbytes = ctx.instance_snapshot_events_bytes(scene.p_stride, PCAP, [EVENT_CAP, EVENT_CAP])
    assert nbytes == 64 + PCAP * scene.p_stride + 8 * EVENT_CAP
    buf = bufs(ctx, nbytes)
    ctx.device_upload(buf, np.full(nbytes // 4, 0xA5A5A5A5, dtype=np.uint32))
    ctx.instance_snapshot_events(scene.p_slab, scene.p_eff, 2, 0, PCAP, scene.evbuf, buf, nbytes)
    want = ref_snapshot_events(scene.pw, 0, scene.events, scene.event_count)
    got = ctx.device_download(buf, nbytes)
    np.testing.assert_array_equal(got[:len(want)], want, err_msg="the snapshot")
    assert (got[len(want):] == 0xA5A5A5A5).all()
    n, d = int(want[3]), int(want[6])
    assert d > 0
    inv = inverse(scene.pw, 0)
    ctx.instance_restore_events(scene.p_slab, scene.p_eff, 2, 0, PCAP, scene.evbuf, buf, nbytes)
    ref_repack_events(scene.pw, 0, scene.events, scene.event_count)
    scene.translate_emitted(inv)
    scene.pw.particles[n + d:] = ctx.slab_download_aos(scene.p_slab, 0, PCAP, scene.p_stride)[n + d:]
    scene.compare("after the restore", draw=False)
    _sync_events(scene, "after the restore")
    for f in range(RELOCATE_AT, RELOCATE_AT + 10):
        scene.step(f)


@TILES
@MODES
def test_move_to_another_context(tiled_ctx, orc, ordered, bufs, native):
    """3. The parent, both children and both event buffers moved into a second context: the parent at slab row 320 of a
    larger slab, the children with version-1 snapshots. The host carries the metadata rows, inserts the child-info rows
    before the restore and points the children's parent_slab_offset at the new slice. Then ten frames there."""
    scene = _scene(tiled_ctx, orc, ordered)
    scene.pending()
    _sync_events(scene, "before the move")
    src = scene.ctx
    ctx2 = native.Context(0)
    try:
        p_first = 320
        p_slab = ctx2.slab_create(p_first + PCAP + 96, scene.p_stride)
        c_slab = [ctx2.slab_create(CCAP, scene.c_stride) for _ in (0, 1)]
        p_eff = ctx2.effect_compile(scene.p_fx)
        c_eff = [ctx2.effect_compile(fx) for fx in scene.c_fx]
        evbuf = [ctx2.event_buffer_create(EVENT_CAP) for _ in (0, 1)]
        for row in (0, 1, 2):
            ctx2.metadata_insert(row, src.read_metadata(row))
            ctx2.draw_args_insert(row)
        for k in (0, 1):
            ctx2.child_info_insert(k, 0, 12345)
        # parent (version 2) and children (version 1) snapshots on the source, restores on the destination
        pbytes = src.instance_snapshot_events_bytes(scene.p_stride, PCAP, [EVENT_CAP, EVENT_CAP])
        pbuf = bufs(src, pbytes)
        src.instance_snapshot_events(scene.p_slab, scene.p_eff, 2, 0, PCAP, scene.evbuf, pbuf, pbytes)
        cbytes = src.instance_snapshot_bytes(scene.c_stride, CCAP)
        cbuf = [bufs(src, cbytes) for _ in (0, 1)]
        for k in (0, 1):
            src.instance_snapshot(scene.c_slab[k], scene.c_eff[k], k, 0, CCAP, cbuf[k], cbytes)
        src.sync()
        snap = ref_snapshot_events(scene.pw, 0, scene.events, scene.event_count)
        np.testing.assert_array_equal(src.device_download(pbuf, len(snap) * 4), snap, err_msg="the parent's snapshot")
        csnap = [ref_snapshot(scene.cw[k], 0) for k in (0, 1)]
        ctx2.instance_restore_events(p_slab, p_eff, 2, p_first, PCAP, evbuf, pbuf, pbytes)
        for k in (0, 1):
            ctx2.instance_restore(c_slab[k], c_eff[k], k, 0, CCAP, cbuf[k], cbytes)
        inv = inverse(scene.pw, 0)
        m, dm, counts = ref_restore_events(scene.pw, 0, snap, scene.events)
        scene.event_count = counts
        scene.translate_emitted(inv)
        assert (m, dm) == (int(snap[3]), int(snap[6]))
        for k in (0, 1):
            ref_restore(scene.cw[k], 0, csnap[k])
        scene.ctx, scene.p_slab, scene.c_slab, scene.p_eff, scene.c_eff, scene.evbuf = ctx2, p_slab, c_slab, p_eff, c_eff, evbuf
        scene.p_first = p_first
        scene.adopt(scene.pw, p_slab, p_first, PCAP, scene.p_stride, m + dm, m)
        for k in (0, 1):
            mc = int(csnap[k][3])
            scene.adopt(scene.cw[k], c_slab[k], 0, CCAP, scene.c_stride, mc, mc)
        scene.compare("after the move", draw=False)
        _sync_events(scene, "after the move")
        for f in range(RELOCATE_AT, RELOCATE_AT + 10):
            scene.step(f)
        ctx2.sync()
    finally:
        ctx2.close()


@MODES
@pytest.mark.parametrize("rows_of", ["n_plus_half_d", "half_n"])
def test_restore_into_fewer_rows(ctx, orc, ordered, rows_of, bufs):
    """4. A restore into an instance of fewer rows than n + D (or than n): the records that fit, the dropped events and the
    resulting event_count, in 128-entry buffers."""
    scene = Scene(ctx, orc, ordered)
    for f in range(RELOCATE_AT):
        scene.step(f)
    scene.pending()
    _sync_events(scene, "before the snapshot")
    nbytes = ctx.instance_snapshot_events_bytes(scene.p_stride, PCAP, [EVENT_CAP, EVENT_CAP])
    buf = bufs(ctx, nbytes)
    ctx.instance_snapshot_events(scene.p_slab, scene.p_eff, 2, 0, PCAP, scene.evbuf, buf, nbytes)
    snap = ref_snapshot_events(scene.pw, 0, scene.events, scene.event_count)
    n, d = int(snap[3]), int(snap[6])
    rows = n + d // 2 if rows_of == "n_plus_half_d" else n // 2
    first = 64
    slab = ctx.slab_create(first + rows + 32, scene.p_stride)
    small = [ctx.event_buffer_create(128) for _ in (0, 1)]
    for k in (0, 1):
        ctx.child_info_insert(4 + k, 0, 777)
    md = R.initial_metadata(rows, 3, scene.p_stride // 4)
    md.base_child_index = 4
    ctx.metadata_insert(3, md)
    ctx.instance_restore_events(slab, scene.p_eff, 3, first, rows, small, buf, nbytes)
    dst = RefWorld(rows, scene.p_stride // 4, [Instance(0, rows)])
    dst.metadata[0] = type(dst.metadata[0]).from_buffer_copy(bytes(md))
    want = [np.zeros(128, dtype=np.uint32) for _ in (0, 1)]
    m, dm, counts = ref_restore_events(dst, 0, snap, want)
    assert m + dm == min(rows, n + d) < n + d
    ctx.sync()
    for k in (0, 1):
        got = ctx.event_buffer_download(small[k], 0, 128)
        kept = min(128, counts[k])
        np.testing.assert_array_equal(got[:kept], want[k][:kept], err_msg=f"channel {k}: kept events")
        assert ctx.read_child_info(4 + k).event_count == counts[k], f"channel {k}: event_count"
    assert any(c > c2 for c, c2 in zip(scene.event_count, counts)), "some events were dropped"
    np.testing.assert_array_equal(np.frombuffer(bytes(ctx.read_metadata(3)), dtype=np.uint32), dst.metadata_rows()[0])
    ind = ctx.slab_download_indirect(slab, first, rows).copy()
    ind[m:, 2] -= np.uint32(first)
    np.testing.assert_array_equal(ind[:m, :2], dst.indirect[:m, :2])
    np.testing.assert_array_equal(ind[m:, 2], dst.indirect[m:, 2])
    np.testing.assert_array_equal(ctx.slab_download_aos(slab, first, rows, scene.p_stride)[:m + dm], dst.particles[:m + dm])


def test_refusals_leave_every_buffer_untouched(ctx, orc, bufs):
    """5. A non-emitting effect, a missing, extra, repeated or invalid channel buffer, a NULL or misaligned buffer and a
    short dst_bytes / src_bytes: HNB_ERR_INVALID_ARG, and the slabs, metadata, event buffers, child infos and the
    snapshot buffer keep every byte."""
    scene = Scene(ctx, orc, False)
    for f in range(RELOCATE_AT):
        scene.step(f)
    scene.pending()
    extra = ctx.event_buffer_create(EVENT_CAP)
    nbytes = ctx.instance_snapshot_events_bytes(scene.p_stride, PCAP, [EVENT_CAP, EVENT_CAP])
    buf = bufs(ctx, nbytes + 16)
    ctx.device_upload(buf, np.full((nbytes + 16) // 4, 0x5A5A5A5A, dtype=np.uint32))

    def state():
        ctx.sync()
        out = [x for _, _, m, ind, p in scene.pulled() for x in (m, ind, p)]
        out += [ctx.event_buffer_download(b, 0, EVENT_CAP) for b in (*scene.evbuf, extra)]
        out += [np.array([ctx.read_child_info(k).event_count for k in (0, 1)])]
        return out + [ctx.device_download(buf, nbytes + 16)]

    before = state()
    ev, p_eff, p_slab = scene.evbuf, scene.p_eff, scene.p_slab
    bad = [("non-emitter", scene.c_slab[0], scene.c_eff[0], 0, CCAP, [ev[0]], buf, nbytes),
           ("missing channel", p_slab, p_eff, 2, PCAP, [ev[0]], buf, nbytes),
           ("extra channel", p_slab, p_eff, 2, PCAP, [ev[0], ev[1], extra], buf, nbytes),
           ("same buffer twice", p_slab, p_eff, 2, PCAP, [ev[0], ev[0]], buf, nbytes),
           ("invalid buffer", p_slab, p_eff, 2, PCAP, [ev[0], 999], buf, nbytes),
           ("rows outside the slab", p_slab, p_eff, 2, PCAP + 1, ev, buf, nbytes),
           ("NULL", p_slab, p_eff, 2, PCAP, ev, 0, nbytes),
           ("misaligned", p_slab, p_eff, 2, PCAP, ev, buf + 8, nbytes)]
    calls = {"repack": lambda s, e, r, n, chans, p, b: ctx.slab_repack_events(s, e, r, 0, n, chans),
             "snapshot": lambda s, e, r, n, chans, p, b: ctx.instance_snapshot_events(s, e, r, 0, n, chans, p, b),
             "restore": lambda s, e, r, n, chans, p, b: ctx.instance_restore_events(s, e, r, 0, n, chans, p, b)}
    cases = [(call, *c) for call in calls for c in bad if not (call == "repack" and c[0] in ("NULL", "misaligned"))]
    cases += [("snapshot", "short dst_bytes", p_slab, p_eff, 2, PCAP, ev, buf, nbytes - 1),
              ("restore", "short src_bytes", p_slab, p_eff, 2, PCAP, ev, buf, 63)]
    for call, why, *args in cases:
        with pytest.raises(N.HanabiError) as e:
            calls[call](*args)
        assert e.value.code == N.HNB_ERR_INVALID_ARG, (call, why, e.value.message)
        for k, (a, b) in enumerate(zip(before, state())):
            np.testing.assert_array_equal(a, b, err_msg=f"{call}, {why}: buffer {k}")
    # 6. the calls without event buffers still refuse the emitter
    for fn, extra_args in ((ctx.slab_repack, ()), (ctx.instance_snapshot, (buf, nbytes)), (ctx.instance_restore, (buf, nbytes))):
        with pytest.raises(N.HanabiError) as e:
            fn(p_slab, p_eff, 2, 0, PCAP, *extra_args)
        assert e.value.code == N.HNB_ERR_INVALID_ARG and "GPU spawn events" in e.value.message
    for k, (a, b) in enumerate(zip(before, state())):
        np.testing.assert_array_equal(a, b, err_msg=f"the calls without events: buffer {k}")
