"""hnb_slab_repack_events, hnb_instance_snapshot_events and hnb_instance_restore_events: their kernels
(hnb_static_kernels.cu: k_repack_inverse, k_events_translate, k_snapshot_gather_dead, k_restore_scatter_dead,
k_restore_events, with the repack's gathers and list writer) under the CPU thread emulation of tests/static_emu.py, in
the host's launch order, against the numpy restatement tests/emitter_relocation_ref.py, which is itself pinned by a
hand-written example."""
import copy
import ctypes as C

import numpy as np
import pytest

from tests import static_emu as S
from tests.emitter_relocation_ref import (EVENTS_VERSION, NONE, dead_count, ref_repack_events, ref_restore_events,
                                          ref_snapshot_events, snapshot_events_bytes)
from tests.helpers import Instance, RefWorld
from tests.kernel_emu import claim
from tests.snapshot_ref import HEADER_WORDS, SNAPSHOT_MAGIC
from tests.static_emu import REPACK_DRIVER, RepackArgs, SoaSlab, churned, expected_bits

pytestmark = pytest.mark.timeout(600)

EVENTS_DRIVER = r"""
extern "C" void semu_repack_inverse(const RepackArgs* a, uint32_t* inv) {
    RepackArgs r = *a;
    emu_run([&] { k_repack_inverse(r, inv); }, (r.rows + RP_THREADS - 1) / RP_THREADS, RP_THREADS, 8);
}
extern "C" void semu_events_translate(const RepackArgs* a, const uint32_t* inv, const EventChannels* ev, uint32_t stride_words, uint32_t* snapshot) {
    RepackArgs r = *a;
    EventChannels e = *ev;
    uint32_t widest = 1;
    for (uint32_t b = 0; b < e.count; ++b) widest = std::max(widest, e.capacity[b]);
    const uint32_t per = (widest + RP_THREADS - 1) / RP_THREADS;
    emu_run([&] { k_events_translate(r, inv, e, per, stride_words, snapshot); }, per * e.count, RP_THREADS, 8);
}
extern "C" void semu_snapshot_gather_dead(const SnapshotArgs* a, const uint32_t* dead, uint32_t* dst) {
    SnapshotArgs s = *a;
    emu_run([&] { k_snapshot_gather_dead(s, dead, dst); }, (s.rows + RP_ROWS_PER_BLOCK - 1) / RP_ROWS_PER_BLOCK, RP_THREADS, 8);
}
extern "C" void semu_restore_scatter_dead(const SnapshotArgs* a, const uint32_t* src, uint32_t channels) {
    SnapshotArgs s = *a;
    emu_run([&] { k_restore_scatter_dead(s, src, channels); }, (s.rows + RP_ROWS_PER_BLOCK - 1) / RP_ROWS_PER_BLOCK, RP_THREADS, 8);
}
extern "C" void semu_restore_events(const SnapshotArgs* a, const uint32_t* src, const EventChannels* ev) {
    SnapshotArgs s = *a;
    EventChannels e = *ev;
    emu_run([&] { k_restore_events(s, src, e); }, e.count, EV_THREADS);
}
extern "C" uint32_t semu_sizeof_event_channels(void) { return sizeof(EventChannels); }
extern "C" uint32_t semu_sizeof_snapshot_args_v2(void) { return sizeof(SnapshotArgs); }
"""


class SnapshotArgs(C.Structure):
    """hnb::SnapshotArgs (hnb_static_kernels.h)"""
    _fields_ = [("metadata", C.c_void_p), ("ping", C.c_void_p), ("pong", C.c_void_p), ("planes", S.PlaneSet),
                ("num_planes", C.c_uint32), ("stride_words", C.c_uint32), ("first", C.c_uint32), ("rows", C.c_uint32),
                ("src_bytes", C.c_uint64)]


class EventChannels(C.Structure):
    """hnb::EventChannels (hnb_static_kernels.h)"""
    _fields_ = [("buffer", C.c_void_p * 4), ("capacity", C.c_uint32 * 4), ("count", C.c_uint32), ("child_infos", C.c_void_p),
                ("num_child_infos", C.c_uint32)]


@pytest.fixture(scope="module")
def elib():
    lib = S.build(REPACK_DRIVER + EVENTS_DRIVER)
    for f in ("semu_repack_inverse", "semu_events_translate", "semu_snapshot_gather_dead", "semu_restore_scatter_dead",
              "semu_restore_events", "semu_repack_gather", "semu_repack_lists"):
        getattr(lib, f).restype = None
    lib.semu_events_translate.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
    lib.semu_restore_scatter_dead.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
    lib.semu_sizeof_event_channels.restype = lib.semu_sizeof_snapshot_args_v2.restype = C.c_uint32
    assert lib.semu_sizeof_event_channels() == C.sizeof(EventChannels)
    assert lib.semu_sizeof_snapshot_args_v2() == C.sizeof(SnapshotArgs)
    return lib


class Emitter:
    """An emitting instance `i` of a SoaSlab: its channels' buffers and the context's child-info rows, channel b's
    event_count at row base + b (the metadata row's base_child_index)."""

    def __init__(self, soa, ref, i, events, counts, base=3):
        self.soa, self.ref, self.i = soa, ref, i
        self.events = [np.array(e, dtype=np.uint32) for e in events]
        self.child = np.zeros((base + len(events) + 2, 2), dtype=np.uint32)
        self.child[:, 1] = 0xDEADBEEF  # rows of other parents keep their words
        self.base = base
        soa.metadata[i].base_child_index = ref.metadata[i].base_child_index = base
        self.counts = list(counts)

    @property
    def counts(self):
        return [int(c) for c in self.child[self.base:self.base + len(self.events), 1]]

    @counts.setter
    def counts(self, counts):
        self.child[self.base:self.base + len(self.events), 1] = counts

    def channels(self):
        ev = EventChannels()
        for b, e in enumerate(self.events):
            ev.buffer[b], ev.capacity[b] = e.ctypes.data, len(e)
        ev.count, ev.child_infos, ev.num_child_infos = len(self.events), self.child.ctypes.data, len(self.child)
        return ev

    def span(self):
        inst = self.ref.instances[self.i]
        return inst.slab_offset, inst.capacity

    def repack_args(self):
        s, (first, rows) = self.soa, self.span()
        return RepackArgs(C.addressof(s.metadata[self.i]), s.cols[0].ctypes.data, s.cols[1].ctypes.data, s.cols[2].ctypes.data,
                          s.bits.ctypes.data, s.claims.ctypes.data, first, rows)

    def snapshot_args(self, src_bytes=0):
        s, (first, rows) = self.soa, self.span()
        ps, off = S.PlaneSet(), 0
        for p, (plane, w) in enumerate(zip(s.planes, s.widths)):
            ps.ptr[p], ps.words[p], ps.word_off[p] = plane.ctypes.data, w // 4, off
            off += w // 4
        return SnapshotArgs(C.addressof(s.metadata[self.i]), s.cols[0].ctypes.data, s.cols[1].ctypes.data, ps, len(s.widths),
                            self.ref.stride_words, first, rows, src_bytes)

    def repack(self, lib):
        """hnb_slab_repack_events' device work, in its order."""
        a, ev, (first, rows) = self.repack_args(), self.channels(), self.span()
        inv = np.zeros(rows, dtype=np.uint32)
        lib.semu_repack_inverse(C.byref(a), inv.ctypes.data)
        scratch = np.zeros(rows * 8 + 8, dtype=np.uint32)
        for plane, w in zip(self.soa.planes, self.soa.widths):
            k = w // 4
            lib.semu_repack_gather(C.byref(a), plane.ctypes.data, scratch.ctypes.data, w)
            plane[first * k:(first + rows) * k] = scratch[:rows * k]
        lib.semu_events_translate(C.byref(a), inv.ctypes.data, C.byref(ev), 0, None)
        lib.semu_repack_lists(C.byref(a))

    def snapshot(self, lib, sentinel=0xA5A5A5A5):
        """hnb_instance_snapshot_events' device work into a buffer of hnb_instance_snapshot_events_bytes."""
        first, rows = self.span()
        dst = np.full(snapshot_events_bytes(self.ref.stride_words * 4, rows, [len(e) for e in self.events]) // 4, sentinel, dtype=np.uint32)
        lib.semu_snapshot_gather_dead(C.byref(self.snapshot_args()), self.soa.cols[2].ctypes.data, dst.ctypes.data)
        a, ev = self.repack_args(), self.channels()
        inv = np.zeros(rows, dtype=np.uint32)
        lib.semu_repack_inverse(C.byref(a), inv.ctypes.data)
        lib.semu_events_translate(C.byref(a), inv.ctypes.data, C.byref(ev), self.ref.stride_words, dst.ctypes.data)
        return dst

    def restore(self, lib, src, src_bytes=None):
        """hnb_instance_restore_events' device work, in its order."""
        a = self.snapshot_args(src.nbytes if src_bytes is None else src_bytes)
        lib.semu_restore_scatter_dead(C.byref(a), src.ctypes.data, len(self.events))
        lib.semu_repack_lists(C.byref(self.repack_args()))
        lib.semu_restore_events(C.byref(a), src.ctypes.data, C.byref(self.channels()))


def _assert_same(em, ref, events, counts, what):
    np.testing.assert_array_equal(em.soa.particles(), ref.particles, err_msg=f"{what}: records")
    np.testing.assert_array_equal(em.soa.indirect(), ref.indirect, err_msg=f"{what}: ping / pong / dead")
    np.testing.assert_array_equal(np.frombuffer(bytes(em.soa.metadata), dtype=np.uint32).reshape(-1, 15), ref.metadata_rows(),
                                  err_msg=f"{what}: metadata")
    for b, (got, want) in enumerate(zip(em.events, events)):
        np.testing.assert_array_equal(got, want, err_msg=f"{what}: event buffer {b}")
    assert em.counts == [c & 0xFFFFFFFF for c in counts], f"{what}: event counts"
    others = np.delete(np.arange(len(em.child)), np.arange(em.base, em.base + len(em.events)))
    assert (em.child[others, 1] == 0xDEADBEEF).all() and (em.child[:, 0] == 0).all(), f"{what}: other child-info words"


def test_oracle_restatement_by_hand():
    """A 6-row instance at slab row 2, records 100 + row. W = 0 lists local slots 4, 0, 5 alive; the dead stack holds slots
    1, 3, 2 from position 3; max_update = 5, so slots 1 and 3 died in the last update (D = 2) and slot 2 earlier. Channel 0
    (capacity 4) overflowed, 6 events: slots 5, 1 (the OnDie event of a dead parent), 4, 4. Channel 1 (capacity 3): slot 3
    and slot 2, which no pending event can name while the invariant holds; its third word is stale."""
    def world():
        ref = RefWorld(8, 1, [Instance(0, 2), Instance(2, 6)])
        ref.particles[:, 0] = 100 + np.arange(8)
        ref.indirect[:, 0] = [0, 1, 4, 0, 5, 70, 71, 72]
        ref.indirect[:, 1] = [0, 1, 60, 61, 62, 63, 64, 65]
        ref.indirect[:, 2] = [0, 1, 90, 91, 92, 3, 5, 4]
        md = ref.metadata[1]
        md.alive_count, md.max_update, md.indirect_write_index, md.particle_counter = 3, 5, 0, 9
        return ref

    def events():
        return [np.array([5, 1, 4, 4], dtype=np.uint32), np.array([3, 2, 9], dtype=np.uint32)]

    ref, ev = world(), events()
    assert ref_repack_events(ref, 1, ev, [6, 2]) == 3
    np.testing.assert_array_equal(ref.particles[:, 0], [100, 101, 106, 102, 107, 103, 105, 104])
    np.testing.assert_array_equal(ev[0], [2, 3, 0, 0])
    np.testing.assert_array_equal(ev[1], [4, 5, 9])

    ref = world()
    snap = ref_snapshot_events(ref, 1, events(), [6, 2])
    np.testing.assert_array_equal(snap, [SNAPSHOT_MAGIC, 2, 4, 3, 9, 6, 2, 2, 6, 2, 0, 0, 4, 2, 0, 0]
                                  + [106, 102, 107, 103, 105] + [2, 3, 0, 0] + [4, NONE])
    assert len(snap) * 4 < snapshot_events_bytes(4, 6, [4, 3])

    for rows, cap0, want in [(6, 4, ([106, 102, 107, 103, 105], 5, [2, 3, 0, 0], [4], [6, 1])),
                             (4, 4, ([106, 102, 107, 103], 4, [2, 3, 0, 0], [], [6, 0])),  # fewer rows than n + D
                             (2, 4, ([106, 102], 2, [0, 0], [], [4, 0])),  # fewer than n: records 2 and 3 go
                             (2, 1, ([106, 102], 2, [0], [], [3, 0]))]:  # ... and a one-entry buffer
        dst = RefWorld(3 + rows, 1, [Instance(0, 3), Instance(3, rows)])
        dst.particles[:, 0] = 200 + np.arange(3 + rows)
        bufs = [np.full(cap0, 77, dtype=np.uint32), np.full(3, 77, dtype=np.uint32)]
        m, dm, counts = ref_restore_events(dst, 1, snap, bufs)
        records, max_update, e0, e1, want_counts = want
        assert (m + dm, dst.metadata[1].max_update, dst.metadata[1].alive_count) == (len(records), max_update, min(3, rows))
        np.testing.assert_array_equal(dst.particles[3:3 + len(records), 0], records)
        np.testing.assert_array_equal(bufs[0][:len(e0)], e0)
        np.testing.assert_array_equal(bufs[1][:len(e1)], e1)
        assert (bufs[1][len(e1):] == 77).all() and counts == want_counts, rows


def _world(rng, stride_words, n, d_extra, rows=1100, first=37, w=1):
    """Instance 1 of a three-instance slab in a churned state with max_update = n + d_extra."""
    ref = RefWorld(first + rows + 50, stride_words, [Instance(0, first), Instance(first, rows), Instance(first + rows, 50)])
    ref.particles[:] = rng.integers(0, 1 << 32, ref.particles.shape, dtype=np.uint64).astype(np.uint32)
    for j, k in enumerate((first // 2, n, 25)):
        churned(rng, ref, j, k, w=(j + w) & 1)
        ref.metadata[j].particle_counter = int(rng.integers(0, 1 << 32))
    ref.metadata[1].max_update = n + d_extra
    return ref


def _pending(rng, ref, i, caps, counts, stale=False):
    """Events naming live slots and slots the last update freed (and, with `stale`, older dead slots), then garbage past
    the stored entries."""
    md, inst = ref.metadata[i], ref.instances[i]
    first, rows = inst.slab_offset, inst.capacity
    n = min(md.alive_count, rows)
    d = dead_count(md, n, rows)
    pool = [ref.indirect[first:first + n, md.indirect_write_index], ref.indirect[first + n:first + n + d, 2] - np.uint32(first)]
    if stale:
        pool.append(ref.indirect[first + n + d:first + rows, 2] - np.uint32(first))
    pool = np.concatenate(pool).astype(np.uint32)
    out = []
    for cap, count in zip(caps, counts):
        buf = rng.integers(0, 1 << 32, cap, dtype=np.uint64).astype(np.uint32)
        stored = min(count, cap)
        if len(pool):
            buf[:stored] = rng.choice(pool, stored)
        out.append(buf)
    return out


# (n, D beyond n, channel capacities, event counts): D = 0, churned, D = rows - n,
# overflowed and empty channels, four channels
CASES = [(700, 0, (256, 256), (40, 300)), (700, 150, (256, 256), (256, 1000)), (300, 800, (256, 64), (0, 65)),
         (1100, 0, (100,), (99,)), (0, 1100, (512, 256), (600, 7)), (512, 200, (64, 64, 300, 16), (64, 1, 299, 17))]


@pytest.mark.parametrize("stride_words,sector", [(1, False), (7, False), (8, True), (12, True)], ids=str)
@pytest.mark.parametrize("n,dx,caps,counts", CASES, ids=str)
def test_repack_matches_the_oracle(elib, stride_words, sector, n, dx, caps, counts):
    rng = np.random.default_rng(n + dx + stride_words)
    ref = _world(rng, stride_words, n, dx)
    events = _pending(rng, ref, 1, caps, counts)
    em = Emitter(SoaSlab(ref, sector, rng), ref, 1, events, counts)
    bits0 = em.soa.bits.copy()
    em.repack(elib)
    want = [e.copy() for e in events]
    assert ref_repack_events(ref, 1, want, counts) == min(n, 1100)
    _assert_same(em, ref, want, counts, "repack")
    np.testing.assert_array_equal(em.soa.bits, expected_bits(bits0, 37, 1100, min(n, 1100)))
    assert em.soa.claims[0] == em.soa.claims[1] == claim(37, min(n, 1100))


@pytest.mark.parametrize("stride_words,sector", [(1, False), (7, False), (8, True)], ids=str)
@pytest.mark.parametrize("n,dx,caps,counts", CASES, ids=str)
def test_snapshot_matches_the_oracle(elib, stride_words, sector, n, dx, caps, counts):
    """The header, n + D records and the entries, with events on slots outside the n + D records; nothing else written,
    the source untouched."""
    rng = np.random.default_rng(7 * n + dx + stride_words)
    ref = _world(rng, stride_words, n, dx)
    events = _pending(rng, ref, 1, caps, counts, stale=True)
    em = Emitter(SoaSlab(ref, sector, rng), ref, 1, events, counts)
    before = copy.deepcopy(ref)
    got = em.snapshot(elib)
    want = ref_snapshot_events(ref, 1, events, counts)
    np.testing.assert_array_equal(got[:len(want)], want)
    assert (got[len(want):] == 0xA5A5A5A5).all(), "words past the complete snapshot were written"
    assert want[1] == EVENTS_VERSION and want[6] == dead_count(ref.metadata[1], min(n, 1100), 1100)
    _assert_same(em, before, events, counts, "the snapshot's source")


@pytest.mark.parametrize("n,dx,caps,counts", CASES, ids=str)
@pytest.mark.parametrize("target", ["same", "moved", "smaller_than_n_plus_d", "smaller_than_n", "small_buffers"])
def test_restore_matches_the_oracle(elib, n, dx, caps, counts, target):
    """Into the instance's own slice (which must leave what the repack leaves), into 1300 rows at slab row 45 of another
    slab, into fewer rows than n + D or than n, and into buffers of a quarter of the capacity."""
    rng = np.random.default_rng(13 * n + dx)
    src_ref = _world(rng, 7, n, dx)
    events = _pending(rng, src_ref, 1, caps, counts)
    src = Emitter(SoaSlab(src_ref, False, rng), src_ref, 1, events, counts)
    snap = src.snapshot(elib)
    n_, d = int(snap[3]), int(snap[6])
    if target == "same":
        repacked, rev = copy.deepcopy(src_ref), [e.copy() for e in events]
        ref_repack_events(repacked, 1, rev, counts)
        ref, em = src_ref, src
    else:
        rows = {"moved": 1300, "smaller_than_n_plus_d": max(1, n_ + d // 2), "smaller_than_n": max(1, n_ // 2)}.get(target, 1100)
        ref = _world(rng, 7, rows // 2, min(20, rows - rows // 2), rows=rows, first=45, w=0)
        dcaps = [max(1, c // 4) for c in caps] if target == "small_buffers" else caps
        em = Emitter(SoaSlab(ref, False, rng), ref, 1, _pending(rng, ref, 1, dcaps, [0] * len(caps)), [5] * len(caps), base=1)
    bits0 = em.soa.bits.copy()
    want = [e.copy() for e in em.events]
    em.restore(elib, snap)
    m, dm, want_counts = ref_restore_events(ref, 1, snap, want)
    _assert_same(em, ref, want, want_counts, target)
    first, rows = em.span()
    np.testing.assert_array_equal(em.soa.bits, expected_bits(bits0, first, rows, m))
    assert em.soa.claims[0] == em.soa.claims[1] == claim(first, m)
    if target == "same":
        np.testing.assert_array_equal(ref.indirect, repacked.indirect)
        np.testing.assert_array_equal(ref.metadata_rows(), repacked.metadata_rows())
        np.testing.assert_array_equal(ref.particles[37:37 + n_ + d], repacked.particles[37:37 + n_ + d])
        for a, b in zip(em.events, rev):
            np.testing.assert_array_equal(a, b)
        assert em.counts == list(counts)
    if target.startswith("smaller"):
        assert m + dm == min(rows, n_ + d)


@pytest.mark.parametrize("corruption", ["magic", "version_1", "stride", "channels", "short_records", "short_events",
                                        "header_only"])
def test_corrupt_or_short_snapshots(elib, corruption):
    """A header that is not a version-2 snapshot of this stride and channel count restores an empty instance with no
    events; a short src_bytes restores the records and entries it holds in full, and nothing past it is read."""
    rng = np.random.default_rng(5)
    src_ref = _world(rng, 5, 400, 100, rows=600, first=0)
    events = _pending(rng, src_ref, 1, (256, 128), (300, 100))
    snap = Emitter(SoaSlab(src_ref, False, rng), src_ref, 1, events, (300, 100)).snapshot(elib)
    full = HEADER_WORDS + 500 * 5 + 256 + 100
    snap, src_bytes = snap[:full].copy(), full * 4
    if corruption == "magic":
        snap[0] ^= 1
    elif corruption == "version_1":
        snap[1] = 1
    elif corruption == "stride":
        snap[2] = 24
    elif corruption == "channels":
        snap[7] = 1
    else:
        src_bytes = {"short_records": 64 + 450 * 20 + 7, "short_events": (full - 150) * 4 + 2, "header_only": 64}[corruption]
        snap = snap[:(src_bytes + 3) // 4].copy()  # the kernels must not read past src_bytes: the array ends there
    ref = _world(rng, 5, 100, 10, rows=700, first=32)
    em = Emitter(SoaSlab(ref, False, rng), ref, 1, [np.full(256, 66, dtype=np.uint32), np.full(128, 66, dtype=np.uint32)], [4, 4])
    want = [e.copy() for e in em.events]
    counter = ref.metadata[1].particle_counter
    em.restore(elib, snap, src_bytes)
    m, dm, counts = ref_restore_events(ref, 1, snap, want, src_bytes)
    _assert_same(em, ref, want, counts, corruption)
    if corruption in ("magic", "version_1", "stride", "channels"):
        assert (m, dm, counts) == (0, 0, [0, 0])
        assert ref.metadata[1].particle_counter == counter and (em.events[0] == 66).all()
    else:  # every entry past src_bytes is dropped: 206 of channel 0's 256 remain readable with short_events
        assert (m, dm, counts) == {"short_records": (400, 50, [44, 0]), "short_events": (400, 100, [250, 0]),
                                   "header_only": (0, 0, [44, 0])}[corruption]
