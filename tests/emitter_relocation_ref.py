"""Oracle restatement of hnb_slab_repack_events, hnb_instance_snapshot_events and hnb_instance_restore_events
(include/hanabi_b200.h) over a RefWorld's reference layouts, built on tests/repack_ref.py and tests/snapshot_ref.py. The
pending events of an instance are given as one uint32 array per channel (its length is the buffer's capacity) and one
unclamped event_count per channel. Test infrastructure only."""
from __future__ import annotations

import numpy as np

from tests.repack_ref import ref_repack
from tests.snapshot_ref import HEADER_WORDS, SNAPSHOT_MAGIC, ref_restore

EVENTS_VERSION = 2
NONE = 0xFFFFFFFF


def snapshot_events_bytes(stride: int, rows: int, capacities) -> int:
    return 4 * HEADER_WORDS + rows * stride + 4 * sum(capacities)


def dead_count(md, n: int, rows: int) -> int:
    """D: the slots the last update freed, at dead-stack positions n .. n+D of the slice."""
    return min(md.max_update - n, rows - n) if md.max_update > n else 0


def _source(ref, i: int, count: int) -> np.ndarray:
    """src[k] for k < count: the repack's source rows (alive slots in list order, then the dead stack), clamped."""
    md, first, rows = ref.metadata[i], ref.instances[i].slab_offset, ref.instances[i].capacity
    n, w = min(md.alive_count, rows), md.indirect_write_index
    src = np.concatenate([ref.indirect[first:first + n, w], ref.indirect[first + n:first + rows, 2] - np.uint32(first)])
    return np.minimum(src, np.uint32(rows - 1))[:count].astype(np.int64)


def inverse(ref, i: int) -> np.ndarray:
    """inv[src[k]] = k over the slice (a permutation when the update invariant holds, which is all this restates)."""
    rows = ref.instances[i].capacity
    inv = np.zeros(rows, dtype=np.uint32)
    inv[_source(ref, i, rows)] = np.arange(rows, dtype=np.uint32)
    return inv


def _lookup(inv, buf, stored, rows):
    return inv[np.minimum(buf[:stored], np.uint32(rows - 1)).astype(np.int64)]


def ref_repack_events(ref, i: int, events, counts) -> int:
    """hnb_slab_repack_events: the stored entries of every channel become inv[e] in place; counts do not change."""
    rows = ref.instances[i].capacity
    if rows == 0:
        return 0
    inv = inverse(ref, i)
    for buf, count in zip(events, counts):
        stored = min(count, len(buf))
        buf[:stored] = np.minimum(_lookup(inv, buf, stored, rows), np.uint32(rows - 1))
    return ref_repack(ref, i)


def ref_snapshot_events(ref, i: int, events, counts) -> np.ndarray:
    """hnb_instance_snapshot_events of instance `i`: the words of the complete version-2 snapshot."""
    md, first, rows = ref.metadata[i], ref.instances[i].slab_offset, ref.instances[i].capacity
    n = min(md.alive_count, rows)
    d = dead_count(md, n, rows)
    stored = [min(c, len(b)) for b, c in zip(events, counts)]
    header = np.zeros(HEADER_WORDS, dtype=np.uint32)
    header[:8] = [SNAPSHOT_MAGIC, EVENTS_VERSION, ref.stride_words * 4, n, md.particle_counter, rows, d, len(events)]
    header[8:8 + len(events)] = [c & 0xFFFFFFFF for c in counts]
    header[12:12 + len(events)] = stored
    parts = [header, ref.particles[first + _source(ref, i, n + d)].reshape(-1)]
    inv = inverse(ref, i)
    for buf, e in zip(events, stored):
        r = _lookup(inv, buf, e, rows)
        parts.append(np.where(r < n + d, r, np.uint32(NONE)).astype(np.uint32))
    return np.concatenate(parts)


def restore_span(ref, i: int, snap: np.ndarray, channels: int, src_bytes: int):
    """(ok, n, D, m, D') of a restore of `snap` into instance `i`."""
    stride, rows = ref.stride_words * 4, ref.instances[i].capacity
    h = snap[:HEADER_WORDS]
    if h[0] != SNAPSHOT_MAGIC or h[1] != EVENTS_VERSION or h[2] != stride or h[7] != channels:
        return False, 0, 0, 0, 0
    n, d = int(h[3]), int(h[6])
    fit = (src_bytes - 4 * HEADER_WORDS) // stride
    m = min(n, rows, fit)
    return True, n, d, m, min(d, rows - m, max(fit - n, 0))


def ref_restore_events(ref, i: int, snap: np.ndarray, events, src_bytes: int | None = None):
    """hnb_instance_restore_events of `snap` (of which `src_bytes` bytes are readable) into instance `i`, whose channels'
    buffers are `events` (written in place). Returns (m, D', the new event counts)."""
    md, first, rows = ref.metadata[i], ref.instances[i].slab_offset, ref.instances[i].capacity
    src_bytes = snap.nbytes if src_bytes is None else src_bytes
    ok, n, d, m, dm = restore_span(ref, i, snap, len(events), src_bytes)
    sw = ref.stride_words
    v1 = snap[:HEADER_WORDS].copy()
    if ok:
        v1[1] = 1
    else:
        v1[0] = 0  # rejected: an empty instance, particle_counter kept
    # the live records, metadata words and lists of a version-1 restore of the same header and records
    assert ref_restore(ref, i, np.concatenate([v1, snap[HEADER_WORDS:(4 * HEADER_WORDS + m * sw * 4) // 4]])) == m
    if not ok:
        md.max_update = 0
        return m, 0, [0] * len(events)
    dead = snap[HEADER_WORDS + n * sw:HEADER_WORDS + (n + dm) * sw].reshape(dm, sw)
    ref.particles[first + m:first + m + dm] = dead
    md.max_update = m + dm
    off, words, counts = HEADER_WORDS + (n + d) * sw, src_bytes // 4, []
    for b, buf in enumerate(events):
        unclamped, stored = int(snap[8 + b]), int(snap[12 + b])
        entries = snap[off:off + max(0, min(stored, words - off))].astype(np.int64)
        live = entries < m
        moved = (entries >= n) & (entries - n < dm)
        kept = np.where(live, entries, m + entries - n)[live | moved][:len(buf)].astype(np.uint32)
        buf[:len(kept)] = kept
        counts.append(max(unclamped - (stored - len(kept)), 0))
        off += stored
    return m, dm, counts
