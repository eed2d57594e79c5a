"""Oracle restatement of hnb_instance_append (include/hanabi_b200.h) over a RefWorld's reference layouts (AoS particles,
interleaved {ping, pong, dead} rows), in the style of tests/snapshot_ref.py. The device state a RefWorld does not hold
(identity claims, alive bits, lifetime floors and common ages) is restated by `append_slots` and `cut_claim`. Test
infrastructure only."""
from __future__ import annotations

import numpy as np

from tests.snapshot_ref import HEADER_WORDS, restore_count


def append_count(ref, i: int, snap: np.ndarray, src_bytes: int | None = None) -> int:
    """m: the records an append of `snap` (of which `src_bytes` bytes are readable) into instance `i` takes."""
    md, rows = ref.metadata[i], ref.instances[i].capacity
    n = min(md.alive_count, rows)
    return min(restore_count(ref, i, snap, src_bytes), md.max_spawn, rows - n)


def append_slots(ref, i: int, snap: np.ndarray, src_bytes: int | None = None) -> np.ndarray:
    """The instance-local slots s_k = dead[first + n + k] - first (clamped to the slice) the m records go to, read before
    the append."""
    md, first, rows = ref.metadata[i], ref.instances[i].slab_offset, ref.instances[i].capacity
    if rows == 0:
        return np.zeros(0, dtype=np.uint32)
    n, m = min(md.alive_count, rows), append_count(ref, i, snap, src_bytes)
    return np.minimum(ref.indirect[first + n:first + n + m, 2] - np.uint32(first), np.uint32(rows - 1)).astype(np.uint32)


def ref_append(ref, i: int, snap: np.ndarray, src_bytes: int | None = None) -> int:
    """hnb_instance_append of `snap` into instance `i` of `ref` over its whole capacity. Returns m."""
    md, first, rows = ref.metadata[i], ref.instances[i].slab_offset, ref.instances[i].capacity
    slots = append_slots(ref, i, snap, src_bytes)
    m = len(slots)
    if m == 0:
        return 0
    n, sw = min(md.alive_count, rows), ref.stride_words
    ref.particles[first + slots.astype(np.int64)] = snap[HEADER_WORDS:HEADER_WORDS + m * sw].reshape(m, sw)
    ref.indirect[first + n:first + n + m, md.indirect_write_index] = slots
    md.alive_count = n + m
    md.max_spawn -= m
    md.particle_counter = (md.particle_counter + m) & 0xFFFFFFFF
    return m


def cut_claim(word: int, first: int, n: int) -> int:
    """The identity claim word of column W after an append of m > 0 records into the instance at `first` with n alive:
    cut to n if it is this instance's and reaches further."""
    base, length = word >> 32, word & 0xFFFFFFFF
    return (first << 32) | n if base == first and length > n else word


def make_snapshot(records: np.ndarray, stride_words: int, count: int | None = None, version: int = 1) -> np.ndarray:
    """A version-1 snapshot written by hand (what a host or a producer kernel writes): the header, then `records`
    (an (k, stride_words) uint32 array). `count` defaults to k."""
    from tests.snapshot_ref import SNAPSHOT_MAGIC
    records = np.asarray(records, dtype=np.uint32).reshape(-1, stride_words)
    header = np.zeros(HEADER_WORDS, dtype=np.uint32)
    header[:4] = [SNAPSHOT_MAGIC, version, stride_words * 4, len(records) if count is None else count]
    return np.concatenate([header, records.reshape(-1)])
