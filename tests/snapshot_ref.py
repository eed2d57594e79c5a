"""Oracle restatement of hnb_instance_snapshot / hnb_instance_restore (include/hanabi_b200.h) over a RefWorld's reference
layouts (AoS particles, interleaved {ping, pong, dead} rows). A snapshot is a uint32 array: the 16 header words, then the
records. Test infrastructure only."""
from __future__ import annotations

import numpy as np

SNAPSHOT_MAGIC = 0x53424E48  # "HNBS"
SNAPSHOT_VERSION = 1
HEADER_WORDS = 16


def snapshot_bytes(stride: int, rows: int) -> int:
    return 4 * HEADER_WORDS + rows * stride


def ref_snapshot(ref, i: int) -> np.ndarray:
    """hnb_instance_snapshot of instance `i` of `ref` (a tests.helpers.RefWorld) over its whole capacity: the
    64 + n * stride bytes the device writes, as words. `ref` is not modified."""
    md, first, rows = ref.metadata[i], ref.instances[i].slab_offset, ref.instances[i].capacity
    n, w = min(md.alive_count, rows), md.indirect_write_index
    header = np.zeros(HEADER_WORDS, dtype=np.uint32)
    header[:6] = [SNAPSHOT_MAGIC, SNAPSHOT_VERSION, ref.stride_words * 4, n, md.particle_counter, rows]
    src = np.minimum(ref.indirect[first:first + n, w], np.uint32(max(rows, 1) - 1)).astype(np.int64)  # clamped as repack_source
    return np.concatenate([header, ref.particles[first + src].reshape(-1)])


def restore_count(ref, i: int, snap: np.ndarray, src_bytes: int | None = None) -> int:
    """m: the records a restore of `snap` (of which `src_bytes` bytes are readable) into instance `i` takes."""
    stride, rows = ref.stride_words * 4, ref.instances[i].capacity
    src_bytes = snap.nbytes if src_bytes is None else src_bytes
    h = snap[:HEADER_WORDS]
    if h[0] != SNAPSHOT_MAGIC or h[1] != SNAPSHOT_VERSION or h[2] != stride:
        return 0
    return int(min(int(h[3]), rows, (src_bytes - 4 * HEADER_WORDS) // stride))


def ref_restore(ref, i: int, snap: np.ndarray, src_bytes: int | None = None) -> int:
    """hnb_instance_restore of `snap` into instance `i` of `ref` over its whole capacity. Returns m."""
    md, first, rows = ref.metadata[i], ref.instances[i].slab_offset, ref.instances[i].capacity
    if rows == 0:
        return 0
    m = restore_count(ref, i, snap, src_bytes)
    sw = ref.stride_words
    ref.particles[first:first + m] = snap[HEADER_WORDS:HEADER_WORDS + m * sw].reshape(m, sw)
    md.alive_count = m
    md.max_spawn = max(md.capacity - m, 0)
    h = snap[:HEADER_WORDS]
    if h[0] == SNAPSHOT_MAGIC and h[1] == SNAPSHOT_VERSION and h[2] == sw * 4:
        md.particle_counter = int(h[4])
    # the lists, dead stack (and, on the device, claims {first, m} and alive bits) that hnb_slab_repack writes for n = m
    ref.indirect[first:first + m, 0] = ref.indirect[first:first + m, 1] = np.arange(m, dtype=np.uint32)
    ref.indirect[first + m:first + rows, 2] = np.arange(first + m, first + rows, dtype=np.uint32)
    return m
