"""Oracle restatement of hnb_slab_repack (include/hanabi_b200.h) over a RefWorld's reference layouts (AoS particles,
interleaved {ping, pong, dead} rows). Test infrastructure only."""
from __future__ import annotations

import numpy as np


def ref_repack(ref, i: int) -> int:
    """hnb_slab_repack of instance `i` of `ref` (a tests.helpers.RefWorld) over its whole capacity. Returns n, the length of
    the identity claims the device writes on both columns (the alive bitmap then has bits [0, n) of the slice set)."""
    md, first, rows = ref.metadata[i], ref.instances[i].slab_offset, ref.instances[i].capacity
    n, w = min(md.alive_count, rows), md.indirect_write_index
    if rows == 0:
        return 0
    # alive slots in list order, then dead slots in stack order; clamped to the slice like the kernel (u32 arithmetic)
    src = np.concatenate([ref.indirect[first:first + n, w], ref.indirect[first + n:first + rows, 2] - np.uint32(first)])
    src = np.minimum(src, np.uint32(rows - 1)).astype(np.int64)
    ref.particles[first:first + rows] = ref.particles[first + src]
    ref.indirect[first:first + n, 0] = ref.indirect[first:first + n, 1] = np.arange(n, dtype=np.uint32)
    ref.indirect[first + n:first + rows, 2] = np.arange(first + n, first + rows, dtype=np.uint32)
    return n
