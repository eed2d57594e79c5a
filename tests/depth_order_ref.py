"""Oracle restatement of hnb_batch_depth_order (include/hanabi_b200.h) over a RefWorld's reference layouts: per instance,
the live entries of its alive list sorted by the depth of `position` against the instance's plane, farthest first, NaN
depths last, equal depths in list order. Works on nothing the device produced. Test infrastructure only."""
from __future__ import annotations

import numpy as np

from tests.bounds_ref import is_nan, ordered_key


def plane_depth(plane, words: np.ndarray) -> np.ndarray:
    """((a*x + b*y) + c*z) + d in float32, every operation rounded on its own; `words` is (n, 3) position bits."""
    a, b, c, d = (np.float32(v) for v in np.asarray(plane, dtype=np.float32))
    p = np.asarray(words, dtype=np.uint32).reshape(-1, 3).view(np.float32)
    with np.errstate(all="ignore"):
        return (((a * p[:, 0]) + (b * p[:, 1])) + (c * p[:, 2])) + d


def sort_keys(depth: np.ndarray) -> np.ndarray:
    """Ascending keys = descending depths in the total order of bounds' key; NaN depths get the largest key."""
    bits = np.asarray(depth, dtype=np.float32).view(np.uint32)
    return np.where(is_nan(bits), np.uint32(0xFFFFFFFF), ~ordered_key(bits)).astype(np.uint32)


def depth_permutation(depth: np.ndarray) -> np.ndarray:
    """pi: depth descending (-0 < +0, infinities included), NaNs last, ties in ascending index."""
    return np.argsort(sort_keys(depth), kind="stable")


def instance_slice(ref, i: int, num_spawners: int | None = None, num_metadata: int | None = None):
    """(first, entries) of spawner row `i`: its clamped slab offset and its live entries in list order (local slots),
    every table word clamped as the device clamps it (tests.bounds_ref.live_rows)."""
    num_spawners = len(ref.spawners) if num_spawners is None else num_spawners
    num_metadata = len(ref.metadata) if num_metadata is None else num_metadata
    sp = ref.spawners[min(i, num_spawners - 1)]
    md = ref.metadata[min(sp.effect_metadata_index, num_metadata - 1)]
    first = min(sp.slab_offset, ref.slab_rows)
    rows = min(md.capacity, ref.slab_rows - first)
    n = min(md.alive_count, rows)
    w = 0 if md.indirect_write_index == 0 else 1
    return first, np.minimum(ref.indirect[first:first + n, w].astype(np.int64), max(rows, 1) - 1).astype(np.uint32)


def ref_depth_order(ref, batch: int, position_word: int, planes: np.ndarray, order: np.ndarray, count: int | None = None,
                    num_spawners: int | None = None, num_metadata: int | None = None) -> np.ndarray:
    """`order` (uint32, slab rows) with the rows hnb_batch_depth_order writes for batch `batch` of `ref` replaced: a copy;
    `planes` is (instances, 4) float32. Returns the copy; `ref` and `order` are not modified."""
    bi = ref.batch_infos[batch]
    out = np.array(order, dtype=np.uint32, copy=True)
    count = bi.prefix_sum_count if count is None else count
    for j in range(count):
        first, entries = instance_slice(ref, bi.spawner_base + j, num_spawners, num_metadata)
        words = ref.particles[first + entries.astype(np.int64), position_word:position_word + 3]
        out[first:first + len(entries)] = entries[depth_permutation(plane_depth(planes[j], words))]
    return out
