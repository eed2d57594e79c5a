"""Oracle restatement of hnb_batch_cull (include/hanabi_b200.h) over a RefWorld's reference layouts: per instance, the
source entries (its alive list, or a given buffer such as a depth order) whose `position` passes all six planes of the
instance's frustum, in source order, and its draw-args row with their count. Works on nothing the device produced.
Test infrastructure only."""
from __future__ import annotations

import numpy as np

from tests.depth_order_ref import instance_slice, plane_depth

DRAW_ARGS_WORDS = 5


def visible_mask(frustum, words: np.ndarray) -> np.ndarray:
    """((a*x + b*y) + c*z) + d >= 0 for all six planes of `frustum` ((6, 4) float32), every operation rounded on its own
    (numpy's float32 multiply and add round each step and never fuse); `words` is (n, 3) position bits. A NaN fails,
    -0 passes."""
    f = np.asarray(frustum, dtype=np.float32).reshape(6, 4)
    inside = np.ones(len(np.asarray(words).reshape(-1, 3)), dtype=bool)
    with np.errstate(invalid="ignore"):
        for plane in f:
            inside &= plane_depth(plane, words) >= np.float32(0.0)
    return inside


def source_entries(ref, i: int, src: np.ndarray | None, num_spawners=None, num_metadata=None):
    """(first, entries) of spawner row `i`: the alive list's live entries, or src[first + k] for k < n, each clamped to
    the slice as the device clamps it."""
    first, entries = instance_slice(ref, i, num_spawners, num_metadata)
    if src is None:
        return first, entries
    n = len(entries)
    sp = ref.spawners[min(i, (len(ref.spawners) if num_spawners is None else num_spawners) - 1)]
    md = ref.metadata[min(sp.effect_metadata_index, (len(ref.metadata) if num_metadata is None else num_metadata) - 1)]
    rows = min(md.capacity, ref.slab_rows - first)
    return first, np.minimum(np.asarray(src[first:first + n], dtype=np.int64), max(rows, 1) - 1).astype(np.uint32)


def ref_cull(ref, batch: int, position_word: int, frusta: np.ndarray, visible: np.ndarray, draw_args: np.ndarray,
             src: np.ndarray | None = None, count: int | None = None, num_spawners=None, num_metadata=None):
    """(visible', args) for batch `batch` of `ref`: `visible` (uint32, slab rows) with the rows hnb_batch_cull writes
    replaced (a copy), and the (count, 5) uint32 args rows. `frusta` is (instances, 6, 4) float32, `draw_args` the
    device draw-args table as (rows, 5) uint32, `src` NULL (None) or a uint32 buffer of slab rows. `count` is the call's
    instance count (the host's batch row); instances past the batch row's own count get args with instance_count 0."""
    bi = ref.batch_infos[batch]
    count = bi.prefix_sum_count if count is None else count
    device_count = min(bi.prefix_sum_count, count)
    num_spawners = len(ref.spawners) if num_spawners is None else num_spawners
    out = np.array(visible, dtype=np.uint32, copy=True)
    table = np.asarray(draw_args, dtype=np.uint32).reshape(-1, DRAW_ARGS_WORDS)
    args = np.zeros((count, DRAW_ARGS_WORDS), dtype=np.uint32)
    for j in range(count):
        m = 0
        if j < device_count:
            first, entries = source_entries(ref, bi.spawner_base + j, src, num_spawners, num_metadata)
            words = ref.particles[first + entries.astype(np.int64), position_word:position_word + 3]
            kept = entries[visible_mask(frusta[j], words)]
            out[first:first + len(kept)] = kept
            m = len(kept)
        sp = ref.spawners[min(bi.spawner_base + j, num_spawners - 1)]
        args[j] = table[min(sp.draw_indirect_index, len(table) - 1)]
        args[j, 1] = m
    return out, args


def frustum_planes(view_proj: np.ndarray, radius: float = 0.0) -> np.ndarray:
    """The six planes (left, right, bottom, top, near, far) of a row-major view-projection matrix M acting on column
    vectors, for a clip volume -w <= x, y <= w, 0 <= z <= w: rows w+x, w-x, w+y, w-y, z, w-z, normalised, with `radius`
    added to d. (6, 4) float32."""
    m = np.asarray(view_proj, dtype=np.float64).reshape(4, 4)
    rows = [m[3] + m[0], m[3] - m[0], m[3] + m[1], m[3] - m[1], m[2], m[3] - m[2]]
    out = []
    for r in rows:
        r = r / np.linalg.norm(r[:3])
        out.append([r[0], r[1], r[2], r[3] + radius])
    return np.array(out, dtype=np.float32)
