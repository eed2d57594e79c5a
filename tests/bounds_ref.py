"""Oracle restatement of hnb_batch_bounds (include/hanabi_b200.h) over a RefWorld's reference layouts (AoS particles,
interleaved {ping, pong, dead} rows, spawner and metadata rows): the per-component minimum and maximum of `position` over
each instance's live particles, in the total order of the float -> unsigned key. Works on nothing the device produced.
Test infrastructure only."""
from __future__ import annotations

import numpy as np

BOUNDS_DTYPE = np.dtype([("min", np.float32, 3), ("count", np.uint32), ("max", np.float32, 3), ("reserved", np.uint32)])
POS_INF, NEG_INF = np.uint32(0x7F800000), np.uint32(0xFF800000)


def ordered_key(bits: np.ndarray) -> np.ndarray:
    """bits ^ (sign ? 0xFFFFFFFF : 0x80000000): unsigned order of the keys = total order of the floats, -0 < +0."""
    bits = np.asarray(bits, dtype=np.uint32)
    return np.where(bits >> np.uint32(31), bits ^ np.uint32(0xFFFFFFFF), bits ^ np.uint32(0x80000000)).astype(np.uint32)


def key_bits(key: np.ndarray) -> np.ndarray:
    key = np.asarray(key, dtype=np.uint32)
    return np.where(key >> np.uint32(31), key ^ np.uint32(0x80000000), key ^ np.uint32(0xFFFFFFFF)).astype(np.uint32)


def is_nan(bits: np.ndarray) -> np.ndarray:
    return (np.asarray(bits, dtype=np.uint32) & np.uint32(0x7FFFFFFF)) > np.uint32(0x7F800000)


def box_of(words: np.ndarray):
    """(min bits[3], max bits[3]) of an (n, 3) array of position words: NaNs skipped, no value -> +inf / -inf."""
    lo, hi = np.full(3, POS_INF, dtype=np.uint32), np.full(3, NEG_INF, dtype=np.uint32)
    for c in range(3):
        b = words[:, c]
        k = ordered_key(b[~is_nan(b)])
        if k.size:
            lo[c], hi[c] = key_bits(k.min()), key_bits(k.max())
    return lo, hi


def live_rows(ref, i: int, num_spawners: int | None = None, num_metadata: int | None = None):
    """Slab rows of the live particles of spawner row `i`, in alive-list order, every table word clamped as the device
    clamps it: the spawner and metadata rows to their tables, the slice to the slab, the list entries to the slice."""
    num_spawners = len(ref.spawners) if num_spawners is None else num_spawners
    num_metadata = len(ref.metadata) if num_metadata is None else num_metadata
    sp = ref.spawners[min(i, num_spawners - 1)]
    md = ref.metadata[min(sp.effect_metadata_index, num_metadata - 1)]
    first = min(sp.slab_offset, ref.slab_rows)
    rows = min(md.capacity, ref.slab_rows - first)
    n = min(md.alive_count, rows)
    w = 0 if md.indirect_write_index == 0 else 1
    src = np.minimum(ref.indirect[first:first + n, w].astype(np.int64), max(rows, 1) - 1)
    return first + src


def ref_bounds(ref, batch: int, position_word: int, out_rows: int | None = None, num_spawners: int | None = None,
               num_metadata: int | None = None) -> np.ndarray:
    """The records hnb_batch_bounds writes for batch `batch` of `ref` (a tests.helpers.RefWorld) whose `position` starts at
    AoS word `position_word`: one per instance of the batch, at most `out_rows`. `ref` is not modified."""
    bi = ref.batch_infos[batch]
    count = bi.prefix_sum_count if out_rows is None else min(bi.prefix_sum_count, out_rows)
    out = np.zeros(count, dtype=BOUNDS_DTYPE)
    for j in range(count):
        rows = live_rows(ref, bi.spawner_base + j, num_spawners, num_metadata)
        lo, hi = box_of(ref.particles[rows, position_word:position_word + 3])
        out[j]["min"], out[j]["max"], out[j]["count"] = lo.view(np.float32), hi.view(np.float32), len(rows)
    return out


def assert_bounds_equal(got: np.ndarray, want: np.ndarray, what: str = ""):
    """Bit for bit, NaN-proof and sign-of-zero-proof: the records are compared as words."""
    np.testing.assert_array_equal(np.ascontiguousarray(got).view(np.uint32).reshape(-1, 8),
                                  np.ascontiguousarray(want).view(np.uint32).reshape(-1, 8), err_msg=f"{what}: bounds records")
