"""ctypes binding of oracle/libvfx_oracle.so (the C restatement). TEST INFRASTRUCTURE ONLY — see the
header of vfx_oracle.c for who may import this."""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

_DIR = Path(__file__).resolve().parent
_LIB = _DIR / "libvfx_oracle.so"

u32, i32, f32 = C.c_uint32, C.c_int32, C.c_float


class SimParams(C.Structure):
    _fields_ = [("delta_time", f32), ("time", f32), ("virtual_delta_time", f32), ("virtual_time", f32),
                ("real_delta_time", f32), ("real_time", f32), ("num_effects", u32)]


class Spawner(C.Structure):
    _fields_ = [("transform", f32 * 12), ("inverse_transform", f32 * 12), ("spawn", i32), ("seed", u32),
                ("render_indirect_read_index", u32), ("effect_metadata_index", u32), ("draw_indirect_index", u32),
                ("slab_offset", u32), ("parent_slab_offset", u32), ("unused", u32)]


class BatchInfo(C.Structure):
    _fields_ = [("total_spawn_count", u32), ("total_update_count", u32), ("spawner_base", u32),
                ("base_particle", u32), ("prefix_sum_offset", u32), ("prefix_sum_count", u32)]


class EffectMetadata(C.Structure):
    _fields_ = [(n, u32) for n in (
        "capacity", "alive_count", "max_update", "max_spawn", "indirect_write_index", "indirect_render_index",
        "init_indirect_dispatch_index", "properties_array_index", "local_child_index", "global_child_index",
        "base_child_index", "particle_stride", "sort_key_offset", "sort_key2_offset", "particle_counter")]


class ChildInfo(C.Structure):
    _fields_ = [("init_indirect_dispatch_index", u32), ("event_count", i32)]


class EffectLocation(C.Structure):
    _fields_ = [("effect_index", u32), ("base_particle", u32), ("update_index", u32)]


class ConstInit(C.Structure):
    _fields_ = [("stride_words", u32), ("words", u32 * 64)]


def _build() -> None:
    subprocess.run(["make", "-s", "-C", str(_DIR)], check=True)


def load() -> C.CDLL:
    if not _LIB.exists():
        _build()
    lib = C.CDLL(str(_LIB))
    P = C.POINTER
    vp = C.c_void_p
    lib.orc_pcg_hash.restype = u32
    lib.orc_pcg_hash.argtypes = [u32]
    lib.orc_to_float01.restype = f32
    lib.orc_to_float01.argtypes = [u32]
    lib.orc_frand.restype = f32
    lib.orc_frand.argtypes = [P(u32)]
    for n in ("orc_frand2", "orc_frand3", "orc_frand4"):
        getattr(lib, n).restype = None
        getattr(lib, n).argtypes = [P(u32), P(f32)]
    lib.orc_find_location_from_particle.restype = EffectLocation
    lib.orc_find_location_from_particle.argtypes = [P(BatchInfo), P(u32), u32]
    lib.orc_indirect.restype = None
    lib.orc_indirect.argtypes = [P(SimParams), P(EffectMetadata), P(u32), P(Spawner), P(u32), P(ChildInfo), u32]
    lib.orc_prefix_sum.restype = None
    lib.orc_prefix_sum.argtypes = [P(BatchInfo), u32, P(u32), P(u32)]
    lib.orc_fill_dispatch_args.restype = None
    lib.orc_fill_dispatch_args.argtypes = [P(u32), P(u32), u32, u32, u32, u32, u32]
    lib.orc_sort_fill.restype = None
    lib.orc_sort_fill.argtypes = [P(C.c_int32), vp, vp, vp, P(EffectMetadata), P(Spawner), u32]
    lib.orc_sort.restype = None
    lib.orc_sort.argtypes = [P(C.c_int32), vp]
    lib.orc_sort_copy.restype = None
    lib.orc_sort_copy.argtypes = [vp, vp, P(EffectMetadata), P(Spawner), u32]
    lib.orc_update.restype = None
    lib.orc_update.argtypes = [P(SimParams), P(u32), vp, u32, vp, P(Spawner), P(u32), P(BatchInfo), P(EffectMetadata),
                               u32, vp, vp]
    lib.orc_init.restype = None
    lib.orc_init.argtypes = [P(SimParams), vp, u32, vp, P(Spawner), P(u32), P(BatchInfo), P(EffectMetadata), u32, vp, vp]
    for n in ("orc_body_update_noop", "orc_body_update_c5", "orc_body_init_const", "orc_body_init_sparks"):
        getattr(lib, n).restype = vp
        getattr(lib, n).argtypes = []
    lib.orc_fill_c5.restype = None
    lib.orc_fill_c5.argtypes = [vp, vp, u32, u32, u32, f32, f32]
    lib.orc_update_c5_parallel.restype = u32
    lib.orc_update_c5_parallel.argtypes = [P(SimParams), P(u32), vp, vp, P(Spawner), P(EffectMetadata), P(f32), vp, C.c_int]
    lib.orc_checksum.restype = C.c_uint64
    lib.orc_checksum.argtypes = [vp, u32, u32, u32]
    lib.orc_fill_c5_ex.restype = None
    lib.orc_fill_c5_ex.argtypes = [vp, vp, u32, u32, u32, f32, f32, u32]
    lib.orc_indirect_reset.restype = None
    lib.orc_indirect_reset.argtypes = [vp, u32, u32]
    lib.orc_checksum_ex.restype = C.c_uint64
    lib.orc_checksum_ex.argtypes = [vp, u32, u32, u32, C.c_uint64]
    lib.orc_row_digests.restype = None
    lib.orc_row_digests.argtypes = [vp, u32, u32, vp]
    lib.orc_set_threads.restype = None
    lib.orc_set_threads.argtypes = [C.c_int]
    lib.orc_max_threads.restype = C.c_int
    lib.orc_max_threads.argtypes = []
    return lib


def ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


def identity_rows():
    return (f32 * 12)(1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0)
