"""ctypes binding of ``libhanabi_b200.so`` (the C ABI declared in ``include/hanabi_b200.h``).

This is the reference-side binding a maintainer would write in Rust with ``extern "C"`` (see
INTEGRATION.md); here it is what the tests and the benchmark call. There is no fallback of any kind:
if the shared library is missing, importing this module raises, and if no GPU is present
``hnb_ctx_create`` returns ``HNB_ERR_NO_DEVICE``.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

_LIB_PATH = Path(__file__).resolve().parent / "libhanabi_b200.so"


class HanabiError(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__(f"hanabi_b200 error {code}: {message}")
        self.code = code
        self.message = message


HNB_OK = 0
HNB_ERR_INVALID_ARG = -1
HNB_ERR_CUDA = -2
HNB_ERR_NVRTC = -3
HNB_ERR_NO_DEVICE = -4
HNB_ERR_OUT_OF_RANGE = -5
HNB_ERR_EXPR = -6
HNB_ERR_LAYOUT = -7
HNB_ERR_NOT_READY = -8
HNB_ERR_BATCH_COVERAGE = -9

INVALID = 0xFFFFFFFF

u32 = C.c_uint32
i32 = C.c_int32
f32 = C.c_float


class SimParams(C.Structure):
    _fields_ = [("delta_time", f32), ("time", f32), ("virtual_delta_time", f32), ("virtual_time", f32),
                ("real_delta_time", f32), ("real_time", f32), ("num_effects", u32)]


class Transform(C.Structure):
    _fields_ = [("x_row", f32 * 4), ("y_row", f32 * 4), ("z_row", f32 * 4)]

    @classmethod
    def identity(cls) -> "Transform":
        return cls((f32 * 4)(1, 0, 0, 0), (f32 * 4)(0, 1, 0, 0), (f32 * 4)(0, 0, 1, 0))


class Spawner(C.Structure):
    _fields_ = [("transform", Transform), ("inverse_transform", Transform), ("spawn", i32), ("seed", u32),
                ("render_pong", u32), ("effect_metadata_index", u32), ("draw_indirect_index", u32),
                ("slab_offset", u32), ("parent_slab_offset", u32), ("_pad", u32)]


class BatchInfo(C.Structure):
    _fields_ = [("total_spawn_count", u32), ("total_update_count", u32), ("spawner_base", u32),
                ("base_particle", u32), ("prefix_sum_offset", u32), ("prefix_sum_count", u32)]


class EffectMetadata(C.Structure):
    _fields_ = [(n, u32) for n in (
        "capacity", "alive_count", "max_update", "max_spawn", "indirect_write_index", "indirect_draw_index",
        "init_indirect_dispatch_index", "properties_array_index", "local_child_index", "global_child_index",
        "base_child_index", "particle_stride", "sort_key_offset", "sort_key2_offset", "particle_counter")]


class DrawIndexedIndirectArgs(C.Structure):
    _fields_ = [("index_count", u32), ("instance_count", u32), ("first_index", u32), ("base_vertex", i32),
                ("first_instance", u32)]


class DispatchIndirectArgs(C.Structure):
    _fields_ = [("x", u32), ("y", u32), ("z", u32)]


class IndirectIndex(C.Structure):
    _fields_ = [("ping", u32), ("pong", u32), ("dead", u32)]


class ChildInfo(C.Structure):
    _fields_ = [("init_indirect_dispatch_index", u32), ("event_count", i32)]


class SlabView(C.Structure):
    _fields_ = [("capacity_rows", u32), ("particle_stride", u32), ("num_planes", u32), ("_pad", u32),
                ("planes", C.c_void_p * 16), ("plane_offset", u32 * 16), ("plane_width", u32 * 16),
                ("ping", C.c_void_p), ("pong", C.c_void_p), ("dead", C.c_void_p)]


class AttrLayout(C.Structure):
    _fields_ = [("name", C.c_char_p), ("value_type", u32), ("offset", u32)]


class EffectDesc(C.Structure):
    _fields_ = [("name", C.c_char_p), ("attrs", C.POINTER(AttrLayout)), ("n_attrs", u32), ("particle_stride", u32),
                ("properties_struct", C.c_char_p), ("properties_size", u32), ("init_code", C.c_char_p),
                ("init_extra", C.c_char_p), ("sim_space_code", C.c_char_p), ("age_code", C.c_char_p),
                ("reap_code", C.c_char_p), ("update_code", C.c_char_p), ("update_extra", C.c_char_p), ("flags", u32),
                ("parent_attrs", C.POINTER(AttrLayout)), ("n_parent_attrs", u32), ("parent_particle_stride", u32),
                ("num_event_bindings", u32)]


class BatchLaunch(C.Structure):
    _fields_ = [("effect", u32), ("slab", u32), ("batch_info_index", u32), ("total_spawn_count", u32),
                ("parent_slab", u32), ("consume_events", u32), ("emit_events", u32 * 4)]

    @classmethod
    def make(cls, effect: int, slab: int, batch_info_index: int = 0, total_spawn_count: int = 0,
             parent_slab: int = INVALID, consume_events: int = INVALID, emit_events=()) -> "BatchLaunch":
        ev = list(emit_events) + [INVALID] * (4 - len(emit_events))
        return cls(effect, slab, batch_info_index, total_spawn_count, parent_slab, consume_events, (u32 * 4)(*ev))


# value types (hnb_value_type)
BOOL, FLOAT, INT, UINT = 0, 1, 2, 3
BVEC2, BVEC3, BVEC4 = 4, 5, 6
VEC2, VEC3, VEC4 = 7, 8, 9
IVEC2, IVEC3, IVEC4 = 10, 11, 12
UVEC2, UVEC3, UVEC4 = 13, 14, 15

EFFECT_LOCAL_SPACE = 1 << 0
EFFECT_CONSUME_GPU_SPAWN_EVENTS = 1 << 1
EFFECT_EMIT_GPU_SPAWN_EVENTS = 1 << 2
EFFECT_READ_PARENT_PARTICLE = 1 << 3
EFFECT_RELAXED_ORDER = 1 << 4
EFFECT_RIBBONS = 1 << 5
EFFECT_FAST_MATH = 1 << 6
EFFECT_ORDERED_EVENTS = 1 << 7
EFFECT_SECTOR_PLANES = 1 << 8
EFFECT_SLOT_ORDER = 1 << 9
SLAB_SECTOR_PLANES = 1 << 0


def _load() -> C.CDLL:
    if not _LIB_PATH.exists():
        raise ImportError(
            f"{_LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'`. "
            "hanabi_b200 has no CPU fallback.")
    return C.CDLL(str(_LIB_PATH))


lib = _load()
P = C.POINTER
vp = C.c_void_p

# name -> (restype, argtypes); every symbol declared in include/hanabi_b200.h
SIGNATURES = {
    "hnb_last_error": (C.c_char_p, []),
    "hnb_version": (C.c_char_p, []),
    "hnb_ctx_create": (i32, [i32, C.c_size_t, P(vp)]),
    "hnb_ctx_destroy": (None, [vp]),
    "hnb_sync": (i32, [vp]),
    "hnb_ctx_stream": (C.c_size_t, [vp]),
    "hnb_ctx_launch_count": (C.c_uint64, [vp]),
    "hnb_ctx_frame_count": (None, [vp, P(C.c_uint64), P(C.c_uint64)]),
    "hnb_slab_create": (i32, [vp, u32, u32, P(u32)]),
    "hnb_slab_create_ex": (i32, [vp, u32, u32, u32, P(u32)]),
    "hnb_slab_destroy": (i32, [vp, u32]),
    "hnb_slab_reset_rows": (i32, [vp, u32, u32, u32]),
    "hnb_slab_rebuild_alive_bits": (i32, [vp, u32, u32, u32, u32, u32]),
    "hnb_slab_upload_aos": (i32, [vp, u32, u32, u32, vp]),
    "hnb_slab_download_aos": (i32, [vp, u32, u32, u32, vp]),
    "hnb_slab_upload_indirect": (i32, [vp, u32, u32, u32, vp]),
    "hnb_slab_download_indirect": (i32, [vp, u32, u32, u32, vp]),
    "hnb_slab_fill_c5": (i32, [vp, u32, u32, u32, u32, f32, f32]),
    "hnb_slab_checksum": (i32, [vp, u32, u32, u32, P(C.c_uint64)]),
    "hnb_slab_checksum_indirect": (i32, [vp, u32, u32, u32, P(C.c_uint64)]),
    "hnb_slab_fill_c5_ex": (i32, [vp, u32, u32, u32, u32, f32, f32, u32]),
    "hnb_slab_repack": (i32, [vp, u32, u32, u32, u32, u32]),
    "hnb_instance_snapshot_bytes": (C.c_size_t, [u32, u32]),
    "hnb_instance_snapshot": (i32, [vp, u32, u32, u32, u32, u32, vp, C.c_size_t]),
    "hnb_instance_restore": (i32, [vp, u32, u32, u32, u32, u32, vp, C.c_size_t]),
    "hnb_slab_checksum_ex": (i32, [vp, u32, u32, u32, C.c_uint64, P(C.c_uint64)]),
    "hnb_slab_device_view": (i32, [vp, u32, P(SlabView)]),
    "hnb_slab_export_aos_device": (i32, [vp, u32, u32, u32, vp]),
    "hnb_slab_import_aos_device": (i32, [vp, u32, u32, u32, vp]),
    "hnb_slab_export_indirect_device": (i32, [vp, u32, u32, u32, vp]),
    "hnb_slab_import_indirect_device": (i32, [vp, u32, u32, u32, vp]),
    "hnb_device_alloc": (vp, [vp, C.c_size_t]),
    "hnb_device_free": (None, [vp, vp]),
    "hnb_device_download": (i32, [vp, vp, vp, C.c_size_t]),
    "hnb_device_upload": (i32, [vp, vp, vp, C.c_size_t]),
    "hnb_effect_compile": (i32, [vp, P(EffectDesc), P(u32)]),
    "hnb_effect_destroy": (i32, [vp, u32]),
    "hnb_compile_job_start": (vp, [P(EffectDesc)]),
    "hnb_compile_job_poll": (i32, [vp]),
    "hnb_compile_job_wait": (i32, [vp]),
    "hnb_compile_job_destroy": (None, [vp]),
    "hnb_effect_create_from_job": (i32, [vp, vp, P(u32)]),
    "hnb_effect_generate_source": (i32, [P(EffectDesc), C.c_char_p, C.c_size_t, P(C.c_size_t)]),
    "hnb_nvrtc_check": (i32, [C.c_char_p, P(C.c_size_t)]),
    "hnb_set_sim_params": (i32, [vp, P(SimParams)]),
    "hnb_upload_spawners": (i32, [vp, P(Spawner), u32]),
    "hnb_upload_batches": (i32, [vp, P(BatchInfo), u32, P(u32), u32]),
    "hnb_metadata_insert": (i32, [vp, u32, P(EffectMetadata)]),
    "hnb_draw_args_insert": (i32, [vp, u32, P(DrawIndexedIndirectArgs)]),
    "hnb_upload_properties": (i32, [vp, u32, u32, vp, u32]),
    "hnb_event_buffer_create": (i32, [vp, u32, P(u32)]),
    "hnb_child_info_insert": (i32, [vp, u32, P(ChildInfo)]),
    "hnb_read_child_info": (i32, [vp, u32, P(ChildInfo)]),
    "hnb_event_buffer_download": (i32, [vp, u32, u32, u32, P(u32)]),
    "hnb_simulate": (i32, [vp, P(BatchLaunch), u32]),
    "hnb_pass_init": (i32, [vp, P(BatchLaunch)]),
    "hnb_pass_indirect": (i32, [vp]),
    "hnb_pass_prefix_sum": (i32, [vp]),
    "hnb_pass_update": (i32, [vp, P(BatchLaunch)]),
    "hnb_pass_sort": (i32, [vp, P(BatchLaunch)]),
    "hnb_pass_fill_dispatch_args": (i32, [vp, P(u32), u32, u32, P(u32), u32, u32, u32, u32]),
    "hnb_read_metadata": (i32, [vp, u32, P(EffectMetadata)]),
    "hnb_read_draw_args": (i32, [vp, u32, P(DrawIndexedIndirectArgs)]),
    "hnb_read_spawner": (i32, [vp, u32, P(Spawner)]),
    "hnb_read_batch_info": (i32, [vp, u32, P(BatchInfo)]),
    "hnb_read_prefix_sum": (i32, [vp, u32, u32, P(u32)]),
    "hnb_read_dispatch_args": (i32, [vp, u32, P(DispatchIndirectArgs)]),
    "hnb_read_tile_size": (i32, [vp, u32, P(u32)]),
    "hnb_read_draw_args_async": (i32, [vp, u32, u32, vp]),
    "hnb_ctx_set_count_mailbox": (i32, [vp, vp, u32, u32]),
    "hnb_ctx_last_epoch": (i32, [vp, P(u32)]),
    "hnb_ctx_tile_state_clears": (i32, [vp, P(C.c_uint64)]),
    "hnb_host_alloc": (vp, [C.c_size_t]),
    "hnb_host_free": (None, [vp]),
    "hnb_ctx_read_debug": (i32, [vp, P(C.c_uint64), i32]),
    "hnb_ctx_read_debug_ring": (i32, [vp, P(C.c_uint64), i32]),
    "hnb_ctx_measure_sm_mhz": (i32, [vp, u32, P(C.c_double)]),
    "hnb_ctx_enable_kernel_timing": (i32, [vp, i32]),
    "hnb_ctx_kernel_time_ms": (i32, [vp, P(C.c_double), P(C.c_uint64)]),
}

for _name, (_res, _args) in SIGNATURES.items():
    _fn = getattr(lib, _name)
    _fn.restype = _res
    _fn.argtypes = _args


def last_error() -> str:
    return (lib.hnb_last_error() or b"").decode(errors="replace")


def check(code: int) -> None:
    if code != HNB_OK:
        raise HanabiError(code, last_error())
