"""Thin object wrapper over the Level-1 C ABI (context, slabs, compiled effects, per-frame tables,
``simulate``). numpy arrays are only used as host buffers for upload / readback.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Iterable, Sequence

import numpy as np

from . import _native as N
from ._native import (BatchInfo, BatchLaunch, ChildInfo, DispatchIndirectArgs, DrawIndexedIndirectArgs,
                      EffectMetadata, SimParams, Spawner, Transform, check, lib)


@dataclass
class AttrField:
    """One field of the reference AoS ``Particle`` record."""
    name: str
    value_type: int
    offset: int


@dataclass
class LoweredEffect:
    """Python mirror of ``hnb_effect_desc``: an effect already lowered to CUDA C snippets."""
    name: str
    attrs: Sequence[AttrField]
    particle_stride: int
    init_code: str = ""
    init_extra: str = ""
    sim_space_code: str = ""
    age_code: str = ""
    reap_code: str = ""
    update_code: str = ""
    update_extra: str = ""
    properties_struct: str = ""
    properties_size: int = 0
    flags: int = 0
    parent_attrs: Sequence[AttrField] = field(default_factory=list)
    parent_particle_stride: int = 0
    num_event_bindings: int = 0

    def to_c(self):
        keep = []  # keep byte strings alive as long as the struct

        def b(s: str):
            v = s.encode()
            keep.append(v)
            return v

        def arr(fields):
            a = (N.AttrLayout * max(1, len(fields)))()
            for i, f in enumerate(fields):
                a[i] = N.AttrLayout(b(f.name), f.value_type, f.offset)
            keep.append(a)
            return a

        d = N.EffectDesc()
        d.name = b(self.name)
        d.attrs = arr(self.attrs)
        d.n_attrs = len(self.attrs)
        d.particle_stride = self.particle_stride
        d.properties_struct = b(self.properties_struct) if self.properties_size else None
        d.properties_size = self.properties_size
        d.init_code = b(self.init_code)
        d.init_extra = b(self.init_extra)
        d.sim_space_code = b(self.sim_space_code)
        d.age_code = b(self.age_code)
        d.reap_code = b(self.reap_code)
        d.update_code = b(self.update_code)
        d.update_extra = b(self.update_extra)
        d.flags = self.flags
        d.parent_attrs = arr(self.parent_attrs)
        d.n_parent_attrs = len(self.parent_attrs)
        d.parent_particle_stride = self.parent_particle_stride
        d.num_event_bindings = self.num_event_bindings
        return d, keep

    def generate_source(self) -> str:
        """Full CUDA C translation unit (no GPU needed)."""
        d, _keep = self.to_c()
        n = C.c_size_t(0)
        check(lib.hnb_effect_generate_source(C.byref(d), None, 0, C.byref(n)))
        buf = C.create_string_buffer(n.value + 1)
        check(lib.hnb_effect_generate_source(C.byref(d), buf, n.value + 1, C.byref(n)))
        return buf.value.decode()


class CompileJob:
    """Background NVRTC compilation of a lowered effect (needs no context and no GPU): `poll()` -> False while
    compiling, True when ready; raises HanabiError with the compiler log if it failed."""

    def __init__(self, fx: LoweredEffect):
        d, _keep = fx.to_c()
        self._h = lib.hnb_compile_job_start(C.byref(d))
        if not self._h:
            raise N.HanabiError(N.HNB_ERR_INVALID_ARG, N.last_error())

    def poll(self) -> bool:
        rc = lib.hnb_compile_job_poll(self._h)
        if rc < 0:
            raise N.HanabiError(rc, N.last_error())
        return rc == 1

    def wait(self) -> None:
        rc = lib.hnb_compile_job_wait(self._h)
        if rc < 0:
            raise N.HanabiError(rc, N.last_error())

    def close(self) -> None:
        if self._h:
            lib.hnb_compile_job_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def nvrtc_check(source: str) -> tuple[int, str]:
    """Compile a translation unit for sm_90a with NVRTC (no GPU needed). Returns (cubin bytes, log)."""
    n = C.c_size_t(0)
    check(lib.hnb_nvrtc_check(source.encode(), C.byref(n)))
    return n.value, N.last_error()


def make_spawner(spawn: int = 0, seed: int = 0, effect_metadata_index: int = 0, draw_indirect_index: int = 0,
                 slab_offset: int = 0, parent_slab_offset: int = N.INVALID, transform: Transform | None = None,
                 inverse_transform: Transform | None = None) -> Spawner:
    s = Spawner()
    s.transform = transform or Transform.identity()
    s.inverse_transform = inverse_transform or Transform.identity()
    s.spawn = spawn
    s.seed = seed & 0xFFFFFFFF
    s.effect_metadata_index = effect_metadata_index
    s.draw_indirect_index = draw_indirect_index
    s.slab_offset = slab_offset
    s.parent_slab_offset = parent_slab_offset
    return s


def initial_metadata(capacity: int, draw_index: int = 0, particle_stride_words: int = 0,
                     properties_array_index: int = N.INVALID) -> EffectMetadata:
    """Initial row written by prepare_effect_metadata (reference mod.rs:6048-6070)."""
    m = EffectMetadata()
    m.capacity = capacity
    m.alive_count = 0
    m.max_update = 0
    m.max_spawn = capacity
    m.indirect_write_index = 0
    m.indirect_draw_index = draw_index
    m.init_indirect_dispatch_index = N.INVALID
    m.properties_array_index = properties_array_index
    m.local_child_index = N.INVALID
    m.global_child_index = N.INVALID
    m.base_child_index = N.INVALID
    m.particle_stride = particle_stride_words
    m.sort_key_offset = N.INVALID
    m.sort_key2_offset = N.INVALID
    m.particle_counter = 0
    return m


class Context:
    """One simulation context on one GPU (≙ the render-world resources of HanabiPlugin)."""

    def __init__(self, device: int = 0, stream: int = 0):
        h = C.c_void_p()
        check(lib.hnb_ctx_create(device, stream, C.byref(h)))
        self._h = h
        self.device = device

    def close(self) -> None:
        if self._h:
            lib.hnb_ctx_destroy(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- misc
    def sync(self) -> None:
        check(lib.hnb_sync(self._h))

    @property
    def stream(self) -> int:
        return lib.hnb_ctx_stream(self._h)

    @property
    def launch_count(self) -> int:
        return lib.hnb_ctx_launch_count(self._h)

    @property
    def frames_simulated(self) -> int:
        f, c = C.c_uint64(0), C.c_uint64(0)
        lib.hnb_ctx_frame_count(self._h, C.byref(f), C.byref(c))
        return f.value

    @property
    def frame_block_copies(self) -> int:
        f, c = C.c_uint64(0), C.c_uint64(0)
        lib.hnb_ctx_frame_count(self._h, C.byref(f), C.byref(c))
        return c.value

    def read_debug(self, clear: bool = True) -> list[int]:
        out = (C.c_uint64 * 16)()
        check(lib.hnb_ctx_read_debug(self._h, out, int(clear)))
        return list(out)

    def read_debug_ring(self, clear: bool = True) -> list[int]:
        out = (C.c_uint64 * 256)()
        check(lib.hnb_ctx_read_debug_ring(self._h, out, int(clear)))
        return list(out)

    def measure_sm_mhz(self, window_us: int = 50) -> float:
        out = C.c_double(0)
        check(lib.hnb_ctx_measure_sm_mhz(self._h, window_us, C.byref(out)))
        return out.value

    def enable_kernel_timing(self, on: bool = True) -> None:
        check(lib.hnb_ctx_enable_kernel_timing(self._h, int(on)))

    def kernel_time_ms(self) -> tuple[float, int]:
        ms, n = C.c_double(0), C.c_uint64(0)
        check(lib.hnb_ctx_kernel_time_ms(self._h, C.byref(ms), C.byref(n)))
        return ms.value, n.value

    # -- slabs
    def slab_create(self, capacity_rows: int, particle_stride: int, sector_planes: bool = False) -> int:
        out = N.u32(0)
        if sector_planes:
            check(lib.hnb_slab_create_ex(self._h, capacity_rows, particle_stride, N.SLAB_SECTOR_PLANES, C.byref(out)))
        else:
            check(lib.hnb_slab_create(self._h, capacity_rows, particle_stride, C.byref(out)))
        return out.value

    def slab_destroy(self, slab: int) -> None:
        check(lib.hnb_slab_destroy(self._h, slab))

    def slab_reset_rows(self, slab: int, first: int, count: int) -> None:
        check(lib.hnb_slab_reset_rows(self._h, slab, first, count))

    def slab_rebuild_alive_bits(self, slab: int, first: int, rows: int, column: int, alive_count: int) -> None:
        check(lib.hnb_slab_rebuild_alive_bits(self._h, slab, first, rows, column, alive_count))

    def slab_upload_aos(self, slab: int, first: int, particles: np.ndarray) -> None:
        a = np.ascontiguousarray(particles)
        count = a.shape[0]
        check(lib.hnb_slab_upload_aos(self._h, slab, first, count, a.ctypes.data_as(C.c_void_p)))

    def slab_download_aos(self, slab: int, first: int, count: int, stride: int) -> np.ndarray:
        out = np.empty((count, stride // 4), dtype=np.uint32)
        check(lib.hnb_slab_download_aos(self._h, slab, first, count, out.ctypes.data_as(C.c_void_p)))
        return out

    def slab_upload_indirect(self, slab: int, first: int, rows: np.ndarray) -> None:
        a = np.ascontiguousarray(rows, dtype=np.uint32).reshape(-1, 3)
        check(lib.hnb_slab_upload_indirect(self._h, slab, first, a.shape[0], a.ctypes.data_as(C.c_void_p)))

    def slab_download_indirect(self, slab: int, first: int, count: int) -> np.ndarray:
        out = np.empty((count, 3), dtype=np.uint32)
        check(lib.hnb_slab_download_indirect(self._h, slab, first, count, out.ctypes.data_as(C.c_void_p)))
        return out

    def slab_fill_c5(self, slab: int, first: int, count: int, seed: int, lifetime_lo: float, lifetime_hi: float,
                     logical_first: int | None = None) -> None:
        """`logical_first`: the slab rows hold logical rows [logical_first, +count) of an instance sharded over devices."""
        check(lib.hnb_slab_fill_c5_ex(self._h, slab, first, count, seed, lifetime_lo, lifetime_hi, first if logical_first is None else logical_first))

    def slab_repack(self, slab: int, effect: int, metadata_row: int, first: int, rows: int) -> None:
        """Move the live particles of the instance at slab rows [first, first+rows) (`rows` = its capacity) to the front of
        its slice in alive-list order; both alive lists and the dead stack become the identity and carry identity claims
        again (hnb_slab_repack). Call between frames; only enqueues work on the context stream."""
        check(lib.hnb_slab_repack(self._h, slab, effect, metadata_row, first, rows))

    @staticmethod
    def instance_snapshot_bytes(particle_stride: int, rows: int) -> int:
        """Bytes a snapshot of a `rows`-row instance may need: the 64-byte header and `rows` records."""
        return lib.hnb_instance_snapshot_bytes(particle_stride, rows)

    def instance_snapshot(self, slab: int, effect: int, metadata_row: int, first: int, rows: int, d_dst: int,
                          dst_bytes: int) -> None:
        """Write the header and the live records, in alive-list order, of the instance at slab rows [first, first+rows) to
        the device buffer `d_dst` (16-byte aligned, at least instance_snapshot_bytes(stride, rows) bytes; a
        hnb_device_alloc pointer or a torch tensor's data_ptr()). The instance is not modified; only enqueues work."""
        check(lib.hnb_instance_snapshot(self._h, slab, effect, metadata_row, first, rows, d_dst, dst_bytes))

    def instance_restore(self, slab: int, effect: int, metadata_row: int, first: int, rows: int, d_src: int,
                         src_bytes: int) -> None:
        """Put the particles of a snapshot at the front of the instance at slab rows [first, first+rows) (any slice, slab
        or context whose effect has the snapshot's stride); its lists, claims and alive bits become what slab_repack
        leaves. `src_bytes`: bytes readable at `d_src` (>= 64). Only enqueues work."""
        check(lib.hnb_instance_restore(self._h, slab, effect, metadata_row, first, rows, d_src, src_bytes))

    def slab_checksum(self, slab: int, first: int, count: int, index_base: int = 0) -> int:
        out = C.c_uint64(0)
        check(lib.hnb_slab_checksum_ex(self._h, slab, first, count, index_base, C.byref(out)))
        return out.value

    # -- device-resident interop (the renderer's view of the state, §8 f-2)
    def slab_device_view(self, slab: int) -> "N.SlabView":
        out = N.SlabView()
        check(lib.hnb_slab_device_view(self._h, slab, C.byref(out)))
        return out

    def device_alloc(self, nbytes: int) -> int:
        p = lib.hnb_device_alloc(self._h, nbytes)
        if not p:
            raise MemoryError(f"hnb_device_alloc({nbytes}) failed")
        return p

    def device_free(self, ptr: int) -> None:
        lib.hnb_device_free(self._h, ptr)

    def device_download(self, ptr: int, nbytes: int) -> np.ndarray:
        out = np.empty(nbytes // 4, dtype=np.uint32)
        check(lib.hnb_device_download(self._h, out.ctypes.data_as(C.c_void_p), ptr, nbytes))
        return out

    def device_upload(self, ptr: int, data: np.ndarray) -> None:
        a = np.ascontiguousarray(data)
        check(lib.hnb_device_upload(self._h, ptr, a.ctypes.data_as(C.c_void_p), a.nbytes))

    def slab_export_aos_device(self, slab: int, first: int, count: int, d_dst: int) -> None:
        check(lib.hnb_slab_export_aos_device(self._h, slab, first, count, d_dst))

    def slab_import_aos_device(self, slab: int, first: int, count: int, d_src: int) -> None:
        check(lib.hnb_slab_import_aos_device(self._h, slab, first, count, d_src))

    def slab_export_indirect_device(self, slab: int, first: int, count: int, d_dst: int) -> None:
        check(lib.hnb_slab_export_indirect_device(self._h, slab, first, count, d_dst))

    def slab_import_indirect_device(self, slab: int, first: int, count: int, d_src: int) -> None:
        check(lib.hnb_slab_import_indirect_device(self._h, slab, first, count, d_src))

    def slab_checksum_indirect(self, slab: int, first: int, count: int) -> int:
        out = C.c_uint64(0)
        check(lib.hnb_slab_checksum_indirect(self._h, slab, first, count, C.byref(out)))
        return out.value

    # -- effects
    def effect_compile(self, fx: LoweredEffect) -> int:
        d, _keep = fx.to_c()
        out = N.u32(0)
        check(lib.hnb_effect_compile(self._h, C.byref(d), C.byref(out)))
        return out.value

    def effect_destroy(self, effect: int) -> None:
        check(lib.hnb_effect_destroy(self._h, effect))

    def effect_create_from_job(self, job: "CompileJob") -> int:
        """Register an effect compiled in the background; raises HanabiError(HNB_ERR_NOT_READY) while the job runs."""
        out = N.u32(0)
        check(lib.hnb_effect_create_from_job(self._h, job._h, C.byref(out)))
        return out.value

    def upload_properties(self, effect: int, array_index: int, blob: bytes) -> None:
        buf = C.create_string_buffer(blob, len(blob))
        check(lib.hnb_upload_properties(self._h, effect, array_index, buf, len(blob)))

    # -- per-frame tables
    def set_sim_params(self, delta_time: float, time: float = 0.0, num_effects: int = 1, virtual_delta_time=None,
                       virtual_time=None, real_delta_time=None, real_time=None) -> None:
        p = SimParams(delta_time, time,
                      delta_time if virtual_delta_time is None else virtual_delta_time,
                      time if virtual_time is None else virtual_time,
                      delta_time if real_delta_time is None else real_delta_time,
                      time if real_time is None else real_time, num_effects)
        check(lib.hnb_set_sim_params(self._h, C.byref(p)))

    def upload_spawners(self, spawners: Sequence[Spawner]) -> None:
        arr = (Spawner * max(1, len(spawners)))(*spawners)
        check(lib.hnb_upload_spawners(self._h, arr, len(spawners)))

    def upload_spawners_raw(self, arr, n: int) -> None:
        check(lib.hnb_upload_spawners(self._h, arr, n))

    def upload_batches(self, batches: Sequence[BatchInfo], prefix_sum: Iterable[int]) -> None:
        barr = (BatchInfo * max(1, len(batches)))(*batches)
        pl = list(prefix_sum)
        parr = (N.u32 * max(1, len(pl)))(*pl)
        check(lib.hnb_upload_batches(self._h, barr, len(batches), parr, len(pl)))

    def upload_batches_raw(self, barr, nb: int, parr, np_: int) -> None:
        check(lib.hnb_upload_batches(self._h, barr, nb, parr, np_))

    def metadata_insert(self, row: int, md: EffectMetadata) -> None:
        check(lib.hnb_metadata_insert(self._h, row, C.byref(md)))

    def draw_args_insert(self, row: int, args: DrawIndexedIndirectArgs | None = None) -> None:
        a = args or DrawIndexedIndirectArgs(6, 0, 0, 0, 0)
        check(lib.hnb_draw_args_insert(self._h, row, C.byref(a)))

    def event_buffer_create(self, capacity: int = 256) -> int:
        out = N.u32(0)
        check(lib.hnb_event_buffer_create(self._h, capacity, C.byref(out)))
        return out.value

    def child_info_insert(self, row: int, init_indirect_dispatch_index: int = 0, event_count: int = 0) -> None:
        ci = ChildInfo(init_indirect_dispatch_index, event_count)
        check(lib.hnb_child_info_insert(self._h, row, C.byref(ci)))

    def read_child_info(self, row: int) -> ChildInfo:
        ci = ChildInfo()
        check(lib.hnb_read_child_info(self._h, row, C.byref(ci)))
        return ci

    def event_buffer_download(self, buf: int, first: int, count: int) -> np.ndarray:
        out = (N.u32 * max(1, count))()
        check(lib.hnb_event_buffer_download(self._h, buf, first, count, out))
        return np.array(out[:count], dtype=np.uint32)

    # -- passes
    # -- count mailbox (pinned host memory written by the update pass; see hnb_ctx_set_count_mailbox)
    def set_count_mailbox(self, rows: int, ring: int = 4):
        """Allocates a pinned mailbox of ring x rows 64-bit words, attaches it and returns a ctypes view of it (None: detach)."""
        if rows == 0:
            check(lib.hnb_ctx_set_count_mailbox(self._h, None, 0, 0))
            return None  # (the pinned block of an earlier attach stays allocated: frames already queued may still post into it)
        p = lib.hnb_host_alloc(rows * ring * 8)
        if not p:
            raise MemoryError("hnb_host_alloc")
        check(lib.hnb_ctx_set_count_mailbox(self._h, p, rows, ring))
        self._mailbox = ((C.c_uint64 * (rows * ring)).from_address(p), rows, ring, p)
        return self._mailbox[0]

    def last_epoch(self) -> int:
        e = N.u32(0)
        check(lib.hnb_ctx_last_epoch(self._h, C.byref(e)))
        return e.value

    def tile_state_clears(self) -> int:
        """How often a batch's look-back tile states were zeroed before an update launch (hnb_ctx_tile_state_clears)."""
        n = C.c_uint64(0)
        check(lib.hnb_ctx_tile_state_clears(self._h, C.byref(n)))
        return n.value

    def mailbox_count(self, epoch: int, row: int = 0, spin: bool = True):
        """instance_count the frame `epoch` published for draw-indirect row `row` (spins until the word has landed)."""
        import time
        view, rows, ring, _ = self._mailbox
        i = (epoch % ring) * rows + row
        deadline = None
        while True:
            w = view[i]
            if (w >> 32) == epoch:
                return w & 0xFFFFFFFF
            if not spin:
                return None
            if deadline is None:
                deadline = time.monotonic() + 10.0
            elif time.monotonic() > deadline:  # e.g. an effect compiled with RELAXED_ORDER (no mailbox), or a later frame reused the slot
                raise TimeoutError(f"count mailbox: frame {epoch} never posted row {row} (slot holds frame {w >> 32})")

    def simulate(self, launches: Sequence[BatchLaunch]) -> None:
        arr = (BatchLaunch * max(1, len(launches)))(*launches)
        check(lib.hnb_simulate(self._h, arr, len(launches)))

    def simulate_raw(self, arr, n: int) -> None:
        check(lib.hnb_simulate(self._h, arr, n))

    def pass_init(self, launch: BatchLaunch) -> None:
        check(lib.hnb_pass_init(self._h, C.byref(launch)))

    def pass_indirect(self) -> None:
        check(lib.hnb_pass_indirect(self._h))

    def pass_prefix_sum(self) -> None:
        check(lib.hnb_pass_prefix_sum(self._h))

    def pass_update(self, launch: BatchLaunch) -> None:
        check(lib.hnb_pass_update(self._h, C.byref(launch)))

    def pass_sort(self, launch: BatchLaunch) -> None:
        """Ribbon sort of every instance of the batch (vfx_sort_fill / vfx_sort / vfx_sort_copy)."""
        check(lib.hnb_pass_sort(self._h, C.byref(launch)))

    def pass_fill_dispatch_args(self, src: Sequence[int], src_offset: int, src_stride: int, dst: Sequence[int],
                                dst_offset: int, dst_stride: int, count: int) -> list[int]:
        s = (N.u32 * max(1, len(src)))(*src)
        d = (N.u32 * max(1, len(dst)))(*dst)
        check(lib.hnb_pass_fill_dispatch_args(self._h, s, src_offset, src_stride, d, len(dst), dst_offset, dst_stride, count))
        return list(d)

    # -- readback
    def read_metadata(self, row: int) -> EffectMetadata:
        m = EffectMetadata()
        check(lib.hnb_read_metadata(self._h, row, C.byref(m)))
        return m

    def read_draw_args(self, row: int) -> DrawIndexedIndirectArgs:
        a = DrawIndexedIndirectArgs()
        check(lib.hnb_read_draw_args(self._h, row, C.byref(a)))
        return a

    def read_spawner(self, row: int) -> Spawner:
        s = Spawner()
        check(lib.hnb_read_spawner(self._h, row, C.byref(s)))
        return s

    def read_batch_info(self, row: int) -> BatchInfo:
        b = BatchInfo()
        check(lib.hnb_read_batch_info(self._h, row, C.byref(b)))
        return b

    def read_prefix_sum(self, first: int, count: int) -> list[int]:
        out = (N.u32 * max(1, count))()
        check(lib.hnb_read_prefix_sum(self._h, first, count, out))
        return list(out[:count])

    def read_dispatch_args(self, row: int) -> DispatchIndirectArgs:
        a = DispatchIndirectArgs()
        check(lib.hnb_read_dispatch_args(self._h, row, C.byref(a)))
        return a

    def read_tile_size(self, row: int) -> int:
        """Rows per update tile of batch `row` at its last launch (the low 16 bits of hnb_read_tile_size's word)."""
        w = N.u32()
        check(lib.hnb_read_tile_size(self._h, row, C.byref(w)))
        return w.value & 0xFFFF
