"""Runs the real `hnb_init` / `hnb_update` kernel templates on the CPU: test infrastructure for `-m "not gpu"` runs.

The full generated translation unit of an effect (vocabulary + tables + generated bodies + hnb_particle_kernels.cuh)
is compiled with g++ behind a small emulation layer: every CUDA thread is an OS thread, a warp is 32 threads with a
barrier and an exchange array (`__ballot_sync`, `__shfl_sync`, `__syncwarp`), a CTA adds a 256-thread barrier, its
dynamic shared memory and its static shared words; atomics are `__atomic` builtins. The three inline-PTX helpers of
the kernels (relaxed 64-bit load / store of a tile state, `%lanemask_lt`) and the two shared-memory declarations are
replaced textually (asserted) — nothing else of the kernel text changes. The grid is a handful of CTAs, so tile
tickets, the look-back chain, deferred compaction, the dead-stack writes and the last-tile bookkeeping all run
exactly as written, under real (OS-scheduled) concurrency.

What is NOT emulated: the effect-independent bookkeeping kernel between init and update (its semantics come from the
C oracle's indirect / prefix-sum restatements plus the deferred init accounting restated in `EmuWorld.frame`), GPU
spawn events, and of course timing. The GPU suite covers those on the device.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
from pathlib import Path

import numpy as np

from oracle import c_oracle as O

ROOT = Path(__file__).resolve().parent.parent
OUT = ROOT / "build" / "kernel_emu"

PRELUDE = r"""
#include <algorithm>
#include <math.h>
#include <pthread.h>
#include <sched.h>
#include <stdint.h>
#include <string.h>
#include <thread>
#include <vector>
#define __device__
#define __forceinline__ inline
#define __global__
#define __launch_bounds__(...)
#define __align__(n)
struct float2 { float x, y; };
struct float4 { float x, y, z, w; };
static inline float2 make_float2(float x, float y) { float2 r = {x, y}; return r; }
static inline float4 make_float4(float x, float y, float z, float w) { float4 r = {x, y, z, w}; return r; }
static inline float __uint_as_float(unsigned int u) { float f; memcpy(&f, &u, 4); return f; }
static inline float __int_as_float(int u) { float f; memcpy(&f, &u, 4); return f; }
static inline unsigned int __float_as_uint(float f) { unsigned int u; memcpy(&u, &f, 4); return u; }
static inline int __float_as_int(float f) { int u; memcpy(&u, &f, 4); return u; }
namespace emu {
struct Warp { pthread_barrier_t bar; unsigned long long slot[32]; };
struct Cta { pthread_barrier_t bar; unsigned char* dyn; unsigned int statics[16]; Warp warps[32]; };
struct Tls { unsigned tid, bid, lane; Cta* cta; Warp* warp; };
static thread_local Tls tls;
struct Dim3 { unsigned x, y, z; };
static inline void warp_sync() { pthread_barrier_wait(&tls.warp->bar); }
static inline unsigned char* dyn_smem() { return tls.cta->dyn; }
static inline unsigned int* static_u32(int i) { return &tls.cta->statics[i]; }
template <typename T> static inline T exchange(T v, unsigned src) {
    unsigned long long raw = 0; memcpy(&raw, &v, sizeof(T));
    tls.warp->slot[tls.lane] = raw;
    warp_sync();
    unsigned long long got = tls.warp->slot[src & 31u];
    warp_sync();
    T out; memcpy(&out, &got, sizeof(T));
    return out;
}
}  // namespace emu
#define threadIdx (emu::Dim3{emu::tls.tid, 0u, 0u})
#define blockIdx (emu::Dim3{emu::tls.bid, 0u, 0u})
static inline void __syncwarp() { emu::warp_sync(); }
static inline void __syncthreads() { pthread_barrier_wait(&emu::tls.cta->bar); }
static inline unsigned __ballot_sync(unsigned, int pred) {
    emu::tls.warp->slot[emu::tls.lane] = pred ? 1ull : 0ull;
    emu::warp_sync();
    unsigned m = 0;
    for (unsigned i = 0; i < 32; ++i) m |= unsigned(emu::tls.warp->slot[i]) << i;
    emu::warp_sync();
    return m;
}
template <typename T> static inline T __shfl_sync(unsigned, T v, int src) { return emu::exchange(v, unsigned(src)); }
template <typename T> static inline T __shfl_xor_sync(unsigned, T v, int d) { return emu::exchange(v, emu::tls.lane ^ unsigned(d)); }
static inline int __popc(unsigned x) { return __builtin_popcount(x); }
static inline int __ffs(unsigned x) { return __builtin_ffs(int(x)); }
static inline void __nanosleep(unsigned) { sched_yield(); }
static inline unsigned atomicAdd(unsigned* p, unsigned v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
static inline int atomicAdd(int* p, int v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
static inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
static inline unsigned atomicSub(unsigned* p, unsigned v) { return __atomic_fetch_sub(p, v, __ATOMIC_SEQ_CST); }
static inline unsigned atomicOr(unsigned* p, unsigned v) { return __atomic_fetch_or(p, v, __ATOMIC_SEQ_CST); }
static inline unsigned atomicAnd(unsigned* p, unsigned v) { return __atomic_fetch_and(p, v, __ATOMIC_SEQ_CST); }
static inline unsigned long long atomicMax(unsigned long long* p, unsigned long long v) {
    unsigned long long old = __atomic_load_n(p, __ATOMIC_SEQ_CST);
    while (old < v && !__atomic_compare_exchange_n(p, &old, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
    return old;
}
"""

# exact kernel-source lines that need a host spelling (asserted to be present: the harness follows the product text)
SUBSTITUTIONS = [
    ('HNB_DI void hnb_st_state(u64* p, u64 v) { asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }',
     'HNB_DI void hnb_st_state(u64* p, u64 v) { __atomic_store_n(p, v, __ATOMIC_RELAXED); }'),
    ('    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");',
     '    v = __atomic_load_n(p, __ATOMIC_RELAXED); sched_yield();  /* a poll: let the OS run somebody else */'),
    ('    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));', '    m = (1u << emu::tls.lane) - 1u;'),
    ('extern __shared__ __align__(16) unsigned char hnb_smem[];', '#define hnb_smem (emu::dyn_smem())'),
    ('    __shared__ u32 sh_first_ticket;', '    u32& sh_first_ticket = *emu::static_u32(0);'),
]

DRIVER = r"""
struct EmuBatch {
    void* frame; void* spawners; uint32_t* spawn_prefix; uint32_t* prefix_sum; uint32_t* tile_prefix; void* batch_info;
    uint32_t* batch_tiles; uint32_t* ticket; unsigned long long* tile_state; void* metadata; uint32_t* draw_args; void* properties;
    void* planes[16]; uint32_t* ping; uint32_t* pong; uint32_t* dead;
    uint32_t capacity, init_thread_count, properties_stride, tile_rows;
    // GPU spawn events (EmuScene)
    void* child_infos; uint32_t* consume_events; uint32_t* emit_events[4]; uint32_t emit_caps[4]; void* parent_planes[16];
    uint32_t* event_counts[4];  // HNB_EFFECT_ORDERED_EVENTS
};
static hnb::BatchParams make_params(const EmuBatch* b) {
    hnb::BatchParams P;
    memset((void*)&P, 0, sizeof(P));
    P.frame = (const hnb::FrameHeader*)b->frame;
    P.spawners = (hnb::Spawner*)b->spawners;
    P.spawn_prefix = b->spawn_prefix;
    P.prefix_sum = b->prefix_sum;
    P.tile_prefix = b->tile_prefix;
    P.batch_info = (const hnb::BatchInfo*)b->batch_info;
    P.bi_spawner_base = P.batch_info->spawner_base; P.bi_prefix_sum_offset = P.batch_info->prefix_sum_offset; P.bi_prefix_sum_count = P.batch_info->prefix_sum_count;
    P.first_md_index = P.spawners[P.bi_spawner_base].effect_metadata_index;
    P.batch_tiles = b->batch_tiles;
    P.ticket = b->ticket;
    P.tile_state = b->tile_state;
    P.metadata = (hnb::EffectMetadata*)b->metadata;
    P.draw_args = b->draw_args;
    P.properties = b->properties;
    for (int p = 0; p < 16; ++p) P.slab.planes[p] = b->planes[p];
    P.slab.particle_index[0] = b->ping;
    P.slab.particle_index[1] = b->pong;
    P.slab.dead_index = b->dead;
    P.slab.capacity_rows = b->capacity;
    P.init_thread_count = b->init_thread_count;
    P.properties_stride = b->properties_stride;
    P.tile_rows = b->tile_rows;
    P.child_infos = (hnb::ChildInfo*)b->child_infos;
    P.consume_events = b->consume_events;
    for (int i = 0; i < 4; ++i) { P.emit_events[i] = b->emit_events[i]; P.emit_events_capacity[i] = b->emit_caps[i]; }
    for (int p = 0; p < 16; ++p) P.parent_slab.planes[p] = b->parent_planes[p];
    for (int i = 0; i < 4; ++i) P.event_counts[i] = b->event_counts[i];
    return P;
}
// `wave`: CTAs running at the same time. hnb_update gets its whole (small) grid at once; hnb_init's CTAs never wait for
// one another, so a large spawn burst runs as successive waves instead of one OS thread per requested spawn.
template <typename K> static void emu_launch(K kernel, const hnb::BatchParams& P, unsigned grid, size_t smem, unsigned wave = 0) {
    if (wave == 0 || wave > grid) wave = grid;
    std::vector<emu::Cta> ctas(wave);
    std::vector<std::vector<unsigned char>> dyn(wave, std::vector<unsigned char>(smem + 64));
    for (unsigned first = 0; first < grid; first += wave) {
        const unsigned n = std::min(wave, grid - first);
        for (unsigned b = 0; b < n; ++b) {
            pthread_barrier_init(&ctas[b].bar, nullptr, HNB_BLOCK);
            ctas[b].dyn = (unsigned char*)(((uintptr_t)dyn[b].data() + 15) & ~(uintptr_t)15);
            memset(ctas[b].statics, 0, sizeof(ctas[b].statics));
            for (int w = 0; w < HNB_BLOCK / 32; ++w) pthread_barrier_init(&ctas[b].warps[w].bar, nullptr, 32);
        }
        std::vector<std::thread> threads;
        threads.reserve(size_t(n) * HNB_BLOCK);
        for (unsigned b = 0; b < n; ++b)
            for (unsigned t = 0; t < HNB_BLOCK; ++t)
                threads.emplace_back([&, b, t] {
                    emu::tls.tid = t; emu::tls.bid = first + b; emu::tls.lane = t & 31u;
                    emu::tls.cta = &ctas[b]; emu::tls.warp = &ctas[b].warps[t >> 5];
                    kernel(P);
                });
        for (auto& th : threads) th.join();
        for (unsigned b = 0; b < n; ++b) {
            pthread_barrier_destroy(&ctas[b].bar);
            for (int w = 0; w < HNB_BLOCK / 32; ++w) pthread_barrier_destroy(&ctas[b].warps[w].bar);
        }
    }
}
extern "C" void emu_init(const EmuBatch* b, uint32_t blocks) { emu_launch(hnb::hnb_init, make_params(b), blocks, HNB_INIT_SMEM_EFFECTS * 4, 8); }
extern "C" void emu_update(const EmuBatch* b, uint32_t blocks, uint32_t smem) { emu_launch(hnb::hnb_update, make_params(b), blocks, smem); }
extern "C" void emu_aos_to_planes(const EmuBatch* b, const uint8_t* aos, uint32_t first, uint32_t count, uint32_t stride) {
    hnb::BatchParams P = make_params(b);
    for (uint32_t r = 0; r < count; ++r) {
        hnb::RawParticle raw; memset((void*)&raw, 0, sizeof(raw));
        memcpy((void*)&raw, aos + size_t(r) * stride, stride);
        hnb::hnb_store_raw(raw, P.slab, first + r);
    }
}
extern "C" void emu_planes_to_aos(const EmuBatch* b, uint8_t* aos, uint32_t first, uint32_t count, uint32_t stride) {
    hnb::BatchParams P = make_params(b);
    for (uint32_t r = 0; r < count; ++r) {
        hnb::RawParticle raw;
        hnb::hnb_load_raw(raw, P.slab, first + r);
        memcpy(aos + size_t(r) * stride, (const void*)&raw, stride);
    }
}
// the look-back's tile state word as this effect's order packs it (`valid` is dropped outside slot order)
extern "C" uint64_t emu_pack_state(uint32_t epoch, uint64_t flag, uint32_t survivors, uint32_t valid) {
#if HNB_SLOT_ORDER
    return hnb::hnb_pack_state(epoch, flag, survivors, valid);
#else
    (void)valid;
    return hnb::hnb_pack_state(epoch, flag, survivors);
#endif
}
extern "C" uint32_t emu_state_flag(uint64_t s, uint32_t epoch) { return hnb::hnb_state_flag(s, epoch); }
extern "C" uint64_t emu_state_value(uint64_t s) { return hnb::hnb_state_value(s); }
extern "C" uint32_t emu_tile_k(void) { return HNB_TILE_K; }
extern "C" uint32_t emu_rows_per_lane(void) { return HNB_ROWS_PER_LANE; }
extern "C" uint32_t emu_init_items(void) { return HNB_INIT_ITEMS; }
"""


# The same driver whose init and update launchers pass the slab's identity claims (SlabView::ident_claim; DRIVER passes
# none), set with emu_set_ident_claim.
_PLAIN_INIT = 'extern "C" void emu_init(const EmuBatch* b, uint32_t blocks) { emu_launch(hnb::hnb_init, make_params(b), blocks, HNB_INIT_SMEM_EFFECTS * 4, 8); }'
_PLAIN_UPDATE = 'extern "C" void emu_update(const EmuBatch* b, uint32_t blocks, uint32_t smem) { emu_launch(hnb::hnb_update, make_params(b), blocks, smem); }'
_CLAIMED_INIT = r"""static unsigned long long* g_ident_claim = nullptr;  // [2]: identity claims of ping / pong
extern "C" void emu_set_ident_claim(unsigned long long* claim) { g_ident_claim = claim; }
extern "C" void emu_init(const EmuBatch* b, uint32_t blocks) {
    hnb::BatchParams P = make_params(b);
    P.slab.ident_claim = g_ident_claim;
    emu_launch(hnb::hnb_init, P, blocks, HNB_INIT_SMEM_EFFECTS * 4, 8);
}"""
_CLAIMED_UPDATE = r"""extern "C" void emu_update(const EmuBatch* b, uint32_t blocks, uint32_t smem) {
    hnb::BatchParams P = make_params(b);
    P.slab.ident_claim = g_ident_claim;
    emu_launch(hnb::hnb_update, P, blocks, smem);
}"""
assert DRIVER.count(_PLAIN_INIT) == 1 and DRIVER.count(_PLAIN_UPDATE) == 1
CLAIMED_DRIVER = DRIVER.replace(_PLAIN_INIT, _CLAIMED_INIT).replace(_PLAIN_UPDATE, _CLAIMED_UPDATE)


class EmuBatch(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("frame", "spawners", "spawn_prefix", "prefix_sum", "tile_prefix", "batch_info", "batch_tiles", "ticket",
                                          "tile_state", "metadata", "draw_args", "properties")] + \
               [("planes", C.c_void_p * 16), ("ping", C.c_void_p), ("pong", C.c_void_p), ("dead", C.c_void_p),
                ("capacity", C.c_uint32), ("init_thread_count", C.c_uint32), ("properties_stride", C.c_uint32), ("tile_rows", C.c_uint32),
                ("child_infos", C.c_void_p), ("consume_events", C.c_void_p), ("emit_events", C.c_void_p * 4), ("emit_caps", C.c_uint32 * 4),
                ("parent_planes", C.c_void_p * 16), ("event_counts", C.c_void_p * 4)]


def build_emulated_effect(lowered, allow_events: bool = False, driver: str = DRIVER) -> C.CDLL:
    """`driver`: the host entry points compiled after the kernels (CLAIMED_DRIVER: launches under identity claims)."""
    src = lowered.generate_source()
    if not allow_events and ("#define HNB_EMIT_EVENTS 1" in src or "#define HNB_READ_PARENT 1" in src or "#define HNB_CONSUME_EVENTS 1" in src):
        raise NotImplementedError("EmuWorld covers effects without GPU spawn events; use EmuScene")
    for old, new in SUBSTITUTIONS:
        assert src.count(old) == 1, f"kernel source changed, update tests/kernel_emu.py: {old!r}"
        src = src.replace(old, new)
    # the remaining `asm` statements sit in #if HNB_PROFILE blocks, which are compiled out (HNB_PROFILE is 0)
    text = PRELUDE + src + driver
    OUT.mkdir(parents=True, exist_ok=True)
    tag = hashlib.sha1(text.encode()).hexdigest()[:16]
    cpp, so = OUT / f"emu_{tag}.{os.getpid()}.cpp", OUT / f"emu_{tag}.so"  # per process: workers may build the same tag at once
    if not so.exists():
        cpp.write_text(text)
        cmd = ["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-pthread", "-w", str(cpp), "-o", str(so) + f".{os.getpid()}.tmp"]
        proc = subprocess.run(cmd, capture_output=True, text=True)
        if proc.returncode != 0:
            raise RuntimeError("host build of the kernel templates failed:\n" + proc.stderr[:6000])
        os.replace(str(so) + f".{os.getpid()}.tmp", so)  # atomic: parallel test workers build the same tag
    lib = C.CDLL(str(so))
    lib.emu_init.argtypes = [C.POINTER(EmuBatch), C.c_uint32]
    lib.emu_update.argtypes = [C.POINTER(EmuBatch), C.c_uint32, C.c_uint32]
    lib.emu_aos_to_planes.argtypes = [C.POINTER(EmuBatch), C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32]
    lib.emu_planes_to_aos.argtypes = [C.POINTER(EmuBatch), C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32]
    for f in ("emu_init", "emu_update", "emu_aos_to_planes", "emu_planes_to_aos"):
        getattr(lib, f).restype = None
    for f in ("emu_tile_k", "emu_rows_per_lane", "emu_init_items"):
        getattr(lib, f).restype = C.c_uint32
    lib.emu_pack_state.argtypes = [C.c_uint32, C.c_uint64, C.c_uint32, C.c_uint32]
    lib.emu_pack_state.restype = C.c_uint64
    lib.emu_state_flag.argtypes = [C.c_uint64, C.c_uint32]
    lib.emu_state_flag.restype = C.c_uint32
    lib.emu_state_value.argtypes = [C.c_uint64]
    lib.emu_state_value.restype = C.c_uint64
    return lib


def tile_count(rows, word: int):
    """hnb_tile_count (hnb_tables.cuh) restated: tiles of an instance with `rows` rows under a tile size word."""
    S = word & 0xFFFF
    rows = np.asarray(rows, dtype=np.int64)
    return (rows + S - 1) // S


class EmuWorld:
    """One batch (all instances of `ref`) simulated by the emulated kernels, starting from `ref`'s current state."""

    def __init__(self, ref, lowered, chunks: int = 1, update_ctas: int = 2, property_blobs=None, static_lib=None, driver=DRIVER):
        """`static_lib` (tests/static_emu.build()): run the real bookkeeping and ribbon-sort kernels too instead of their
        restatements."""
        self.ref, self.lib = ref, build_emulated_effect(lowered, driver=driver)
        self.static_lib = static_lib
        self.ribbons = bool(lowered.flags & (1 << 5))  # HNB_EFFECT_RIBBONS
        self.stride = ref.stride_words * 4
        assert lowered.particle_stride == self.stride
        n, rows = len(ref.instances), ref.slab_rows
        self.n, self.rows = n, rows
        k = self.lib.emu_tile_k()
        assert chunks * k <= self.lib.emu_rows_per_lane()
        self.tile = 32 * k * chunks
        self.tile_word, small = self.tile, self.tile
        self.update_ctas = update_ctas
        u32 = np.uint32
        self.planes = [np.zeros(rows * 8, dtype=u32) for _ in range(16)]          # room for 32-byte-wide (sector) columns
        self.sector = bool(lowered.flags & (1 << 8))                               # HNB_EFFECT_SECTOR_PLANES
        self.cols = [np.ascontiguousarray(ref.indirect[:, c]).copy() for c in range(3)]
        self.metadata = (O.EffectMetadata * n).from_buffer_copy(bytes(ref.metadata))
        self.spawners = (O.Spawner * n).from_buffer_copy(bytes(ref.spawners))
        self.draw = ref.draw.copy()
        self.spawn_prefix = np.zeros(n, dtype=u32)
        self.prefix_sum = np.zeros(n, dtype=u32)
        self.tile_prefix = np.zeros(n + 1, dtype=u32)
        self.batch_info = (O.BatchInfo * 1)(O.BatchInfo(0, 0, 0, 0, 0, n))
        self.batch_tiles = np.zeros(1, dtype=u32)
        self.ticket = np.zeros(1, dtype=u32)
        self.tile_state = np.zeros(rows // small + n + 2, dtype=np.uint64)
        self.frame = np.zeros(16, dtype=u32)                                       # FrameHeader: SimParams (7 words) | epoch | num_batches
        self.dispatch = np.zeros(3, dtype=u32)
        self.spawn_range = np.zeros(n, dtype=u32)
        self.tile_size = np.array([self.tile_word], dtype=u32)
        self.epoch = 0
        self.props = None
        self.props_stride = 0
        if property_blobs:
            self.props_stride = (len(property_blobs[0]) + 15) // 16 * 16
            buf = bytearray(self.props_stride * len(property_blobs))
            for i, b in enumerate(property_blobs):
                buf[i * self.props_stride: i * self.props_stride + len(b)] = b
            self.props = np.frombuffer(bytes(buf), dtype=np.uint8).copy()
        self.b = EmuBatch()
        self._bind()
        aos = np.ascontiguousarray(ref.particles)
        self.lib.emu_aos_to_planes(C.byref(self.b), aos.ctypes.data, 0, rows, self.stride)

    def _bind(self):
        b, ptr = self.b, lambda a: a.ctypes.data
        b.frame, b.spawners, b.spawn_prefix, b.prefix_sum, b.tile_prefix = ptr(self.frame), C.addressof(self.spawners), ptr(self.spawn_prefix), ptr(self.prefix_sum), ptr(self.tile_prefix)
        b.batch_info, b.batch_tiles, b.ticket, b.tile_state = C.addressof(self.batch_info), ptr(self.batch_tiles), ptr(self.ticket), ptr(self.tile_state)
        b.metadata, b.draw_args = C.addressof(self.metadata), ptr(self.draw)
        b.properties = ptr(self.props) if self.props is not None else None
        for p in range(16):
            b.planes[p] = ptr(self.planes[p])
        b.ping, b.pong, b.dead = ptr(self.cols[0]), ptr(self.cols[1]), ptr(self.cols[2])
        b.capacity, b.properties_stride, b.tile_rows = self.rows, self.props_stride, self.tile_word

    def frame_step(self, orc, sim, spawns, seeds):
        """One simulate(): init kernel -> bookkeeping (restated) -> update kernel. `sim`: the oracle world's SimParams."""
        u32p = C.POINTER(C.c_uint32)
        n = self.n
        self.frame[:7] = np.frombuffer(bytes(sim), dtype=np.uint32)
        self.epoch += 1
        self.frame[7], self.frame[8] = self.epoch, 1
        run = 0
        for i in range(n):
            self.spawners[i].spawn, self.spawners[i].seed = int(spawns[i]), int(seeds[i]) & 0xFFFFFFFF
            self.spawn_prefix[i] = run
            run += max(0, int(spawns[i]))
        self.prefix_sum[:] = self.spawn_prefix
        # ---- init (vfx_init.wgsl): ceil64(total) logical threads, HNB_INIT_ITEMS of them per emulated thread
        threads = (run + 63) // 64 * 64
        self.b.init_thread_count = threads
        if threads:
            per_block = 256 * self.lib.emu_init_items()
            self.lib.emu_init(C.byref(self.b), (threads + per_block - 1) // per_block)
        if self.static_lib is not None:
            # ---- bookkeeping by the real fused kernel (k_bookkeeping): per-instance init thread ranges as bind_launch writes them
            for i in range(n):
                end = int(self.spawn_prefix[i + 1]) if i + 1 < n else threads
                self.spawn_range[i] = max(0, end - int(self.spawn_prefix[i])) if threads else 0
            self.static_lib.semu_bookkeeping(C.byref(self._static_tables()), 1)
        else:
            # ---- bookkeeping restated: deferred init accounting (the kernel assigned ranks instead of bumping the counters) ...
            for i in range(n):
                md = self.metadata[i]
                passed = min(max(0, int(spawns[i])), md.max_spawn)
                md.alive_count += passed
                md.particle_counter += passed
            # ... then vfx_indirect + vfx_prefix_sum as restated by the C oracle, and the tile prefix of this launch
            orc.orc_indirect(self.frame.ctypes.data_as(C.POINTER(O.SimParams)), self.metadata, self.draw.ctypes.data_as(u32p), self.spawners,
                             self.prefix_sum.ctypes.data_as(u32p), None, 0)
            alive = self.prefix_sum.copy()
            orc.orc_prefix_sum(self.batch_info, 1, self.prefix_sum.ctypes.data_as(u32p), self.dispatch.ctypes.data_as(u32p))
            tiles = tile_count(alive, self.tile_word)
            self.tile_prefix[:n] = np.concatenate([[0], np.cumsum(tiles)[:-1]]) if n else []
            self.tile_prefix[n] = tiles.sum()
            self.batch_tiles[0] = tiles.sum()
            self.ticket[0] = 0
        # ---- update (vfx_update.wgsl): a persistent grid of a few CTAs
        self.lib.emu_update(C.byref(self.b), self.update_ctas, 160 * 1024)
        if self.ribbons:
            self._sort_ribbons(orc)

    def _static_tables(self):
        from tests.static_emu import StaticTables
        T, p = StaticTables(), lambda a: a.ctypes.data
        T.frame, T.spawners, T.spawn_range, T.prefix_sum, T.tile_prefix = p(self.frame), C.addressof(self.spawners), p(self.spawn_range), p(self.prefix_sum), p(self.tile_prefix)
        T.batch_infos, T.batch_tile_size, T.dispatch_args, T.batch_tiles, T.tickets = C.addressof(self.batch_info), p(self.tile_size), p(self.dispatch), p(self.batch_tiles), p(self.ticket)
        T.metadata, T.draw_args, T.child_infos, T.num_child_infos = C.addressof(self.metadata), p(self.draw), None, 0
        return T

    def _sort_ribbons(self, orc):
        """Passes "hanabi:sort_prefix_sum" + "hanabi:sort" of hnb_simulate (needs the static kernels library)."""
        assert self.static_lib is not None, "ribbon effects need static_lib"
        from tests.static_emu import RibbonSortArgs
        lib = self.static_lib
        lib.semu_prefix_sum(C.byref(self._static_tables()), 1)
        a = RibbonSortArgs()
        words = self.stride // 4
        assert words % 4 == 0, "effect records are multiples of 16 bytes"
        pieces = words // 4
        col, p = 0, 0
        while p < pieces:                         # physical columns (effect_source.cpp::physical_planes)
            width = 8 if (self.sector and p + 1 < pieces) else 4
            a.planes.ptr[col], a.planes.words[col], a.planes.word_off[col] = self.planes[col].ctypes.data, width, 4 * p
            for k in range(width):
                a.planes.word_to_plane[4 * p + k] = col
            p += width // 4
            col += 1
        a.ping, a.pong, a.spawners, a.metadata = self.cols[0].ctypes.data, self.cols[1].ctypes.data, C.addressof(self.spawners), C.addressof(self.metadata)
        a.spawner_base, a.instance_count = 0, self.n
        grid = 2
        self._sort_scratch = ([np.zeros(self.rows, dtype=np.uint64) for _ in range(2)], [np.zeros(self.rows, dtype=np.uint32) for _ in range(2)],
                              np.zeros(lib.semu_hist_words(grid), dtype=np.uint32))
        for i in range(2):
            a.scratch_keys[i], a.scratch_vals[i] = self._sort_scratch[0][i].ctypes.data, self._sort_scratch[1][i].ctypes.data
        a.scratch_hist, a.scratch_rows = self._sort_scratch[2].ctypes.data, self.rows
        lib.semu_ribbon_sort_small(C.byref(a))
        if self.rows > 2048:
            lib.semu_ribbon_sort_large(C.byref(a), grid)

    def pull(self):
        aos = np.zeros((self.rows, self.stride // 4), dtype=np.uint32)
        self.lib.emu_planes_to_aos(C.byref(self.b), aos.ctypes.data, 0, self.rows, self.stride)
        return {"particles": aos, "indirect": np.stack(self.cols, axis=1),
                "metadata": np.frombuffer(bytes(self.metadata), dtype=np.uint32).reshape(self.n, 15).copy(), "draw": self.draw.copy(),
                "prefix": self.prefix_sum.copy(), "total_update": self.batch_info[0].total_update_count}


class EmuScene:
    """Several single-instance batches with shared global tables — spawners, metadata, prefix sums, child infos, event
    buffers — i.e. what one hnb_ctx holds, so that parents can emit GPU spawn events and children consume them. A frame is
    hnb_simulate(): init of every batch in order, the real fused bookkeeping kernel (+ event clear), update of every batch.

    members: list of dicts  {ref: RefWorld (1 instance), lowered, parent: member index or None,
                             consume: event buffer index or None, emit: [event buffer indices], child_row: ChildInfo row or None}
    """

    def __init__(self, members, event_caps, static_lib, chunks: int = 1, update_ctas: int = 2):
        from tests.static_emu import StaticTables
        self.static, self.members, n = static_lib, members, len(members)
        u32 = np.uint32
        self.n = n
        self.metadata = (O.EffectMetadata * n)()
        self.spawners = (O.Spawner * n)()
        self.draw = np.zeros(5 * n, dtype=u32)
        self.spawn_prefix, self.prefix_sum, self.spawn_range = np.zeros(n, dtype=u32), np.zeros(n, dtype=u32), np.zeros(n, dtype=u32)
        self.tile_prefix = np.zeros(n + 1, dtype=u32)
        self.batch_infos = (O.BatchInfo * n)()
        self.tile_size, self.dispatch = np.zeros(n, dtype=u32), np.zeros(3 * n, dtype=u32)
        self.batch_tiles, self.tickets = np.zeros(n, dtype=u32), np.zeros(n, dtype=u32)
        self.frame = np.zeros(16, dtype=u32)
        self.child_infos = np.zeros((max(1, len(event_caps)), 2), dtype=np.int32)     # {init_indirect_dispatch_index, event_count}
        self.events = [np.zeros(c, dtype=u32) for c in event_caps]
        self.epoch = 0
        self.update_ctas = update_ctas
        self.slabs = []
        for b, m in enumerate(members):
            ref, lib = m["ref"], build_emulated_effect(m["lowered"], allow_events=True)
            assert len(ref.instances) == 1
            k = lib.emu_tile_k()
            tile = 32 * k * chunks
            self.tile_size[b] = tile
            rows = ref.slab_rows
            slab = dict(lib=lib, rows=rows, stride=ref.stride_words * 4, tile=tile, planes=[np.zeros(rows * 4, dtype=u32) for _ in range(16)],
                        cols=[np.ascontiguousarray(ref.indirect[:, c]).copy() for c in range(3)], tile_state=np.zeros(rows // tile + 4, dtype=np.uint64), b=EmuBatch())
            self.slabs.append(slab)
            md = O.EffectMetadata.from_buffer_copy(bytes(ref.metadata[0]))
            md.indirect_render_index = b
            if m.get("consume") is not None:
                md.global_child_index, md.local_child_index = m["child_row"], 0
            if m.get("emit"):
                md.base_child_index = m["base_child_row"]
            self.metadata[b] = md
            sp = O.Spawner.from_buffer_copy(bytes(ref.spawners[0]))
            sp.effect_metadata_index, sp.draw_indirect_index = b, b
            if m.get("parent") is not None:
                sp.parent_slab_offset = 0
            self.spawners[b] = sp
            self.batch_infos[b] = O.BatchInfo(0, 0, b, 0, b, 1)
        for b, m in enumerate(members):
            self._bind(b)
            slab = self.slabs[b]
            aos = np.ascontiguousarray(m["ref"].particles)
            slab["lib"].emu_aos_to_planes(C.byref(slab["b"]), aos.ctypes.data, 0, slab["rows"], slab["stride"])
        T, p = StaticTables(), lambda a: a.ctypes.data
        T.frame, T.spawners, T.spawn_range, T.prefix_sum, T.tile_prefix = p(self.frame), C.addressof(self.spawners), p(self.spawn_range), p(self.prefix_sum), p(self.tile_prefix)
        T.batch_infos, T.batch_tile_size, T.dispatch_args, T.batch_tiles, T.tickets = C.addressof(self.batch_infos), p(self.tile_size), p(self.dispatch), p(self.batch_tiles), p(self.tickets)
        T.metadata, T.draw_args, T.child_infos, T.num_child_infos = C.addressof(self.metadata), p(self.draw), p(self.child_infos), len(event_caps)
        self.T = T

    def _bind(self, b):
        slab, m, ptr = self.slabs[b], self.members[b], lambda a: a.ctypes.data
        e = slab["b"]
        e.frame, e.spawners, e.spawn_prefix, e.prefix_sum, e.tile_prefix = ptr(self.frame), C.addressof(self.spawners), ptr(self.spawn_prefix), ptr(self.prefix_sum), ptr(self.tile_prefix)
        e.batch_info = C.addressof(self.batch_infos) + b * C.sizeof(O.BatchInfo)
        e.batch_tiles, e.ticket, e.tile_state = ptr(self.batch_tiles) + 4 * b, ptr(self.tickets) + 4 * b, ptr(slab["tile_state"])
        e.metadata, e.draw_args, e.properties = C.addressof(self.metadata), ptr(self.draw), None
        for p in range(16):
            e.planes[p] = ptr(slab["planes"][p])
        e.ping, e.pong, e.dead = (ptr(c) for c in slab["cols"])
        e.capacity, e.properties_stride, e.tile_rows = slab["rows"], 0, slab["tile"]
        e.child_infos = ptr(self.child_infos)
        if m.get("consume") is not None:
            e.consume_events = ptr(self.events[m["consume"]])
        for i, ev in enumerate(m.get("emit") or []):
            e.emit_events[i], e.emit_caps[i] = ptr(self.events[ev]), len(self.events[ev])
            if m.get("ordered"):
                slab.setdefault("event_counts", {})[i] = np.zeros(slab["rows"], dtype=np.uint32)
                slab.setdefault("event_block_sums", {})[i] = np.zeros(slab["rows"] // 2048 + 2, dtype=np.uint32)
                e.event_counts[i] = ptr(slab["event_counts"][i])
        if m.get("parent") is not None:
            for p in range(16):
                e.parent_planes[p] = ptr(self.slabs[m["parent"]]["planes"][p])

    def frame_step(self, sim, spawns, seeds):
        n = self.n
        self.frame[:7] = np.frombuffer(bytes(sim), dtype=np.uint32)
        self.frame[6] = n                       # sim.num_effects of the shared context
        self.epoch += 1
        self.frame[7], self.frame[8] = self.epoch, n
        threads = []
        for b, m in enumerate(self.members):
            self.spawners[b].spawn, self.spawners[b].seed = int(spawns[b]), int(seeds[b]) & 0xFFFFFFFF
            self.spawn_prefix[b] = self.prefix_sum[b] = 0
            if m.get("consume") is not None:
                t = (len(self.events[m["consume"]]) + 63) // 64 * 64    # dispatch sized by the buffer, capped on the device by event_count
                self.spawn_range[b] = t | 0x80000000
            else:
                t = (max(0, int(spawns[b])) + 63) // 64 * 64
                self.spawn_range[b] = t
            threads.append(t)
        for b, slab in enumerate(self.slabs):       # pass "hanabi:init"
            slab["b"].init_thread_count = threads[b]
            if threads[b]:
                per_block = 256 * slab["lib"].emu_init_items()
                slab["lib"].emu_init(C.byref(slab["b"]), (threads[b] + per_block - 1) // per_block)
        self.static.semu_bookkeeping(C.byref(self.T), n)   # indirect + prefix sums (+ deferred init accounting), then the event clear
        self.static.semu_clear_events(C.byref(self.T), n)
        for slab in self.slabs:                     # pass "hanabi:update"
            slab["lib"].emu_update(C.byref(slab["b"]), self.update_ctas, 160 * 1024)
        from tests.static_emu import EventAppendArgs
        for b, m in enumerate(self.members):        # HNB_EFFECT_ORDERED_EVENTS: the three k_events_* launches per channel
            if not m.get("ordered"):
                continue
            slab = self.slabs[b]
            for i, ev in enumerate(m.get("emit") or []):
                a = EventAppendArgs()
                a.counts, a.ping, a.pong = slab["event_counts"][i].ctypes.data, slab["cols"][0].ctypes.data, slab["cols"][1].ctypes.data
                a.spawner = C.addressof(self.spawners) + b * C.sizeof(O.Spawner)
                a.metadata = C.addressof(self.metadata) + b * C.sizeof(O.EffectMetadata)
                a.block_sums, a.child_infos, a.binding = slab["event_block_sums"][i].ctypes.data, self.child_infos.ctypes.data, i
                a.buffer, a.capacity = self.events[ev].ctypes.data, len(self.events[ev])
                self.static.semu_ordered_event_append(C.byref(a), slab["rows"])

    def pull(self, b):
        slab = self.slabs[b]
        aos = np.zeros((slab["rows"], slab["stride"] // 4), dtype=np.uint32)
        slab["lib"].emu_planes_to_aos(C.byref(slab["b"]), aos.ctypes.data, 0, slab["rows"], slab["stride"])
        return {"particles": aos, "indirect": np.stack(slab["cols"], axis=1), "metadata": np.frombuffer(bytes(self.metadata[b]), dtype=np.uint32).copy(),
                "instance_count": int(self.draw[5 * b + 1])}


# ---- shared by the emulation tests ------------------------------------------------------------------------------------
def assert_same(ref, got, what):
    """Every buffer of an EmuWorld bit for bit against the oracle world."""
    np.testing.assert_array_equal(got["metadata"], ref.metadata_rows(), err_msg=f"{what}: metadata")
    np.testing.assert_array_equal(got["draw"], ref.draw, err_msg=f"{what}: draw args")
    np.testing.assert_array_equal(got["prefix"], ref.prefix, err_msg=f"{what}: prefix sums")
    assert got["total_update"] == ref.batch_infos[0].total_update_count
    np.testing.assert_array_equal(got["indirect"], ref.indirect, err_msg=f"{what}: ping / pong / dead")
    np.testing.assert_array_equal(got["particles"], ref.particles, err_msg=f"{what}: particles")


def c5_world(rng, insts):
    """A C5 world of `insts`, back to back, their alive rows with random motion and lifetimes of 0.02 to 0.15 s."""
    from tests.helpers import RefWorld
    ref = RefWorld(sum(i.capacity for i in insts), 8, insts)
    for inst in ref.instances:
        n = inst.alive
        p = np.zeros((n, 8), dtype=np.float32)
        p[:, 0:3] = rng.uniform(-1, 1, (n, 3)); p[:, 4:7] = rng.uniform(-1, 1, (n, 3)); p[:, 7] = rng.uniform(0.02, 0.15, n)
        ref.particles[inst.slab_offset:inst.slab_offset + n] = p.view(np.uint32)
    return ref


def claim(base, length):
    """An identity-claim word: rows [0, length) of the column starting at slab row `base` hold their own index."""
    return np.uint64((base << 32) | length)


def claimed(ref, chunks, claim_len):
    """The emulated C5 world of `ref` with a claim of `claim_len` rows on both alive-list columns; returns (EmuWorld, the
    two claim words, which the kernels update in place)."""
    from bevy_hanabi_b200 import recipes
    emu = EmuWorld(ref, recipes.c5_lowered(), chunks=chunks, update_ctas=2, driver=CLAIMED_DRIVER)
    claims = np.array([claim(0, claim_len)] * 2, dtype=np.uint64)
    emu.lib.emu_set_ident_claim.argtypes = [C.c_void_p]
    emu.lib.emu_set_ident_claim.restype = None
    emu.lib.emu_set_ident_claim(claims.ctypes.data)
    return emu, claims


def c5_frame(orc, ref, emu, spawn=0):
    """One frame of the single-instance C5 world `ref` with its constant init, in the oracle and in `emu`."""
    from tests.effects import ACCEL_DRAG, c5_init
    ref.set_spawns([spawn])
    ref.oracle_frame(orc, orc.orc_body_update_c5(), ACCEL_DRAG, orc.orc_body_init_const(), C.byref(c5_init()))
    emu.frame_step(orc, ref.sim, [spawn], [42])


def random_event_scene(orc, ordered, seed):
    """A randomised parent / two-children scene (emission probability, events per death, lifetimes, spawn schedule,
    tile size, grid). Default mode: event buffers as multisets (sub-multisets on overflow), the oracle adopts the
    buffer's order; ordered mode: exact buffers. Everything else exact in both."""
    from collections import Counter

    from bevy_hanabi_b200 import graph as G
    from oracle.hanabi_oracle import EffectOracle, pcg_hash
    from tests import static_emu
    from tests.effects import EVENT_CAP
    from tests.helpers import Instance, RefWorld, oracle_append_events, oracle_child_init
    A = G.Attribute
    rng = np.random.default_rng(700 + seed)
    p_cap, c_cap = int(rng.choice([300, 1024, 1500])), 4096
    wp = G.ExprWriter()
    parent = (G.EffectAsset(p_cap, wp.module, name="emitter")
              .init(G.SetAttributeModifier(A.POSITION, wp.rand(G.VEC3) * wp.lit(2.) - wp.lit(1.)))
              .init(G.SetAttributeModifier(A.VELOCITY, wp.rand(G.VEC3) - wp.lit(0.5)))
              .init(G.SetAttributeModifier(A.AGE, wp.lit(0.)))
              .init(G.SetAttributeModifier(A.LIFETIME, wp.lit(float(rng.choice([0.05, 0.1]))).uniform(wp.lit(float(rng.choice([0.3, 0.6]))))))
              .update(G.EmitSpawnEventModifier(G.ALWAYS, (wp.rand(G.FLOAT) * wp.lit(float(rng.choice([1.0625, 1.25, 1.5])))).cast(G.UINT), 0))
              .update(G.EmitSpawnEventModifier(G.ON_DIE, wp.lit(G.U32(int(rng.integers(1, 6)))), 1)))
    children = []
    for tag in (0, 1):
        wc = G.ExprWriter()
        children.append(G.EffectAsset(c_cap, wc.module, name=f"child{tag}")
                        .init(G.InheritAttributeModifier(A.POSITION))
                        .init(G.SetAttributeModifier(A.VELOCITY, wc.parent_attr(A.VELOCITY) * wc.lit(0.5 + tag) + (wc.rand(G.VEC3) - wc.lit(0.5))))
                        .init(G.SetAttributeModifier(A.AGE, wc.lit(0.)))
                        .init(G.SetAttributeModifier(A.LIFETIME, wc.lit(0.15 + 0.1 * tag)))
                        .init(G.SetAttributeModifier(A.U32_0, wc.parent_attr(A.ID))))
    p_fx = parent.generate(num_event_bindings=2, ordered_events=ordered)
    c_fx = [c.generate(parent=parent) for c in children]
    dt = 1.0 / 30.0
    pw = RefWorld(p_cap, p_fx.particle_stride // 4, [Instance(0, p_cap, alive=0, seed=1)], dt=dt)
    cw = [RefWorld(c_cap, c_fx[0].particle_stride // 4, [Instance(0, c_cap, alive=0, seed=2 + k)], dt=dt) for k in (0, 1)]
    po, co = EffectOracle(parent), [EffectOracle(c) for c in children]
    scene = EmuScene([dict(ref=cw[0], lowered=c_fx[0], parent=2, consume=0, child_row=0),
                      dict(ref=cw[1], lowered=c_fx[1], parent=2, consume=1, child_row=1),
                      dict(ref=pw, lowered=p_fx, emit=[0, 1], base_child_row=0, ordered=ordered)], [EVENT_CAP, EVENT_CAP], static_emu.build(),
                     chunks=int(rng.choice([1, 2])), update_ctas=int(rng.integers(1, 4)))
    events = [np.zeros(EVENT_CAP, dtype=np.uint32) for _ in (0, 1)]
    event_count, all_emitted = [0, 0], [[], []]
    for f in range(10):
        spawn = int(rng.integers(0, p_cap)) if rng.random() < 0.4 else 0
        seed_p = int(pcg_hash(np.array([seed * 1000 + f], dtype=np.uint32))[0])
        seed_c = [int(pcg_hash(np.array([seed * 1000 + 500 + 10 * f + k], dtype=np.uint32))[0]) for k in (0, 1)]
        n_valid = []
        for k in (0, 1):
            assert int(scene.child_infos[k, 1]) == event_count[k]
            nv = min(event_count[k], EVENT_CAP)
            got = scene.events[k].copy()
            if ordered:
                np.testing.assert_array_equal(got[:nv], events[k][:nv], err_msg=f"frame {f} channel {k}: event order")
            elif event_count[k] <= EVENT_CAP:
                assert sorted(got[:nv].tolist()) == sorted(events[k][:nv].tolist())
            else:
                emitted, kept = Counter(all_emitted[k]), Counter(got.tolist())
                assert all(kept[p] <= emitted[p] for p in kept)
            events[k][:nv] = got[:nv]
            n_valid.append(nv)
        t = np.float32(f * dt)
        pw.sim.time = t
        for k in (0, 1):
            cw[k].sim.time = t
            cw[k].set_spawns([0], [seed_c[k]])
            oracle_child_init(children[k], co[k], cw[k], po, pw, events[k], n_valid[k], seed_c[k])
        pw.set_spawns([spawn], [seed_p])
        po.init_pass(pw)
        event_count = [0, 0]
        for w in (cw[0], cw[1], pw):
            w.oracle_indirect(orc)
            w.oracle_prefix_sum(orc)
        for k in (0, 1):
            co[k].update_pass(cw[k])
        po.update_pass(pw)
        for channel, counts in po.last_emitted:
            event_count[channel] = oracle_append_events(pw, counts, events[channel], event_count[channel])
            rows_read = pw.indirect[:pw.metadata[0].max_update, 1 - pw.metadata[0].indirect_write_index]
            all_emitted[channel] = np.repeat(rows_read, counts[:len(rows_read)]).tolist()
        scene.frame_step(pw.sim, [0, 0, spawn], [seed_c[0], seed_c[1], seed_p])
        for b, world in enumerate((cw[0], cw[1], pw)):
            got = scene.pull(b)
            want_md = world.metadata_rows()[0].copy()
            want_md[5] = b
            for fld in (7, 8, 9, 10):
                want_md[fld] = got["metadata"][fld]
            np.testing.assert_array_equal(got["metadata"], want_md, err_msg=f"frame {f} member {b}: metadata")
            np.testing.assert_array_equal(got["indirect"], world.indirect, err_msg=f"frame {f} member {b}: lists")
            np.testing.assert_array_equal(got["particles"], world.particles, err_msg=f"frame {f} member {b}: particles")
