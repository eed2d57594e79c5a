"""Runs the effect-independent kernels (hnb_static_kernels.cu: indirect, prefix sum, fused bookkeeping, tile prefix;
hnb_ribbon_sort.cu: shared-memory bitonic sort and the cooperative radix sort) on the CPU — same thread-level emulation
as tests/kernel_emu.py, extended with what these files use: `blockDim` / `gridDim`, `__shfl_up_sync`,
`__match_any_sync`, `__syncthreads_or`, cooperative-groups `grid.sync()` (a barrier over every thread of the launch)
and `__shared__` declarations, which are rewritten into per-CTA allocations so that CTAs can run concurrently.

The kernel sources are taken verbatim up to their host-side launchers; test infrastructure only.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import re
import os
import subprocess
from pathlib import Path

from tests.kernel_emu import PRELUDE

ROOT = Path(__file__).resolve().parent.parent
KERNELS = ROOT / "bevy_hanabi_b200" / "csrc" / "kernels"
OUT = ROOT / "build" / "kernel_emu"

EXTRA_PRELUDE = r"""
#include <algorithm>
#include <map>
#include <mutex>
typedef int cudaError_t;
#define __grid_constant__
typedef void* cudaStream_t;
namespace emu {
struct Launch { pthread_barrier_t grid_bar; unsigned grid, block; };
struct CtaExtra { std::mutex mu; std::map<int, void*> shared; int or_acc; };
static thread_local Launch* launch;
static thread_local CtaExtra* cta_extra;
static inline void* cta_alloc(int key, size_t bytes) {
    std::lock_guard<std::mutex> lock(cta_extra->mu);
    void*& p = cta_extra->shared[key];
    if (!p) p = calloc(1, bytes + 16);
    return p;
}
}  // namespace emu
#define blockDim (emu::Dim3{emu::launch->block, 1u, 1u})
#define gridDim (emu::Dim3{emu::launch->grid, 1u, 1u})
template <typename T> static inline T __shfl_up_sync(unsigned, T v, int d) {
    T got = emu::exchange(v, emu::tls.lane >= unsigned(d) ? emu::tls.lane - unsigned(d) : emu::tls.lane);
    return emu::tls.lane >= unsigned(d) ? got : v;
}
static inline unsigned __match_any_sync(unsigned, unsigned v) {
    emu::tls.warp->slot[emu::tls.lane] = v;
    emu::warp_sync();
    unsigned m = 0;
    for (unsigned i = 0; i < 32; ++i) m |= (unsigned(emu::tls.warp->slot[i]) == v ? 1u : 0u) << i;
    emu::warp_sync();
    return m;
}
static inline int __syncthreads_or(int pred) {
    __syncthreads();
    if (pred) __atomic_store_n(&emu::cta_extra->or_acc, 1, __ATOMIC_SEQ_CST);
    __syncthreads();
    const int r = __atomic_load_n(&emu::cta_extra->or_acc, __ATOMIC_SEQ_CST);
    __syncthreads();
    if (emu::tls.tid == 0) emu::cta_extra->or_acc = 0;
    __syncthreads();
    return r;
}
namespace cooperative_groups {
struct grid_group { void sync() const { pthread_barrier_wait(&emu::launch->grid_bar); } };
static inline grid_group this_grid() { return grid_group(); }
}
// `wave`: how many CTAs run at the same time (0 = the whole grid, required when the kernel has grid-wide barriers)
template <typename F> static void emu_run(F body, unsigned grid, unsigned block, unsigned wave = 0) {
    if (wave == 0 || wave > grid) wave = grid;
    emu::Launch L;
    L.grid = grid; L.block = block;
    pthread_barrier_init(&L.grid_bar, nullptr, grid * block);
    for (unsigned first = 0; first < grid; first += wave) {
        const unsigned count = std::min(wave, grid - first);
        std::vector<emu::Cta> ctas(count);
        std::vector<emu::CtaExtra> extra(count);
        for (unsigned b = 0; b < count; ++b) {
            pthread_barrier_init(&ctas[b].bar, nullptr, block);
            ctas[b].dyn = nullptr;
            extra[b].or_acc = 0;
            for (unsigned w = 0; w < (block + 31) / 32; ++w) pthread_barrier_init(&ctas[b].warps[w].bar, nullptr, 32);
        }
        std::vector<std::thread> threads;
        for (unsigned b = 0; b < count; ++b)
            for (unsigned t = 0; t < block; ++t)
                threads.emplace_back([&, b, t] {
                    emu::tls.tid = t; emu::tls.bid = first + b; emu::tls.lane = t & 31u;
                    emu::tls.cta = &ctas[b]; emu::tls.warp = &ctas[b].warps[t >> 5];
                    emu::launch = &L; emu::cta_extra = &extra[b];
                    body();
                });
        for (auto& th : threads) th.join();
        for (auto& e : extra) for (auto& kv : e.shared) free(kv.second);
    }
}
"""

DRIVER = r"""
using namespace hnb;
extern "C" void semu_indirect(const StaticTables* T, uint32_t n) { StaticTables t = *T; emu_run([&] { k_indirect(t); }, (n + 63) / 64, 64); }
extern "C" void semu_clear_events(const StaticTables* T, uint32_t n) { StaticTables t = *T; emu_run([&] { k_clear_events(t); }, (n + 63) / 64, 64); }
extern "C" void semu_prefix_sum(const StaticTables* T, uint32_t nb) { StaticTables t = *T; emu_run([&] { k_prefix_sum(t); }, (nb + 63) / 64, 64); }
extern "C" void semu_bookkeeping(const StaticTables* T, uint32_t nb) { StaticTables t = *T; emu_run([&] { k_bookkeeping<16>(t, FrameBlock<16>{}, 0u); }, nb, 256, 8); }
extern "C" void semu_tile_prefix(const StaticTables* T, uint32_t batch, uint32_t tile) { StaticTables t = *T; emu_run([&] { k_tile_prefix(t, batch, tile); }, 1, 256); }
extern "C" void semu_ribbon_sort_small(const RibbonSortArgs* a) { RibbonSortArgs r = *a; emu_run([&] { k_ribbon_sort_small(r); }, r.instance_count, 1024, 3); }
extern "C" void semu_ribbon_sort_large(const RibbonSortArgs* a, uint32_t grid) { RibbonSortArgs r = *a; r.scratch_grid = grid; emu_run([&] { k_ribbon_sort_large(r); }, grid, 512); }
extern "C" void semu_ordered_event_append(const EventAppendArgs* a, uint32_t capacity_rows) {
    EventAppendArgs e = *a;
    const unsigned blocks = (capacity_rows + EV_ROWS_PER_BLOCK - 1) / EV_ROWS_PER_BLOCK;
    emu_run([&] { k_events_block_sums(e); }, blocks, EV_THREADS, 8);
    emu_run([&] { k_events_scan_blocks(e, blocks); }, 1, EV_THREADS);
    emu_run([&] { k_events_write(e); }, blocks, EV_THREADS, 8);
}
extern "C" void semu_events_scan_blocks(const EventAppendArgs* a, uint32_t blocks) { EventAppendArgs e = *a; emu_run([&] { k_events_scan_blocks(e, blocks); }, 1, EV_THREADS); }
extern "C" uint32_t semu_sizeof_event_args(void) { return sizeof(EventAppendArgs); }
extern "C" uint32_t semu_sizeof_static_tables(void) { return sizeof(StaticTables); }
extern "C" uint32_t semu_sizeof_ribbon_args(void) { return sizeof(RibbonSortArgs); }
extern "C" uint32_t semu_hist_words(uint32_t grid) { return 2 * 8 * 256 + 256 * grid; }
"""


def _strip_includes(text: str) -> str:
    return "\n".join(l for l in text.splitlines() if not l.lstrip().startswith("#include") and l.strip() != "#pragma once")


def _rewrite_shared(text: str) -> str:
    """`__shared__ T a[N], b;`  ->  per-CTA allocations shared by the CTA's threads (keys are unique per declarator)."""
    counter = [0]

    def repl(m):
        indent, ctype, decls = m.group(1), m.group(2).strip(), m.group(3)
        out = []
        for d in re.split(r",\s*(?![^\[]*\])", decls):
            d = d.strip()
            counter[0] += 1
            am = re.match(r"(\w+)\[(.+)\]$", d)
            if am:
                out.append(f"{indent}{ctype}* const {am.group(1)} = ({ctype}*)emu::cta_alloc({counter[0]}, sizeof({ctype}) * ({am.group(2)}));")
            else:
                out.append(f"{indent}{ctype}& {d} = *({ctype}*)emu::cta_alloc({counter[0]}, sizeof({ctype}));")
        return "\n".join(out)

    new = re.sub(r"^([ \t]*)__shared__\s+((?:unsigned\s+)?\w+)\s+([^;]+);[^\n]*$", repl, text, flags=re.M)
    assert "__shared__" not in re.sub(r"//[^\n]*", "", new), "an unhandled __shared__ declaration is left"
    return new


def build() -> C.CDLL:
    wgsl = _strip_includes((KERNELS / "hnb_wgsl.cuh").read_text())
    tables = _strip_includes((KERNELS / "hnb_tables.cuh").read_text())
    header = _strip_includes((KERNELS / "hnb_static_kernels.h").read_text())
    static = (KERNELS / "hnb_static_kernels.cu").read_text()
    static = _strip_includes(static[:static.index("cudaError_t launch_indirect(")]) + "\n}  // namespace hnb\n"
    ribbon = (KERNELS / "hnb_ribbon_sort.cu").read_text()
    ribbon = _strip_includes(ribbon[:ribbon.index("cudaError_t launch_ribbon_sort(")])
    # the sort kernels sit in an anonymous namespace that is closed just before the launcher
    assert ribbon.rstrip().endswith("}  // namespace"), "hnb_ribbon_sort.cu layout changed"
    ribbon += "\n}  // namespace hnb\n"
    # k_measure_sm_clock reads %globaltimer: not needed here
    static = re.sub(r"__global__ void k_measure_sm_clock.*?\n}\n", "", static, flags=re.S)
    body = _rewrite_shared(static + "\n" + ribbon)
    text = PRELUDE + EXTRA_PRELUDE + wgsl + "\n" + tables + "\n" + header + "\n" + body + DRIVER
    OUT.mkdir(parents=True, exist_ok=True)
    tag = hashlib.sha1(text.encode()).hexdigest()[:16]
    cpp, so = OUT / f"static_{tag}.{os.getpid()}.cpp", OUT / f"static_{tag}.so"  # per process: workers may build the same tag at once
    if not so.exists():
        cpp.write_text(text)
        cmd = ["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-w", str(cpp), "-o", str(so) + f".{os.getpid()}.tmp"]
        proc = subprocess.run(cmd, capture_output=True, text=True)
        if proc.returncode != 0:
            raise RuntimeError("host build of the static kernels failed:\n" + proc.stderr[:6000])
        os.replace(str(so) + f".{os.getpid()}.tmp", so)  # atomic: parallel test workers build the same tag
    lib = C.CDLL(str(so))
    for f in ("semu_sizeof_static_tables", "semu_sizeof_ribbon_args", "semu_sizeof_event_args"):
        getattr(lib, f).restype = C.c_uint32
    lib.semu_hist_words.restype = C.c_uint32
    lib.semu_hist_words.argtypes = [C.c_uint32]
    return lib


class StaticTables(C.Structure):
    """hnb::StaticTables (hnb_static_kernels.h)"""
    _fields_ = [(n, C.c_void_p) for n in ("frame", "spawners", "spawn_range", "prefix_sum", "tile_prefix", "batch_infos", "batch_tile_size",
                                          "dispatch_args", "batch_tiles", "tickets", "metadata", "draw_args", "child_infos")] + [("num_child_infos", C.c_uint32)]


class PlaneSet(C.Structure):
    _fields_ = [("ptr", C.c_void_p * 16), ("words", C.c_uint32 * 16), ("word_off", C.c_uint32 * 16), ("word_to_plane", C.c_ubyte * 64)]


class RibbonSortArgs(C.Structure):
    _fields_ = [("planes", PlaneSet), ("ping", C.c_void_p), ("pong", C.c_void_p), ("spawners", C.c_void_p), ("metadata", C.c_void_p),
                ("spawner_base", C.c_uint32), ("instance_count", C.c_uint32), ("scratch_keys", C.c_void_p * 2), ("scratch_vals", C.c_void_p * 2),
                ("scratch_hist", C.c_void_p), ("scratch_rows", C.c_uint32), ("scratch_grid", C.c_uint32)]


class EventAppendArgs(C.Structure):
    """hnb::EventAppendArgs (hnb_static_kernels.h)"""
    _fields_ = [("counts", C.c_void_p), ("ping", C.c_void_p), ("pong", C.c_void_p), ("spawner", C.c_void_p), ("metadata", C.c_void_p),
                ("block_sums", C.c_void_p), ("child_infos", C.c_void_p), ("binding", C.c_uint32), ("buffer", C.c_void_p), ("capacity", C.c_uint32)]
