// hnb_static_kernels.cu — effect-independent kernels, compiled ahead of time by nvcc for sm_90a.
//
//   k_indirect        ≙ src/render/vfx_indirect.wgsl main()   (:31-90)
//   k_prefix_sum      ≙ src/render/vfx_prefix_sum.wgsl main() (:14-43)
//   k_bookkeeping     = both of the above fused into one launch (one CTA per batch), used by
//                       hnb_simulate(); results identical to running them back to back
//   k_fill_dispatch_args ≙ src/render/vfx_utils.wgsl fill_dispatch_args (:54-67)
//   slab helpers: reset (effect_cache.rs:300-323), AoS<->SoA transposes, synthetic fill, checksum
//
// In addition to the reference's outputs the indirect step (a) applies the alive_count /
// particle_counter increments that the reference's init pass performs with per-particle atomics
// (vfx_init.wgsl:141,151) — our init kernel assigns ranks instead and defers the counter update to
// this per-instance step — and (b) the prefix step also scans the per-instance update TILE counts
// consumed by the persistent update kernel.
#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <cuda_runtime.h>

#include "hnb_wgsl.cuh"
#include "hnb_tables.cuh"
#include "hnb_static_kernels.h"

namespace hnb {

// ---------------------------------------------------------------------------------------------
// Per-instance step shared by k_indirect and k_bookkeeping.
// ---------------------------------------------------------------------------------------------
// The words of a spawner row that only the HOST writes (GpuSpawnerParams is uploaded by the CPU every frame, mod.rs:4679-4705; the
// device writes `render_indirect_read_index` only): they may be read before the programmatic-dependency wait.
struct SpawnerHostWords {
    u32 effect_metadata_index, draw_indirect_index;
    i32 spawn;
};
__device__ __forceinline__ SpawnerHostWords load_spawner_host_words(const StaticTables& T, u32 global_effect_index) {
    const Spawner* spawner = &T.spawners[global_effect_index];
    SpawnerHostWords w;
    w.effect_metadata_index = spawner->effect_metadata_index;
    w.draw_indirect_index = spawner->draw_indirect_index;
    w.spawn = spawner->spawn;
    return w;
}
// The frame block (header + every host-written table of the frame arena: batch infos, tile size words, spawner rows, spawn
// ranges, spawn prefix) as a kernel parameter: small frames reach the device inside the launch itself, with no copy-engine
// operation between two kernels of the frame chain (which would cost its own latency AND the programmatic overlap).
template <int NW> struct FrameBlock { u32 w[NW]; };
static_assert(offsetof(Spawner, render_indirect_read_index) == 26 * 4 && sizeof(Spawner) == 128, "k_bookkeeping skips this word when it stores a frame block");
static_assert(offsetof(BatchInfo, total_update_count) == 4 && sizeof(BatchInfo) == 24, "k_bookkeeping skips this word when it stores a frame block");
// a host-written arena word: from the parameter block when this launch carries the tables, else from the arena
template <int NW> __device__ __forceinline__ u32 host_word(const StaticTables& T, const FrameBlock<NW>& block, bool from_block, const void* arena_address) {
    if (from_block) return block.w[u32((const char*)arena_address - (const char*)T.frame) >> 2u];
    return *(const u32*)arena_address;
}
template <int NW> __device__ __forceinline__ SpawnerHostWords load_spawner_host_words(const StaticTables& T, const FrameBlock<NW>& block, bool from_block, u32 global_effect_index) {
    const Spawner* spawner = &T.spawners[global_effect_index];
    SpawnerHostWords w;
    w.effect_metadata_index = host_word(T, block, from_block, &spawner->effect_metadata_index);
    w.draw_indirect_index = host_word(T, block, from_block, &spawner->draw_indirect_index);
    w.spawn = i32(host_word(T, block, from_block, &spawner->spawn));
    return w;
}

// Loads of one instance's step (phase 1), separated from its arithmetic and stores (phase 2) so that a thread handling
// several instances has all their (dependent, latency-bound) loads in flight together.
struct EffectLoads {
    u32 range, alive_count, max_spawn, capacity, write_index, particle_counter, global_child_index;
};
__device__ __forceinline__ EffectLoads load_effect(const StaticTables& T, u32 global_effect_index, const SpawnerHostWords& hw) {
    const EffectMetadata* md = &T.metadata[hw.effect_metadata_index];
    EffectLoads L;
    L.range = T.spawn_range[global_effect_index];
    L.alive_count = md->alive_count;
    L.max_spawn = md->max_spawn;
    L.capacity = md->capacity;
    L.write_index = md->indirect_write_index;
    L.particle_counter = md->particle_counter;
    L.global_child_index = md->global_child_index;
    return L;
}
__device__ __forceinline__ u32 apply_effect(const StaticTables& T, u32 global_effect_index, const SpawnerHostWords& hw, const EffectLoads& L, u32* capacity_out = nullptr) {
    Spawner* spawner = &T.spawners[global_effect_index];
    EffectMetadata* md = &T.metadata[hw.effect_metadata_index];

    // (a) deferred init accounting: number of init threads of this instance that passed the caps of
    // vfx_init.wgsl:115-137 in the init launch that preceded this pass (0 if there was none).
    u32 alive_count = L.alive_count;
    if (L.range != 0u) {
        u32 requested;
        if (L.range & 0x80000000u) {
            // GPU-event driven instance: requested = event_count (vfx_init.wgsl:123-129)
            requested = u32(T.child_infos[L.global_child_index].event_count);
        } else {
            requested = u32(hw.spawn);
        }
        u32 n = min(L.range & 0x7fffffffu, requested);
        n = min(n, L.max_spawn);
        alive_count += n;
        md->alive_count = alive_count;
        md->particle_counter = L.particle_counter + n;
        T.spawn_range[global_effect_index] = 0u;
    }

    // vfx_indirect.wgsl:52-89
    const u32 dri_base = HNB_DRAW_INDEXED_INDIRECT_STRIDE * hw.draw_indirect_index;
    T.draw_args[dri_base + 1u] = 0u;
    const u32 capacity = L.capacity;
    if (capacity_out) *capacity_out = capacity;
    const u32 dead_count = capacity - alive_count;
    T.prefix_sum[global_effect_index] = alive_count;
    md->max_update = alive_count;
    md->max_spawn = dead_count;
    const u32 ping = L.write_index;
    const u32 pong = 1u - ping;
    md->indirect_write_index = pong;
    spawner->render_indirect_read_index = pong;
    return alive_count;
}
__device__ __forceinline__ u32 indirect_one_effect(const StaticTables& T, u32 global_effect_index, const SpawnerHostWords& hw, u32* capacity_out = nullptr) {
    return apply_effect(T, global_effect_index, hw, load_effect(T, global_effect_index, hw), capacity_out);
}

__global__ void k_indirect(StaticTables T) {
    const u32 global_effect_index = blockIdx.x * blockDim.x + threadIdx.x;
    if (global_effect_index >= T.frame->sim.num_effects) return;
    // HAS_GPU_SPAWN_EVENTS: clear the event counts AFTER they were consumed by init (:38-46). The
    // reference indexes the child-info array with the effect index; we do the same.
    // NOTE: the deferred accounting above needs event_count, so it is read before being cleared
    // only when the clearing thread and the reading thread are the same; to stay race-free the clear
    // happens in a second kernel phase (see k_clear_events).
    indirect_one_effect(T, global_effect_index, load_spawner_host_words(T, global_effect_index));
}

__global__ void k_clear_events(StaticTables T) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= T.frame->sim.num_effects) return;
    if (i < T.num_child_infos) T.child_infos[i].event_count = 0;
}

// Serial scan of one batch by one thread, exactly like the reference (vfx_prefix_sum.wgsl:27-42).
__global__ void k_prefix_sum(StaticTables T) {
    const u32 batch_index = blockIdx.x * blockDim.x + threadIdx.x;
    if (batch_index >= T.frame->num_batches) return;
    BatchInfo* bi = &T.batch_infos[batch_index];
    const u32 offset = bi->prefix_sum_offset;
    const u32 end = offset + bi->prefix_sum_count;
    const u32 tile = T.batch_tile_size[batch_index];
    u32 sum = 0u, tiles = 0u;
    for (u32 i = offset; i < end; i += 1u) {
        const u32 count = T.prefix_sum[i];
        T.prefix_sum[i] = sum;
        T.tile_prefix[i] = tiles;
        sum += count;
        // slot order: the update pass walks the instance's slots, not its alive rows
        const u32 rows = (tile & HNB_TILE_SLOT_ORDER) ? T.metadata[T.spawners[bi->spawner_base + (i - offset)].effect_metadata_index].capacity : count;
        tiles += hnb_tile_count(rows, tile);
    }
    bi->total_update_count = sum;
    T.dispatch_args[batch_index * 3u + 0u] = (sum + 63u) >> 6u;
    T.dispatch_args[batch_index * 3u + 1u] = 1u;
    T.dispatch_args[batch_index * 3u + 2u] = 1u;
    T.batch_tiles[batch_index] = tiles;
    T.tickets[batch_index] = 0u;
}

// Fused indirect + prefix-sum: CTA b owns batch b. Requires that the batches tile the spawner table
// (checked on the host: HNB_ERR_BATCH_COVERAGE), which Batcher::push guarantees in the reference
// (prefix sums and spawners are allocated in sync, vfx_indirect.wgsl:66).
//
// Launched with programmatic stream serialization (see hnb_pdl_wait): the CTA becomes resident during the tail of the
// previous frame's update kernel and lets this frame's update grid follow it onto the SMs, so that the frame chain
// update(N) -> bookkeeping(N+1) -> update(N+1) pays no launch latency. `header_words` != NULL: the 64-byte frame header
// (sim params, epoch, batch count) travels as a kernel parameter and CTA 0 stores it into the device frame block —
// frames whose tables did not change need no host->device copy at all.
#define BK_THREADS 256
#define BK_ITEMS 4  // instances per thread and pass of the many-instance path
#define BK_HEADER_WORDS u32(sizeof(FrameHeader) / 4)
// `block_words`: 0 = the host copied the frame block; BK_HEADER_WORDS = only the 64-byte header rides in `block` (tables unchanged
// since the last frame); more = `block` holds the first `block_words` words of the frame arena, i.e. the header AND every
// host-written table (frames without init launches whose tables fit the parameter space).
template <int NW>
__global__ void __launch_bounds__(BK_THREADS) k_bookkeeping(StaticTables T, const __grid_constant__ FrameBlock<NW> block, u32 block_words) {
    __shared__ u32 s_warp_a[BK_THREADS / 32], s_warp_t[BK_THREADS / 32];
    __shared__ u32 s_carry_a, s_carry_t;
    hnb_pdl_launch_dependents();
    // ---- Before the dependency wait: everything that only the HOST writes (batch infos, tile size word, the spawner rows'
    // CPU words). These came with a stream-ordered copy that completed before this grid could start, and no kernel touches
    // them, so the loads (and their DRAM / L2 round trips: batch info -> spawner row are DEPENDENT) overlap the tail of the
    // previous frame's update kernel instead of sitting on the frame chain's critical path. Device-written state (metadata
    // rows, spawn ranges, child infos, the frame header) is read after the wait only.
    const u32 batch_index = blockIdx.x;
    const bool from_block = block_words > BK_HEADER_WORDS;  // the tables travel with this launch: never read them from the arena
    BatchInfo* bi = &T.batch_infos[batch_index];
    const u32 offset = host_word(T, block, from_block, &bi->prefix_sum_offset);
    const u32 count = host_word(T, block, from_block, &bi->prefix_sum_count);
    const u32 tile = host_word(T, block, from_block, &T.batch_tile_size[batch_index]);
    const u32 tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5u;
    // Batches of at most 32 instances (every single-effect batch) need one warp and no barrier.
    const bool one_warp = count <= 32u;
    // (the other warps of CTA 0 stay for the store of a large parameter block)
    const bool block_helpers = blockIdx.x == 0 && block_words > 64u;
    if (one_warp && warp != 0u && !block_helpers) return;
    SpawnerHostWords first_hw[BK_ITEMS];
#pragma unroll
    for (int k = 0; k < BK_ITEMS; ++k) {
        first_hw[k] = SpawnerHostWords();
        const u32 i = one_warp ? (k == 0 ? tid : count) : tid * BK_ITEMS + k;
        if (i < count) first_hw[k] = load_spawner_host_words(T, block, from_block, offset + i);
    }
    hnb_pdl_wait();
    // CTA 0 puts the block into the device arena for the kernels that follow (the update pass reads spawner rows, the frame
    // header, ...). Nobody reads those words concurrently: the previous frame's kernels are complete (the wait above), the other
    // CTAs of this grid take their host words from `block`, and the next frame's grids cannot become resident before the
    // update kernel of THIS frame has passed its own wait (it signals its dependents after it), i.e. after this grid is done.
    // The two word classes of the block's range that the DEVICE writes — `total_update_count` of a batch info and
    // `render_indirect_read_index` of a spawner row, both written further down by whichever CTA owns the row — are left out of
    // the store: every stored word is host-only, so the store races with nothing in this grid.
    if (blockIdx.x == 0) {
        const u32 bi0 = u32((const u32*)T.batch_infos - (const u32*)T.frame), bi1 = u32((const u32*)T.batch_tile_size - (const u32*)T.frame);
        const u32 sp0 = u32((const u32*)T.spawners - (const u32*)T.frame), sp1 = u32((const u32*)T.spawn_range - (const u32*)T.frame);
        for (u32 i = tid; i < block_words; i += ((one_warp && !block_helpers) ? 32u : BK_THREADS)) {
            const bool device_word = (i >= bi0 && i < bi1 && (i - bi0) % u32(sizeof(BatchInfo) / 4) == 1u) ||
                                     (i >= sp0 && i < sp1 && (i - sp0) % u32(sizeof(Spawner) / 4) == 26u);
            if (!device_word) ((u32*)T.frame)[i] = block.w[i];
        }
    }
    if (one_warp && warp != 0u) return;
    if (one_warp) {
        u32 a = 0u, t = 0u;
        if (lane < count) {
            u32 capacity;
            a = indirect_one_effect(T, offset + lane, first_hw[0], &capacity);
            t = hnb_tile_count((tile & HNB_TILE_SLOT_ORDER) ? capacity : a, tile);
        }
        u32 ia = a, it = t;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const u32 ua = __shfl_up_sync(0xffffffffu, ia, d), ut = __shfl_up_sync(0xffffffffu, it, d);
            if (lane >= d) { ia += ua; it += ut; }
        }
        if (lane < count) {
            T.prefix_sum[offset + lane] = ia - a;
            T.tile_prefix[offset + lane] = it - t;
        }
        const u32 sum = __shfl_sync(0xffffffffu, ia, 31), tiles = __shfl_sync(0xffffffffu, it, 31);
        if (lane == 0) {
            bi->total_update_count = sum;
            T.dispatch_args[batch_index * 3u + 0u] = (sum + 63u) >> 6u;
            T.dispatch_args[batch_index * 3u + 1u] = 1u;
            T.dispatch_args[batch_index * 3u + 2u] = 1u;
            T.batch_tiles[batch_index] = tiles;
            T.tickets[batch_index] = 0u;
        }
        return;
    }
    if (tid == 0) { s_carry_a = 0u; s_carry_t = 0u; }
    __syncthreads();
    // Each thread owns BK_ITEMS CONSECUTIVE instances per pass (1024 instances = one pass): phase 1 issues the loads of all of
    // them, phase 2 does their arithmetic and stores, then one block-wide scan over the per-thread sums.
    for (u32 chunk = 0; chunk < count; chunk += BK_THREADS * BK_ITEMS) {
        const u32 i0 = chunk + tid * BK_ITEMS;
        SpawnerHostWords hw[BK_ITEMS];
        EffectLoads L[BK_ITEMS];
#pragma unroll
        for (int k = 0; k < BK_ITEMS; ++k) {
            hw[k] = first_hw[k];
            if (chunk != 0u && i0 + k < count) hw[k] = load_spawner_host_words(T, block, from_block, offset + i0 + k);
        }
#pragma unroll
        for (int k = 0; k < BK_ITEMS; ++k)
            if (i0 + k < count) L[k] = load_effect(T, offset + i0 + k, hw[k]);
        u32 a[BK_ITEMS], t[BK_ITEMS], sa = 0u, st = 0u;
#pragma unroll
        for (int k = 0; k < BK_ITEMS; ++k) {
            a[k] = 0u; t[k] = 0u;
            if (i0 + k < count) {
                u32 capacity;
                a[k] = apply_effect(T, offset + i0 + k, hw[k], L[k], &capacity);
                t[k] = hnb_tile_count((tile & HNB_TILE_SLOT_ORDER) ? capacity : a[k], tile);
            }
            sa += a[k]; st += t[k];
        }
        // block-wide exclusive scan of the per-thread sums (sa, st)
        u32 ia = sa, it = st;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const u32 ua = __shfl_up_sync(0xffffffffu, ia, d), ut = __shfl_up_sync(0xffffffffu, it, d);
            if (lane >= d) { ia += ua; it += ut; }
        }
        if (lane == 31) { s_warp_a[warp] = ia; s_warp_t[warp] = it; }
        __syncthreads();
        u32 wa = 0u, wt = 0u;
        for (u32 w = 0; w < warp; ++w) { wa += s_warp_a[w]; wt += s_warp_t[w]; }
        const u32 carry_a = s_carry_a, carry_t = s_carry_t;
        u32 base_a = carry_a + wa + ia - sa, base_t = carry_t + wt + it - st;
#pragma unroll
        for (int k = 0; k < BK_ITEMS; ++k) {
            if (i0 + k < count) {
                T.prefix_sum[offset + i0 + k] = base_a;
                T.tile_prefix[offset + i0 + k] = base_t;
            }
            base_a += a[k]; base_t += t[k];
        }
        __syncthreads();
        if (tid == BK_THREADS - 1) { s_carry_a = carry_a + wa + ia; s_carry_t = carry_t + wt + it; }
        __syncthreads();
    }
    if (tid == 0) {
        const u32 sum = s_carry_a;
        bi->total_update_count = sum;
        T.dispatch_args[batch_index * 3u + 0u] = (sum + 63u) >> 6u;
        T.dispatch_args[batch_index * 3u + 1u] = 1u;
        T.dispatch_args[batch_index * 3u + 2u] = 1u;
        T.batch_tiles[batch_index] = s_carry_t;
        T.tickets[batch_index] = 0u;
    }
}

// Tile prefix of ONE batch for a given tile size, from the max_update values already published by the
// indirect pass. Used by the stand-alone hnb_pass_update(), whose tile size (a property of the compiled
// effect and of the launch) is unknown to a stand-alone prefix-sum pass.
__global__ void __launch_bounds__(BK_THREADS) k_tile_prefix(StaticTables T, u32 batch_index, u32 tile) {
    __shared__ u32 s_warp_t[BK_THREADS / 32];
    __shared__ u32 s_carry_t;
    const BatchInfo* bi = &T.batch_infos[batch_index];
    const u32 offset = bi->prefix_sum_offset, count = bi->prefix_sum_count;
    const u32 tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5u;
    if (tid == 0) s_carry_t = 0u;
    __syncthreads();
    for (u32 chunk = 0; chunk < count; chunk += BK_THREADS) {
        const u32 i = chunk + tid;
        u32 t = 0u;
        if (i < count) {
            const Spawner* sp = &T.spawners[bi->spawner_base + i];
            const EffectMetadata* md = &T.metadata[sp->effect_metadata_index];
            t = hnb_tile_count((tile & HNB_TILE_SLOT_ORDER) ? md->capacity : md->max_update, tile);
        }
        u32 it = t;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const u32 ut = __shfl_up_sync(0xffffffffu, it, d);
            if (lane >= d) it += ut;
        }
        if (lane == 31) s_warp_t[warp] = it;
        __syncthreads();
        u32 wt = 0u;
        for (u32 w = 0; w < warp; ++w) wt += s_warp_t[w];
        const u32 carry_t = s_carry_t;
        if (i < count) T.tile_prefix[offset + i] = carry_t + wt + it - t;
        __syncthreads();
        if (tid == BK_THREADS - 1) s_carry_t = carry_t + wt + it;
        __syncthreads();
    }
    if (tid == 0) {
        T.batch_tiles[batch_index] = s_carry_t;
        T.tickets[batch_index] = 0u;
    }
}

// vfx_utils.wgsl:54-67
__global__ void k_fill_dispatch_args(const u32* src, u32* dst, u32 src_offset, u32 src_stride, u32 dst_offset,
                                     u32 dst_stride, u32 count) {
    const u32 thread_index = blockIdx.x * blockDim.x + threadIdx.x;
    if (thread_index >= count) return;
    const u32 s = src_offset + thread_index * src_stride;
    const u32 d = dst_offset + thread_index * dst_stride;
    const u32 thread_count = src[s];
    dst[d] = (thread_count + 63u) >> 6u;
    dst[d + 1u] = 1u;
    dst[d + 2u] = 1u;
}

// ---------------------------------------------------------------------------------------------
// Slab helpers
// ---------------------------------------------------------------------------------------------
__global__ void k_slab_reset(u32* ping, u32* pong, u32* dead, u32 first, u32 count) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    ping[first + i] = 0u;
    pong[first + i] = 0u;
    dead[first + i] = first + i;  // effect_cache.rs:317-319
}

// Alive bitmap of a slab (one bit per row, HNB_EFFECT_SLOT_ORDER): set or clear the bits of rows [first, first+count).
// One thread per 32-row word; words only partly inside the range are updated atomically.
__global__ void k_bits_range(u32* bits, u32 first, u32 count, u32 set) {
    const u32 w0 = first >> 5u;
    const u32 w = w0 + blockIdx.x * blockDim.x + threadIdx.x;
    const u64 end = u64(first) + count;
    if (u64(w) * 32u >= end) return;
    const u64 lo = u64(w) * 32u > first ? u64(w) * 32u : u64(first);
    const u64 hi = u64(w) * 32u + 32u < end ? u64(w) * 32u + 32u : end;
    const u32 n = u32(hi - lo), sh = u32(lo - u64(w) * 32u);
    const u32 mask = (n == 32u ? 0xffffffffu : ((1u << n) - 1u)) << sh;
    if (mask == 0xffffffffu) bits[w] = set ? 0xffffffffu : 0u;
    else if (set) atomicOr(&bits[w], mask);
    else atomicAnd(&bits[w], ~mask);
}
// ... and the bits of the rows an alive list names: list[i] (instance-local) + base, i < alive_count
__global__ void k_bits_from_list(u32* bits, const u32* list, u32 base, u32 alive_count) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= alive_count) return;
    const u32 row = base + list[i];
    atomicOr(&bits[row >> 5u], 1u << (row & 31u));
}

// Synthetic C5 state (SURVEY §8d): counter-based so that the CPU oracle can regenerate any row.
//   s = pcg_hash(row ^ seed); six successive pcg_hash -> position, velocity in [-1,1); one more -> lifetime
// `logical_first`: row of the LOGICAL instance stored at slab row `first` (a shard of an instance split by index range
// over several devices holds the unsharded instance's values under shard-local indices).
__global__ void k_fill_c5(float4* pos_age, float4* vel_life, u32* ping, u32* pong, u64* claim, u32 first, u32 count, u32 seed,
                          f32 lifetime_lo, f32 lifetime_hi, u32 logical_first) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    if (i == 0u) {
        hnb_claim_store(&claim[0], hnb_claim_pack(first, count));
        hnb_claim_store(&claim[1], hnb_claim_pack(first, count));
    }
    const u32 row = first + i;
    u32 s = pcg_hash((logical_first + i) ^ seed);
    f32 v[7];
    for (int k = 0; k < 7; ++k) { s = pcg_hash(s); v[k] = to_float01(s); }
    pos_age[row] = make_float4(v[0] * 2.0f - 1.0f, v[1] * 2.0f - 1.0f, v[2] * 2.0f - 1.0f, 0.0f);
    vel_life[row] = make_float4(v[3] * 2.0f - 1.0f, v[4] * 2.0f - 1.0f, v[5] * 2.0f - 1.0f,
                                lifetime_lo + v[6] * (lifetime_hi - lifetime_lo));
    ping[row] = i;  // instance-local identity alive list in both columns
    pong[row] = i;
}

// ---------------------------------------------------------------------------------------------
// Repack of one instance (hnb_slab_repack): local row i receives the record of local row src[i], the alive slots first in
// alive-list order, then the dead slots in stack order; afterwards both alive lists and the dead stack are the identity.
// One gather launch per physical column (into a scratch of `rows` elements, copied back over the slice by the host), then
// one launch for the lists, the claims and the alive bitmap. n and W come from the device metadata row.
// ---------------------------------------------------------------------------------------------
#define RP_THREADS 256
#define RP_ITEMS 4  // rows per thread in flight: a gather is bound by latency (as hnb_init, DESIGN.md §4.2)
#define RP_ROWS_PER_BLOCK (RP_THREADS * RP_ITEMS)

// One element of a physical column: 1, 2, 4 or 8 words (4, 8, 16 or 32 bytes; 32 = a sector-plane column).
template <int W> struct alignas(W >= 4 ? 16 : W * 4) RepackPiece { u32 w[W]; };

// src[i], clamped to the slice: a state that breaks the update invariant gives an unspecified result, never an access
// outside the slice.
__device__ __forceinline__ u32 repack_source(const RepackArgs& a, const u32* list, u32 n, u32 i) {
    const u32 s = i < n ? list[a.first + i] : a.dead[a.first + i] - a.first;
    return min(s, a.rows - 1u);
}

template <int W>
__global__ void __launch_bounds__(RP_THREADS) k_repack_gather(RepackArgs a, const RepackPiece<W>* col, RepackPiece<W>* scratch) {
    const u32 n = min(a.metadata->alive_count, a.rows);
    const u32* list = a.metadata->indirect_write_index == 0u ? a.ping : a.pong;
    const u32 i0 = blockIdx.x * RP_ROWS_PER_BLOCK + threadIdx.x;
    u32 src[RP_ITEMS];
#pragma unroll
    for (u32 k = 0; k < RP_ITEMS; ++k) {
        const u32 i = i0 + k * RP_THREADS;
        src[k] = i < a.rows ? repack_source(a, list, n, i) : 0u;
    }
    RepackPiece<W> v[RP_ITEMS];
#pragma unroll
    for (u32 k = 0; k < RP_ITEMS; ++k)
        if (i0 + k * RP_THREADS < a.rows) v[k] = col[u64(a.first) + src[k]];
#pragma unroll
    for (u32 k = 0; k < RP_ITEMS; ++k)
        if (i0 + k * RP_THREADS < a.rows) scratch[i0 + k * RP_THREADS] = v[k];
}

// After every gather (they read the lists): ping = pong = identity below n, dead = identity from n, both claims
// {first, n}, alive bits set below n and cleared above. Thread t owns row t and, for t < words, bitmap word t of the slice.
__global__ void __launch_bounds__(RP_THREADS) k_repack_lists(RepackArgs a) {
    const u32 n = min(a.metadata->alive_count, a.rows);
    const u32 i = blockIdx.x * RP_THREADS + threadIdx.x;
    if (i == 0u) {
        hnb_claim_store(&a.claim[0], hnb_claim_pack(a.first, n));
        hnb_claim_store(&a.claim[1], hnb_claim_pack(a.first, n));
    }
    if (i < a.rows) {
        if (i < n) {
            a.ping[a.first + i] = i;
            a.pong[a.first + i] = i;
        } else {
            a.dead[a.first + i] = a.first + i;
        }
    }
    const u32 w0 = a.first >> 5u;
    const u64 end = u64(a.first) + a.rows, alive_end = u64(a.first) + n;
    const u32 w = w0 + i;
    if (u64(w) * 32u >= end) return;
    const u64 lo = u64(w) * 32u > a.first ? u64(w) * 32u : u64(a.first);
    const u64 hi = u64(w) * 32u + 32u < end ? u64(w) * 32u + 32u : end;
    const u64 alive_hi = hi < alive_end ? hi : alive_end;
    const u32 sh = u32(lo - u64(w) * 32u);
    const u32 span = u32(hi - lo), alive = alive_hi > lo ? u32(alive_hi - lo) : 0u;
    const u32 inside = (span == 32u ? 0xffffffffu : ((1u << span) - 1u)) << sh;
    const u32 set = (alive == 32u ? 0xffffffffu : ((1u << alive) - 1u)) << sh;
    if (inside == 0xffffffffu) {
        a.alive_bits[w] = set;
    } else {  // a word shared with a neighbouring instance: change only the slice's bits
        atomicAnd(&a.alive_bits[w], ~inside | set);
        if (set) atomicOr(&a.alive_bits[w], set);
    }
}

// ---------------------------------------------------------------------------------------------
// Snapshot / restore of one instance (hnb_instance_snapshot / hnb_instance_restore). A snapshot is a 64-byte header
// followed by reference AoS records in alive-list order: record i sits at word HNB_SNAPSHOT_HEADER_WORDS + i * stride_words.
// Both kernels move one physical column at a time, RP_ITEMS rows in flight per thread, and split a piece into the widest
// accesses the record stride and the piece's offset in the record allow (16, 8 or 4 bytes; the buffer is 16-byte aligned).
// ---------------------------------------------------------------------------------------------
template <int Q, int W> __device__ __forceinline__ void snapshot_store(u32* dst, const RepackPiece<W>& v) {
#pragma unroll
    for (int j = 0; j < W / Q; ++j) {
        RepackPiece<Q> q;
#pragma unroll
        for (int k = 0; k < Q; ++k) q.w[k] = v.w[j * Q + k];
        ((RepackPiece<Q>*)dst)[j] = q;
    }
}
template <int Q, int W> __device__ __forceinline__ void snapshot_load(const u32* src, RepackPiece<W>& v) {
#pragma unroll
    for (int j = 0; j < W / Q; ++j) {
        const RepackPiece<Q> q = ((const RepackPiece<Q>*)src)[j];
#pragma unroll
        for (int k = 0; k < Q; ++k) v.w[j * Q + k] = q.w[k];
    }
}
// words of alignment shared by every record's piece at word `off`: 4, 2 or 1
__device__ __forceinline__ u32 snapshot_align(u32 stride_words, u32 off) {
    const u32 m = stride_words | off;
    return (m & 3u) == 0u ? 4u : ((m & 1u) == 0u ? 2u : 1u);
}

// records i0 + k * RP_THREADS < n of column p: local rows src[k] -> AoS records in `dst`
template <int W>
__device__ __forceinline__ void snapshot_column(const SnapshotArgs& a, u32 p, const u32 (&src)[RP_ITEMS], u32 i0, u32 n, u32* dst) {
    const RepackPiece<W>* col = (const RepackPiece<W>*)a.planes.ptr[p] + a.first;
    const u32 off = a.planes.word_off[p], al = snapshot_align(a.stride_words, off);
    RepackPiece<W> v[RP_ITEMS];
#pragma unroll
    for (u32 k = 0; k < RP_ITEMS; ++k)
        if (i0 + k * RP_THREADS < n) v[k] = col[src[k]];
#pragma unroll
    for (u32 k = 0; k < RP_ITEMS; ++k) {
        const u32 i = i0 + k * RP_THREADS;
        if (i >= n) continue;
        u32* d = dst + HNB_SNAPSHOT_HEADER_WORDS + u64(i) * a.stride_words + off;
        if (W >= 4 && al == 4u) snapshot_store<4>(d, v[k]);
        else if (W >= 2 && al >= 2u) snapshot_store<2>(d, v[k]);
        else snapshot_store<1>(d, v[k]);
    }
}

// Header by the first 16 threads, then record i < n = min(alive_count, rows) from local row list_W[i] (clamped to the
// slice as repack_source clamps it). Reads nothing but the metadata row, column W and the planes.
__global__ void __launch_bounds__(RP_THREADS) k_snapshot_gather(SnapshotArgs a, u32* dst) {
    const EffectMetadata* md = a.metadata;
    const u32 n = min(md->alive_count, a.rows);
    if (blockIdx.x == 0u && threadIdx.x < HNB_SNAPSHOT_HEADER_WORDS) {
        const u32 t = threadIdx.x;
        dst[t] = t == 0u ? HNB_SNAPSHOT_MAGIC_WORD
               : t == 1u ? HNB_SNAPSHOT_VERSION_WORD
               : t == 2u ? a.stride_words * 4u
               : t == 3u ? n
               : t == 4u ? md->particle_counter
               : t == 5u ? a.rows
               : 0u;
    }
    const u32* list = md->indirect_write_index == 0u ? a.ping : a.pong;
    const u32 i0 = blockIdx.x * RP_ROWS_PER_BLOCK + threadIdx.x;
    if (i0 >= n) return;
    u32 src[RP_ITEMS];
#pragma unroll
    for (u32 k = 0; k < RP_ITEMS; ++k) {
        const u32 i = i0 + k * RP_THREADS;
        src[k] = i < n ? min(list[a.first + i], a.rows - 1u) : 0u;
    }
    for (u32 p = 0; p < a.num_planes; ++p) {
        switch (a.planes.words[p]) {
        case 1: snapshot_column<1>(a, p, src, i0, n, dst); break;
        case 2: snapshot_column<2>(a, p, src, i0, n, dst); break;
        case 4: snapshot_column<4>(a, p, src, i0, n, dst); break;
        default: snapshot_column<8>(a, p, src, i0, n, dst); break;
        }
    }
}

// m = min(count, rows, records the buffer holds); 0 for a header that is not a version-1 snapshot of this stride
__device__ __forceinline__ u32 restore_count(const SnapshotArgs& a, const u32* src) {
    if (src[0] != HNB_SNAPSHOT_MAGIC_WORD || src[1] != HNB_SNAPSHOT_VERSION_WORD || src[2] != a.stride_words * 4u) return 0u;
    const u64 fit = (a.src_bytes - HNB_SNAPSHOT_HEADER_WORDS * 4u) / (a.stride_words * 4u);
    const u64 m = src[3] < a.rows ? src[3] : a.rows;
    return u32(m < fit ? m : fit);
}

template <int W>
__device__ __forceinline__ void restore_column(const SnapshotArgs& a, u32 p, u32 i0, u32 m, const u32* src) {
    RepackPiece<W>* col = (RepackPiece<W>*)a.planes.ptr[p] + a.first;
    const u32 off = a.planes.word_off[p], al = snapshot_align(a.stride_words, off);
    RepackPiece<W> v[RP_ITEMS];
#pragma unroll
    for (u32 k = 0; k < RP_ITEMS; ++k) {
        const u32 i = i0 + k * RP_THREADS;
        if (i >= m) continue;
        const u32* s = src + HNB_SNAPSHOT_HEADER_WORDS + u64(i) * a.stride_words + off;
        if (W >= 4 && al == 4u) snapshot_load<4>(s, v[k]);
        else if (W >= 2 && al >= 2u) snapshot_load<2>(s, v[k]);
        else snapshot_load<1>(s, v[k]);
    }
#pragma unroll
    for (u32 k = 0; k < RP_ITEMS; ++k)
        if (i0 + k * RP_THREADS < m) col[i0 + k * RP_THREADS] = v[k];
}

// Record i < m -> local row i of every column; thread 0 writes alive_count = m, max_spawn = capacity - m (0 if the row's
// capacity is below m) and, for an accepted header, particle_counter. k_repack_lists follows and reads m back.
__global__ void __launch_bounds__(RP_THREADS) k_restore_scatter(SnapshotArgs a, const u32* src) {
    const u32 m = restore_count(a, src);
    const u32 i0 = blockIdx.x * RP_ROWS_PER_BLOCK + threadIdx.x;
    if (i0 == 0u) {
        EffectMetadata* md = a.metadata;
        md->alive_count = m;
        md->max_spawn = md->capacity > m ? md->capacity - m : 0u;
        if (src[0] == HNB_SNAPSHOT_MAGIC_WORD && src[1] == HNB_SNAPSHOT_VERSION_WORD && src[2] == a.stride_words * 4u)
            md->particle_counter = src[4];
    }
    if (i0 >= m) return;
    for (u32 p = 0; p < a.num_planes; ++p) {
        switch (a.planes.words[p]) {
        case 1: restore_column<1>(a, p, i0, m, src); break;
        case 2: restore_column<2>(a, p, i0, m, src); break;
        case 4: restore_column<4>(a, p, i0, m, src); break;
        default: restore_column<8>(a, p, i0, m, src); break;
        }
    }
}

// Order-independent checksum: sum over rows of a 64-bit mix of the row's AoS words and row index.
__global__ void k_checksum(PlaneSet planes, u32 first, u32 count, u32 stride_words, u64 index_base, u64* out) {
    u64 acc = 0;
    for (u64 i = u64(blockIdx.x) * blockDim.x + threadIdx.x; i < count; i += u64(gridDim.x) * blockDim.x) {
        u64 h = 0xcbf29ce484222325ull ^ (index_base + u64(i));
        for (u32 w = 0; w < stride_words; ++w) {
            const u32 p = planes.word_to_plane[w];
            const u32 lane = w - planes.word_off[p];
            const u32 x = ((const u32*)planes.ptr[p])[u64(first + i) * planes.words[p] + lane];
            h = (h ^ u64(x)) * 0x100000001b3ull;
        }
        h ^= h >> 29; h *= 0xbf58476d1ce4e5b9ull; h ^= h >> 32;
        acc += h;
    }
    for (int d = 16; d > 0; d >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, d);
    if ((threadIdx.x & 31u) == 0) atomicAdd((unsigned long long*)out, (unsigned long long)acc);
}

// ---------------------------------------------------------------------------------------------
// Ordered event append (HNB_EFFECT_ORDERED_EVENTS). The update kernel stored, per update row, how many events the
// particle asked for on a channel; these three launches append them in row order — the order a serial execution of the
// reference's threads would produce (append_spawn_events_N, lib.rs:976-993): position = exclusive prefix of the counts,
// clamped to the buffer capacity; ChildInfo.event_count receives the unclamped total like the reference's atomicAdd.
// ---------------------------------------------------------------------------------------------
#define EV_THREADS 256
#define EV_ITEMS 8
#define EV_ROWS_PER_BLOCK (EV_THREADS * EV_ITEMS)

__device__ __forceinline__ u32 ev_block_exclusive_scan(u32 v, u32* s_warp, u32* total) {
    const u32 lane = threadIdx.x & 31u, warp = threadIdx.x >> 5u;
    u32 incl = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const u32 up = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += up;
    }
    if (lane == 31u) s_warp[warp] = incl;
    __syncthreads();
    u32 before = 0u, all = 0u;
    for (u32 w = 0; w < EV_THREADS / 32; ++w) {
        const u32 x = s_warp[w];
        before += w < warp ? x : 0u;
        all += x;
    }
    __syncthreads();
    if (total) *total = all;
    return before + incl - v;
}

__global__ void __launch_bounds__(EV_THREADS) k_events_block_sums(EventAppendArgs a) {
    __shared__ u32 s_warp[EV_THREADS / 32];
    const u32 rows = a.metadata->max_update;
    const u32 first = blockIdx.x * EV_ROWS_PER_BLOCK + threadIdx.x * EV_ITEMS;
    u32 sum = 0u;
#pragma unroll
    for (u32 k = 0; k < EV_ITEMS; ++k)
        if (first + k < rows) sum += a.counts[first + k];
    u32 total;
    ev_block_exclusive_scan(sum, s_warp, &total);
    if (threadIdx.x == 0) a.block_sums[blockIdx.x] = total;
}

// one CTA: exclusive scan of the block sums in place, total into the child's event count
__global__ void __launch_bounds__(EV_THREADS) k_events_scan_blocks(EventAppendArgs a, u32 num_blocks) {
    __shared__ u32 s_warp[EV_THREADS / 32];
    __shared__ u32 s_carry;
    if (threadIdx.x == 0) s_carry = 0u;
    __syncthreads();
    for (u32 chunk = 0; chunk < num_blocks; chunk += EV_THREADS) {
        const u32 i = chunk + threadIdx.x;
        const u32 v = i < num_blocks ? a.block_sums[i] : 0u;
        u32 total;
        const u32 excl = ev_block_exclusive_scan(v, s_warp, &total);
        const u32 carry = s_carry;
        if (i < num_blocks) a.block_sums[i] = carry + excl;
        __syncthreads();
        if (threadIdx.x == 0) s_carry = carry + total;
        __syncthreads();
    }
    if (threadIdx.x == 0) atomicAdd(&a.child_infos[a.metadata->base_child_index + a.binding].event_count, i32(s_carry));
}

__global__ void __launch_bounds__(EV_THREADS) k_events_write(EventAppendArgs a) {
    __shared__ u32 s_warp[EV_THREADS / 32];
    const u32 rows = a.metadata->max_update;
    // the alive list the update pass READ: the column that is not indirect_write_index, instance-local rows
    const u32* read_col = (a.metadata->indirect_write_index == 0u ? a.pong : a.ping) + a.spawner->slab_offset;
    const u32 first = blockIdx.x * EV_ROWS_PER_BLOCK + threadIdx.x * EV_ITEMS;
    u32 c[EV_ITEMS], sum = 0u;
#pragma unroll
    for (u32 k = 0; k < EV_ITEMS; ++k) {
        c[k] = first + k < rows ? a.counts[first + k] : 0u;
        sum += c[k];
    }
    u32 pos = a.block_sums[blockIdx.x] + ev_block_exclusive_scan(sum, s_warp, nullptr);
#pragma unroll
    for (u32 k = 0; k < EV_ITEMS; ++k) {
        if (c[k] == 0u) continue;
        const u32 particle_index = read_col[first + k];
        for (u32 i = 0; i < c[k] && pos + i < a.capacity; ++i) a.buffer[pos + i] = particle_index;
        pos += c[k];
    }
}

// Effective SM clock: cycles elapsed on one SM over ~`window_ns` of the global timer.
__global__ void k_measure_sm_clock(u64* out, u64 window_ns) {
    u64 t0, t1;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    const long long c0 = clock64();
    do {
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
    } while (t1 - t0 < window_ns);
    const long long c1 = clock64();
    out[0] = u64(c1 - c0);
    out[1] = t1 - t0;
}

// ---------------------------------------------------------------------------------------------
// Host-callable launchers (declared in hnb_static_kernels.h)
// ---------------------------------------------------------------------------------------------
static inline unsigned blocks_for(u64 n, unsigned bs) { return (unsigned)((n + bs - 1) / bs); }

cudaError_t launch_indirect(const StaticTables& T, u32 num_effects, cudaStream_t st) {
    if (num_effects == 0) return cudaSuccess;
    k_indirect<<<blocks_for(num_effects, 64), 64, 0, st>>>(T);
    if (T.num_child_infos) k_clear_events<<<blocks_for(num_effects, 64), 64, 0, st>>>(T);
    return cudaGetLastError();
}
cudaError_t launch_prefix_sum(const StaticTables& T, u32 num_batches, cudaStream_t st) {
    if (num_batches == 0) return cudaSuccess;
    k_prefix_sum<<<blocks_for(num_batches, 64), 64, 0, st>>>(T);
    return cudaGetLastError();
}
cudaError_t launch_tile_prefix(const StaticTables& T, u32 batch_index, u32 tile, cudaStream_t st) {
    k_tile_prefix<<<1, BK_THREADS, 0, st>>>(T, batch_index, tile);
    return cudaGetLastError();
}
// The frame block of a frame WITH an init pass: init reads the tables before the bookkeeping kernel runs, so the block gets a
// kernel of its own at the head of the frame (one CTA; the store happens after the dependency wait, like in k_bookkeeping).
template <int NW>
__global__ void __launch_bounds__(BK_THREADS) k_frame_block(u32* arena, const __grid_constant__ FrameBlock<NW> block, u32 block_words) {
    hnb_pdl_wait();
    hnb_pdl_launch_dependents();
    for (u32 i = threadIdx.x; i < block_words; i += BK_THREADS) arena[i] = block.w[i];
}
template <int NW>
static cudaError_t launch_frame_block_t(u32* arena, const u32* src, u32 words, cudaStream_t st) {
    FrameBlock<NW> blk;
    memcpy(blk.w, src, size_t(words) * 4);
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(1);
    cfg.blockDim = dim3(BK_THREADS);
    cfg.stream = st;
    cudaLaunchAttribute attr{};
    attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr.val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, k_frame_block<NW>, arena, blk, words);
}
cudaError_t launch_frame_block(void* device_arena, const void* frame_block, u32 block_bytes, cudaStream_t st) {
    if (!frame_block || block_bytes == 0 || (block_bytes & 3u) || block_bytes > HNB_FRAME_BLOCK_MAX_BYTES) return cudaErrorInvalidValue;
    const u32 words = block_bytes / 4u;
    if (words <= 64u) return launch_frame_block_t<64>((u32*)device_arena, (const u32*)frame_block, words, st);
    if (words <= HNB_FRAME_BLOCK_MID_BYTES / 4u) return launch_frame_block_t<HNB_FRAME_BLOCK_MID_BYTES / 4>((u32*)device_arena, (const u32*)frame_block, words, st);
    return launch_frame_block_t<HNB_FRAME_BLOCK_MAX_BYTES / 4>((u32*)device_arena, (const u32*)frame_block, words, st);
}

template <int NW>
static cudaError_t launch_bookkeeping_t(const StaticTables& T, u32 num_batches, const u32* block_words_src, u32 block_words, cudaStream_t st) {
    FrameBlock<NW> blk;
    if (block_words) memcpy(blk.w, block_words_src, size_t(block_words) * 4);
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(num_batches);
    cfg.blockDim = dim3(BK_THREADS);
    cfg.stream = st;
    cudaLaunchAttribute attr{};
    attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr.val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, k_bookkeeping<NW>, T, blk, block_words);
}
cudaError_t launch_bookkeeping(const StaticTables& T, u32 num_effects, u32 num_batches, const void* frame_block, u32 block_bytes, cudaStream_t st) {
    if (num_batches == 0) return cudaSuccess;
    if (block_bytes & 3u) return cudaErrorInvalidValue;
    const u32 words = frame_block ? block_bytes / 4u : 0u;
    cudaError_t e;
    if (words <= BK_HEADER_WORDS) e = launch_bookkeeping_t<int(sizeof(FrameHeader) / 4)>(T, num_batches, (const u32*)frame_block, words, st);
    else if (words <= 64u) e = launch_bookkeeping_t<64>(T, num_batches, (const u32*)frame_block, words, st);
    else if (words <= HNB_FRAME_BLOCK_MID_BYTES / 4u) e = launch_bookkeeping_t<HNB_FRAME_BLOCK_MID_BYTES / 4>(T, num_batches, (const u32*)frame_block, words, st);
    else if (words <= HNB_FRAME_BLOCK_MAX_BYTES / 4u) e = launch_bookkeeping_t<HNB_FRAME_BLOCK_MAX_BYTES / 4>(T, num_batches, (const u32*)frame_block, words, st);
    else return cudaErrorInvalidValue;
    if (e != cudaSuccess) return e;
    if (T.num_child_infos) k_clear_events<<<blocks_for(num_effects, 64), 64, 0, st>>>(T);
    return cudaGetLastError();
}
cudaError_t launch_ordered_event_append(const EventAppendArgs& a, u32 capacity_rows, cudaStream_t st) {
    const u32 blocks = (capacity_rows + EV_ROWS_PER_BLOCK - 1) / EV_ROWS_PER_BLOCK;
    if (blocks == 0) return cudaSuccess;
    k_events_block_sums<<<blocks, EV_THREADS, 0, st>>>(a);
    k_events_scan_blocks<<<1, EV_THREADS, 0, st>>>(a, blocks);
    k_events_write<<<blocks, EV_THREADS, 0, st>>>(a);
    return cudaGetLastError();
}
cudaError_t launch_fill_dispatch_args(const u32* src, u32* dst, u32 src_offset, u32 src_stride, u32 dst_offset,
                                      u32 dst_stride, u32 count, cudaStream_t st) {
    if (count == 0) return cudaSuccess;
    k_fill_dispatch_args<<<blocks_for(count, 64), 64, 0, st>>>(src, dst, src_offset, src_stride, dst_offset, dst_stride, count);
    return cudaGetLastError();
}
cudaError_t launch_slab_reset(u32* ping, u32* pong, u32* dead, u32 first, u32 count, cudaStream_t st) {
    if (count == 0) return cudaSuccess;
    k_slab_reset<<<blocks_for(count, 256), 256, 0, st>>>(ping, pong, dead, first, count);
    return cudaGetLastError();
}
cudaError_t launch_bits_range(u32* bits, u32 first, u32 count, bool set, cudaStream_t st) {
    if (count == 0) return cudaSuccess;
    const u32 words = u32(((u64(first) + count + 31u) >> 5u) - (first >> 5u));
    k_bits_range<<<blocks_for(words, 256), 256, 0, st>>>(bits, first, count, set ? 1u : 0u);
    return cudaGetLastError();
}
cudaError_t launch_bits_from_list(u32* bits, const u32* list, u32 base, u32 alive_count, cudaStream_t st) {
    if (alive_count == 0) return cudaSuccess;
    k_bits_from_list<<<blocks_for(alive_count, 256), 256, 0, st>>>(bits, list, base, alive_count);
    return cudaGetLastError();
}
cudaError_t launch_fill_c5(void* pos_age, void* vel_life, u32* ping, u32* pong, u64* claim, u32 first, u32 count, u32 seed, f32 lo, f32 hi, u32 logical_first, cudaStream_t st) {
    if (count == 0) return cudaSuccess;
    k_fill_c5<<<blocks_for(count, 256), 256, 0, st>>>((float4*)pos_age, (float4*)vel_life, ping, pong, claim, first, count, seed, lo, hi, logical_first);
    return cudaGetLastError();
}
cudaError_t launch_repack_gather(const RepackArgs& a, const void* col, void* scratch, u32 width, cudaStream_t st) {
    if (a.rows == 0) return cudaSuccess;
    const unsigned blocks = blocks_for(a.rows, RP_ROWS_PER_BLOCK);
    switch (width) {
    case 4: k_repack_gather<1><<<blocks, RP_THREADS, 0, st>>>(a, (const RepackPiece<1>*)col, (RepackPiece<1>*)scratch); break;
    case 8: k_repack_gather<2><<<blocks, RP_THREADS, 0, st>>>(a, (const RepackPiece<2>*)col, (RepackPiece<2>*)scratch); break;
    case 16: k_repack_gather<4><<<blocks, RP_THREADS, 0, st>>>(a, (const RepackPiece<4>*)col, (RepackPiece<4>*)scratch); break;
    case 32: k_repack_gather<8><<<blocks, RP_THREADS, 0, st>>>(a, (const RepackPiece<8>*)col, (RepackPiece<8>*)scratch); break;
    default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}
cudaError_t launch_repack_lists(const RepackArgs& a, cudaStream_t st) {
    if (a.rows == 0) return cudaSuccess;
    k_repack_lists<<<blocks_for(a.rows, RP_THREADS), RP_THREADS, 0, st>>>(a);
    return cudaGetLastError();
}
cudaError_t launch_snapshot_gather(const SnapshotArgs& a, u32* dst, cudaStream_t st) {
    if (a.rows == 0) return cudaSuccess;
    k_snapshot_gather<<<blocks_for(a.rows, RP_ROWS_PER_BLOCK), RP_THREADS, 0, st>>>(a, dst);
    return cudaGetLastError();
}
cudaError_t launch_restore_scatter(const SnapshotArgs& a, const u32* src, cudaStream_t st) {
    if (a.rows == 0) return cudaSuccess;
    k_restore_scatter<<<blocks_for(a.rows, RP_ROWS_PER_BLOCK), RP_THREADS, 0, st>>>(a, src);
    return cudaGetLastError();
}
cudaError_t launch_measure_sm_clock(u64* out2, u64 window_ns, cudaStream_t st) {
    k_measure_sm_clock<<<1, 1, 0, st>>>(out2, window_ns);
    return cudaGetLastError();
}
cudaError_t launch_checksum(const PlaneSet& planes, u32 first, u32 count, u32 stride_words, u64 index_base, u64* out, cudaStream_t st) {
    if (count == 0) return cudaSuccess;
    k_checksum<<<132 * 4, 256, 0, st>>>(planes, first, count, stride_words, index_base, out);
    return cudaGetLastError();
}

}  // namespace hnb
