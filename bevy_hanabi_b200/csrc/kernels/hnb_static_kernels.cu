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
// Common ages of a slab's 32-row groups [g0, g0 + groups) (DESIGN.md §3), one thread per group. A deferred word's age goes
// back into record word `age_word` of all 32 rows of its group (rows past `capacity` excepted), wherever the column plan
// keeps it: the warp writes the rows of its deferred groups one group at a time, one row per lane. Then, with `clear` (for
// writers of records), every word of the range and its lifetime floor become the sentinel; without (for readers), a
// deferred word becomes the word known at `epoch`, and every other word stays.
__global__ void k_flush_group_ages(PlaneSet planes, u32 age_word, u64* group_age, u32* life_floor, u32 g0, u32 groups, u32 capacity,
                                   u32 clear, u32 epoch) {
    const u32 t = blockIdx.x * blockDim.x + threadIdx.x, lane = threadIdx.x & 31u;
    const bool mine = t < groups;
    const u32 g = g0 + t;
    const u64 word = mine ? group_age[g] : HNB_GROUP_AGE_NONE;
    const bool deferred = hnb_group_age_deferred(word);
    const u32 p = planes.word_to_plane[age_word], wl = hnb_word_lane(planes, age_word);
    const u32 deferred_mask = __ballot_sync(0xffffffffu, deferred);
    if (lane == 0u && deferred_mask != 0u)  // every deferred word of the range stops being deferred below
        atomicAdd((unsigned long long*)hnb_deferred_groups(group_age, capacity), 0ull - u64(__popc(deferred_mask)));
    for (u32 pending = deferred_mask; pending; pending &= pending - 1u) {
        const int src = __ffs(pending) - 1;
        const u32 row = __shfl_sync(0xffffffffu, g, src) * 32u + lane;
        const u32 age = __shfl_sync(0xffffffffu, u32(word), src);
        if (row < capacity) ((u32*)planes.ptr[p])[u64(row) * planes.words[p] + wl] = age;
    }
    if (!mine) return;
    if (clear) {
        group_age[g] = HNB_GROUP_AGE_NONE;
        life_floor[g] = HNB_LIFE_FLOOR_NONE;
    } else if (deferred) {
        group_age[g] = (u64(epoch) << 32) | u32(word);
    }
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
// The eight record words go to whatever columns the slab's plan gives them.
__global__ void k_fill_c5(PlaneSet planes, u32* ping, u32* pong, u64* claim, u32 first, u32 count, u32 seed,
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
    const f32 rec[8] = {v[0] * 2.0f - 1.0f, v[1] * 2.0f - 1.0f, v[2] * 2.0f - 1.0f, 0.0f,
                        v[3] * 2.0f - 1.0f, v[4] * 2.0f - 1.0f, v[5] * 2.0f - 1.0f, lifetime_lo + v[6] * (lifetime_hi - lifetime_lo)};
#pragma unroll
    for (u32 w = 0; w < 8; ++w) {
        const u32 p = planes.word_to_plane[w];
        ((f32*)planes.ptr[p])[u64(row) * planes.words[p] + hnb_word_lane(planes, w)] = rec[w];
    }
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
        u32* d = dst + HNB_SNAPSHOT_HEADER_WORDS + u64(i) * a.stride_words;
        if (off & HNB_PLANE_WORD_LIST) {  // a word map: each lane to its own record word
#pragma unroll
            for (u32 l = 0; l < W; ++l) d[hnb_plane_word(a.planes, p, l)] = v[k].w[l];
            continue;
        }
        d += off;
        if (W >= 4 && al == 4u) snapshot_store<4>(d, v[k]);
        else if (W >= 2 && al >= 2u) snapshot_store<2>(d, v[k]);
        else snapshot_store<1>(d, v[k]);
    }
}

// D of an emitting instance: the slots its last update freed sit at dead-stack positions n .. n+D of its slice
// (deaths are pushed to dead[max_update-1-rank]), and a pending OnDie event may name any of them.
__device__ __forceinline__ u32 last_dead_count(const EffectMetadata* md, u32 n, u32 rows) {
    const u32 updated = md->max_update;
    return updated > n ? min(updated - n, rows - n) : 0u;
}

// Header by the first 16 threads, then record i < n = min(alive_count, rows) from local row list_W[i] (clamped to the
// slice as repack_source clamps it). Reads nothing but the metadata row, column W and the planes. DEAD (version 2): the
// header names version 2 and D in word 6, and records n .. n+D come from local rows dead[first+i] - first.
template <bool DEAD>
__device__ __forceinline__ void snapshot_gather(const SnapshotArgs& a, const u32* dead, u32* dst) {
    const EffectMetadata* md = a.metadata;
    const u32 n = min(md->alive_count, a.rows);
    const u32 d = DEAD ? last_dead_count(md, n, a.rows) : 0u;
    if (blockIdx.x == 0u && threadIdx.x < HNB_SNAPSHOT_HEADER_WORDS) {
        const u32 t = threadIdx.x;
        dst[t] = t == 0u ? HNB_SNAPSHOT_MAGIC_WORD
               : t == 1u ? (DEAD ? HNB_SNAPSHOT_EVENTS_VERSION_WORD : HNB_SNAPSHOT_VERSION_WORD)
               : t == 2u ? a.stride_words * 4u
               : t == 3u ? n
               : t == 4u ? md->particle_counter
               : t == 5u ? a.rows
               : t == 6u ? d
               : 0u;
    }
    const u32* list = md->indirect_write_index == 0u ? a.ping : a.pong;
    const u32 i0 = blockIdx.x * RP_ROWS_PER_BLOCK + threadIdx.x;
    if (i0 >= n + d) return;
    u32 src[RP_ITEMS];
#pragma unroll
    for (u32 k = 0; k < RP_ITEMS; ++k) {
        const u32 i = i0 + k * RP_THREADS;
        src[k] = i < n ? min(list[a.first + i], a.rows - 1u) : (DEAD && i < n + d) ? min(dead[a.first + i] - a.first, a.rows - 1u) : 0u;
    }
    for (u32 p = 0; p < a.num_planes; ++p) {
        switch (a.planes.words[p]) {
        case 1: snapshot_column<1>(a, p, src, i0, n + d, dst); break;
        case 2: snapshot_column<2>(a, p, src, i0, n + d, dst); break;
        case 4: snapshot_column<4>(a, p, src, i0, n + d, dst); break;
        default: snapshot_column<8>(a, p, src, i0, n + d, dst); break;
        }
    }
}
__global__ void __launch_bounds__(RP_THREADS) k_snapshot_gather(SnapshotArgs a, u32* dst) { snapshot_gather<false>(a, nullptr, dst); }
// version 2: words 7-15 of the header and the events follow from k_events_translate
__global__ void __launch_bounds__(RP_THREADS) k_snapshot_gather_dead(SnapshotArgs a, const u32* dead, u32* dst) { snapshot_gather<true>(a, dead, dst); }

// m = min(count, rows, records the buffer holds); 0 for a header that is not a version-1 snapshot of this stride
__device__ __forceinline__ u32 restore_count(const SnapshotArgs& a, const u32* src) {
    if (src[0] != HNB_SNAPSHOT_MAGIC_WORD || src[1] != HNB_SNAPSHOT_VERSION_WORD || src[2] != a.stride_words * 4u) return 0u;
    const u64 fit = (a.src_bytes - HNB_SNAPSHOT_HEADER_WORDS * 4u) / (a.stride_words * 4u);
    const u64 m = src[3] < a.rows ? src[3] : a.rows;
    return u32(m < fit ? m : fit);
}

// What a restore takes from a version-2 snapshot: live records [0, m) to rows [0, m) and dead records [n, n+dm) to rows
// [m, m+dm), with m = min(n, rows, records the buffer holds) and dm = min(D, rows - m, dead records the buffer holds).
// All zero for a header that is not a version-2 snapshot of this stride with `channels` event channels.
struct RestoreSpan {
    u32 n, d, m, dm;
    bool ok;
};
__device__ __forceinline__ RestoreSpan restore_span(const SnapshotArgs& a, const u32* src, u32 channels) {
    RestoreSpan s{0u, 0u, 0u, 0u, false};
    if (src[0] != HNB_SNAPSHOT_MAGIC_WORD || src[1] != HNB_SNAPSHOT_EVENTS_VERSION_WORD || src[2] != a.stride_words * 4u ||
        src[7] != channels)
        return s;
    s.ok = true;
    s.n = src[3];
    s.d = src[6];
    const u64 fit = (a.src_bytes - HNB_SNAPSHOT_HEADER_WORDS * 4u) / (a.stride_words * 4u);
    const u64 m = s.n < a.rows ? s.n : a.rows;
    s.m = u32(m < fit ? m : fit);
    const u64 dead_fit = fit > s.n ? fit - s.n : 0u;
    const u64 dm = s.d < a.rows - s.m ? s.d : a.rows - s.m;
    s.dm = u32(dm < dead_fit ? dm : dead_fit);
    return s;
}

// column p's piece of record r of the snapshot at `src`; `al` = snapshot_align(stride_words, word_off[p])
template <int W>
__device__ __forceinline__ void snapshot_piece(const SnapshotArgs& a, u32 p, u32 off, u32 al, const u32* src, u32 r, RepackPiece<W>& v) {
    const u32* s = src + HNB_SNAPSHOT_HEADER_WORDS + u64(r) * a.stride_words;
    if (off & HNB_PLANE_WORD_LIST) {  // a word map: each lane from its own record word
#pragma unroll
        for (u32 l = 0; l < W; ++l) v.w[l] = s[hnb_plane_word(a.planes, p, l)];
        return;
    }
    s += off;
    if (W >= 4 && al == 4u) snapshot_load<4>(s, v);
    else if (W >= 2 && al >= 2u) snapshot_load<2>(s, v);
    else snapshot_load<1>(s, v);
}

// rows i0 + k * RP_THREADS < m + dm of column p from records i (i < m) and n + i - m (the dead records)
template <int W>
__device__ __forceinline__ void restore_column(const SnapshotArgs& a, u32 p, u32 i0, u32 m, u32 dm, u32 n, const u32* src) {
    RepackPiece<W>* col = (RepackPiece<W>*)a.planes.ptr[p] + a.first;
    const u32 off = a.planes.word_off[p], al = snapshot_align(a.stride_words, off);
    RepackPiece<W> v[RP_ITEMS];
#pragma unroll
    for (u32 k = 0; k < RP_ITEMS; ++k) {
        const u32 i = i0 + k * RP_THREADS;
        if (i >= m + dm) continue;
        snapshot_piece<W>(a, p, off, al, src, i < m ? i : n + (i - m), v[k]);
    }
#pragma unroll
    for (u32 k = 0; k < RP_ITEMS; ++k)
        if (i0 + k * RP_THREADS < m + dm) col[i0 + k * RP_THREADS] = v[k];
}

// Record i < m -> local row i of every column; thread 0 writes alive_count = m, max_spawn = capacity - m (0 if the row's
// capacity is below m) and, for an accepted header, particle_counter. k_repack_lists follows and reads m back.
// DEAD (version 2): also dead record n + j -> row m + j for j < dm, and max_update = m + dm.
template <bool DEAD>
__device__ __forceinline__ void restore_scatter(const SnapshotArgs& a, const u32* src, u32 channels) {
    u32 m, dm = 0u, n = 0u;
    bool ok;
    if (DEAD) {
        const RestoreSpan s = restore_span(a, src, channels);
        m = s.m; dm = s.dm; n = s.n; ok = s.ok;
    } else {
        m = restore_count(a, src);
        ok = src[0] == HNB_SNAPSHOT_MAGIC_WORD && src[1] == HNB_SNAPSHOT_VERSION_WORD && src[2] == a.stride_words * 4u;
    }
    const u32 i0 = blockIdx.x * RP_ROWS_PER_BLOCK + threadIdx.x;
    if (i0 == 0u) {
        EffectMetadata* md = a.metadata;
        md->alive_count = m;
        md->max_spawn = md->capacity > m ? md->capacity - m : 0u;
        if (ok) md->particle_counter = src[4];
        if (DEAD) md->max_update = m + dm;
    }
    if (i0 >= m + dm) return;
    for (u32 p = 0; p < a.num_planes; ++p) {
        switch (a.planes.words[p]) {
        case 1: restore_column<1>(a, p, i0, m, dm, n, src); break;
        case 2: restore_column<2>(a, p, i0, m, dm, n, src); break;
        case 4: restore_column<4>(a, p, i0, m, dm, n, src); break;
        default: restore_column<8>(a, p, i0, m, dm, n, src); break;
        }
    }
}
__global__ void __launch_bounds__(RP_THREADS) k_restore_scatter(SnapshotArgs a, const u32* src) { restore_scatter<false>(a, src, 0u); }
__global__ void __launch_bounds__(RP_THREADS) k_restore_scatter_dead(SnapshotArgs a, const u32* src, u32 channels) {
    restore_scatter<true>(a, src, channels);
}

// ---------------------------------------------------------------------------------------------
// Append to one instance (hnb_instance_append): record k < m takes the slot the k-th spawn of an init would take,
// s_k = dead[first + n + k] - first, with m = min(count, max_spawn, rows - n, records the buffer holds) and n =
// min(alive_count, rows). The scatter reads n and max_spawn, so the metadata words and the claim cut follow in a second
// launch (k_append_commit).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ u32 append_count(const AppendArgs& a, const u32* src, u32 n) {
    return min(min(restore_count(a.s, src), a.s.metadata->max_spawn), a.s.rows - n);
}

// records i0 + k * RP_THREADS < m of column p -> local rows slot[k]
template <int W>
__device__ __forceinline__ void append_column(const SnapshotArgs& a, u32 p, const u32 (&slot)[RP_ITEMS], u32 i0, u32 m, const u32* src) {
    RepackPiece<W>* col = (RepackPiece<W>*)a.planes.ptr[p] + a.first;
    const u32 off = a.planes.word_off[p], al = snapshot_align(a.stride_words, off);
    RepackPiece<W> v[RP_ITEMS];
#pragma unroll
    for (u32 k = 0; k < RP_ITEMS; ++k)
        if (i0 + k * RP_THREADS < m) snapshot_piece<W>(a, p, off, al, src, i0 + k * RP_THREADS, v[k]);
#pragma unroll
    for (u32 k = 0; k < RP_ITEMS; ++k)
        if (i0 + k * RP_THREADS < m) col[slot[k]] = v[k];
}

// What the store half of an init does for each appended record (hnb_particle_kernels.cuh, hnb_init): the record in every
// column, list_W[first + n + k] = s_k, the alive bit (slot order) and the slot's group words the sentinel.
__global__ void __launch_bounds__(RP_THREADS) k_append_scatter(AppendArgs a, const u32* src) {
    const EffectMetadata* md = a.s.metadata;
    const u32 n = min(md->alive_count, a.s.rows);
    const u32 m = append_count(a, src, n);
    const u32 i0 = blockIdx.x * RP_ROWS_PER_BLOCK + threadIdx.x;
    if (i0 >= m) return;
    const u32 base = a.s.first;
    u32 slot[RP_ITEMS];
#pragma unroll
    for (u32 k = 0; k < RP_ITEMS; ++k) {
        const u32 i = i0 + k * RP_THREADS;
        slot[k] = i < m ? min(a.dead[base + n + i] - base, a.s.rows - 1u) : 0u;  // clamped as repack_source
    }
    for (u32 p = 0; p < a.s.num_planes; ++p) {
        switch (a.s.planes.words[p]) {
        case 1: append_column<1>(a.s, p, slot, i0, m, src); break;
        case 2: append_column<2>(a.s, p, slot, i0, m, src); break;
        case 4: append_column<4>(a.s, p, slot, i0, m, src); break;
        default: append_column<8>(a.s, p, slot, i0, m, src); break;
        }
    }
    u32* list = md->indirect_write_index == 0u ? a.ping : a.pong;
#pragma unroll
    for (u32 k = 0; k < RP_ITEMS; ++k) {
        const u32 i = i0 + k * RP_THREADS;
        if (i >= m) continue;
        const u32 row = base + slot[k];
        list[base + n + i] = slot[k];
        if (a.alive_bits) atomicOr(&a.alive_bits[row >> 5u], 1u << (row & 31u));
        // the slot's lifetime and age changed: its group's floor and common age prove nothing until an update stores them
        a.life_floor[row >> 5u] = HNB_LIFE_FLOOR_NONE;
        a.group_age[row >> 5u] = HNB_GROUP_AGE_NONE;
    }
}

// After the scatter: alive_count = n + m, max_spawn -= m, particle_counter += m, and the identity claim of column W cut to
// n (the first appended row ends what it can cover). Nothing for m = 0.
__global__ void k_append_commit(AppendArgs a, const u32* src) {
    EffectMetadata* md = a.s.metadata;
    const u32 n = min(md->alive_count, a.s.rows);
    const u32 m = append_count(a, src, n);
    if (m == 0u) return;
    md->alive_count = n + m;
    md->max_spawn -= m;
    md->particle_counter += m;
    u64* const claim = &a.claim[md->indirect_write_index];
    if (hnb_claim_len(hnb_claim_load(claim), a.s.first) > n) hnb_claim_store(claim, hnb_claim_pack(a.s.first, n));
}

// ---------------------------------------------------------------------------------------------
// Pending GPU spawn events of an emitting instance (hnb_slab_repack_events, hnb_instance_snapshot_events,
// hnb_instance_restore_events). Between frames an event is an instance-local parent slot: a live slot or one of the D
// slots the last update freed. The repack and the snapshot move slot src[i] to row / record i, so both translate an event
// through inv[src[i]] = i.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ ChildInfo* channel_info(const EventChannels& ev, const EffectMetadata* md, u32 b) {
    const u64 row = u64(md->base_child_index) + b;
    return row < ev.num_child_infos ? &ev.child_infos[row] : nullptr;
}
// entries of channel b that hold an event: min(event_count, capacity)
__device__ __forceinline__ u32 channel_stored(const EventChannels& ev, const EffectMetadata* md, u32 b) {
    const ChildInfo* ci = channel_info(ev, md, b);
    return ci ? min(u32(ci->event_count), ev.capacity[b]) : 0u;
}

// inv[src[i]] = i over the slice; before k_repack_lists, which rewrites the lists
__global__ void __launch_bounds__(RP_THREADS) k_repack_inverse(RepackArgs a, u32* inv) {
    const u32 n = min(a.metadata->alive_count, a.rows);
    const u32* list = a.metadata->indirect_write_index == 0u ? a.ping : a.pong;
    const u32 i = blockIdx.x * RP_THREADS + threadIdx.x;
    if (i < a.rows) inv[repack_source(a, list, n, i)] = i;
}

// Entry k of channel b = blockIdx.x / blocks_per_channel. `snapshot` NULL (repack): e -> inv[e] in place. Otherwise the
// entry goes to the snapshot as the record index inv[e], or 0xFFFFFFFF when that is not below n + D, after the channels
// before it; block 0 writes header words 7-15. Clamped to the slice, like repack_source.
__global__ void __launch_bounds__(RP_THREADS) k_events_translate(RepackArgs a, const u32* inv, EventChannels ev, u32 blocks_per_channel,
                                                                 u32 stride_words, u32* snapshot) {
    const EffectMetadata* md = a.metadata;
    const u32 b = blockIdx.x / blocks_per_channel;
    const u32 k = (blockIdx.x % blocks_per_channel) * RP_THREADS + threadIdx.x;
    const u32 stored = channel_stored(ev, md, b);
    if (!snapshot) {
        if (k < stored) ev.buffer[b][k] = min(inv[min(ev.buffer[b][k], a.rows - 1u)], a.rows - 1u);
        return;
    }
    const u32 n = min(md->alive_count, a.rows);
    const u32 records = n + last_dead_count(md, n, a.rows);
    if (blockIdx.x == 0u && threadIdx.x < 1u + 2u * HNB_MAX_EVENT_BINDINGS) {
        const u32 t = threadIdx.x, c = (t - 1u) % HNB_MAX_EVENT_BINDINGS;
        const ChildInfo* ci = c < ev.count ? channel_info(ev, md, c) : nullptr;
        snapshot[7u + t] = t == 0u ? ev.count
                         : t <= HNB_MAX_EVENT_BINDINGS ? (ci ? u32(ci->event_count) : 0u)
                         : (c < ev.count ? channel_stored(ev, md, c) : 0u);
    }
    if (k >= stored) return;
    u64 off = HNB_SNAPSHOT_HEADER_WORDS + u64(records) * stride_words;
    for (u32 c = 0; c < b; ++c) off += channel_stored(ev, md, c);
    const u32 r = inv[min(ev.buffer[b][k], a.rows - 1u)];
    snapshot[off + k] = r < records ? r : 0xFFFFFFFFu;
}

// Order-independent checksum: sum over rows of a 64-bit mix of the row's AoS words and row index.
__global__ void k_checksum(PlaneSet planes, u32 first, u32 count, u32 stride_words, u64 index_base, u64* out) {
    u64 acc = 0;
    for (u64 i = u64(blockIdx.x) * blockDim.x + threadIdx.x; i < count; i += u64(gridDim.x) * blockDim.x) {
        u64 h = 0xcbf29ce484222325ull ^ (index_base + u64(i));
        for (u32 w = 0; w < stride_words; ++w) {
            const u32 p = planes.word_to_plane[w];
            const u32 x = ((const u32*)planes.ptr[p])[u64(first + i) * planes.words[p] + hnb_word_lane(planes, w)];
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

// CTA b compacts channel b of a version-2 snapshot into its buffer: record index r -> row r (r < m) or m + r - n
// (n <= r < n + dm), any other entry dropped, as is every entry past the capacity; order kept. event_count becomes the
// stored unclamped count minus the dropped entries (0 for a rejected header). Reads nothing past src_bytes.
__global__ void __launch_bounds__(EV_THREADS) k_restore_events(SnapshotArgs a, const u32* src, EventChannels ev) {
    __shared__ u32 s_warp[EV_THREADS / 32];
    __shared__ u32 s_carry;
    const u32 b = blockIdx.x;
    const RestoreSpan s = restore_span(a, src, ev.count);
    ChildInfo* ci = channel_info(ev, a.metadata, b);
    if (!s.ok) {
        if (threadIdx.x == 0u && ci) ci->event_count = 0;
        return;
    }
    const u32 unclamped = src[8u + b], stored = src[12u + b], cap = ev.capacity[b];
    u64 off = HNB_SNAPSHOT_HEADER_WORDS + (u64(s.n) + s.d) * a.stride_words;
    for (u32 c = 0; c < b; ++c) off += src[12u + c];
    const u64 words = a.src_bytes / 4u;
    const u32 readable = off < words ? (words - off < stored ? u32(words - off) : stored) : 0u;
    if (threadIdx.x == 0u) s_carry = 0u;
    __syncthreads();
    for (u32 k0 = 0; k0 < readable; k0 += EV_THREADS) {
        const u32 carry = s_carry;
        if (carry >= cap) break;  // uniform: every thread read s_carry after the same barrier
        const u32 k = k0 + threadIdx.x;
        u32 row = 0xFFFFFFFFu;
        if (k < readable) {
            const u32 r = src[off + k];
            if (r < s.m) row = r;
            else if (r >= s.n && r - s.n < s.dm) row = s.m + (r - s.n);
        }
        u32 total;
        const u32 pos = carry + ev_block_exclusive_scan(row != 0xFFFFFFFFu ? 1u : 0u, s_warp, &total);
        if (row != 0xFFFFFFFFu && pos < cap) ev.buffer[b][pos] = row;
        if (threadIdx.x == 0u) s_carry = carry + total;
        __syncthreads();
    }
    if (threadIdx.x == 0u && ci) {
        const u32 dropped = stored - min(s_carry, cap);
        ci->event_count = i32(unclamped >= dropped ? unclamped - dropped : 0u);
    }
}

// ---------------------------------------------------------------------------------------------
// Bounds of every instance of a batch (hnb_batch_bounds): a pure read of the `position` column(s). One persistent launch
// reduces all instances, one small launch writes the records.
//
// Floats are compared through the usual order-preserving key (bounds_key), so -0 < +0, the infinities take part and the
// result is the same whatever the order of the reduction. A NaN is skipped. Every partial result is kept as a MAXIMUM:
// `hi` of the keys and `lo` of the inverted keys. No float has key 0 or 0xFFFFFFFF (those bit patterns are NaNs), so 0
// means "no value" in both, and an accumulator of zeroes is the reset state.
// ---------------------------------------------------------------------------------------------
#define BD_THREADS 256
#define BD_ITEMS 4  // rows per thread in flight (as RP_ITEMS)
#define BD_TILE (BD_THREADS * BD_ITEMS)

__device__ __forceinline__ u32 bounds_key(u32 bits) { return bits ^ ((bits >> 31u) ? 0xFFFFFFFFu : 0x80000000u); }
__device__ __forceinline__ u32 bounds_bits(u32 key) { return key ^ ((key >> 31u) ? 0x80000000u : 0xFFFFFFFFu); }

struct BoundsAcc { u32 lo[3], hi[3]; };
__device__ __forceinline__ void bounds_take(BoundsAcc& r, int c, u32 bits) {
    if ((bits & 0x7FFFFFFFu) > 0x7F800000u) return;  // NaN
    const u32 k = bounds_key(bits);
    r.lo[c] = max(r.lo[c], ~k);
    r.hi[c] = max(r.hi[c], k);
}

// Instance j of the batch as the device tables of the last simulated frame describe it, every word clamped: the spawner
// and metadata rows to their tables, the slice to the slab, n = min(alive_count, rows) as hnb_instance_snapshot defines it.
struct BoundsInstance { u32 first, rows, n, w; };
__device__ __forceinline__ u32 bounds_count(const BoundsArgs& a) { return min(a.batch_info->prefix_sum_count, a.max_instances); }
__device__ __forceinline__ BoundsInstance bounds_instance(const BoundsArgs& a, u32 j) {
    const u64 row = u64(a.batch_info->spawner_base) + j;
    const Spawner* sp = &a.spawners[row < a.num_spawners ? row : a.num_spawners - 1u];
    const EffectMetadata* md = &a.metadata[min(sp->effect_metadata_index, a.num_metadata - 1u)];
    BoundsInstance b;
    b.first = min(sp->slab_offset, a.capacity_rows);
    b.rows = min(md->capacity, a.capacity_rows - b.first);
    b.n = min(md->alive_count, b.rows);
    b.w = md->indirect_write_index == 0u ? 0u : 1u;
    return b;
}

// Persistent grid. Every CTA walks the instances (their descriptions staged BD_THREADS at a time in shared memory, so the
// dependent table loads of 1024 instances cost four rounds, not 1024) and takes the tiles t with t + j = blockIdx (mod
// gridDim) of instance j: one 64 Mi-row instance and 1024 instances of 64 tiles both spread evenly, with no prefix of
// counts the host would have to know. Rows below the identity claim of column W take pidx = i without a list load; the
// slab's two claim words are read once per thread, they do not change under the kernel.
// FAST: position's three words sit in one 16-byte column, or in one half of a 32-byte sector-plane column: one 16-byte
// load per row. Otherwise one 4-byte load per word from whatever columns the plan gave them.
// Per (warp, instance) that had a tile: registers -> shuffles -> six atomicMax into the accumulator by lanes 0-5. The
// warps of a CTA never wait for one another inside a staging round, so one warp's gather overlaps another's reduction.
template <bool FAST>
__global__ void __launch_bounds__(BD_THREADS) k_bounds_reduce(BoundsArgs a) {
    __shared__ u32 s_first[BD_THREADS], s_rows[BD_THREADS], s_n[BD_THREADS], s_w[BD_THREADS];
    const u32 count = bounds_count(a);
    const u32 tid = threadIdx.x, lane = tid & 31u, G = gridDim.x;
    const u64 claim0 = hnb_claim_load(&a.claim[0]), claim1 = hnb_claim_load(&a.claim[1]);
    u32 rot = 0u;  // j mod G of the instance at hand
    for (u32 chunk = 0; chunk < count; chunk += BD_THREADS) {
        __syncthreads();
        if (chunk + tid < count) {
            const BoundsInstance b = bounds_instance(a, chunk + tid);
            s_first[tid] = b.first; s_rows[tid] = b.rows; s_n[tid] = b.n; s_w[tid] = b.w;
        }
        __syncthreads();
        const u32 staged = min(count - chunk, u32(BD_THREADS));
        for (u32 jj = 0; jj < staged; ++jj, rot = rot + 1u == G ? 0u : rot + 1u) {
            const u32 n = s_n[jj], tiles = (n + BD_TILE - 1u) / BD_TILE;
            u32 t = blockIdx.x >= rot ? blockIdx.x - rot : blockIdx.x + G - rot;
            if (t >= tiles) continue;
            const u32 first = s_first[jj], last_row = s_rows[jj] - 1u, w = s_w[jj];
            const u32* list = (w == 0u ? a.ping : a.pong) + first;
            const u32 claimed = min(hnb_claim_len(w == 0u ? claim0 : claim1, first), n);
            BoundsAcc r = {{0u, 0u, 0u}, {0u, 0u, 0u}};
            for (; t < tiles; t += G) {
                const u32 i0 = t * BD_TILE + tid;
                u32 p[BD_ITEMS];
#pragma unroll
                for (u32 k = 0; k < BD_ITEMS; ++k) {
                    const u32 i = i0 + k * BD_THREADS;
                    p[k] = i < claimed ? i : (i < n ? min(list[i], last_row) : 0u);
                }
                if (FAST) {
                    const RepackPiece<4>* col = (const RepackPiece<4>*)a.col[0];
                    const u32 quads = a.col_words[0] >> 2u, quad = a.col_lane[0] >> 2u;
                    RepackPiece<4> v[BD_ITEMS];
#pragma unroll
                    for (u32 k = 0; k < BD_ITEMS; ++k)
                        if (i0 + k * BD_THREADS < n) v[k] = col[(u64(first) + p[k]) * quads + quad];
#pragma unroll
                    for (u32 k = 0; k < BD_ITEMS; ++k) {
                        if (i0 + k * BD_THREADS >= n) continue;
#pragma unroll
                        for (int c = 0; c < 3; ++c) bounds_take(r, c, v[k].w[c]);
                    }
                } else {
                    u32 v[BD_ITEMS][3];
#pragma unroll
                    for (u32 k = 0; k < BD_ITEMS; ++k) {
                        if (i0 + k * BD_THREADS >= n) continue;
#pragma unroll
                        for (int c = 0; c < 3; ++c) v[k][c] = a.col[c][(u64(first) + p[k]) * a.col_words[c] + a.col_lane[c]];
                    }
#pragma unroll
                    for (u32 k = 0; k < BD_ITEMS; ++k) {
                        if (i0 + k * BD_THREADS >= n) continue;
#pragma unroll
                        for (int c = 0; c < 3; ++c) bounds_take(r, c, v[k][c]);
                    }
                }
            }
#pragma unroll
            for (int c = 0; c < 3; ++c) {
#pragma unroll
                for (int d = 16; d > 0; d >>= 1) {
                    r.lo[c] = max(r.lo[c], __shfl_xor_sync(0xffffffffu, r.lo[c], d));
                    r.hi[c] = max(r.hi[c], __shfl_xor_sync(0xffffffffu, r.hi[c], d));
                }
            }
            // every lane holds the warp's six maxima: lane s < 6 publishes slot s (0: a warp whose rows had no value)
            const u32 m = lane == 0u ? r.lo[0] : lane == 1u ? r.lo[1] : lane == 2u ? r.lo[2] : lane == 3u ? r.hi[0] : lane == 4u ? r.hi[1] : r.hi[2];
            if (lane < 6u && m) atomicMax(&a.acc[u64(chunk + jj) * 8u + (lane < 3u ? lane : lane + 1u)], u64(m));
        }
    }
}

// Record j of every instance the call covers (those past the batch's device-side count get an empty one), and the
// accumulator back to zeroes for the next call.
__global__ void __launch_bounds__(BD_THREADS) k_bounds_write(BoundsArgs a) {
    const u32 j = blockIdx.x * BD_THREADS + threadIdx.x;
    if (j >= a.max_instances) return;
    const u32 n = j < bounds_count(a) ? bounds_instance(a, j).n : 0u;
    u64* acc = a.acc + u64(j) * 8u;
    RepackPiece<4> lo, hi;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const u32 l = u32(acc[c]), h = u32(acc[4 + c]);
        lo.w[c] = l ? bounds_bits(~l) : 0x7F800000u;  // +inf: no value
        hi.w[c] = h ? bounds_bits(h) : 0xFF800000u;   // -inf
        acc[c] = 0ull;
        acc[4 + c] = 0ull;
    }
    lo.w[3] = n;
    hi.w[3] = 0u;
    RepackPiece<4>* out = (RepackPiece<4>*)a.out + u64(j) * 2u;
    out[0] = lo;
    out[1] = hi;
}

// ---------------------------------------------------------------------------------------------
// Draw order of every instance of a batch (hnb_batch_depth_order): the live entries of each instance sorted back to
// front by the depth of `position` against the instance's plane. A pure read of the instance, like bounds.
//
// Sort key: ~bounds_key(depth bits), and 0xFFFFFFFF for a NaN depth. Ascending keys are descending depths in bounds'
// total order; no non-NaN depth has key 0xFFFFFFFF (bounds_key 0 is the NaN 0xFFFFFFFF), so NaNs go last. Every sort
// below is stable and starts from the live entries in ascending i, so equal keys keep ascending i.
//
// Tiles of DO_TILE rows belong to one instance (tile t of instance j: rows [t*DO_TILE, (t+1)*DO_TILE) of its live list).
// Thirteen launches, whatever the batch holds:
//   k_do_plan      tiles per instance and their prefix over the batch (one CTA), digit totals zeroed (every CTA)
//   k_do_keys      per tile: entries, positions, keys. An instance of one tile is sorted whole in shared memory (four
//                  8-bit LSD passes) and written to the order; a larger one writes (key, entry) at its own slab rows of
//                  scratch buffer 0, the tile's digit-0 histogram, and the instance's totals of all four digits
//   4 x (k_do_scan, k_do_scatter), with k_do_hist before the scan of passes 1-3: an LSD pass over 8 bits. The scan
//                  makes the per-tile histograms exclusive offsets in (digit, tile) order, one warp per (instance,
//                  digit); the scatter ranks each tile's digits stably and moves its pairs to the other buffer, or
//                  writes the entries to the order in the instance's last pass that runs.
// A pass whose digit is the same for all n keys of an instance (one total equals n) does not run for it; an instance
// for which no pass runs has its scratch entries copied to the order by the last scatter.
// ---------------------------------------------------------------------------------------------
#define DO_THREADS 256  // also the number of digit values: thread d owns digit d in every histogram step
#define DO_WARPS (DO_THREADS / 32)
#define DO_ITEMS 16
#define DO_WARP_ROWS (32 * DO_ITEMS)
#define DO_TILE (DO_THREADS * DO_ITEMS)
#define DO_CTAS_PER_SM 4  // tile kernels loop over tiles: more CTAs than fit would only wait

// ((a*x + b*y) + c*z) + d, every step rounded on its own (no contraction).
#ifdef __CUDA_ARCH__
__device__ __forceinline__ float do_mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float do_add(float a, float b) { return __fadd_rn(a, b); }
#else
__device__ __forceinline__ float do_mul(float a, float b) { return a * b; }
__device__ __forceinline__ float do_add(float a, float b) { return a + b; }
#endif
__device__ __forceinline__ u32 depth_sort_key(const float* plane, u32 x, u32 y, u32 z) {
    const float depth = do_add(do_add(do_add(do_mul(plane[0], __uint_as_float(x)), do_mul(plane[1], __uint_as_float(y))),
                                      do_mul(plane[2], __uint_as_float(z))), plane[3]);
    const u32 bits = __float_as_uint(depth);
    return (bits & 0x7FFFFFFFu) > 0x7F800000u ? 0xFFFFFFFFu : ~bounds_key(bits);
}

// Instance j as the tile plan (do_tile_plan) recorded it in `info`: 8 words.
struct DepthInstance { u32 first, n, tile_base, tiles, w, rows, mask; };
__device__ __forceinline__ DepthInstance do_instance(const u32* info, u32 j) {
    const u32* in = info + u64(j) * 8u;
    return DepthInstance{in[0], in[1], in[2], in[3], in[4], in[5], in[6]};
}
// The instance that owns tile g of the call: the largest j with tile_base <= g (tile_base is non-decreasing in j, and
// instances without tiles share the base of the next one). The caller checks g - tile_base < tiles.
__device__ __forceinline__ u32 do_find(const u32* info, u32 count, u32 g) {
    u32 lo = 0u, hi = count - 1u;
    while (lo < hi) {
        const u32 mid = hi - (hi - lo) / 2u;
        if (info[u64(mid) * 8u + 2u] <= g) lo = mid;
        else hi = mid - 1u;
    }
    return lo;
}
// The buffer pass p reads: one flip per pass that ran before it.
__device__ __forceinline__ u32 do_src(u32 mask, u32 pass) { return __popc(mask & ((1u << pass) - 1u)) & 1u; }

// Stable rank of every item of a tile among the items of its digit. Item k of a warp is tile row
// warp * DO_WARP_ROWS + k * 32 + lane, so a warp ranks its items k = 0, 1, ... in turn with __match_any_sync, and the
// per-warp digit counts are then scanned in warp order. Digit 256 marks an item past the instance's end (no rank).
// On return rank[k] is the number of earlier items of the tile with the same digit, and s_tot[d] the tile's count of d.
__device__ __forceinline__ void do_rank(const u32 (&dig)[DO_ITEMS], u32 (&rank)[DO_ITEMS], u32* s_cnt, u32* s_tot) {
    const u32 tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    __syncthreads();  // the previous tile's readers of s_cnt are done
    for (u32 k = tid; k < DO_WARPS * 256u; k += DO_THREADS) s_cnt[k] = 0u;
    __syncthreads();
    u32* cnt = s_cnt + warp * 256u;
    const u32 lt = (1u << lane) - 1u;
#pragma unroll
    for (u32 k = 0; k < DO_ITEMS; ++k) {
        const u32 peers = __match_any_sync(0xffffffffu, dig[k]);
        const u32 before = dig[k] < 256u ? cnt[dig[k]] : 0u;
        rank[k] = before + __popc(peers & lt);
        __syncwarp();
        if (dig[k] < 256u && (peers & lt) == 0u) cnt[dig[k]] = before + __popc(peers);
        __syncwarp();
    }
    __syncthreads();
    u32 run = 0u;
    for (u32 w = 0; w < DO_WARPS; ++w) {
        const u32 c = s_cnt[w * 256u + tid];
        s_cnt[w * 256u + tid] = run;
        run += c;
    }
    s_tot[tid] = run;
    __syncthreads();
#pragma unroll
    for (u32 k = 0; k < DO_ITEMS; ++k)
        if (dig[k] < 256u) rank[k] += s_cnt[warp * 256u + dig[k]];
}

// Exclusive prefix of v over the CTA's threads in thread order.
__device__ __forceinline__ u32 do_block_exclusive(u32 v, u32* s_warp) {
    const u32 tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    u32 x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const u32 y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= u32(d)) x += y;
    }
    __syncthreads();  // s_warp of an earlier call is read
    if (lane == 31u) s_warp[warp] = x;
    __syncthreads();
    u32 before = 0u;
    for (u32 w = 0; w < warp; ++w) before += s_warp[w];
    return before + x - v;
}

// Tiles of DO_TILE rows per instance and their prefix over the batch, kept in `info` (8 words per instance) for the
// later launches of a call, and the call's tile count in `total_tiles`; run by one CTA of DO_THREADS threads. An instance
// whose tiles would pass `max_tiles` (only possible when the tables describe overlapping slices) gets none: it is not
// processed, and nothing outside the buffers is touched.
__device__ __forceinline__ void do_tile_plan(const BoundsArgs& src, u32* info, u32* total_tiles, u32 max_tiles, u32* s_warp) {
    const u32 count = bounds_count(src), tid = threadIdx.x;
    u64 carry = 0u;
    for (u32 chunk = 0; chunk < count; chunk += DO_THREADS) {
        const u32 j = chunk + tid;
        BoundsInstance b = {0u, 0u, 0u, 0u};
        if (j < count) b = bounds_instance(src, j);
        const u32 tiles = u32((u64(b.n) + DO_TILE - 1u) / DO_TILE);
        const u32 excl = do_block_exclusive(tiles, s_warp);
        const u64 base = carry + excl;
        if (j < count) {
            u32* in = info + u64(j) * 8u;
            const bool fits = base + tiles <= max_tiles;
            in[0] = b.first; in[1] = b.n; in[2] = u32(base < max_tiles ? base : max_tiles); in[3] = fits ? tiles : 0u;
            in[4] = b.w; in[5] = b.rows; in[6] = 0u; in[7] = 0u;
        }
        __syncthreads();
        if (tid == DO_THREADS - 1u) s_warp[0] = excl + tiles;
        __syncthreads();
        carry += s_warp[0];
    }
    if (tid == 0u) *total_tiles = u32(carry < max_tiles ? carry : max_tiles);
}

// The tile plan (CTA 0); the digit totals of the call's instances back to zero (every CTA).
__global__ void __launch_bounds__(DO_THREADS) k_do_plan(DepthOrderArgs a) {
    __shared__ u32 s_warp[DO_WARPS];
    const u32 count = bounds_count(a.src), tid = threadIdx.x;
    for (u64 k = u64(blockIdx.x) * DO_THREADS + tid; k < u64(count) * 1024u; k += u64(gridDim.x) * DO_THREADS) a.totals[k] = 0u;
    if (blockIdx.x != 0u) return;
    do_tile_plan(a.src, a.info, a.total_tiles, a.max_tiles, s_warp);
}

// Entry, position and key of every live row of the tile; rows below the identity claim of column W load no list entry.
template <bool FAST>
__device__ __forceinline__ void do_tile_keys(const DepthOrderArgs& a, const DepthInstance& in, u32 claimed, const float* plane,
                                             u32 i0, u32 (&key)[DO_ITEMS], u32 (&val)[DO_ITEMS]) {
    const BoundsArgs& s = a.src;
    const u32* list = (in.w == 0u ? s.ping : s.pong) + in.first;
    const u32 last_row = in.rows - 1u;
#pragma unroll
    for (u32 k = 0; k < DO_ITEMS; ++k) {
        const u32 i = i0 + k * 32u;
        val[k] = i < claimed ? i : (i < in.n ? min(list[i], last_row) : 0u);
    }
    if (FAST) {
        const RepackPiece<4>* col = (const RepackPiece<4>*)s.col[0];
        const u32 quads = s.col_words[0] >> 2u, quad = s.col_lane[0] >> 2u;
        RepackPiece<4> v[DO_ITEMS];
#pragma unroll
        for (u32 k = 0; k < DO_ITEMS; ++k)
            if (i0 + k * 32u < in.n) v[k] = col[(u64(in.first) + val[k]) * quads + quad];
#pragma unroll
        for (u32 k = 0; k < DO_ITEMS; ++k)
            key[k] = i0 + k * 32u < in.n ? depth_sort_key(plane, v[k].w[0], v[k].w[1], v[k].w[2]) : 0xFFFFFFFFu;
    } else {
        u32 v[DO_ITEMS][3];
#pragma unroll
        for (u32 k = 0; k < DO_ITEMS; ++k) {
            if (i0 + k * 32u >= in.n) continue;
#pragma unroll
            for (int c = 0; c < 3; ++c) v[k][c] = s.col[c][(u64(in.first) + val[k]) * s.col_words[c] + s.col_lane[c]];
        }
#pragma unroll
        for (u32 k = 0; k < DO_ITEMS; ++k)
            key[k] = i0 + k * 32u < in.n ? depth_sort_key(plane, v[k][0], v[k][1], v[k][2]) : 0xFFFFFFFFu;
    }
}

// Persistent grid over the call's tiles (the count is read from the plan). One-tile instances are sorted here whole;
// larger ones get their pairs, histograms and totals for the passes.
template <bool FAST>
__global__ void __launch_bounds__(DO_THREADS) k_do_keys(DepthOrderArgs a) {
    __shared__ u32 s_key[DO_TILE], s_val[DO_TILE];
    __shared__ u32 s_cnt[DO_WARPS * 256], s_tot[256], s_warp[DO_WARPS];
    const u32 count = bounds_count(a.src), total = *a.total_tiles, tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    const u64 claim0 = hnb_claim_load(&a.src.claim[0]), claim1 = hnb_claim_load(&a.src.claim[1]);
    for (u32 g = blockIdx.x; g < total; g += gridDim.x) {
        const u32 j = do_find(a.info, count, g);
        const DepthInstance in = do_instance(a.info, j);
        const u32 t = g - in.tile_base;
        if (t >= in.tiles) continue;  // CTA-uniform
        const u32 claimed = min(hnb_claim_len(in.w == 0u ? claim0 : claim1, in.first), in.n);
        const u32 r0 = warp * DO_WARP_ROWS + lane, i0 = t * DO_TILE + r0;
        u32 key[DO_ITEMS], val[DO_ITEMS];
        do_tile_keys<FAST>(a, in, claimed, a.planes + u64(j) * 4u, i0, key, val);
        if (in.tiles == 1u) {
            u32 dig[DO_ITEMS], rank[DO_ITEMS];
            for (u32 pass = 0; pass < 4u; ++pass) {
#pragma unroll
                for (u32 k = 0; k < DO_ITEMS; ++k) dig[k] = i0 + k * 32u < in.n ? (key[k] >> (8u * pass)) & 255u : 256u;
                do_rank(dig, rank, s_cnt, s_tot);
                const u32 base = do_block_exclusive(s_tot[tid], s_warp);
                __syncthreads();  // every thread has read s_tot
                s_tot[tid] = base;
                __syncthreads();
#pragma unroll
                for (u32 k = 0; k < DO_ITEMS; ++k) {
                    if (dig[k] >= 256u) continue;
                    const u32 r = s_tot[dig[k]] + rank[k];
                    s_key[r] = key[k];
                    s_val[r] = val[k];
                }
                __syncthreads();
#pragma unroll
                for (u32 k = 0; k < DO_ITEMS; ++k) {
                    if (r0 + k * 32u >= in.n) continue;
                    key[k] = s_key[r0 + k * 32u];
                    val[k] = s_val[r0 + k * 32u];
                }
            }
#pragma unroll
            for (u32 k = 0; k < DO_ITEMS; ++k)
                if (r0 + k * 32u < in.n) a.order[u64(in.first) + r0 + k * 32u] = val[k];
            continue;
        }
        __syncthreads();  // the previous tile's readers of s_cnt are done
        for (u32 k = tid; k < 4u * 256u; k += DO_THREADS) s_cnt[k] = 0u;
        __syncthreads();
#pragma unroll
        for (u32 k = 0; k < DO_ITEMS; ++k) {
            const u32 i = i0 + k * 32u;
            if (i >= in.n) continue;
            a.keys[0][u64(in.first) + i] = key[k];
            a.vals[0][u64(in.first) + i] = val[k];
#pragma unroll
            for (u32 p = 0; p < 4u; ++p) atomicAdd(&s_cnt[p * 256u + ((key[k] >> (8u * p)) & 255u)], 1u);
        }
        __syncthreads();
        a.hist[u64(in.tile_base) * 256u + u64(tid) * in.tiles + t] = s_cnt[tid];
#pragma unroll
        for (u32 p = 0; p < 4u; ++p)
            if (s_cnt[p * 256u + tid]) atomicAdd(&a.totals[u64(j) * 1024u + p * 256u + tid], s_cnt[p * 256u + tid]);
    }
}

// Pass `pass`, one warp per (instance, digit d): the row of tile counts of d becomes exclusive offsets into the
// instance's order, starting at the count of the smaller digits. Pass 0 also decides, from the totals, which passes run.
__global__ void __launch_bounds__(DO_THREADS) k_do_scan(DepthOrderArgs a, u32 pass) {
    const u32 lane = threadIdx.x & 31u;
    const u64 row = u64(blockIdx.x) * DO_WARPS + (threadIdx.x >> 5);
    const u32 count = bounds_count(a.src);
    if (row >= u64(count) * 256u) return;  // warp-uniform
    const u32 j = u32(row >> 8), d = u32(row & 255u);
    const DepthInstance in = do_instance(a.info, j);
    if (in.tiles < 2u) return;
    const u32* tot = a.totals + u64(j) * 1024u;
    u32 run;
    if (pass == 0u) {
        u32 mask = 0u;
        for (u32 p = 0; p < 4u; ++p) {
            bool constant = false;
#pragma unroll
            for (u32 q = 0; q < 8u; ++q) constant |= tot[p * 256u + q * 32u + lane] == in.n;
            if (__ballot_sync(0xffffffffu, constant) == 0u) mask |= 1u << p;
        }
        if (d == 0u && lane == 0u) a.info[u64(j) * 8u + 6u] = mask;
        run = mask & 1u;
    } else {
        run = (in.mask >> pass) & 1u;
    }
    if (!run) return;
    u32 base = 0u;
#pragma unroll
    for (u32 q = 0; q < 8u; ++q) {
        const u32 e = q * 32u + lane;
        if (e < d) base += tot[pass * 256u + e];
    }
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) base += __shfl_xor_sync(0xffffffffu, base, s);
    u32* h = a.hist + u64(in.tile_base) * 256u + u64(d) * in.tiles;
    for (u32 t0 = 0; t0 < in.tiles; t0 += 256u) {
        u32 v[8];
#pragma unroll
        for (u32 q = 0; q < 8u; ++q) v[q] = t0 + q * 32u + lane < in.tiles ? h[t0 + q * 32u + lane] : 0u;
#pragma unroll
        for (u32 q = 0; q < 8u; ++q) {
            u32 x = v[q];
#pragma unroll
            for (int s = 1; s < 32; s <<= 1) {
                const u32 y = __shfl_up_sync(0xffffffffu, x, s);
                if (lane >= u32(s)) x += y;
            }
            if (t0 + q * 32u + lane < in.tiles) h[t0 + q * 32u + lane] = base + x - v[q];
            base += __shfl_sync(0xffffffffu, x, 31);
        }
    }
}

// Pass `pass` over every tile of the instances it runs for: stable digit ranks within the tile plus the tile's offsets
// give each pair its place in the instance's slice of the other buffer (of the order, in the last pass that runs).
// Places are clamped to the instance's n: only tables that describe overlapping slices could produce another.
__global__ void __launch_bounds__(DO_THREADS) k_do_scatter(DepthOrderArgs a, u32 pass) {
    __shared__ u32 s_cnt[DO_WARPS * 256], s_tot[256];
    const u32 count = bounds_count(a.src), total = *a.total_tiles, tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    for (u32 g = blockIdx.x; g < total; g += gridDim.x) {
        const DepthInstance in = do_instance(a.info, do_find(a.info, count, g));
        const u32 t = g - in.tile_base;
        if (in.tiles < 2u || t >= in.tiles) continue;  // CTA-uniform
        const u32 i0 = t * DO_TILE + warp * DO_WARP_ROWS + lane;
        if (!((in.mask >> pass) & 1u)) {
            if (pass == 3u && in.mask == 0u) {  // every digit constant: the keys are all equal, the entries in order
#pragma unroll
                for (u32 k = 0; k < DO_ITEMS; ++k) {
                    const u32 i = i0 + k * 32u;
                    if (i < in.n) a.order[u64(in.first) + i] = a.vals[0][u64(in.first) + i];
                }
            }
            continue;
        }
        const u32 src = do_src(in.mask, pass), last = (in.mask >> (pass + 1u)) == 0u;
        u32 key[DO_ITEMS], val[DO_ITEMS], dig[DO_ITEMS], rank[DO_ITEMS];
#pragma unroll
        for (u32 k = 0; k < DO_ITEMS; ++k) {
            const u32 i = i0 + k * 32u;
            key[k] = i < in.n ? a.keys[src][u64(in.first) + i] : 0u;
            val[k] = i < in.n ? a.vals[src][u64(in.first) + i] : 0u;
            dig[k] = i < in.n ? (key[k] >> (8u * pass)) & 255u : 256u;
        }
        do_rank(dig, rank, s_cnt, s_tot);
        s_tot[tid] = a.hist[u64(in.tile_base) * 256u + u64(tid) * in.tiles + t];
        __syncthreads();
#pragma unroll
        for (u32 k = 0; k < DO_ITEMS; ++k) {
            if (dig[k] >= 256u) continue;
            const u64 r = u64(in.first) + min(s_tot[dig[k]] + rank[k], in.n - 1u);
            if (last) {
                a.order[r] = val[k];
            } else {
                a.keys[src ^ 1u][r] = key[k];
                a.vals[src ^ 1u][r] = val[k];
            }
        }
    }
}

// Tile histograms of pass `pass` (1-3) over the buffer that pass reads.
__global__ void __launch_bounds__(DO_THREADS) k_do_hist(DepthOrderArgs a, u32 pass) {
    __shared__ u32 s_cnt[256];
    const u32 count = bounds_count(a.src), total = *a.total_tiles, tid = threadIdx.x;
    for (u32 g = blockIdx.x; g < total; g += gridDim.x) {
        const DepthInstance in = do_instance(a.info, do_find(a.info, count, g));
        const u32 t = g - in.tile_base;
        if (in.tiles < 2u || t >= in.tiles || !((in.mask >> pass) & 1u)) continue;  // CTA-uniform
        const u32* keys = a.keys[do_src(in.mask, pass)] + in.first;
        __syncthreads();
        s_cnt[tid] = 0u;
        __syncthreads();
        const u32 end = u64(t + 1u) * DO_TILE < in.n ? (t + 1u) * DO_TILE : in.n;
        for (u32 i = t * DO_TILE + tid; i < end; i += DO_THREADS)
            atomicAdd(&s_cnt[(keys[i] >> (8u * pass)) & 255u], 1u);
        __syncthreads();
        a.hist[u64(in.tile_base) * 256u + u64(tid) * in.tiles + t] = s_cnt[tid];
    }
}

// ---------------------------------------------------------------------------------------------
// Visible particles of every instance of a batch (hnb_batch_cull): the source entries of each instance whose `position`
// lies inside the instance's six frustum planes, compacted in source order, and the instance's draw arguments with that
// count. A pure read of the instance, like bounds and depth order.
//
// The tiles are depth order's (DO_TILE rows of one instance, planned by do_tile_plan). Row i of a tile is tested by
// lane i % 32 of warp (i % DO_TILE) / DO_WARP_ROWS, as item (i % DO_WARP_ROWS) / 32, so one ballot per item is one word
// of the tile's visibility mask. Four launches, whatever the batch holds:
//   k_cull_plan   the tile plan (one CTA)
//   k_cull_test   per tile: source entries, positions, the six plane tests; the tile's mask and visible count
//   k_cull_scan   per instance (one CTA): tile counts -> exclusive prefixes; the instance's draw-args row with its count
//   k_cull_write  per tile: each visible entry to first + prefix + its rank in the mask, so a warp's stores are consecutive
// Several views with one source (hnb_batch_cull_views) take the same plan and the same tile bodies for every view at
// once: k_cull_views_test loads each row's entry and position once and keeps a mask and a count per (tile, view),
// k_cull_views_scan runs per (instance, view), and k_cull_views_write loads an entry once for all views that see it.
// ---------------------------------------------------------------------------------------------
#define CULL_PLANES 6
#define CULL_WORDS (DO_TILE / 32)  // mask words per tile: DO_ITEMS per warp
static_assert(CULL_WORDS == HNB_BATCH_CULL_MASK_WORDS && CULL_WORDS == DO_WARPS * DO_ITEMS, "one mask word per item of a warp");
#define CULL_ITEMS 8               // items of a thread with loads in flight together (DO_ITEMS / CULL_ITEMS rounds per tile)
#define CULL_SCAN_ITEMS 16         // tile counts per thread per round of k_cull_scan

// ((a*x + b*y) + c*z) + d >= 0 for plane q = (a, b, c, d), each step rounded on its own: a NaN fails, -0 passes.
__device__ __forceinline__ bool cull_plane(const float* q, u32 x, u32 y, u32 z) {
    const float v = do_add(do_add(do_add(do_mul(q[0], __uint_as_float(x)), do_mul(q[1], __uint_as_float(y))),
                                  do_mul(q[2], __uint_as_float(z))), q[3]);
    return v >= 0.0f;
}
__device__ __forceinline__ bool cull_inside(const float* f, u32 x, u32 y, u32 z) {
    bool inside = true;
#pragma unroll
    for (int p = 0; p < CULL_PLANES; ++p) inside &= cull_plane(f + 4 * p, x, y, z);
    return inside;
}

// Where the source entries of an instance come from: d_src at the instance's rows, or its alive-list column W, whose rows
// below the identity claim are i (no load). Every entry is clamped to the slice.
struct CullSource { const u32* list; u32 claimed, last_row; };
__device__ __forceinline__ CullSource cull_source(const CullArgs& a, const DepthInstance& in, u64 claim0, u64 claim1) {
    if (a.src_list) return CullSource{a.src_list + in.first, 0u, in.rows - 1u};
    return CullSource{(in.w == 0u ? a.src.ping : a.src.pong) + in.first, min(hnb_claim_len(in.w == 0u ? claim0 : claim1, in.first), in.n),
                      in.rows - 1u};
}
__device__ __forceinline__ u32 cull_entry(const CullSource& s, u32 i) { return i < s.claimed ? i : min(s.list[i], s.last_row); }

__global__ void __launch_bounds__(DO_THREADS) k_cull_plan(CullArgs a) {
    __shared__ u32 s_warp[DO_WARPS];
    do_tile_plan(a.src, a.info, a.total_tiles, a.max_tiles, s_warp);
}

// The tile passes below serve one view (hnb_batch_cull: NV = 1, views = 1) and up to NV views (hnb_batch_cull_views)
// with one body. View v's scratch is block v of `mask` and `prefix` (max_tiles tiles each); view 0's block is the whole
// single-view scratch. Only views < `views` are touched.

// Persistent grid over the call's tiles. The instance's frusta, one per view, `frustum_stride` floats apart, are staged
// in shared memory when a CTA's instance changes (they may sit in pinned host memory). Each row's entry and position are
// loaded once and tested against every view; each view gets the tile's mask and visible count. FAST: position in one
// 16-byte load per row, as k_bounds_reduce.
template <bool FAST, u32 NV>
__device__ __forceinline__ void cull_test_tiles(const CullArgs& a, u32 views, u64 frustum_stride, float* s_frustum, u32* s_count) {
    static_assert(4 * CULL_PLANES * NV <= DO_THREADS, "one thread stages one frustum word");
    const u32 count = bounds_count(a.src), total = *a.total_tiles, tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    const u64 claim0 = hnb_claim_load(&a.src.claim[0]), claim1 = hnb_claim_load(&a.src.claim[1]);
    const BoundsArgs& s = a.src;
    u32 staged = 0xFFFFFFFFu;
    for (u32 g = blockIdx.x; g < total; g += gridDim.x) {
        const u32 j = do_find(a.info, count, g);
        const DepthInstance in = do_instance(a.info, j);
        const u32 t = g - in.tile_base;
        if (t >= in.tiles) continue;  // CTA-uniform
        __syncthreads();              // the previous tile's readers of s_frustum and s_count are done
        if (j != staged && tid < 4u * CULL_PLANES * views) {
            const u32 v = tid / (4u * CULL_PLANES), k = tid % (4u * CULL_PLANES);
            s_frustum[tid] = a.frusta[u64(v) * frustum_stride + u64(j) * (4u * CULL_PLANES) + k];
        }
        if (tid < views) s_count[tid] = 0u;
        staged = j;
        __syncthreads();
        const CullSource src = cull_source(a, in, claim0, claim1);
        const u32 i0 = t * DO_TILE + warp * DO_WARP_ROWS + lane;
        u32 word[NV], seen[NV];
#pragma unroll
        for (u32 v = 0; v < NV; ++v) word[v] = seen[v] = 0u;
#pragma unroll
        for (u32 h = 0; h < DO_ITEMS; h += CULL_ITEMS) {
            u32 e[CULL_ITEMS], p[CULL_ITEMS][3];
#pragma unroll
            for (u32 k = 0; k < CULL_ITEMS; ++k) {
                const u32 i = i0 + (h + k) * 32u;
                e[k] = i < in.n ? cull_entry(src, i) : 0u;
            }
            if (FAST) {
                const RepackPiece<4>* col = (const RepackPiece<4>*)s.col[0];
                const u32 quads = s.col_words[0] >> 2u, quad = s.col_lane[0] >> 2u;
#pragma unroll
                for (u32 k = 0; k < CULL_ITEMS; ++k) {
                    if (i0 + (h + k) * 32u >= in.n) continue;
                    const RepackPiece<4> q = col[(u64(in.first) + e[k]) * quads + quad];
#pragma unroll
                    for (int c = 0; c < 3; ++c) p[k][c] = q.w[c];
                }
            } else {
#pragma unroll
                for (u32 k = 0; k < CULL_ITEMS; ++k) {
                    if (i0 + (h + k) * 32u >= in.n) continue;
#pragma unroll
                    for (int c = 0; c < 3; ++c) p[k][c] = s.col[c][(u64(in.first) + e[k]) * s.col_words[c] + s.col_lane[c]];
                }
            }
#pragma unroll
            for (u32 v = 0; v < NV; ++v) {
                if (v >= views) break;  // CTA-uniform
                bool vis[CULL_ITEMS];
                if (NV == 1) {
                    // one view: its planes stay in registers for the whole tile
#pragma unroll
                    for (u32 k = 0; k < CULL_ITEMS; ++k)
                        vis[k] = i0 + (h + k) * 32u < in.n && cull_inside(s_frustum, p[k][0], p[k][1], p[k][2]);
                } else {
                    // plane by plane over the items: one read of a plane from shared memory serves CULL_ITEMS rows
#pragma unroll
                    for (u32 k = 0; k < CULL_ITEMS; ++k) vis[k] = i0 + (h + k) * 32u < in.n;
#pragma unroll
                    for (u32 pl = 0; pl < CULL_PLANES; ++pl) {
                        float q[4];
#pragma unroll
                        for (int c = 0; c < 4; ++c) q[c] = s_frustum[4u * (CULL_PLANES * v + pl) + c];
#pragma unroll
                        for (u32 k = 0; k < CULL_ITEMS; ++k) vis[k] = vis[k] && cull_plane(q, p[k][0], p[k][1], p[k][2]);
                    }
                }
#pragma unroll
                for (u32 k = 0; k < CULL_ITEMS; ++k) {
                    const u32 b = __ballot_sync(0xffffffffu, vis[k]);
                    if (lane == h + k) word[v] = b;
                    seen[v] += __popc(b);
                }
            }
        }
#pragma unroll
        for (u32 v = 0; v < NV; ++v) {
            if (v >= views) break;
            if (lane < DO_ITEMS) a.mask[(u64(v) * a.max_tiles + g) * CULL_WORDS + warp * DO_ITEMS + lane] = word[v];
            if (lane == 0u && seen[v]) atomicAdd(&s_count[v], seen[v]);
        }
        __syncthreads();
        if (tid < views) a.prefix[u64(tid) * a.max_tiles + g] = s_count[tid];
    }
}

template <bool FAST>
__global__ void __launch_bounds__(DO_THREADS) k_cull_test(CullArgs a) {
    __shared__ float s_frustum[4 * CULL_PLANES];
    __shared__ u32 s_count[1];
    cull_test_tiles<FAST, 1>(a, 1u, 0u, s_frustum, s_count);
}

// One CTA: the visible counts of instance j's tiles in a view's `prefix` block become exclusive prefixes within the
// instance, and args[j] (of that view's args rows) receives the draw-args row its spawner row names (clamped to the
// table) with instance_count = the instance's visible total (0 for a j past the batch's device-side count).
__device__ __forceinline__ void cull_scan_instance(const CullArgs& a, u32 j, u32* prefix, u32* args, u32* s_warp, u32* s_round) {
    const u32 tid = threadIdx.x;
    u32 m = 0u;
    if (j < bounds_count(a.src)) {  // CTA-uniform
        const DepthInstance in = do_instance(a.info, j);
        u32* c = prefix + in.tile_base;
        for (u32 t0 = 0; t0 < in.tiles; t0 += DO_THREADS * CULL_SCAN_ITEMS) {
            const u32 tb = t0 + tid * CULL_SCAN_ITEMS;
            u32 v[CULL_SCAN_ITEMS], sum = 0u;
#pragma unroll
            for (u32 q = 0; q < CULL_SCAN_ITEMS; ++q) {
                v[q] = tb + q < in.tiles ? c[tb + q] : 0u;
                sum += v[q];
            }
            u32 run = m + do_block_exclusive(sum, s_warp);
#pragma unroll
            for (u32 q = 0; q < CULL_SCAN_ITEMS; ++q) {
                if (tb + q < in.tiles) c[tb + q] = run;
                run += v[q];
            }
            __syncthreads();  // s_round of the previous round is read
            if (tid == DO_THREADS - 1u) *s_round = run;
            __syncthreads();
            m = *s_round;
        }
    }
    if (tid < HNB_DRAW_INDEXED_INDIRECT_STRIDE) {
        const u64 row = u64(a.src.batch_info->spawner_base) + j;
        const Spawner* sp = &a.src.spawners[row < a.src.num_spawners ? row : a.src.num_spawners - 1u];
        const u32 dri = min(sp->draw_indirect_index, a.num_draw_args - 1u);
        args[u64(j) * HNB_DRAW_INDEXED_INDIRECT_STRIDE + tid] = tid == 1u ? m : a.draw_args[u64(dri) * HNB_DRAW_INDEXED_INDIRECT_STRIDE + tid];
    }
}

// CTA j, one per instance the call covers.
__global__ void __launch_bounds__(DO_THREADS) k_cull_scan(CullArgs a) {
    __shared__ u32 s_warp[DO_WARPS];
    __shared__ u32 s_round;
    cull_scan_instance(a, blockIdx.x, a.prefix, a.args, s_warp, &s_round);
}

// Persistent grid over the call's tiles: a visible row's place in a view is its tile's prefix there plus the visible rows
// before it in the view's mask. A row's entry is loaded again, once, where any view's mask bit is set, and stored to every
// such view, whose entries lie `visible_stride` words after the previous view's; places are clamped to the instance's n.
template <u32 NV>
__device__ __forceinline__ void cull_write_tiles(const CullArgs& a, u32 views, u64 visible_stride, u32* s_warp) {
    const u32 count = bounds_count(a.src), total = *a.total_tiles, tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    const u64 claim0 = hnb_claim_load(&a.src.claim[0]), claim1 = hnb_claim_load(&a.src.claim[1]);
    const u32 lt = (1u << lane) - 1u;
    for (u32 g = blockIdx.x; g < total; g += gridDim.x) {
        const DepthInstance in = do_instance(a.info, do_find(a.info, count, g));
        const u32 t = g - in.tile_base;
        if (t >= in.tiles) continue;  // CTA-uniform
        // lane k < DO_ITEMS holds mask word k of its warp in each view and the view's visible rows of the tile before it
        u32 word[NV], before[NV];
#pragma unroll
        for (u32 v = 0; v < NV; ++v) {
            if (v >= views) break;  // CTA-uniform
            const u64 vg = u64(v) * a.max_tiles + g;
            word[v] = lane < DO_ITEMS ? a.mask[vg * CULL_WORDS + warp * DO_ITEMS + lane] : 0u;
            before[v] = a.prefix[vg] + do_block_exclusive(__popc(word[v]), s_warp);
        }
        const CullSource src = cull_source(a, in, claim0, claim1);
        const u32 i0 = t * DO_TILE + warp * DO_WARP_ROWS + lane;
#pragma unroll
        for (u32 k = 0; k < DO_ITEMS; ++k) {
            u32 wk[NV], bk[NV], any = 0u;
#pragma unroll
            for (u32 v = 0; v < NV; ++v) {
                if (v >= views) break;
                wk[v] = __shfl_sync(0xffffffffu, word[v], k);
                bk[v] = __shfl_sync(0xffffffffu, before[v], k);
                any |= wk[v];
            }
            if (!((any >> lane) & 1u)) continue;
            const u32 e = cull_entry(src, i0 + k * 32u);
#pragma unroll
            for (u32 v = 0; v < NV; ++v) {
                if (v >= views) break;
                if (!((wk[v] >> lane) & 1u)) continue;
                const u32 r = min(bk[v] + __popc(wk[v] & lt), in.n - 1u);
                a.visible[u64(v) * visible_stride + in.first + r] = e;
            }
        }
    }
}

__global__ void __launch_bounds__(DO_THREADS) k_cull_write(CullArgs a) {
    __shared__ u32 s_warp[DO_WARPS];
    cull_write_tiles<1>(a, 1u, 0u, s_warp);
}

// hnb_batch_cull_views: the same passes for a.views views, after the same k_cull_plan.
template <bool FAST>
__global__ void __launch_bounds__(DO_THREADS, 2) k_cull_views_test(CullViewsArgs a) {
    __shared__ float s_frustum[4 * CULL_PLANES * HNB_BATCH_CULL_MAX_VIEWS];
    __shared__ u32 s_count[HNB_BATCH_CULL_MAX_VIEWS];
    cull_test_tiles<FAST, HNB_BATCH_CULL_MAX_VIEWS>(a.c, a.views, u64(a.frustum_rows) * (4u * CULL_PLANES), s_frustum, s_count);
}

// CTA v * max_instances + j: instance j in view v.
__global__ void __launch_bounds__(DO_THREADS) k_cull_views_scan(CullViewsArgs a) {
    __shared__ u32 s_warp[DO_WARPS];
    __shared__ u32 s_round;
    const u32 j = blockIdx.x % a.c.src.max_instances, v = blockIdx.x / a.c.src.max_instances;
    cull_scan_instance(a.c, j, a.c.prefix + u64(v) * a.c.max_tiles, a.c.args + u64(v) * a.args_rows * HNB_DRAW_INDEXED_INDIRECT_STRIDE,
                       s_warp, &s_round);
}

__global__ void __launch_bounds__(DO_THREADS) k_cull_views_write(CullViewsArgs a) {
    __shared__ u32 s_warp[DO_WARPS];
    cull_write_tiles<HNB_BATCH_CULL_MAX_VIEWS>(a.c, a.views, a.visible_rows, s_warp);
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
cudaError_t launch_flush_group_ages(const PlaneSet& planes, u32 age_word, u64* group_age, u32* life_floor, u32 first, u32 count,
                                    u32 capacity, bool clear, u32 epoch, cudaStream_t st) {
    if (count == 0) return cudaSuccess;
    const u32 g0 = first >> 5u, groups = u32(((u64(first) + count + 31u) >> 5u) - g0);
    k_flush_group_ages<<<blocks_for(groups, 256), 256, 0, st>>>(planes, age_word, group_age, life_floor, g0, groups, capacity,
                                                                           clear ? 1u : 0u, epoch);
    return cudaGetLastError();
}
cudaError_t launch_bits_from_list(u32* bits, const u32* list, u32 base, u32 alive_count, cudaStream_t st) {
    if (alive_count == 0) return cudaSuccess;
    k_bits_from_list<<<blocks_for(alive_count, 256), 256, 0, st>>>(bits, list, base, alive_count);
    return cudaGetLastError();
}
cudaError_t launch_fill_c5(const PlaneSet& planes, u32* ping, u32* pong, u64* claim, u32 first, u32 count, u32 seed, f32 lo, f32 hi, u32 logical_first, cudaStream_t st) {
    if (count == 0) return cudaSuccess;
    k_fill_c5<<<blocks_for(count, 256), 256, 0, st>>>(planes, ping, pong, claim, first, count, seed, lo, hi, logical_first);
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
cudaError_t launch_snapshot_gather(const SnapshotArgs& a, u32* dst, cudaStream_t st, const u32* dead) {
    if (a.rows == 0) return cudaSuccess;
    if (dead) k_snapshot_gather_dead<<<blocks_for(a.rows, RP_ROWS_PER_BLOCK), RP_THREADS, 0, st>>>(a, dead, dst);
    else k_snapshot_gather<<<blocks_for(a.rows, RP_ROWS_PER_BLOCK), RP_THREADS, 0, st>>>(a, dst);
    return cudaGetLastError();
}
cudaError_t launch_restore_scatter(const SnapshotArgs& a, const u32* src, cudaStream_t st, const u32* channels) {
    if (a.rows == 0) return cudaSuccess;
    if (channels) k_restore_scatter_dead<<<blocks_for(a.rows, RP_ROWS_PER_BLOCK), RP_THREADS, 0, st>>>(a, src, *channels);
    else k_restore_scatter<<<blocks_for(a.rows, RP_ROWS_PER_BLOCK), RP_THREADS, 0, st>>>(a, src);
    return cudaGetLastError();
}
cudaError_t launch_append(const AppendArgs& a, const u32* src, cudaStream_t st, u32* launches) {
    // m is at most the records the buffer holds and at most rows: no more threads than the smaller of the two
    const u64 held = (a.s.src_bytes - HNB_SNAPSHOT_HEADER_WORDS * 4u) / (a.s.stride_words * 4u);
    const u32 bound = u32(held < a.s.rows ? held : a.s.rows);
    if (bound == 0u) return cudaSuccess;
    k_append_scatter<<<blocks_for(bound, RP_ROWS_PER_BLOCK), RP_THREADS, 0, st>>>(a, src);
    ++*launches;
    cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) return err;
    k_append_commit<<<1, 1, 0, st>>>(a, src);
    ++*launches;
    return cudaGetLastError();
}
cudaError_t launch_repack_inverse(const RepackArgs& a, u32* inv, cudaStream_t st) {
    if (a.rows == 0) return cudaSuccess;
    k_repack_inverse<<<blocks_for(a.rows, RP_THREADS), RP_THREADS, 0, st>>>(a, inv);
    return cudaGetLastError();
}
cudaError_t launch_events_translate(const RepackArgs& a, const u32* inv, const EventChannels& ev, u32 stride_words, u32* snapshot,
                                    cudaStream_t st) {
    if (a.rows == 0 || ev.count == 0) return cudaSuccess;
    u32 widest = 1u;
    for (u32 b = 0; b < ev.count; ++b) widest = std::max(widest, ev.capacity[b]);
    const u32 per_channel = blocks_for(widest, RP_THREADS);
    k_events_translate<<<per_channel * ev.count, RP_THREADS, 0, st>>>(a, inv, ev, per_channel, stride_words, snapshot);
    return cudaGetLastError();
}
cudaError_t launch_restore_events(const SnapshotArgs& a, const u32* src, const EventChannels& ev, cudaStream_t st) {
    if (a.rows == 0 || ev.count == 0) return cudaSuccess;
    k_restore_events<<<ev.count, EV_THREADS, 0, st>>>(a, src, ev);
    return cudaGetLastError();
}
// CTAs of k_bounds_reduce<FAST> that one SM holds
template <bool FAST> static cudaError_t bounds_blocks_per_sm(int* out) {
    static int cached = 0;
    if (cached == 0) {
        int n = 0;
        const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, k_bounds_reduce<FAST>, BD_THREADS, 0);
        if (e != cudaSuccess) return e;
        cached = std::max(n, 1);
    }
    *out = cached;
    return cudaSuccess;
}
cudaError_t launch_batch_bounds(const BoundsArgs& a, bool fast, u32 sm_count, cudaStream_t st) {
    if (a.max_instances == 0) return cudaSuccess;
    int per_sm = 1;
    const cudaError_t e = fast ? bounds_blocks_per_sm<true>(&per_sm) : bounds_blocks_per_sm<false>(&per_sm);
    if (e != cudaSuccess) return e;
    // no more CTAs than the slab can have tiles: a small batch is a small launch
    const u64 max_tiles = u64(a.capacity_rows) / BD_TILE + a.max_instances;
    const unsigned grid = (unsigned)std::min<u64>(max_tiles, u64(sm_count) * u64(per_sm));
    if (fast) k_bounds_reduce<true><<<grid, BD_THREADS, 0, st>>>(a);
    else k_bounds_reduce<false><<<grid, BD_THREADS, 0, st>>>(a);
    k_bounds_write<<<blocks_for(a.max_instances, BD_THREADS), BD_THREADS, 0, st>>>(a);
    return cudaGetLastError();
}
u64 depth_order_max_tiles(u32 capacity_rows, u32 max_instances) { return u64(capacity_rows) / DO_TILE + max_instances; }
cudaError_t launch_batch_depth_order(const DepthOrderArgs& a, bool fast, u32 sm_count, cudaStream_t st) {
    if (a.src.max_instances == 0) return cudaSuccess;
    // tile kernels: no more CTAs than the call can have tiles; the plan zeroes 1024 totals per instance
    const unsigned tiles = (unsigned)std::max<u64>(1, std::min<u64>(a.max_tiles, u64(sm_count) * DO_CTAS_PER_SM));
    const unsigned plan = std::min(blocks_for(u64(a.src.max_instances) * 1024u, DO_THREADS * 16u), 1024u);
    const unsigned rows = blocks_for(u64(a.src.max_instances) * 256u, DO_WARPS);
    k_do_plan<<<plan, DO_THREADS, 0, st>>>(a);
    if (fast) k_do_keys<true><<<tiles, DO_THREADS, 0, st>>>(a);
    else k_do_keys<false><<<tiles, DO_THREADS, 0, st>>>(a);
    for (u32 pass = 0; pass < 4u; ++pass) {
        if (pass) k_do_hist<<<tiles, DO_THREADS, 0, st>>>(a, pass);
        k_do_scan<<<rows, DO_THREADS, 0, st>>>(a, pass);
        k_do_scatter<<<tiles, DO_THREADS, 0, st>>>(a, pass);
    }
    return cudaGetLastError();
}
// CTAs of `kernel` (DO_THREADS threads) that one SM holds, asked once per kernel
template <typename K> static cudaError_t do_ctas_per_sm(K kernel, int* cached, u32* out) {
    if (*cached == 0) {
        int n = 0;
        const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, DO_THREADS, 0);
        if (e != cudaSuccess) return e;
        *cached = std::max(n, 1);
    }
    *out = u32(*cached);
    return cudaSuccess;
}
// The four launches of a cull over args `a` (`c`: its single-view part): tile kernels with every CTA resident at once and
// no more CTAs than the call can have tiles; `scan_ctas` CTAs of `scan`.
template <typename A>
static cudaError_t cull_launches(const A& a, const CullArgs& c, void (*test)(A), int* test_cached, void (*scan)(A), u64 scan_ctas,
                                 void (*write)(A), int* write_cached, u32 sm_count, cudaStream_t st) {
    if (c.src.max_instances == 0) return cudaSuccess;
    u32 per_test = 1, per_write = 1;
    cudaError_t e = do_ctas_per_sm(test, test_cached, &per_test);
    if (e == cudaSuccess) e = do_ctas_per_sm(write, write_cached, &per_write);
    if (e != cudaSuccess) return e;
    const unsigned test_grid = (unsigned)std::max<u64>(1, std::min<u64>(c.max_tiles, u64(sm_count) * per_test));
    const unsigned write_grid = (unsigned)std::max<u64>(1, std::min<u64>(c.max_tiles, u64(sm_count) * per_write));
    k_cull_plan<<<1, DO_THREADS, 0, st>>>(c);
    test<<<test_grid, DO_THREADS, 0, st>>>(a);
    scan<<<(unsigned)scan_ctas, DO_THREADS, 0, st>>>(a);
    write<<<write_grid, DO_THREADS, 0, st>>>(a);
    return cudaGetLastError();
}
cudaError_t launch_batch_cull(const CullArgs& a, bool fast, u32 sm_count, cudaStream_t st) {
    static int test_fast = 0, test_any = 0, write = 0;
    return cull_launches(a, a, fast ? k_cull_test<true> : k_cull_test<false>, fast ? &test_fast : &test_any, k_cull_scan,
                         a.src.max_instances, k_cull_write, &write, sm_count, st);
}
cudaError_t launch_batch_cull_views(const CullViewsArgs& a, bool fast, u32 sm_count, cudaStream_t st) {
    static int test_fast = 0, test_any = 0, write = 0;
    return cull_launches(a, a.c, fast ? k_cull_views_test<true> : k_cull_views_test<false>, fast ? &test_fast : &test_any,
                         k_cull_views_scan, u64(a.c.src.max_instances) * a.views, k_cull_views_write, &write, sm_count, st);
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
