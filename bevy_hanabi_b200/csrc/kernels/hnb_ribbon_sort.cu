// hnb_ribbon_sort.cu — ribbon sort (SURVEY.md §8f-4), compiled ahead of time by nvcc for sm_90a.
//
// Replaces the reference's three dispatches per ribbon effect instance (mod.rs:7444-7610):
//     vfx_sort_fill.wgsl :38-57   pairs[k] = {particle[RIBBON_ID], particle[AGE], particle_index}
//     vfx_sort.wgsl      :18-55   ONE thread insertion-sorts the pairs by (key, key2), u32 compare
//     vfx_sort_copy.wgsl :30-46   the sorted particle indices go back into the SAME alive-list column
// The reference's result is the STABLE sort of the alive-list entries by the 64-bit key
// (ribbon_id << 32 | age bits) — stable with respect to the order the fill threads appended in, which
// we fix to the canonical (thread index) order like everywhere else. Two kernels produce exactly that:
//
//   k_ribbon_sort_small  one CTA per instance, n <= 2048: keys staged in shared memory, bitonic network
//                        on (key, rank) — the rank tie-break makes the network's result the stable one.
//   k_ribbon_sort_large  cooperative grid, n > 2048: LSD radix sort, 8-bit digits over the 64-bit key,
//                        digit histograms of all eight passes taken while filling, passes whose digit is
//                        constant skipped (ribbon ids are small and ages share their exponent byte, so
//                        typically 3-4 of 8 passes run), per-CTA contiguous chunks + digit-major
//                        (digit, CTA) offsets keep every pass stable.
//
// Both gather the keys straight from the slab's SoA planes through the AoS word -> plane map; no key
// buffer exists outside the large path's scratch.
#include <cstdint>
#include <cooperative_groups.h>
#include <cuda_runtime.h>

#include "hnb_tables.cuh"
#include "hnb_static_kernels.h"

namespace cg = cooperative_groups;

namespace hnb {

namespace {

constexpr u32 kSmallMax = HNB_RIBBON_SORT_SMALL_MAX;  // 2048
constexpr u32 kSmallThreads = 1024;
constexpr u32 kLargeThreads = 512;
constexpr u32 kLargeWarps = kLargeThreads / 32;

__device__ __forceinline__ u32 load_word(const PlaneSet& planes, u32 row, u32 word) {
    const u32 p = planes.word_to_plane[word];
    return ((const u32*)planes.ptr[p])[u64(row) * planes.words[p] + (word - planes.word_off[p])];
}

struct Instance {
    u32 n, base, k1, k2;
    u32* column;
};
__device__ __forceinline__ Instance load_instance(const RibbonSortArgs& a, u32 i) {
    const Spawner& sp = a.spawners[a.spawner_base + i];
    const EffectMetadata& md = a.metadata[sp.effect_metadata_index];
    Instance r;
    r.n = md.alive_count;
    r.base = sp.slab_offset;
    r.k1 = md.sort_key_offset;
    r.k2 = md.sort_key2_offset;
    // the column the update pass wrote this frame (vfx_sort_fill.wgsl:49-50); sorted in place
    r.column = (md.indirect_write_index == 0u ? a.ping : a.pong) + r.base;
    return r;
}
__device__ __forceinline__ u64 load_key(const RibbonSortArgs& a, const Instance& in, u32 particle_index) {
    const u32 row = in.base + particle_index;
    return (u64(load_word(a.planes, row, in.k1)) << 32) | u64(load_word(a.planes, row, in.k2));
}

// ---------------------------------------------------------------------------------------------
// n <= 2048: one CTA, shared memory, bitonic network on (key, rank)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kSmallThreads) k_ribbon_sort_small(RibbonSortArgs a) {
    __shared__ u64 s_key[kSmallMax];
    __shared__ u32 s_val[kSmallMax];
    __shared__ unsigned short s_rank[kSmallMax];
    const Instance in = load_instance(a, blockIdx.x);
    if (in.n < 2u || in.n > kSmallMax) return;  // CTA-uniform
    u32 m = 2u;
    while (m < in.n) m <<= 1;
    for (u32 r = threadIdx.x; r < m; r += kSmallThreads) {
        if (r < in.n) {
            const u32 e = in.column[r];
            s_val[r] = e;
            s_key[r] = load_key(a, in, e);
        } else {
            s_key[r] = ~u64(0);  // padding sorts last: a real pair with the same key has a smaller rank
        }
        s_rank[r] = (unsigned short)r;
    }
    __syncthreads();
    for (u32 k = 2u; k <= m; k <<= 1) {
        for (u32 j = k >> 1; j > 0u; j >>= 1) {
            for (u32 t = threadIdx.x; t < (m >> 1); t += kSmallThreads) {
                const u32 lo = ((t & ~(j - 1u)) << 1) | (t & (j - 1u));  // insert a 0 bit at position log2(j)
                const u32 hi = lo | j;
                const bool ascending = (lo & k) == 0u;
                const u64 ka = s_key[lo], kb = s_key[hi];
                const unsigned short ra = s_rank[lo], rb = s_rank[hi];
                const bool a_greater = ka > kb || (ka == kb && ra > rb);
                if (a_greater == ascending) {
                    s_key[lo] = kb; s_key[hi] = ka;
                    s_rank[lo] = rb; s_rank[hi] = ra;
                }
            }
            __syncthreads();
        }
    }
    // every entry was read into s_val before the first store (barriers above)
    for (u32 r = threadIdx.x; r < in.n; r += kSmallThreads) in.column[r] = s_val[s_rank[r]];
}

// ---------------------------------------------------------------------------------------------
// n > 2048: cooperative LSD radix sort
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kLargeThreads) k_ribbon_sort_large(RibbonSortArgs a) {
    cg::grid_group grid = cg::this_grid();
    __shared__ u32 s_hist[8 * 256];                 // fill: the eight digit histograms; passes: [0,256) chunk histogram
    __shared__ u32 s_offset[256];                   // running output position of each digit for this CTA
    __shared__ u32 s_scan[256];
    __shared__ unsigned short s_warp_cnt[kLargeWarps * 256];
    const u32 G = gridDim.x, cta = blockIdx.x, tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    // scratch_hist: two copies of the [8][256] digit histograms (used alternately by successive large instances;
    // both zero at launch), then the digit-major [256][G] per-CTA histogram table of the current pass
    u32* const cta_hist = a.scratch_hist + 2 * 8 * 256;
    u32 seq = 0u;

    for (u32 inst = 0; inst < a.instance_count; ++inst) {
        const Instance in = load_instance(a, inst);
        if (in.n <= kSmallMax || in.n > a.scratch_rows) continue;  // grid-uniform
        u32* const ghist = a.scratch_hist + (seq & 1u) * 8u * 256u;
        u32* const ghist_next = a.scratch_hist + ((seq + 1u) & 1u) * 8u * 256u;
        ++seq;
        const u32 n = in.n;
        // contiguous chunk of this CTA, a whole number of 512-key tiles
        const u32 tiles = (n + kLargeThreads - 1u) / kLargeThreads;
        const u32 tiles_per_cta = (tiles + G - 1u) / G;
        const u32 chunk_begin = min(n, cta * tiles_per_cta * kLargeThreads);
        const u32 chunk_end = min(n, chunk_begin + tiles_per_cta * kLargeThreads);

        // ---- fill (vfx_sort_fill.wgsl) + histograms of all eight digits
        for (u32 i = tid; i < 8u * 256u; i += kLargeThreads) s_hist[i] = 0u;
        __syncthreads();
        for (u32 r = chunk_begin + tid; r < chunk_end; r += kLargeThreads) {
            const u32 e = in.column[r];
            const u64 key = load_key(a, in, e);
            a.scratch_keys[0][r] = key;
            a.scratch_vals[0][r] = e;
#pragma unroll
            for (u32 p = 0; p < 8u; ++p) atomicAdd(&s_hist[p * 256u + u32((key >> (8u * p)) & 0xFFu)], 1u);
        }
        __syncthreads();
        for (u32 i = tid; i < 8u * 256u; i += kLargeThreads)
            if (s_hist[i]) atomicAdd(&ghist[i], s_hist[i]);
        grid.sync();
        // a digit shared by every key leaves the order unchanged: such passes are skipped (grid-uniform mask)
        u32 skip_mask = 0u;
        for (u32 p = 0; p < 8u; ++p)
            if (__syncthreads_or(tid < 256u && ghist[p * 256u + tid] == n)) skip_mask |= 1u << p;
        // the other histogram copy was last read before the previous instance's final grid.sync: reset it for the next one
        if (cta == 0u)
            for (u32 i = tid; i < 8u * 256u; i += kLargeThreads) ghist_next[i] = 0u;

        u32 cur = 0u;
        for (u32 p = 0; p < 8u; ++p) {
            if (skip_mask & (1u << p)) continue;
            const u64* src_k = a.scratch_keys[cur];
            const u32* src_v = a.scratch_vals[cur];
            u64* dst_k = a.scratch_keys[cur ^ 1u];
            u32* dst_v = a.scratch_vals[cur ^ 1u];
            const u32 shift = 8u * p;

            // (a) digit histogram of this CTA's chunk
            if (tid < 256u) s_hist[tid] = 0u;
            __syncthreads();
            for (u32 r = chunk_begin + tid; r < chunk_end; r += kLargeThreads) atomicAdd(&s_hist[u32((src_k[r] >> shift) & 0xFFu)], 1u);
            __syncthreads();
            if (tid < 256u) cta_hist[tid * G + cta] = s_hist[tid];
            grid.sync();

            // (b) output position of (digit d, this CTA) = keys with a smaller digit + keys of digit d in earlier CTAs
            {
                const u32 d = tid >> 1, half = tid & 1u;
                const u32 c0 = half ? (G + 1u) / 2u : 0u, c1 = half ? G : (G + 1u) / 2u;
                u32 total = 0u, before = 0u;
                for (u32 c = c0; c < c1; ++c) {
                    const u32 h = cta_hist[d * G + c];
                    total += h;
                    before += c < cta ? h : 0u;
                }
                total += __shfl_xor_sync(0xffffffffu, total, 1);
                before += __shfl_xor_sync(0xffffffffu, before, 1);
                if (half == 0u) { s_scan[d] = total; s_offset[d] = before; }
            }
            __syncthreads();
            if (warp == 0u) {  // exclusive scan of the 256 digit totals
                u32 v[8], sum = 0u;
#pragma unroll
                for (u32 k = 0; k < 8u; ++k) { v[k] = s_scan[lane * 8u + k]; sum += v[k]; }
                u32 incl = sum;
#pragma unroll
                for (u32 dlt = 1u; dlt < 32u; dlt <<= 1) {
                    const u32 up = __shfl_up_sync(0xffffffffu, incl, dlt);
                    if (lane >= dlt) incl += up;
                }
                u32 run = incl - sum;
#pragma unroll
                for (u32 k = 0; k < 8u; ++k) { s_scan[lane * 8u + k] = run; run += v[k]; }
            }
            __syncthreads();
            if (tid < 256u) s_offset[tid] += s_scan[tid];
            __syncthreads();

            // (c) stable scatter, one 512-key tile at a time
            for (u32 tile = chunk_begin; tile < chunk_end; tile += kLargeThreads) {
                for (u32 i = tid; i < kLargeWarps * 256u; i += kLargeThreads) s_warp_cnt[i] = 0;
                __syncthreads();
                const u32 r = tile + tid;
                const bool valid = r < chunk_end;
                u64 key = 0;
                u32 val = 0u, d = 256u + lane;  // invalid lanes: a digit nobody shares
                if (valid) { key = src_k[r]; val = src_v[r]; d = u32((key >> shift) & 0xFFu); }
                const u32 peers = __match_any_sync(0xffffffffu, d);
                const u32 rank_in_warp = __popc(peers & ((1u << lane) - 1u));
                if (valid && rank_in_warp == 0u) s_warp_cnt[warp * 256u + d] = (unsigned short)__popc(peers);
                __syncthreads();
                if (valid) {
                    u32 pos = s_offset[d] + rank_in_warp;
                    for (u32 w = 0; w < warp; ++w) pos += s_warp_cnt[w * 256u + d];
                    dst_k[pos] = key;
                    dst_v[pos] = val;
                }
                __syncthreads();
                if (tid < 256u) {
                    u32 t = 0u;
#pragma unroll
                    for (u32 w = 0; w < kLargeWarps; ++w) t += s_warp_cnt[w * 256u + tid];
                    s_offset[tid] += t;
                }
                __syncthreads();
            }
            grid.sync();
            cur ^= 1u;
        }

        // ---- copy back (vfx_sort_copy.wgsl); the scratch is reused by the next instance after the barrier
        {
            const u32* out_v = a.scratch_vals[cur];
            for (u32 r = chunk_begin + tid; r < chunk_end; r += kLargeThreads) in.column[r] = out_v[r];
        }
        grid.sync();
    }
}

}  // namespace

cudaError_t launch_ribbon_sort(const RibbonSortArgs& args, bool any_large, u32 sm_count, cudaStream_t st, u32* launches) {
    if (args.instance_count == 0) return cudaSuccess;
    k_ribbon_sort_small<<<args.instance_count, kSmallThreads, 0, st>>>(args);
    cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) return err;
    *launches += 1;
    if (!any_large) return cudaSuccess;
    int per_sm = 0;
    err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_ribbon_sort_large, (int)kLargeThreads, 0);
    if (err != cudaSuccess) return err;
    if (per_sm < 1) return cudaErrorLaunchOutOfResources;
    // one CTA per SM: enough parallelism for a sort that is off the metric, and the (digit, CTA) table stays small
    u32 grid = sm_count < args.scratch_grid ? sm_count : args.scratch_grid;
    RibbonSortArgs a = args;
    void* params[] = {&a};
    err = cudaLaunchCooperativeKernel((const void*)k_ribbon_sort_large, dim3(grid), dim3(kLargeThreads), params, 0, st);
    if (err != cudaSuccess) return err;
    *launches += 1;
    return cudaSuccess;
}

size_t ribbon_sort_hist_words(u32 grid) { return size_t(2 * 8 * 256) + size_t(256) * grid; }

}  // namespace hnb
