// hnb_interop_kernels.cu — layout conversion between the slab's SoA storage and the reference's buffer layouts
// (SURVEY.md §8 f-2): AoS `Particle` records (ParticleLayout, attributes.rs:1807-1913) and interleaved `IndirectEntry`
// rows {particle_index[2], dead_index} (vfx_common.wgsl:66-78, mod.rs:139-146). Compiled ahead of time by nvcc for
// sm_90a. Used by the host up/download entry points and by the device-to-device export a renderer binds.
#include <algorithm>
#include <cstdint>
#include <cuda_runtime.h>

#include "hnb_wgsl.cuh"
#include "hnb_tables.cuh"
#include "hnb_static_kernels.h"

namespace hnb {

static inline unsigned blocks_for(u64 n, unsigned bs) { return (unsigned)((n + bs - 1) / bs); }

// AoS rows (stride_words u32 each) <-> planes. Plane p covers words [word_off[p], word_off[p]+words[p]).
// The reference's render pass reads particles as AoS records through the alive list (vfx_render.wgsl:228-231,
// mod.rs:139-146), so this transpose is the per-frame interop path (§8 f-2), not only a test helper: a CTA stages
// TR_ROWS whole records in shared memory — plane side moved as float4/float2/u32 columns (consecutive lanes =
// consecutive rows, fully coalesced), AoS side moved as one contiguous run of float4 — so both sides of the copy use
// full 128-byte lines.
#define TR_THREADS 256
template <bool TO_AOS>
__global__ void __launch_bounds__(TR_THREADS) k_transpose(u32* __restrict__ aos, PlaneSet planes, u32 first, u32 count, u32 stride_words,
                                                          u32 rows_per_cta, u32 num_planes) {
    extern __shared__ __align__(16) u32 tr_tile[];  // [rows_per_cta][stride_words], the AoS image of the tile
    const u32 row0 = blockIdx.x * rows_per_cta;
    if (row0 >= count) return;
    const u32 rows = min(rows_per_cta, count - row0);
    const u32 tile_words = rows * stride_words;
    u32* const g_tile = aos + u64(row0) * stride_words;
    const bool vec_ok = (tile_words & 3u) == 0u && ((u64)(uintptr_t)g_tile & 15ull) == 0ull;
    if (!TO_AOS) {
        if (vec_ok) for (u32 i = threadIdx.x; i < tile_words / 4u; i += TR_THREADS) ((uint4*)tr_tile)[i] = ((const uint4*)g_tile)[i];
        else for (u32 i = threadIdx.x; i < tile_words; i += TR_THREADS) tr_tile[i] = g_tile[i];
        __syncthreads();
    }
    for (u32 p = 0; p < num_planes; ++p) {
        const u32 w = planes.words[p], off = planes.word_off[p];
        const bool aligned16 = ((stride_words | off) & 3u) == 0u;
        for (u32 r = threadIdx.x; r < rows; r += TR_THREADS) {
            const u64 grow = u64(first) + row0 + r;
            if (off & HNB_PLANE_WORD_LIST) {  // a word map: lane l <-> its own record word
                u32* const rec = tr_tile + r * stride_words;
                u32* const g = (u32*)planes.ptr[p] + grow * w;
                for (u32 l = 0; l < w; ++l) {
                    if (TO_AOS) rec[hnb_plane_word(planes, p, l)] = g[l];
                    else g[l] = rec[hnb_plane_word(planes, p, l)];
                }
                continue;
            }
            u32* t = tr_tile + r * stride_words + off;
            if (w == 4u) {
                uint4* g = (uint4*)planes.ptr[p] + grow;
                if (aligned16) {  // record stride and piece offset multiples of 16 bytes: one 128-bit shared-memory access
                    if (TO_AOS) *(uint4*)t = *g; else *g = *(const uint4*)t;
                } else if (TO_AOS) { const uint4 v = *g; t[0] = v.x; t[1] = v.y; t[2] = v.z; t[3] = v.w; }
                else *g = make_uint4(t[0], t[1], t[2], t[3]);
            } else if (w == 8u) {  // sector planes: two 16-byte pieces per element
                uint4* g = (uint4*)planes.ptr[p] + 2ull * grow;
                if (TO_AOS) { const uint4 a = g[0], b = g[1]; t[0] = a.x; t[1] = a.y; t[2] = a.z; t[3] = a.w; t[4] = b.x; t[5] = b.y; t[6] = b.z; t[7] = b.w; }
                else { g[0] = make_uint4(t[0], t[1], t[2], t[3]); g[1] = make_uint4(t[4], t[5], t[6], t[7]); }
            } else if (w == 2u) {
                uint2* g = (uint2*)planes.ptr[p] + grow;
                if (TO_AOS) { const uint2 v = *g; t[0] = v.x; t[1] = v.y; }
                else *g = make_uint2(t[0], t[1]);
            } else {
                u32* g = (u32*)planes.ptr[p] + grow;
                if (TO_AOS) t[0] = *g; else *g = t[0];
            }
        }
    }
    if (TO_AOS) {
        __syncthreads();
        if (vec_ok) for (u32 i = threadIdx.x; i < tile_words / 4u; i += TR_THREADS) ((uint4*)g_tile)[i] = ((const uint4*)tr_tile)[i];
        else for (u32 i = threadIdx.x; i < tile_words; i += TR_THREADS) g_tile[i] = tr_tile[i];
    }
}
// {ping, pong, dead} columns <-> interleaved 12-byte IndirectEntry rows, staged the same way (3 words per row).
#define IL_ROWS 1024
template <bool INTERLEAVE>
__global__ void __launch_bounds__(TR_THREADS) k_indirect_rows(u32* __restrict__ rows3, u32* ping, u32* pong, u32* dead, u32 first, u32 count) {
    __shared__ __align__(16) u32 tile[IL_ROWS * 3];
    const u32 row0 = blockIdx.x * IL_ROWS;
    if (row0 >= count) return;
    const u32 rows = min((u32)IL_ROWS, count - row0);
    u32* const g_tile = rows3 + u64(row0) * 3u;
    const bool vec_ok = ((rows * 3u) & 3u) == 0u && ((u64)(uintptr_t)g_tile & 15ull) == 0ull;
    if (!INTERLEAVE) {
        if (vec_ok) for (u32 i = threadIdx.x; i < rows * 3u / 4u; i += TR_THREADS) ((uint4*)tile)[i] = ((const uint4*)g_tile)[i];
        else for (u32 i = threadIdx.x; i < rows * 3u; i += TR_THREADS) tile[i] = g_tile[i];
        __syncthreads();
    }
    for (u32 r = threadIdx.x; r < rows; r += TR_THREADS) {
        const u64 g = u64(first) + row0 + r;
        if (INTERLEAVE) { tile[3u * r] = ping[g]; tile[3u * r + 1u] = pong[g]; tile[3u * r + 2u] = dead[g]; }
        else { ping[g] = tile[3u * r]; pong[g] = tile[3u * r + 1u]; dead[g] = tile[3u * r + 2u]; }
    }
    if (INTERLEAVE) {
        __syncthreads();
        if (vec_ok) for (u32 i = threadIdx.x; i < rows * 3u / 4u; i += TR_THREADS) ((uint4*)g_tile)[i] = ((const uint4*)tile)[i];
        else for (u32 i = threadIdx.x; i < rows * 3u; i += TR_THREADS) g_tile[i] = tile[i];
    }
}

// rows per CTA of the record transposes: as many as fit 48 KB of shared memory, at most 1024
// (1024 rows of 32 bytes: every thread moves four records per plane, enough loads in flight to cover the two barriers)
static inline u32 transpose_rows(u32 stride_words) { return std::max(1u, std::min(1024u, (48u * 1024u) / (stride_words * 4u))); }
static inline u32 count_planes(const PlaneSet& planes, u32 stride_words) {
    u32 n = 0, covered = 0;
    while (n < HNB_MAX_PLANES && covered < stride_words && planes.words[n]) covered += planes.words[n++];
    return n;
}
cudaError_t launch_aos_to_planes(const u32* aos, const PlaneSet& planes, u32 first, u32 count, u32 stride_words, cudaStream_t st) {
    if (count == 0) return cudaSuccess;
    const u32 rows = transpose_rows(stride_words);
    k_transpose<false><<<blocks_for(count, rows), TR_THREADS, size_t(rows) * stride_words * 4, st>>>(const_cast<u32*>(aos), planes, first, count, stride_words, rows,
                                                                                                   count_planes(planes, stride_words));
    return cudaGetLastError();
}
cudaError_t launch_planes_to_aos(u32* aos, const PlaneSet& planes, u32 first, u32 count, u32 stride_words, cudaStream_t st) {
    if (count == 0) return cudaSuccess;
    const u32 rows = transpose_rows(stride_words);
    k_transpose<true><<<blocks_for(count, rows), TR_THREADS, size_t(rows) * stride_words * 4, st>>>(aos, planes, first, count, stride_words, rows,
                                                                                                  count_planes(planes, stride_words));
    return cudaGetLastError();
}
cudaError_t launch_indirect_interleave(u32* rows3, const u32* ping, const u32* pong, const u32* dead, u32 first, u32 count, cudaStream_t st) {
    if (count == 0) return cudaSuccess;
    k_indirect_rows<true><<<blocks_for(count, IL_ROWS), TR_THREADS, 0, st>>>(rows3, const_cast<u32*>(ping), const_cast<u32*>(pong), const_cast<u32*>(dead), first, count);
    return cudaGetLastError();
}
cudaError_t launch_indirect_deinterleave(const u32* rows3, u32* ping, u32* pong, u32* dead, u32 first, u32 count, cudaStream_t st) {
    if (count == 0) return cudaSuccess;
    k_indirect_rows<false><<<blocks_for(count, IL_ROWS), TR_THREADS, 0, st>>>(const_cast<u32*>(rows3), ping, pong, dead, first, count);
    return cudaGetLastError();
}

}  // namespace hnb
