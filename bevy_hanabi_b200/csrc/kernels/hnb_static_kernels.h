// hnb_static_kernels.h — host-callable launchers of the ahead-of-time compiled kernels
// (hnb_static_kernels.cu). Includable from plain C++ (g++) and from nvcc.
#pragma once
#include <cuda_runtime.h>

#include "hnb_tables.cuh"

namespace hnb {

// Device pointers of the context-wide tables used by the per-instance / per-batch passes.
struct StaticTables {
    const FrameHeader* frame;
    Spawner* spawners;
    u32* spawn_range;        // per instance: init threads mapped to it this frame (bit31: event driven); zeroed after use
    u32* prefix_sum;
    u32* tile_prefix;
    BatchInfo* batch_infos;
    const u32* batch_tile_size;  // per batch: tile size word (hnb_tile_word) of the batch's compiled effect and launch
    u32* dispatch_args;      // DispatchIndirectArgs rows as u32[3]
    u32* batch_tiles;
    u32* tickets;
    EffectMetadata* metadata;
    u32* draw_args;
    ChildInfo* child_infos;
    u32 num_child_infos;
};

// SoA planes of one slab, with the word -> plane map used by the AoS <-> SoA transposes.
struct PlaneSet {
    void* ptr[HNB_MAX_PLANES];
    u32 words[HNB_MAX_PLANES];     // u32 words per row of plane p (4, 2 or 1)
    u32 word_off[HNB_MAX_PLANES];  // first AoS word covered by plane p
    unsigned char word_to_plane[HNB_MAX_PLANES * 4];
};

// Ribbon sort of one batch (hnb_ribbon_sort.cu): every instance of the batch has its freshly written alive-list
// column stably sorted by (particle[sort_key_offset], particle[sort_key2_offset]).
#define HNB_RIBBON_SORT_SMALL_MAX 2048u
struct RibbonSortArgs {
    PlaneSet planes;            // particle planes of the slab
    u32* ping;                  // alive-list columns of the slab (row 0 of the slab)
    u32* pong;
    const Spawner* spawners;
    const EffectMetadata* metadata;
    u32 spawner_base;           // first instance of the batch (BatchInfo::spawner_base)
    u32 instance_count;         // BatchInfo::prefix_sum_count
    // scratch of the large path (unused when every instance has <= HNB_RIBBON_SORT_SMALL_MAX rows)
    u64* scratch_keys[2];
    u32* scratch_vals[2];
    u32* scratch_hist;          // ribbon_sort_hist_words(scratch_grid) words; the first 2*8*256 zero at launch
    u32 scratch_rows;
    u32 scratch_grid;
};
cudaError_t launch_ribbon_sort(const RibbonSortArgs& args, bool any_large, u32 sm_count, cudaStream_t st, u32* launches);
size_t ribbon_sort_hist_words(u32 grid);

// Ordered event append of one emitting instance and one channel (HNB_EFFECT_ORDERED_EVENTS).
struct EventAppendArgs {
    const u32* counts;              // events requested by update row r (written by hnb_update)
    const u32* ping;                // alive-list columns of the parent's slab
    const u32* pong;
    const Spawner* spawner;         // the emitting instance (slab_offset)
    const EffectMetadata* metadata; // its row: max_update rows were updated, indirect_write_index tells the read column
    u32* block_sums;                // scratch: one word per 2048 rows of slab capacity
    ChildInfo* child_infos;         // event_count of row metadata->base_child_index + binding += total
    u32 binding;                    // event channel
    u32* buffer;                    // the child's event buffer
    u32 capacity;                   // ... and its length
};
cudaError_t launch_ordered_event_append(const EventAppendArgs& a, u32 capacity_rows, cudaStream_t st);
inline u32 ordered_event_blocks(u32 capacity_rows) { return (capacity_rows + 2047u) / 2048u; }

// Repack of one instance (hnb_slab_repack): slab rows [first, first+rows), its metadata row (alive_count, and
// indirect_write_index naming the alive list to follow). Pointers are the slab's row-0 columns.
struct RepackArgs {
    const EffectMetadata* metadata;
    u32* ping;
    u32* pong;
    u32* dead;
    u32* alive_bits;
    u64* claim;  // [2]: the slab's identity claims
    u32 first, rows;
};
// scratch[i] = col[first + src[i]] for i < rows, `width` = bytes per element of the column (4, 8, 16 or 32)
cudaError_t launch_repack_gather(const RepackArgs& a, const void* col, void* scratch, u32 width, cudaStream_t st);
// lists, claims and alive bits; enqueue after every gather of the instance
cudaError_t launch_repack_lists(const RepackArgs& a, cudaStream_t st);

// Snapshot / restore of one instance (hnb_instance_snapshot / hnb_instance_restore): the header words of
// hnb_instance_snapshot_header (include/hanabi_b200.h), then reference AoS records of stride_words words each.
#define HNB_SNAPSHOT_HEADER_WORDS 16u
#define HNB_SNAPSHOT_MAGIC_WORD 0x53424E48u  // "HNBS" in little-endian byte order
#define HNB_SNAPSHOT_VERSION_WORD 1u
struct SnapshotArgs {
    EffectMetadata* metadata;  // the instance's row: read by a snapshot, written by a restore
    const u32* ping;           // alive-list columns of the slab (row 0), read by a snapshot
    const u32* pong;
    PlaneSet planes;           // the slab's physical columns (row 0)
    u32 num_planes;
    u32 stride_words;          // the effect's record stride
    u32 first, rows;           // the slice
    u64 src_bytes;             // restore: bytes readable at the source (>= 64)
};
// header + records i < min(alive_count, rows) in alive-list order
cudaError_t launch_snapshot_gather(const SnapshotArgs& a, u32* dst, cudaStream_t st);
// records i < m to local rows i, and alive_count / max_spawn / particle_counter; enqueue launch_repack_lists after it
cudaError_t launch_restore_scatter(const SnapshotArgs& a, const u32* src, cudaStream_t st);

cudaError_t launch_indirect(const StaticTables& T, u32 num_effects, cudaStream_t st);
cudaError_t launch_prefix_sum(const StaticTables& T, u32 num_batches, cudaStream_t st);
cudaError_t launch_tile_prefix(const StaticTables& T, u32 batch_index, u32 tile, cudaStream_t st);
// `frame_block` / `block_bytes`: the first bytes of the HOST frame arena to carry in the kernel's parameter space and store into
// T.frame from there — NULL / 0: the host copied the frame block; sizeof(FrameHeader): the header only; up to
// HNB_FRAME_BLOCK_MAX_BYTES: header + every host-written table. Launched with programmatic stream serialization.
#define HNB_FRAME_BLOCK_MID_BYTES 3840u    // fits the classic 4 KB parameter space together with the table pointers
#define HNB_FRAME_BLOCK_MAX_BYTES 30720u   // CUDA 12.1+ on sm_70+: 32764 bytes of kernel parameters
cudaError_t launch_bookkeeping(const StaticTables& T, u32 num_effects, u32 num_batches, const void* frame_block, u32 block_bytes, cudaStream_t st);
// the same block at the head of a frame that has an init pass (a one-CTA kernel stores it into the device arena)
cudaError_t launch_frame_block(void* device_arena, const void* frame_block, u32 block_bytes, cudaStream_t st);
cudaError_t launch_fill_dispatch_args(const u32* src, u32* dst, u32 src_offset, u32 src_stride, u32 dst_offset,
                                      u32 dst_stride, u32 count, cudaStream_t st);
cudaError_t launch_slab_reset(u32* ping, u32* pong, u32* dead, u32 first, u32 count, cudaStream_t st);
// alive bitmap of a slab (HNB_EFFECT_SLOT_ORDER): set / clear the bits of a row range; set the bits an alive list names
cudaError_t launch_bits_range(u32* bits, u32 first, u32 count, bool set, cudaStream_t st);
cudaError_t launch_bits_from_list(u32* bits, const u32* list, u32 base, u32 alive_count, cudaStream_t st);
cudaError_t launch_aos_to_planes(const u32* aos, const PlaneSet& planes, u32 first, u32 count, u32 stride_words, cudaStream_t st);
cudaError_t launch_planes_to_aos(u32* aos, const PlaneSet& planes, u32 first, u32 count, u32 stride_words, cudaStream_t st);
cudaError_t launch_indirect_interleave(u32* rows3, const u32* ping, const u32* pong, const u32* dead, u32 first, u32 count, cudaStream_t st);
cudaError_t launch_indirect_deinterleave(const u32* rows3, u32* ping, u32* pong, u32* dead, u32 first, u32 count, cudaStream_t st);
// also sets the identity claims `claim[2]` of both columns to {first, count}
cudaError_t launch_fill_c5(void* pos_age, void* vel_life, u32* ping, u32* pong, u64* claim, u32 first, u32 count, u32 seed, f32 lo, f32 hi, u32 logical_first, cudaStream_t st);
cudaError_t launch_measure_sm_clock(u64* out2, u64 window_ns, cudaStream_t st);
cudaError_t launch_checksum(const PlaneSet& planes, u32 first, u32 count, u32 stride_words, u64 index_base, u64* out, cudaStream_t st);

}  // namespace hnb
