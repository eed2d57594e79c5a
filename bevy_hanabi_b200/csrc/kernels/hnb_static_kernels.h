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
    // The record words plane p holds, in lane order. A plane of consecutive words: the first one. A word map (a column
    // plan whose column holds words that are not consecutive, DESIGN.md §4.1): HNB_PLANE_WORD_LIST, and lane l's word in
    // bits [6l, 6l + 6).
    u32 word_off[HNB_MAX_PLANES];
    unsigned char word_to_plane[HNB_MAX_PLANES * 4];
};
#define HNB_PLANE_WORD_LIST 0x80000000u
// record word of lane `lane` of plane p
HNB_HD u32 hnb_plane_word(const PlaneSet& s, u32 p, u32 lane) {
    const u32 o = s.word_off[p];
    return (o & HNB_PLANE_WORD_LIST) ? (o >> (6u * lane)) & 63u : o + lane;
}
// lane of record word w in its plane word_to_plane[w]
HNB_HD u32 hnb_word_lane(const PlaneSet& s, u32 w) {
    const u32 o = s.word_off[s.word_to_plane[w]];
    if (!(o & HNB_PLANE_WORD_LIST)) return w - o;
    u32 lane = 0;
    while (lane < 3u && ((o >> (6u * lane)) & 63u) != w) ++lane;
    return lane;
}

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
// header + records i < min(alive_count, rows) in alive-list order. `dead` (the slab's dead stack, row 0): a version-2
// header, and the D records of the slots the last update freed after them; launch_events_translate completes it.
cudaError_t launch_snapshot_gather(const SnapshotArgs& a, u32* dst, cudaStream_t st, const u32* dead = nullptr);
// records i < m to local rows i, and alive_count / max_spawn / particle_counter; enqueue launch_repack_lists after it.
// `channels` != NULL: a version-2 snapshot of that many event channels; also the dead records and max_update.
cudaError_t launch_restore_scatter(const SnapshotArgs& a, const u32* src, cudaStream_t st, const u32* channels = nullptr);

// Append of a version-1 snapshot to one instance (hnb_instance_append): its records go to the slots the next spawns of an
// init would take. Pointers are the slab's row-0 columns; the group words are indexed by slab row / 32.
struct AppendArgs {
    SnapshotArgs s;    // the slice, its planes, its metadata row (read, then written by the commit) and src_bytes
    u32* ping;         // alive-list columns: entries [first + n, first + n + m) of column W are written
    u32* pong;
    const u32* dead;   // dead stack: entries [first + n, first + n + m) name the slots
    u32* alive_bits;   // NULL unless the effect has HNB_EFFECT_SLOT_ORDER
    u32* life_floor;   // the slab's lifetime floors and common ages: the written slots' groups become the sentinel
    u64* group_age;
    u64* claim;        // [2]: the slab's identity claims; column W's is cut to n
};
// The scatter (records, list entries, bits, group words), then one thread for the metadata words and the claim cut.
// Nothing is launched when src_bytes holds no record; `launches` counts the launches made.
cudaError_t launch_append(const AppendArgs& a, const u32* src, cudaStream_t st, u32* launches);

// The event buffers an emitting instance appends to (hnb_batch_launch.emit_events), channels b < count. Channel b's
// pending count is child_infos[metadata->base_child_index + b].event_count (none when that row does not exist).
#define HNB_SNAPSHOT_EVENTS_VERSION_WORD 2u
struct EventChannels {
    u32* buffer[HNB_MAX_EVENT_BINDINGS];
    u32 capacity[HNB_MAX_EVENT_BINDINGS];
    u32 count;
    ChildInfo* child_infos;
    u32 num_child_infos;
};
// inv[src[i]] = i for the repack's source rows (rows words); enqueue before launch_repack_lists
cudaError_t launch_repack_inverse(const RepackArgs& a, u32* inv, cudaStream_t st);
// every pending event e -> inv[e]: in place (`snapshot` NULL), or as record indices into a version-2 snapshot whose
// records launch_snapshot_gather wrote (header words 7-15 and the entries)
cudaError_t launch_events_translate(const RepackArgs& a, const u32* inv, const EventChannels& ev, u32 stride_words, u32* snapshot,
                                    cudaStream_t st);
// the events of a version-2 snapshot into the channels' buffers and event counts; after launch_restore_scatter
cudaError_t launch_restore_events(const SnapshotArgs& a, const u32* src, const EventChannels& ev, cudaStream_t st);

// Bounds of every instance of one batch (hnb_batch_bounds): per component of `position`, the minimum and maximum over the
// instance's live particles in the total order of bounds_key. Everything about the instances is read on the device; the
// host only names the batch's row, the slab's columns and where `position` sits in them.
struct BoundsArgs {
    const BatchInfo* batch_info;     // the batch's row of the device frame block (spawner_base, prefix_sum_count)
    const Spawner* spawners;         // device spawner table, `num_spawners` rows
    const EffectMetadata* metadata;  // device metadata table, `num_metadata` rows
    u32 num_spawners, num_metadata;
    const u32* ping;                 // alive-list columns of the slab (row 0)
    const u32* pong;
    const u64* claim;                // [2]: the slab's identity claims, only read
    u32 capacity_rows;               // rows of the slab
    u32 max_instances;               // records `out` and `acc` hold for this call
    // Word c of `position` is word col_lane[c] of the col_words[c]-word elements of column col[c] (row 0 of the slab).
    // The fast kernel needs the three words in one column at a 16-byte boundary: col[0], col_words[0] and col_lane[0].
    const u32* col[3];
    u32 col_words[3], col_lane[3];
    // 8 slots per instance, all zero between calls: max(~key) of x y z, -, max(key) of x y z, -. A slot is a 64-bit word
    // with the 32-bit key in its low half: 64 bits is the atomicMax width the project's kernels and their CPU emulation use.
    u64* acc;
    void* out;                       // hnb_instance_bounds records (32 bytes each, 16-byte aligned)
};
// One persistent launch that reduces every instance into `acc`, then one that writes the records and zeroes `acc` again.
// `fast`: position's three words share one 16- or 32-byte column. `sm_count`: SMs of the device.
cudaError_t launch_batch_bounds(const BoundsArgs& a, bool fast, u32 sm_count, cudaStream_t st);
#define HNB_BATCH_BOUNDS_LAUNCHES 2u

// Draw order of every instance of one batch (hnb_batch_depth_order): per instance, its live entries sorted by the depth of
// `position` against the instance's plane, farthest first, NaN last, ties in list order, written at its own slab rows of
// `order`. The instances and `position` are found as BoundsArgs describes (its acc and out are not used).
struct DepthOrderArgs {
    BoundsArgs src;
    const float* planes;  // (a, b, c, d) per instance of the batch
    u32* order;           // d_order: indexed by slab row
    // Scratch, one context-owned buffer: 16 bytes per slab row, 1 KiB per tile of the call, 4 KiB + 32 bytes per instance.
    u32* keys[2];         // LSD pass buffers of (key, entry), indexed by slab row
    u32* vals[2];
    u32* hist;            // 256 words per tile: instance j's block at 256 * tile_base, digit-major [digit][tile]
    u32* totals;          // [instance][pass][digit]: digit counts of each instance of more than one tile
    u32* info;            // 8 words per instance (k_do_plan): first, n, tile_base, tiles, W, rows, mask of passes that run
    u32* total_tiles;     // [1]: tiles of the call
    u32 max_tiles;        // depth_order_max_tiles(capacity_rows, max_instances): `hist` holds 256 words per tile
};
// Tiles a call can have: disjoint slices of n_j rows need sum ceil(n_j / tile) <= capacity_rows / tile + instances.
u64 depth_order_max_tiles(u32 capacity_rows, u32 max_instances);
// A fixed sequence of launches whatever the batch holds. `fast`: position's three words share one 16- or 32-byte column.
cudaError_t launch_batch_depth_order(const DepthOrderArgs& a, bool fast, u32 sm_count, cudaStream_t st);
#define HNB_BATCH_DEPTH_ORDER_LAUNCHES 13u

// Visible particles of every instance of one batch (hnb_batch_cull): per instance, the source entries whose `position`
// passes all six planes of the instance's frustum, in source order, at its own slab rows of `visible`, and its draw-args
// row with that count. The instances and `position` are found as BoundsArgs describes (its acc and out are not used);
// the tiles are depth order's (depth_order_max_tiles).
struct CullArgs {
    BoundsArgs src;
    const float* frusta;     // 6 planes (a, b, c, d) per instance of the batch
    const u32* src_list;     // d_src, indexed by slab row; NULL: the alive-list column W
    u32* visible;            // d_visible: indexed by slab row
    u32* args;               // d_args: 5 words (a draw-args row) per instance of the batch, 4-byte aligned
    const u32* draw_args;    // device draw-args table, 5 words per row, `num_draw_args` rows (at least one)
    u32 num_draw_args;
    // Scratch, one context-owned buffer: (DO_TILE / 32 + 1) words per tile of the call, 8 words per instance, 1 word.
    u32* mask;               // DO_TILE / 32 words per tile: bit l of word w = row 32w + l of the tile is visible
    u32* prefix;             // 1 word per tile: its visible count (k_cull_test), then its exclusive prefix in the instance
    u32* info;               // 8 words per instance (the tile plan): first, n, tile_base, tiles, W, rows
    u32* total_tiles;        // [1]: tiles of the call
    u32 max_tiles;           // depth_order_max_tiles(capacity_rows, max_instances)
};
// A fixed sequence of launches whatever the batch holds. `fast`: position's three words share one 16- or 32-byte column.
cudaError_t launch_batch_cull(const CullArgs& a, bool fast, u32 sm_count, cudaStream_t st);
#define HNB_BATCH_CULL_LAUNCHES 4u
#define HNB_BATCH_CULL_MASK_WORDS 128u  // DO_TILE / 32: mask words per tile

// Visible particles of every instance of one batch in up to HNB_BATCH_CULL_MAX_VIEWS views (hnb_batch_cull_views), with
// one shared source: view v's part of each stacked buffer is what a CullArgs with v's frusta, visible and args would
// name. The scratch holds `views` blocks of masks, then `views` blocks of prefixes (max_tiles tiles each), then the
// plan: c.mask, c.prefix = c.mask + views * DO_TILE / 32 * max_tiles, c.info = c.prefix + views * max_tiles.
struct CullViewsArgs {
    CullArgs c;              // view 0's frusta, visible and args, the shared source and the scratch
    u32 views;               // 1 .. HNB_BATCH_CULL_MAX_VIEWS
    u32 frustum_rows;        // view v's frusta: c.frusta + 24 * v * frustum_rows
    u32 visible_rows;        // view v's entries: c.visible + v * visible_rows
    u32 args_rows;           // view v's args rows: c.args + 5 * v * args_rows
};
// The launches of launch_batch_cull (HNB_BATCH_CULL_LAUNCHES), whatever `views` is.
cudaError_t launch_batch_cull_views(const CullViewsArgs& a, bool fast, u32 sm_count, cudaStream_t st);
#define HNB_BATCH_CULL_MAX_VIEWS 8u

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
// common ages of the 32-row groups rows [first, first + count) touch (DESIGN.md §3): deferred ages back into the age word of
// their rows; then, with `clear`, every word and lifetime floor of the range the sentinel, else deferred words known at `epoch`
cudaError_t launch_flush_group_ages(const PlaneSet& planes, u32 age_word, u64* group_age, u32* life_floor, u32 first, u32 count,
                                    u32 capacity, bool clear, u32 epoch, cudaStream_t st);
cudaError_t launch_aos_to_planes(const u32* aos, const PlaneSet& planes, u32 first, u32 count, u32 stride_words, cudaStream_t st);
cudaError_t launch_planes_to_aos(u32* aos, const PlaneSet& planes, u32 first, u32 count, u32 stride_words, cudaStream_t st);
cudaError_t launch_indirect_interleave(u32* rows3, const u32* ping, const u32* pong, const u32* dead, u32 first, u32 count, cudaStream_t st);
cudaError_t launch_indirect_deinterleave(const u32* rows3, u32* ping, u32* pong, u32* dead, u32 first, u32 count, cudaStream_t st);
// also sets the identity claims `claim[2]` of both columns to {first, count}
cudaError_t launch_fill_c5(const PlaneSet& planes, u32* ping, u32* pong, u64* claim, u32 first, u32 count, u32 seed, f32 lo, f32 hi, u32 logical_first, cudaStream_t st);
cudaError_t launch_measure_sm_clock(u64* out2, u64 window_ns, cudaStream_t st);
cudaError_t launch_checksum(const PlaneSet& planes, u32 first, u32 count, u32 stride_words, u64 index_base, u64* out, cudaStream_t st);

}  // namespace hnb
