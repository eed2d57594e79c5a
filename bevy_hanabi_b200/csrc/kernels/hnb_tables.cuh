// hnb_tables.cuh — device-side view of the GPU tables shared by all kernels. Tight C layouts of the
// reference structs (src/render/mod.rs:135-622, src/render/vfx_common.wgsl:3-255; byte layouts in
// SURVEY.md Appendix A), identical to the host structs in include/hanabi_b200.h.
//
// Compiled by NVRTC (after hnb_wgsl.cuh, which provides u32/i32/f32) and by nvcc.
#pragma once

#ifndef HNB_SCALAR_TYPEDEFS
#define HNB_SCALAR_TYPEDEFS
typedef float f32;
typedef int i32;
typedef unsigned int u32;
typedef unsigned long long u64;
#endif

namespace hnb {

struct SimParams {  // GpuSimParams, mod.rs:218
    f32 delta_time, time, virtual_delta_time, virtual_time, real_delta_time, real_time;
    u32 num_effects;
};

struct Spawner {  // GpuSpawnerParams, mod.rs:381; 128 B
    f32 transform[12];          // rows x,y,z of the affine matrix
    f32 inverse_transform[12];
    i32 spawn;
    u32 seed;
    u32 render_indirect_read_index;
    u32 effect_metadata_index;
    u32 draw_indirect_index;
    u32 slab_offset;
    u32 parent_slab_offset;
    u32 unused;
};

struct BatchInfo {  // GpuBatchInfo, mod.rs:537; 24 B
    u32 total_spawn_count, total_update_count, spawner_base, base_particle, prefix_sum_offset, prefix_sum_count;
};

struct EffectMetadata {  // GpuEffectMetadata, mod.rs:566; 60 B
    u32 capacity, alive_count, max_update, max_spawn, indirect_write_index, indirect_render_index,
        init_indirect_dispatch_index, properties_array_index, local_child_index, global_child_index,
        base_child_index, particle_stride, sort_key_offset, sort_key2_offset, particle_counter;
};

struct ChildInfo {  // GpuChildInfo, event.rs:204
    u32 init_indirect_dispatch_index;
    i32 event_count;
};

// ---- update tile size word (BatchParams::tile_rows, StaticTables::batch_tile_size) -----------------------------
//   [15:0]  S  rows of a tile, a multiple of 32*K
//   [31]    slot order (HNB_EFFECT_SLOT_ORDER): tiles cut the instance's SLOTS [0, capacity), not its alive-list rows
// An instance with `rows` rows (alive particles, or slots in slot order) has ceil(rows / S) tiles; the bookkeeping
// kernels and hnb_update share this rule.
#if defined(__CUDACC__) || defined(__CUDACC_RTC__)
#define HNB_HD __host__ __device__ __forceinline__
#else
#define HNB_HD inline
#endif
#define HNB_TILE_SLOT_ORDER 0x80000000u
HNB_HD u32 hnb_tile_rows(u32 word) { return word & 0xffffu; }
HNB_HD u32 hnb_tile_count(u32 rows, u32 word) {
    const u32 S = hnb_tile_rows(word);
    return (rows + S - 1u) / S;
}

// ---- identity claim of an alive-list column (SlabView::ident_claim, DESIGN.md §3) ------------------------------
// One 64-bit word per index column: (base << 32) | len means  particle_index[c][base + i] == i  for every i < len that lies
// in the slice of the instance whose slab offset is `base` (0: no claim). An ordered update pass reads no alive-list entry the
// claim covers and stores no entry that already holds its value. Every writer of an index column keeps the claim true or
// shrinks it, in stream order, before any later reader. The word is always read and written as ONE aligned 64-bit access:
// update passes of other batches on side streams may read it concurrently and must never see a new base with an old length.
HNB_HD u64 hnb_claim_pack(u32 base, u32 len) { return (u64(base) << 32) | u64(len); }
HNB_HD u64 hnb_claim_load(const u64* claim) { return *(const volatile u64*)claim; }
HNB_HD void hnb_claim_store(u64* claim, u64 word) { *(volatile u64*)claim = word; }
// length of the claim `word` for the instance at slab offset `base` (0 when the claim is another instance's)
HNB_HD u32 hnb_claim_len(u64 word, u32 base) { return u32(word >> 32) == base ? u32(word) : 0u; }

#define HNB_DRAW_INDEXED_INDIRECT_STRIDE 5u  // vfx_common.wgsl:146
#define HNB_MAX_PLANES 16
#define HNB_MAX_EVENT_BINDINGS 4
#define HNB_INVALID 0xFFFFFFFFu

// Header of the per-frame block the host uploads with ONE copy before each simulate():
// sim params + frame epoch, followed (at fixed capacity-derived offsets) by the spawner rows, the
// per-effect init thread ranges, the CPU spawn prefix sums and the batch infos.
struct FrameHeader {
    SimParams sim;
    u32 epoch;        // monotonically increasing, never 0: validates decoupled look-back tile states
    u32 num_batches;
    u32 _pad[7];
};  // 64 B

// Slab columns: SoA planes of the AoS record + the three u32 indirection columns
// (IndirectEntry {particle_index[2], dead_index}, vfx_common.wgsl:66-78, stored column-wise).
struct SlabView {
    void* planes[HNB_MAX_PLANES];
    u32* particle_index[2];  // ping / pong alive lists (instance-local particle indices)
    u32* dead_index;         // dead stack (slab-global rows)
    u32* alive_bits;         // one bit per slab row: the row holds a particle (kept current by HNB_EFFECT_SLOT_ORDER effects)
    u64* ident_claim;        // [2]: identity claim of particle_index[0] / [1] (see hnb_claim_pack); NULL = no claims
    u32 capacity_rows;
    u32 _pad;
};

// Everything one init/update launch needs. Passed by value as the single kernel parameter.
struct BatchParams {
    const FrameHeader* frame;
    Spawner* spawners;               // whole table; batch rows start at batch_info->spawner_base
    const u32* spawn_prefix;         // CPU prefix sums of spawn counts (never rewritten on device)
    const u32* prefix_sum;           // GPU-rewritten prefix (alive counts) — same indexing
    const u32* tile_prefix;          // exclusive scan of per-effect update tile counts — same indexing
    const BatchInfo* batch_info;     // this batch's row
    const u32* batch_tiles;          // this batch's total update tile count
    u32* ticket;                     // this batch's dynamic tile ticket counter
    unsigned long long* tile_state;  // this batch's decoupled look-back states
    EffectMetadata* metadata;
    u32* draw_args;                  // DrawIndexedIndirectArgs rows as u32[5]
    ChildInfo* child_infos;
    const void* properties;          // array<Properties> of the effect
    SlabView slab;
    SlabView parent_slab;
    const u32* consume_events;       // event buffer read by init
    u32* emit_events[HNB_MAX_EVENT_BINDINGS];
    u32 emit_events_capacity[HNB_MAX_EVENT_BINDINGS];
    u32 init_thread_count;           // ceil64(total_spawn_count): logical init threads of this launch
    u32 properties_stride;           // bytes
    u32 tile_rows;                   // tile size word of this launch (see hnb_tile_rows): rows per tile (multiple of 32*K, <= 32*K*HNB_MAX_CHUNKS) + flags
    u32 _pad0;
    unsigned long long* debug;       // 16 counters, written only by kernels compiled with HNB_PROFILE=1
    u32* event_counts[HNB_MAX_EVENT_BINDINGS];  // HNB_EFFECT_ORDERED_EVENTS: events requested by update row r on channel b (else NULL)
    // Count mailbox (hnb_ctx_set_count_mailbox; NULL = none): pinned HOST memory, `mailbox_ring` slots of `mailbox_rows` 64-bit
    // words. The last tile of an instance stores (epoch << 32) | instance_count at [(epoch % ring) * rows + draw-indirect row]:
    // the host learns a frame's counts by reading its own memory — no copy, no event, nothing between two kernels of the chain.
    unsigned long long* mailbox;
    u32 mailbox_rows, mailbox_ring;
    u32 late_tables;
    // this batch's GpuBatchInfo words the kernels need (the host knows them when it launches: no dependent load for them)
    u32 bi_spawner_base, bi_prefix_sum_offset, bi_prefix_sum_count;
    u32 first_md_index;              // effect_metadata_index of the batch's first instance (used when the batch has exactly one)          // 1: the host-written tables are stored by the kernel just ahead (k_frame_block): read them after the wait
    // 1: the update may leave common-age words deferred (HNB_GROUP_AGE_DEFERRED) and consumes the deferred words it meets.
    // 0: no word is deferred and none is made so.
    u32 defer_ages;
    // Lifetime floors of the slab (HNB_LIFE_FLOOR effects, DESIGN.md §3): one f32 per 32 slab rows, a lower bound of the
    // lifetimes of the group's particles, or HNB_LIFE_FLOOR_NONE. NULL: the slab uses no floors. Kept out of SlabView so
    // that the parameter offsets, and the code, of effects without floors stay as they were.
    f32* life_floor;
    // Common ages of the slab (HNB_GROUP_AGE effects, DESIGN.md §3): one 64-bit word per 32 slab rows, (epoch << 32) | the
    // age bits every row of the group held after the update of frame `epoch`. Only a word of the previous frame's epoch is
    // known; all bits set: unknown. NULL: the slab keeps none (always NULL when life_floor is).
    // Deferred (bits 63:62 = 01, with defer_ages): bits 31:0 are the age of every row of the group, whose age column is
    // stale; bits 37:32 count the rows an update outside a floor tile has already taken the age from (see hnb_update).
    // The array ends with one more word past the groups' (hnb_deferred_groups): how many words are deferred.
    u64* group_age;
};
#define HNB_GROUP_AGE_DEFERRED (1ull << 62)
HNB_HD bool hnb_group_age_deferred(u64 word) { return (word >> 62) == 1ull; }
// The count of deferred words of a slab of `capacity_rows` rows: never below the number of deferred words that a walker
// other than the one that stored them may meet. Updates outside floor tiles read no word while it is 0.
HNB_HD u64* hnb_deferred_groups(u64* group_age, u32 capacity_rows) { return group_age + (capacity_rows >> 5) + 1u; }
// All bits set: a NaN, against which every comparison is false, so it proves nothing (0.0 would: ages can be negative).
// Also the unknown common age (an age column whose bits are all ones never has a known common age).
#define HNB_LIFE_FLOOR_NONE 0xffffffffu
#define HNB_GROUP_AGE_NONE 0xffffffffffffffffull

}  // namespace hnb
