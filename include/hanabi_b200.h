/*
 * hanabi_b200.h — C ABI of the H100-native Hanabi particle simulation backend.
 *
 * This is the drop-in boundary for the hot path of djeedai/bevy_hanabi: it replaces the
 * wgpu compute dispatch recorded by `simulate()` (reference src/render/mod.rs:6942-7613)
 * and the GPU buffers that function touches.  A Rust `HanabiRenderPlugin` replacement
 * would bind exactly these entry points with `extern "C"` (see INTEGRATION.md); in this
 * repository they are bound by ctypes (bevy_hanabi_b200/_native.py).
 *
 * Conventions
 *   - every function returns int32_t: 0 = HNB_OK, negative = hnb_status error
 *   - no exceptions cross the boundary; hnb_last_error() returns a thread-local message
 *   - all pointers are caller-owned host memory unless stated otherwise
 *   - one context per GPU; a context is NOT thread-safe (one caller thread, like the
 *     reference's render thread)
 *   - struct layouts are the tight C versions of the reference's GPU structs
 *     (reference src/render/mod.rs:135-622); WebGPU alignment padding is not reproduced
 *
 * Two layers:
 *   Level 1 (runtime, sections 1-6): what `simulate()` and the buffer caches bind.
 *   Level 2 (authoring/codegen, section 7+): replaces src/graph + src/modifier +
 *     EffectShaderSources::generate, lowering to CUDA C instead of WGSL. It exists in
 *     this library because the Rust toolchain is absent; a Rust host could keep its own
 *     Module/Expr and call only Level 1 with already-lowered code.
 */
#ifndef HANABI_B200_H
#define HANABI_B200_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HNB_API __attribute__((visibility("default")))

/* ------------------------------------------------------------------------------------ */
/* 0. Status codes                                                                       */
/* ------------------------------------------------------------------------------------ */
typedef enum hnb_status {
    HNB_OK = 0,
    HNB_ERR_INVALID_ARG = -1,
    HNB_ERR_CUDA = -2,          /* CUDA runtime/driver failure, see hnb_last_error() */
    HNB_ERR_NVRTC = -3,         /* generated kernel failed to compile, log in hnb_last_error() */
    HNB_ERR_NO_DEVICE = -4,     /* no CUDA device / driver: the product path never falls back to CPU */
    HNB_ERR_OUT_OF_RANGE = -5,
    HNB_ERR_EXPR = -6,          /* expression / modifier evaluation error (ExprError in the reference) */
    HNB_ERR_LAYOUT = -7,        /* invalid particle or property layout */
    HNB_ERR_NOT_READY = -8,     /* resource missing: simulate() skips instead of desynchronising buffers
                                   (reference mod.rs:6994-7022) */
    HNB_ERR_BATCH_COVERAGE = -9 /* batches must tile [0,num_effects) of the spawner table */
} hnb_status;

/** Thread-local message describing the last error returned on this thread. */
HNB_API const char* hnb_last_error(void);
/** Library version string. */
HNB_API const char* hnb_version(void);

/* ------------------------------------------------------------------------------------ */
/* 1. GPU table rows (reference src/render/mod.rs, SURVEY Appendix A)                    */
/* ------------------------------------------------------------------------------------ */

/** GpuSimParams (reference mod.rs:218-243, vfx_common.wgsl:3-20). 28 bytes. */
typedef struct hnb_sim_params {
    float delta_time, time, virtual_delta_time, virtual_time, real_delta_time, real_time;
    uint32_t num_effects;
} hnb_sim_params;

/** GpuCompressedTransform (reference mod.rs:291): three rows of the 4x4 affine matrix. */
typedef struct hnb_transform {
    float x_row[4], y_row[4], z_row[4];
} hnb_transform;

/** GpuSpawnerParams (reference mod.rs:381-415, vfx_common.wgsl:22-57). 128 bytes. */
typedef struct hnb_spawner {
    hnb_transform transform;
    hnb_transform inverse_transform;
    int32_t spawn;
    uint32_t seed;
    uint32_t render_pong; /* written by the indirect pass */
    uint32_t effect_metadata_index;
    uint32_t draw_indirect_index;
    uint32_t slab_offset;
    uint32_t parent_slab_offset; /* 0xFFFFFFFF if none */
    uint32_t _pad;
} hnb_spawner;

/** GpuBatchInfo (reference mod.rs:537-555, vfx_common.wgsl:149-170). 24 bytes. */
typedef struct hnb_batch_info {
    uint32_t total_spawn_count;
    uint32_t total_update_count; /* written by the prefix-sum pass */
    uint32_t spawner_base;
    uint32_t base_particle;
    uint32_t prefix_sum_offset;
    uint32_t prefix_sum_count;
} hnb_batch_info;

/** GpuEffectMetadata (reference mod.rs:566-622, vfx_common.wgsl:186-255). 60 bytes. */
typedef struct hnb_effect_metadata {
    uint32_t capacity;
    uint32_t alive_count;
    uint32_t max_update;
    uint32_t max_spawn;
    uint32_t indirect_write_index;
    uint32_t indirect_draw_index;
    uint32_t init_indirect_dispatch_index;
    uint32_t properties_array_index;
    uint32_t local_child_index;
    uint32_t global_child_index;
    uint32_t base_child_index;
    uint32_t particle_stride; /* in u32 */
    uint32_t sort_key_offset;
    uint32_t sort_key2_offset;
    uint32_t particle_counter;
} hnb_effect_metadata;

/** GpuDrawIndexedIndirectArgs (reference mod.rs:514-520); stride 5 u32. */
typedef struct hnb_draw_indexed_indirect_args {
    uint32_t index_count;
    uint32_t instance_count; /* written by the update pass */
    uint32_t first_index;
    int32_t base_vertex;
    uint32_t first_instance;
} hnb_draw_indexed_indirect_args;

/** GpuDispatchIndirectArgs (reference mod.rs:462). */
typedef struct hnb_dispatch_indirect_args {
    uint32_t x, y, z;
} hnb_dispatch_indirect_args;

/** GpuIndirectIndex (reference mod.rs:139-146): one interleaved row of the indirect buffer. */
typedef struct hnb_indirect_index {
    uint32_t ping, pong, dead;
} hnb_indirect_index;

/** GpuChildInfo (reference event.rs:204). */
typedef struct hnb_child_info {
    uint32_t init_indirect_dispatch_index;
    int32_t event_count;
} hnb_child_info;

/* ------------------------------------------------------------------------------------ */
/* 2. Context                                                                            */
/* ------------------------------------------------------------------------------------ */
typedef struct hnb_ctx hnb_ctx;

/**
 * Create a context on CUDA device `cuda_device`. `external_stream` is a cudaStream_t cast to
 * uintptr_t on which all work is enqueued (0 = the context creates its own non-blocking
 * stream). Fails with HNB_ERR_NO_DEVICE when no GPU/driver is present: there is no CPU path.
 */
HNB_API int32_t hnb_ctx_create(int32_t cuda_device, uintptr_t external_stream, hnb_ctx** out);
HNB_API void hnb_ctx_destroy(hnb_ctx* ctx);
/** Block until all work enqueued on the context stream has completed. */
HNB_API int32_t hnb_sync(hnb_ctx* ctx);
/** The cudaStream_t (as uintptr_t) work is enqueued on. */
HNB_API uintptr_t hnb_ctx_stream(hnb_ctx* ctx);
/** Number of kernels launched by this context since creation (for bench `gpu_launches`). */
HNB_API uint64_t hnb_ctx_launch_count(hnb_ctx* ctx);
/** hnb_simulate() calls so far, and how many of them had to copy the frame block host->device (the others carried the
 *  64-byte frame header in kernel parameter space: no table row, tile size or init range had changed). */
HNB_API void hnb_ctx_frame_count(hnb_ctx* ctx, uint64_t* frames, uint64_t* frame_block_copies);

/* ------------------------------------------------------------------------------------ */
/* 3. Particle slabs ≙ ParticleSlab::new (reference src/render/effect_cache.rs:246-356)  */
/* ------------------------------------------------------------------------------------ */
typedef uint32_t hnb_slab;
typedef uint32_t hnb_effect;  /* a compiled effect registered with a context (section 4) */
typedef uint32_t hnb_event_buffer;  /* an event buffer of GPU spawn events (section 5) */

/**
 * Allocate a slab of `capacity_rows` particles whose reference AoS record is
 * `particle_stride_bytes` (ParticleLayout::min_binding_size, attributes.rs:1837).
 * Storage is SoA: one zero-filled block of capacity_rows x stride bytes, carved into columns (float4, float2 or u32
 * elements) by a column plan (hnb_effect_column_plan), plus three u32 columns ping/pong/dead. dead[i] = i
 * (effect_cache.rs:309-322); ping/pong = 0. Every plan fits the same block, so the plan is chosen late: the first effect
 * bound to the slab (its first init/update launch, hnb_slab_repack or hnb_instance_restore) fixes that effect's plan.
 * Before that the slab is in the default cut (what hnb_slab_device_view shows, and where hnb_slab_fill_c5 and the AoS
 * uploads write); records written before the first bind move to the effect's columns then, once, after the launches of
 * that call were validated (a device copy through a second block of capacity x stride bytes, and one synchronisation; if
 * the block cannot be allocated the slab keeps the default cut). hnb_slab_device_view pins the plan it shows. A child
 * reads its parent slab in whatever plan the slab has. An effect bound later to a slab of another plan runs a
 * module compiled for the slab's plan (hnb_ctx_plan_compiles). Slabs of HNB_SLAB_SECTOR_PLANES keep the sector cut.
 * A plan with columns narrower than 16 bytes costs more DRAM sectors per gathered record once an effect's alive list has
 * become a permutation of its slice (C5: 4 sectors read and 3 written instead of 2 and 2); hnb_slab_repack or
 * HNB_EFFECT_SLOT_ORDER restore coalesced access, sector planes halve the sectors of 16-byte pieces.
 */
HNB_API int32_t hnb_slab_create(hnb_ctx* ctx, uint32_t capacity_rows, uint32_t particle_stride_bytes,
                                hnb_slab* out);
/** Slab layout options. HNB_SLAB_SECTOR_PLANES: pairs of 16-byte record pieces share one 32-byte-wide column, so the
 *  two pieces a gather reads are ONE full DRAM sector. For long-running effects whose alive list has become a permutation
 *  of the slab (spawning into recycled slots) 16-byte-wide columns waste half of every sector (DESIGN.md §10); coalesced
 *  access is unchanged. Effects for such a slab are compiled with HNB_EFFECT_SECTOR_PLANES. Experimental: validated under
 *  the CPU kernel emulation, not yet measured on a GPU. */
enum { HNB_SLAB_SECTOR_PLANES = 1u << 0 };
HNB_API int32_t hnb_slab_create_ex(hnb_ctx* ctx, uint32_t capacity_rows, uint32_t particle_stride_bytes, uint32_t flags, hnb_slab* out);
HNB_API int32_t hnb_slab_destroy(hnb_ctx* ctx, hnb_slab slab);
/** Re-initialise dead[i]=i, ping=pong=0 for rows [first,first+count) (SURVEY App. D item 5). */
HNB_API int32_t hnb_slab_reset_rows(hnb_ctx* ctx, hnb_slab slab, uint32_t first, uint32_t count);
/** Rebuild the slab's alive bitmap (HNB_EFFECT_SLOT_ORDER) for the instance occupying rows [first,first+rows) from its
 *  alive list: the first `alive_count` entries of indirection column `column` (0 = ping, 1 = pong). Needed only after state
 *  was brought in from outside (hnb_slab_upload_* / import); the init and update passes keep the bitmap current. */
HNB_API int32_t hnb_slab_rebuild_alive_bits(hnb_ctx* ctx, hnb_slab slab, uint32_t first, uint32_t rows, uint32_t column,
                                            uint32_t alive_count);
/** Upload/download particles in the reference AoS layout (rows [first,first+count)). */
HNB_API int32_t hnb_slab_upload_aos(hnb_ctx* ctx, hnb_slab slab, uint32_t first, uint32_t count,
                                    const void* particles_aos);
HNB_API int32_t hnb_slab_download_aos(hnb_ctx* ctx, hnb_slab slab, uint32_t first, uint32_t count,
                                      void* particles_aos);
/** Upload/download the interleaved {ping,pong,dead} rows of the reference IndirectBuffer. */
HNB_API int32_t hnb_slab_upload_indirect(hnb_ctx* ctx, hnb_slab slab, uint32_t first, uint32_t count,
                                         const hnb_indirect_index* rows);
HNB_API int32_t hnb_slab_download_indirect(hnb_ctx* ctx, hnb_slab slab, uint32_t first, uint32_t count,
                                           hnb_indirect_index* rows);
/**
 * Device-side fill used by benchmarks and large-scale property tests (no host buffer):
 * rows [first,first+count) become alive with alive-list = identity, position/velocity
 * ~U(-1,1)^3 from a counter-based PCG stream seeded by `seed`, age 0, lifetime uniform in
 * [lifetime_lo, lifetime_hi]. Only valid for the 32-byte {position,age,velocity,lifetime}
 * layout (SURVEY §8d config C5). Does not touch metadata rows.
 */
HNB_API int32_t hnb_slab_fill_c5(hnb_ctx* ctx, hnb_slab slab, uint32_t first, uint32_t count,
                                 uint32_t seed, float lifetime_lo, float lifetime_hi);
/** The same fill for a SHARD of a logical instance split by index range over several devices (SURVEY.md §8e): slab rows
 *  [first,first+count) receive the values of logical rows [logical_first, logical_first+count) — what a single-GPU slab
 *  holding the whole instance would have there — under shard-local particle indices. */
HNB_API int32_t hnb_slab_fill_c5_ex(hnb_ctx* ctx, hnb_slab slab, uint32_t first, uint32_t count,
                                    uint32_t seed, float lifetime_lo, float lifetime_hi, uint32_t logical_first);
/**
 * Repack one instance so that its particles are contiguous again and the update pass reads its alive list as the identity
 * (coalesced record access, and the 64 B per particle-step path of DESIGN.md §4.1). A long-running effect spawns into
 * whatever slots died, so its alive list drifts into a permutation of its slice; call this between frames, for example
 * every few seconds for each long-running instance.
 *
 * The instance occupies slab rows [first, first+rows) (`rows` must be its capacity: a precondition, not checked on the
 * device), its metadata row is `metadata_row`, and `effect` is the effect it runs. Call it between hnb_simulate calls,
 * where the update invariant holds. With W = indirect_write_index and n = min(alive_count, rows) read from the DEVICE
 * metadata row, list = column W (instance-local values) and dead = the dead stack (slab-global values):
 *   - local row i takes the record of local row src[i], for every plane and all `rows` rows (dead ones too):
 *     src[i] = list[first+i] for i < n, dead[first+i] - first for n <= i < rows (alive slots in list order, then dead slots
 *     in stack order; a bijection when the invariant holds);
 *   - ping[first+i] = pong[first+i] = i for i < n (rows >= n of both columns are left as they are);
 *     dead[first+i] = first+i for n <= i < rows (rows < n are left as they are), so later spawns take slots n, n+1, ...;
 *   - both identity claims of the slab become {first, n} (a claim another instance of the slab held is dropped);
 *   - the alive bitmap of the slice has bits < n set and the rest cleared (HNB_EFFECT_SLOT_ORDER).
 * Metadata, draw args, spawners, counters and the count mailbox do not change. Ribbon effects may be repacked: the
 * repack makes the sorted order the slot order, and PREV/NEXT words move with their record unchanged (no pass maintains
 * links: they keep the value init gave them).
 *
 * Work is only enqueued on the context stream (no host synchronisation, no device->host read): it is ordered after
 * every launch of the previous hnb_simulate and before the next one. A state that breaks the invariant gives an
 * unspecified result, but no access outside the slice. The scratch (rows x the widest physical column: 1 GiB for a
 * 64 Mi-row 32-byte instance) comes from cudaMallocAsync on the context stream and is released the same way.
 * HNB_ERR_INVALID_ARG, with nothing enqueued, when the rows lie outside the slab, the metadata row is out of range, the
 * effect's stride or HNB_EFFECT_SECTOR_PLANES flag does not match the slab, or the effect has
 * HNB_EFFECT_EMIT_GPU_SPAWN_EVENTS (pending events name parent slots that the child's next init reads).
 */
HNB_API int32_t hnb_slab_repack(hnb_ctx* ctx, hnb_slab slab, hnb_effect effect, uint32_t metadata_row, uint32_t first,
                                uint32_t rows);

/**
 * Snapshots of one instance's live particles, in a device buffer the caller owns: a 64-byte header written on the device,
 * then `count` reference AoS `Particle` records (the effect's particle_stride bytes each) in alive-list order. The first
 * 64 + count * particle_stride bytes are a complete snapshot: a host may read the header, then copy just that prefix.
 * A snapshot carries records and particle_counter only: properties, spawners, clocks and pending GPU spawn events are
 * the host's to carry.
 */
#define HNB_SNAPSHOT_MAGIC 0x53424E48u /* "HNBS" in little-endian byte order */
#define HNB_SNAPSHOT_VERSION 1u
typedef struct hnb_instance_snapshot_header {
    uint32_t magic;            /* HNB_SNAPSHOT_MAGIC */
    uint32_t version;          /* HNB_SNAPSHOT_VERSION */
    uint32_t particle_stride;  /* bytes per record = the effect's reference AoS stride */
    uint32_t count;            /* n: records that follow, in alive-list order */
    uint32_t particle_counter; /* the metadata row's particle_counter */
    uint32_t rows;             /* the source slice's rows (informational) */
    uint32_t reserved[10];     /* zero */
} hnb_instance_snapshot_header;

/** Bytes a snapshot of a `rows`-row slice may need: 64 + rows * particle_stride. */
HNB_API size_t hnb_instance_snapshot_bytes(uint32_t particle_stride, uint32_t rows);
/**
 * Snapshot the instance at slab rows [first, first+rows) (`rows` = its capacity), metadata row `metadata_row`, running
 * `effect`, into `d_dst` (`dst_bytes` >= hnb_instance_snapshot_bytes(stride, rows)). With n = min(alive_count, rows),
 * W = indirect_write_index and particle_counter read from the DEVICE metadata row, record i < n is the record of local
 * row list_W[first+i] (clamped to the slice, as hnb_slab_repack does); bytes past 64 + n * stride are not written. The
 * instance is not modified. Call between hnb_simulate calls; work is only enqueued on the context stream.
 */
HNB_API int32_t hnb_instance_snapshot(hnb_ctx* ctx, hnb_slab slab, hnb_effect effect, uint32_t metadata_row, uint32_t first,
                                      uint32_t rows, void* d_dst, size_t dst_bytes);
/**
 * Restore a snapshot into the instance at slab rows [first, first+rows) (`rows` = its capacity; any slice, slab or
 * context whose effect has the snapshot's stride). `d_src` is read on this context's device (any allocation that device
 * can read); `src_bytes` >= 64 is how many bytes it holds. On the device, m = min(count, rows, (src_bytes - 64) / stride),
 * or 0 when magic, version or particle_stride do not match the effect (a corrupt snapshot restores an empty instance and
 * is never read out of bounds). Then:
 *   - record i < m goes to slab row first+i of every plane; rows >= m of the planes are left as they are;
 *   - the metadata row gets alive_count = m, max_spawn = capacity - m (its own capacity word; 0 if that is below m) and,
 *     for an accepted header, particle_counter = header.particle_counter; no other metadata word or draw argument
 *     changes (the next frame's indirect pass rewrites instance_count);
 *   - the lists, dead stack, both identity claims {first, m} and the alive bits are what hnb_slab_repack writes for n = m.
 * So restore(snapshot(X)) into X's own slice leaves the lists, claims, bits, metadata and live records that
 * hnb_slab_repack(X) leaves; into another slice, slab or context, the same state shifted to the new `first`. With
 * rows < n the first `rows` particles in alive-list order are kept, as the reference drops spawns beyond capacity.
 *
 * Both calls return HNB_ERR_INVALID_ARG, with nothing enqueued, when the rows lie outside the slab, the metadata row is
 * out of range, the effect's stride or HNB_EFFECT_SECTOR_PLANES flag does not match the slab, the effect has
 * HNB_EFFECT_EMIT_GPU_SPAWN_EVENTS, the buffer is NULL or not 16-byte aligned, dst_bytes is below
 * hnb_instance_snapshot_bytes(stride, rows), or src_bytes is below 64. rows == 0 is a no-op. Neither call synchronises
 * or allocates.
 */
HNB_API int32_t hnb_instance_restore(hnb_ctx* ctx, hnb_slab slab, hnb_effect effect, uint32_t metadata_row, uint32_t first,
                                     uint32_t rows, const void* d_src, size_t src_bytes);

/**
 * Append the records of a version-1 snapshot to the live particles of the instance at slab rows [first, first+rows)
 * (`rows` = its capacity), as spawns would take them: sparks at many explicit points in one frame, or the particles of a
 * dying instance handed to a shared one (append its hnb_instance_snapshot). The arguments are hnb_instance_restore's;
 * `d_src` may be written by the host or by a kernel, since every count is read on the DEVICE. With n = min(alive_count,
 * rows), W = indirect_write_index and `dead` the slab's dead stack:
 *   - m = min(header.count, max_spawn, rows - n, (src_bytes - 64) / stride), or 0 when magic, version (1 only) or
 *     particle_stride do not match the effect. An append of m = 0 writes nothing.
 *   - Record k < m goes where the k-th spawn of an init would put it: slot s_k = dead[first + n + k] - first (clamped to
 *     the slice), slab row first + s_k of every column, and list_W[first + n + k] = s_k.
 *   - As after a spawn: the identity claim of column W is cut to n if it reaches further, the alive bit of each written
 *     slot is set (HNB_EFFECT_SLOT_ORDER), and the lifetime floor and common age of each written slot's 32-row group
 *     become unknown. Floors and common ages of other groups are kept: a free slot never lies in a deferred group.
 *   - The metadata row gets alive_count = n + m, max_spawn -= m and particle_counter += m (the header's particle_counter
 *     and rows are ignored).
 * Nothing else changes: dead-stack entries, max_update, draw args, spawners, the other list column and claim, the count
 * mailbox (the next frame's indirect pass rewrites instance_count). Bounds, depth order, cull and snapshot calls made
 * before the next hnb_simulate see the appended particles, and two appends in a row compose. Ribbon, slot-order,
 * relaxed-order and sector-plane effects and children of GPU events are accepted; appended records keep their own
 * RIBBON_ID and PREV/NEXT words.
 *
 * Call between hnb_simulate calls; work is only enqueued on the context stream (no synchronisation, no allocation). No
 * access leaves the slice or d_src[0, src_bytes), whatever the device holds. HNB_ERR_INVALID_ARG, with nothing enqueued,
 * on every input hnb_instance_restore refuses, HNB_EFFECT_EMIT_GPU_SPAWN_EVENTS effects included (their pending events
 * name the dead slots an append would fill). rows == 0 is a no-op.
 */
HNB_API int32_t hnb_instance_append(hnb_ctx* ctx, hnb_slab slab, hnb_effect effect, uint32_t metadata_row, uint32_t first,
                                    uint32_t rows, const void* d_src, size_t src_bytes);

/**
 * Repack, snapshot and restore of an instance whose effect has HNB_EFFECT_EMIT_GPU_SPAWN_EVENTS, together with the events
 * it appended in its last update, which the children's next init consumes. Between frames a pending event is an
 * instance-local parent slot: a live slot, or one of the D = min(max_update - n, rows - n) slots the last update freed,
 * which sit at dead-stack positions n .. n+D of the slice (an OnDie parent keeps its record there). Each call takes
 * `emit_events`, the instance's hnb_batch_launch.emit_events: a valid event buffer for every channel b <
 * num_event_bindings, each buffer once, and 0xFFFFFFFF for the other channels. Channel b's pending count is the context's
 * child_infos[base_child_index + b].event_count, base_child_index read from the DEVICE metadata row (a channel whose row
 * does not exist has none). The calls keep every rule of the calls without events (between frames, work only enqueued,
 * nothing read out of the slice) and return HNB_ERR_INVALID_ARG, with nothing enqueued, on the same inputs, and also when
 * the effect does not emit or `emit_events` does not match its channels.
 *
 * hnb_slab_repack_events does what hnb_slab_repack does, and rewrites entries [0, min(event_count, capacity)) of every
 * channel in place as e -> inv[e], where inv[src[i]] = i: each event names the row its parent's record moved to.
 * event_count (its overflow surplus included) and the order of the entries do not change. Its scratch grows by rows x 4
 * bytes.
 *
 * hnb_instance_snapshot_events writes a version-2 snapshot (HNB_SNAPSHOT_EVENTS_VERSION) into `d_dst`, of at least
 * hnb_instance_snapshot_events_bytes(stride, rows, capacities) bytes (event_capacity[b]: the capacity of channel b's
 * buffer, 0 past the effect's channels):
 *   - header words 0-5 as in version 1; reserved[0] = D, reserved[1] = the channel count C, reserved[2 + b] = channel b's
 *     unclamped event_count and reserved[6 + b] = e_b = min(event_count, capacity) (0 past C);
 *   - the n live records in alive-list order, as in version 1, then D dead records: record n + j is local row
 *     dead[first + n + j] - first;
 *   - then, channel after channel, e_b entries: the record index of the event's slot, or 0xFFFFFFFF when that slot is
 *     not one of the n + D records.
 * The first 64 + (n + D) * stride + 4 * sum(e_b) bytes are the complete snapshot. The call takes a scratch of rows x 4
 * bytes with cudaMallocAsync on the context stream and releases it the same way.
 *
 * hnb_instance_restore_events restores a version-2 snapshot whose stride and channel count match the effect. With m as
 * for version 1, live record i < m goes to row i and dead record n + j to row m + j for j < D', where D' = min(D, rows - m,
 * dead records within src_bytes). The lists, dead stack, claims and alive bits are those of hnb_instance_restore; the
 * metadata row gets what hnb_instance_restore writes, plus max_update = m + D'. Record index r becomes row r (r < m) or
 * m + r - n (n <= r < n + D'); any other entry is dropped, and so is every entry past the destination buffer's capacity
 * or past src_bytes. The kept entries fill the channel's buffer in their order, and this context's
 * child_infos[base_child_index + b].event_count becomes the stored unclamped count minus the dropped entries. A header
 * that does not match restores an empty instance with event_count = 0 on every channel. Restoring into X's own slice
 * leaves what hnb_slab_repack_events(X) leaves, except on rows >= n + D.
 */
#define HNB_SNAPSHOT_EVENTS_VERSION 2u
HNB_API int32_t hnb_slab_repack_events(hnb_ctx* ctx, hnb_slab slab, hnb_effect effect, uint32_t metadata_row, uint32_t first,
                                       uint32_t rows, const hnb_event_buffer emit_events[4]);
/** Bytes a version-2 snapshot of a `rows`-row slice may need: 64 + rows * particle_stride + 4 * sum(event_capacity[b]). */
HNB_API size_t hnb_instance_snapshot_events_bytes(uint32_t particle_stride, uint32_t rows, const uint32_t event_capacity[4]);
HNB_API int32_t hnb_instance_snapshot_events(hnb_ctx* ctx, hnb_slab slab, hnb_effect effect, uint32_t metadata_row,
                                             uint32_t first, uint32_t rows, const hnb_event_buffer emit_events[4], void* d_dst,
                                             size_t dst_bytes);
HNB_API int32_t hnb_instance_restore_events(hnb_ctx* ctx, hnb_slab slab, hnb_effect effect, uint32_t metadata_row,
                                            uint32_t first, uint32_t rows, const hnb_event_buffer emit_events[4],
                                            const void* d_src, size_t src_bytes);
/** 64-bit FNV-style checksum of the AoS bytes of rows [first,first+count), computed on device
 *  (order-independent sum of per-row hashes), for whole-slab comparisons at sizes the host
 *  cannot download cheaply. */
HNB_API int32_t hnb_slab_checksum(hnb_ctx* ctx, hnb_slab slab, uint32_t first, uint32_t count,
                                  uint64_t* out);

/** The same with row i hashed as logical row `index_base + i`: the checksums of the shards of a logical instance then
 *  add up (mod 2^64) to the checksum of the unsharded instance. */
HNB_API int32_t hnb_slab_checksum_ex(hnb_ctx* ctx, hnb_slab slab, uint32_t first, uint32_t count, uint64_t index_base,
                                     uint64_t* out);
/** Same checksum over the interleaved {ping,pong,dead} rows of the slab's indirection columns. */
HNB_API int32_t hnb_slab_checksum_indirect(hnb_ctx* ctx, hnb_slab slab, uint32_t first, uint32_t count,
                                           uint64_t* out);

/* Device-resident interop (SURVEY.md §8 f-2). The only consumer of the simulated state is the render pass, which binds
 * the particle buffer as AoS `Particle` records and the indirect buffer as interleaved rows on the DEVICE
 * (vfx_render.wgsl:228-231 reads particle_buffer[indirect_buffer[i].particle_index[render_pong]], mod.rs:139-146).
 * A renderer sharing the CUDA device (Vulkan/D3D12 external memory, or a CUDA rasteriser) either reads the SoA columns in
 * place (hnb_slab_device_view) or asks for the reference layouts in its own device buffer; both are asynchronous on the
 * context stream and involve no host copy. `d_*` pointers are DEVICE pointers. */
typedef struct hnb_slab_view {
    uint32_t capacity_rows, particle_stride, num_planes, _pad;
    void* planes[16];          /* column p holds bytes [plane_offset[p], +plane_width[p]) of every record, capacity_rows elements;
                                  in a word map (hnb_effect_column_plan) it holds the words hnb_effect_column_words names */
    uint32_t plane_offset[16];
    uint32_t plane_width[16];  /* 16, 8 or 4 bytes (32 with HNB_SLAB_SECTOR_PLANES: two 16-byte pieces per element) */
    uint32_t *ping, *pong, *dead; /* the three u32 columns of IndirectEntry */
} hnb_slab_view;
/** A read path for renderers. The pointers, offsets and widths stay valid for the slab's lifetime: a slab whose plan no
 * effect has fixed yet (section 3) is pinned to the default cut by this call, and effects bound to it later run modules
 * generated for that cut. Take the view after the first hnb_simulate that binds the slab to see the effect's own plan.
 * Writing the index columns (ping / pong) through it is not supported: the update pass may
 * skip alive-list loads and stores where it knows a column to be the identity, and a write through the view does not
 * drop that knowledge. Use hnb_slab_import_indirect_device or hnb_slab_upload_indirect to change the lists.
 * The same holds for records: the update pass of an effect with HNB_ATTR_REAP_ONLY keeps a lifetime floor per 32 rows,
 * and every call of this API that writes records clears the floors it covers. A write through the view would not, so a
 * slab whose view has been handed out stops using floors for good. */
HNB_API int32_t hnb_slab_device_view(hnb_ctx* ctx, hnb_slab slab, hnb_slab_view* out);
/** Rows [first,first+count) as AoS records into `d_dst` (count * particle_stride bytes). */
HNB_API int32_t hnb_slab_export_aos_device(hnb_ctx* ctx, hnb_slab slab, uint32_t first, uint32_t count, void* d_dst);
HNB_API int32_t hnb_slab_import_aos_device(hnb_ctx* ctx, hnb_slab slab, uint32_t first, uint32_t count, const void* d_src);
/** Rows [first,first+count) of the indirection columns as interleaved {ping,pong,dead} rows (12 bytes each). */
HNB_API int32_t hnb_slab_export_indirect_device(hnb_ctx* ctx, hnb_slab slab, uint32_t first, uint32_t count, hnb_indirect_index* d_dst);
HNB_API int32_t hnb_slab_import_indirect_device(hnb_ctx* ctx, hnb_slab slab, uint32_t first, uint32_t count, const hnb_indirect_index* d_src);
/** Plain device memory on the context's GPU for callers without their own CUDA allocator (tests, examples). */
HNB_API void* hnb_device_alloc(hnb_ctx* ctx, size_t bytes);
HNB_API void hnb_device_free(hnb_ctx* ctx, void* d_ptr);
HNB_API int32_t hnb_device_download(hnb_ctx* ctx, void* host_dst, const void* d_src, size_t bytes);
HNB_API int32_t hnb_device_upload(hnb_ctx* ctx, void* d_dst, const void* host_src, size_t bytes);

/* ------------------------------------------------------------------------------------ */
/* 4. Compiled effects ≙ pipeline specialisation (reference mod.rs:1758,1866;            */
/*    templates vfx_init.wgsl / vfx_update.wgsl)                                          */
/* ------------------------------------------------------------------------------------ */
/* hnb_effect: declared with hnb_slab above */

/** Value types of attributes/properties (reference src/graph/mod.rs ValueType). */
typedef enum hnb_value_type {
    HNB_BOOL = 0, HNB_FLOAT = 1, HNB_INT = 2, HNB_UINT = 3,
    HNB_BVEC2 = 4, HNB_BVEC3 = 5, HNB_BVEC4 = 6,
    HNB_VEC2 = 7, HNB_VEC3 = 8, HNB_VEC4 = 9,
    HNB_IVEC2 = 10, HNB_IVEC3 = 11, HNB_IVEC4 = 12,
    HNB_UVEC2 = 13, HNB_UVEC3 = 14, HNB_UVEC4 = 15,
    /* float matrices matCxR<f32> (C columns of R rows; values are C*R words, column by column) */
    HNB_MAT2 = 16, HNB_MAT3 = 17, HNB_MAT4 = 18,
    HNB_MAT2X3 = 19, HNB_MAT2X4 = 20, HNB_MAT3X2 = 21, HNB_MAT3X4 = 22, HNB_MAT4X2 = 23, HNB_MAT4X3 = 24
} hnb_value_type;

/** One field of the reference's AoS `Particle` record (ParticleLayout, attributes.rs:1807-1913). */
typedef struct hnb_attr_layout {
    const char* name;    /* field name, e.g. "position" */
    uint32_t value_type; /* hnb_value_type */
    uint32_t offset;     /* byte offset in the AoS record */
    uint32_t flags;      /* HNB_ATTR_* (0 = the update may write the attribute) */
} hnb_attr_layout;

/**
 * HNB_ATTR_UPDATE_READ_ONLY: no code of the update body (age, reap, update code and UPDATE_EXTRA) assigns this attribute.
 * The effect's column plan then gives the read-only words columns of their own, and the update pass stores only the
 * columns that hold a word it writes: C5 ({position, age, velocity, lifetime}, lifetime read-only) moves 32 B read + 28 B
 * written per particle-step instead of 32 + 32. The runtime trusts the declaration: an update that assigns a read-only
 * attribute has the assignment dropped wherever the attribute sits in an unstored column. The graph lowering
 * (hnb_asset_generate) sets the flag from the code it emits. Ignored for parent layouts.
 */
enum { HNB_ATTR_UPDATE_READ_ONLY = 1u << 0 };
/**
 * HNB_ATTR_REAP_ONLY (on "lifetime" only, together with HNB_ATTR_UPDATE_READ_ONLY): the update reads the lifetime only in
 * the standard age and reap code (`was_alive = age < lifetime; age = age + delta_time; is_alive = age < lifetime`), no
 * other code of the update body (update code, UPDATE_EXTRA) reads it and nothing else writes AGE. When, in addition, the
 * lifetime sits in a 4-byte column of its own, the update pass keeps a lifetime floor per 32 slab rows and skips the
 * lifetime load of every particle the floor proves alive this frame (DESIGN.md §3). The results are bit-identical
 * either way. The graph lowering sets the flag; hand-written descriptors that set it must honour the conditions.
 */
enum { HNB_ATTR_REAP_ONLY = 1u << 1 };

enum {
    HNB_EFFECT_LOCAL_SPACE = 1u << 0,          /* LayoutFlags::LOCAL_SPACE_SIMULATION */
    HNB_EFFECT_CONSUME_GPU_SPAWN_EVENTS = 1u << 1,
    HNB_EFFECT_EMIT_GPU_SPAWN_EVENTS = 1u << 2,
    HNB_EFFECT_READ_PARENT_PARTICLE = 1u << 3,
    HNB_EFFECT_RELAXED_ORDER = 1u << 4,        /* alive/dead lists in atomic order (sets exact,
                                                  order scheduling-dependent like the reference) */
    HNB_EFFECT_RIBBONS = 1u << 5,              /* LayoutFlags::RIBBONS (lib.rs:1018-1019): the layout has RIBBON_ID;
                                                  hnb_simulate() sorts the alive list by (RIBBON_ID, AGE) after the update */
    HNB_EFFECT_FAST_MATH = 1u << 6,            /* compile the effect with FMA contraction and approximate division /
                                                  square root — the latitude a WGSL compiler has. fp32 results stay within
                                                  the 1e-5 relative bound but are no longer bit-identical to the oracle;
                                                  integer bookkeeping is unaffected. Pays off for ALU-bound effects. */
    HNB_EFFECT_ORDERED_EVENTS = 1u << 7,       /* with EMIT_GPU_SPAWN_EVENTS: events are appended after the update pass in
                                                  the canonical (row) order instead of with per-particle atomics, so the
                                                  event buffer and what an overflow drops are deterministic (the
                                                  reference's order is scheduling-dependent, lib.rs:976-993). The batch must
                                                  hold one instance (parents of GPU-event children never merge). Costs
                                                  12 B of traffic per updated particle and channel. */
    HNB_EFFECT_SECTOR_PLANES = 1u << 8,        /* the effect addresses slabs created with HNB_SLAB_SECTOR_PLANES (must match) */
    HNB_EFFECT_SLOT_ORDER = 1u << 9            /* the update pass visits the instance's particles in ascending SLOT order (guided
                                                  by an alive bitmap of the slab) instead of alive-list order: the result is what
                                                  the reference computes when its alive list happens to be sorted by particle
                                                  index — same sets, same counts, lists in ascending-slot serial order — and
                                                  every warp touches one contiguous span of each column however long the effect
                                                  has been recycling slots (an alive list that has become a permutation of the
                                                  slab costs 4-8x in DRAM sectors otherwise, for the reference's AoS layout as
                                                  well). Needs instances on 32-row boundaries and < 2^28 slots; not combinable
                                                  with RELAXED_ORDER, ORDERED_EVENTS, SECTOR_PLANES. */
};

/**
 * Lowered effect, i.e. the substitutions EffectShaderSources::generate (reference
 * src/lib.rs:805-1335) makes into vfx_init.wgsl / vfx_update.wgsl, with the code strings
 * in CUDA C instead of WGSL. Any code pointer may be NULL (= empty).
 */
typedef struct hnb_effect_desc {
    const char* name;
    const hnb_attr_layout* attrs; /* {{ATTRIBUTES}}: fields in AoS order, pads excluded */
    uint32_t n_attrs;
    uint32_t particle_stride;       /* bytes */
    const char* properties_struct;  /* {{PROPERTIES}}: body of `struct Properties { ... }` or NULL */
    uint32_t properties_size;       /* bytes of one Properties record (0 = none) */
    const char* init_code;          /* {{INIT_CODE}} */
    const char* init_extra;         /* {{INIT_EXTRA}} */
    const char* sim_space_code;     /* {{SIMULATION_SPACE_TRANSFORM_PARTICLE}} */
    const char* age_code;           /* {{AGE_CODE}} */
    const char* reap_code;          /* {{REAP_CODE}} */
    const char* update_code;        /* {{UPDATE_CODE}} (Euler integration already inserted) */
    const char* update_extra;       /* {{UPDATE_EXTRA}} */
    uint32_t flags;
    const hnb_attr_layout* parent_attrs; /* {{PARENT_ATTRIBUTES}} when READ_PARENT_PARTICLE */
    uint32_t n_parent_attrs;
    uint32_t parent_particle_stride;
    uint32_t num_event_bindings;    /* number of child event buffers this effect appends to */
} hnb_effect_desc;

/** Compile (NVRTC, sm_90a, cached by source hash ≙ ShaderCache) the init+update kernels. */
HNB_API int32_t hnb_effect_compile(hnb_ctx* ctx, const hnb_effect_desc* desc, hnb_effect* out);
HNB_API int32_t hnb_effect_destroy(hnb_ctx* ctx, hnb_effect effect);

/* Background compilation. The reference compiles pipelines asynchronously and neither ticks nor batches an effect
 * until both are ready (spawn.rs:968-973, mod.rs:3853-3894). A job runs the NVRTC step on its own thread and needs no
 * context (it also works without a GPU); hnb_effect_create_from_job() then only loads the finished binary. */
typedef struct hnb_compile_job hnb_compile_job;
/** Copies the descriptor and starts compiling. NULL (message in hnb_last_error()) if the descriptor is invalid. */
HNB_API hnb_compile_job* hnb_compile_job_start(const hnb_effect_desc* desc);
/** 0 = still compiling, 1 = ready, HNB_ERR_NVRTC = failed (compiler log in hnb_last_error()). Never blocks. */
HNB_API int32_t hnb_compile_job_poll(hnb_compile_job* job);
/** Blocks until the job has finished; returns like hnb_compile_job_poll. */
HNB_API int32_t hnb_compile_job_wait(hnb_compile_job* job);
HNB_API void hnb_compile_job_destroy(hnb_compile_job* job);
/** Register the compiled effect with a context: HNB_ERR_NOT_READY while the job runs (simulate nothing for that
 *  effect meanwhile, like the reference), HNB_ERR_NVRTC if it failed. The job can be reused for other contexts. */
HNB_API int32_t hnb_effect_create_from_job(hnb_ctx* ctx, hnb_compile_job* job, hnb_effect* out);
/**
 * Generate the full CUDA C translation unit for `desc` without a GPU (works with ctx=NULL):
 * writes a NUL-terminated string of at most `cap` bytes into `out`, returns its full length
 * in *len. Used by the CPU test-suite (≙ the reference's naga validation tests).
 */
HNB_API int32_t hnb_effect_generate_source(const hnb_effect_desc* desc, char* out, size_t cap, size_t* len);
/** The effect's column plan (no GPU needed): *n columns, column p taking widths[p] bytes per row at capacity x offsets[p]
 *  bytes of the slab's block (at most 16; `offsets` / `widths` may be NULL to ask for *n only). Unless the plan is a word
 *  map (below), column p holds bytes [offsets[p], offsets[p] + widths[p]) of every record. A pure function of the stride,
 *  the attributes' offsets and flags, and the effect flags:
 *   - no read-only attribute, HNB_EFFECT_SECTOR_PLANES or HNB_EFFECT_EMIT_GPU_SPAWN_EVENTS: the default cut (as many
 *     16-byte columns as fit, then an 8- and/or 4-byte tail; 32-byte-wide pairs with sector planes). Children read a
 *     parent slab in the default cut;
 *   - an effect that keeps lifetime floors (an ordered pass, an f32 age, an f32 lifetime flagged
 *     HNB_ATTR_UPDATE_READ_ONLY | HNB_ATTR_REAP_ONLY): a word map. The age and the lifetime get 4-byte columns of their
 *     own, the other words the update may write are packed in record order into 16-, 8- and 4-byte columns, then the
 *     other words the same way; columns are laid out widest first. hnb_effect_column_words tells which record words each
 *     column holds. The authored C5: [0,16) = position, velocity.x; [16,24) = velocity.yz; [24,28) = age;
 *     [28,32) = lifetime. When the map would take more columns than the rule below, that rule applies;
 *   - otherwise every maximal run of words of one class (written by the update, or not: read-only attributes and
 *     padding) is cut into 16-, 8- and 4-byte columns, each at an offset that is a multiple of its width.
 *     C5 with a read-only lifetime: [0,16) [16,24) [24,28) [28,32). A plan of more than 16 columns falls back to the
 *     default cut. */
HNB_API int32_t hnb_effect_column_plan(const hnb_effect_desc* desc, uint32_t* offsets, uint32_t* widths, uint32_t* n);
/** The record words (4-byte words of the reference AoS record) the columns of hnb_effect_column_plan hold: words[k] for
 *  k < *n = particle_stride / 4, column 0's lanes first, then column 1's, and so on (widths[p] / 4 lanes each). `words`
 *  may be NULL to ask for *n only. */
HNB_API int32_t hnb_effect_column_words(const hnb_effect_desc* desc, uint32_t* words, uint32_t* n);
/** hnb_effect_generate_source for the module a context compiles when the effect is bound to a slab whose plan is
 *  `n_planes` columns (`offsets`, `widths`) other than its own: the update stores every column holding a word it may
 *  write. The columns named here hold the record bytes [offsets[p], offsets[p] + widths[p]): a word map cannot be named,
 *  so for a word-map effect, passing its own hnb_effect_column_plan gives the module of a slab cut that way, not its own
 *  module (which hnb_effect_generate_source gives). */
HNB_API int32_t hnb_effect_generate_source_for_plan(const hnb_effect_desc* desc, uint32_t n_planes, const uint32_t* offsets,
                                                    const uint32_t* widths, char* out, size_t cap, size_t* len);
/** NVRTC-compile a translation unit for sm_90a without loading it (no GPU needed). On failure
 *  the compiler log is available from hnb_last_error(). `cubin_size` may be NULL. */
HNB_API int32_t hnb_nvrtc_check(const char* source, size_t* cubin_size);

/* ------------------------------------------------------------------------------------ */
/* 5. Per-frame tables ≙ spawner_buffer / effect_metadata_buffer / batch_info + prefix   */
/*    sums / draw_indirect / sim_params / properties (mod.rs:4679-4705, :6960-6973)       */
/* ------------------------------------------------------------------------------------ */
HNB_API int32_t hnb_set_sim_params(hnb_ctx* ctx, const hnb_sim_params* params);
HNB_API int32_t hnb_upload_spawners(hnb_ctx* ctx, const hnb_spawner* rows, uint32_t n);
/** Batch infos + the CPU prefix sums of spawn counts built by Batcher::push (batch.rs:348-386). */
HNB_API int32_t hnb_upload_batches(hnb_ctx* ctx, const hnb_batch_info* rows, uint32_t n_batches,
                                   const uint32_t* prefix_sum, uint32_t n_prefix);
/** Insert/overwrite one metadata row; like the reference (mod.rs:6074-6087) this resets the
 *  instance. Does not touch slab rows (call hnb_slab_reset_rows). */
HNB_API int32_t hnb_metadata_insert(hnb_ctx* ctx, uint32_t row, const hnb_effect_metadata* md);
HNB_API int32_t hnb_draw_args_insert(hnb_ctx* ctx, uint32_t row, const hnb_draw_indexed_indirect_args* args);
/** Upload the serialized property blob (EffectProperties::serialize, properties.rs:437) of one
 *  instance into the effect's `array<Properties>` at `array_index`. */
HNB_API int32_t hnb_upload_properties(hnb_ctx* ctx, hnb_effect effect, uint32_t array_index,
                                      const void* blob, uint32_t bytes);

/* GPU spawn events (reference src/render/event.rs) */
/** Allocate an event buffer of `capacity` SpawnEvent entries (reference hard-codes 256, event.rs:266). */
HNB_API int32_t hnb_event_buffer_create(hnb_ctx* ctx, uint32_t capacity, hnb_event_buffer* out);
HNB_API int32_t hnb_child_info_insert(hnb_ctx* ctx, uint32_t row, const hnb_child_info* info);
HNB_API int32_t hnb_read_child_info(hnb_ctx* ctx, uint32_t row, hnb_child_info* out);
HNB_API int32_t hnb_event_buffer_download(hnb_ctx* ctx, hnb_event_buffer buf, uint32_t first, uint32_t count,
                                          uint32_t* particle_indices);

/* ------------------------------------------------------------------------------------ */
/* 6. The hot path ≙ simulate() (reference mod.rs:6942-7613)                             */
/* ------------------------------------------------------------------------------------ */
/** One batch = one init dispatch + one update dispatch (reference EffectBatch, batch.rs). */
typedef struct hnb_batch_launch {
    hnb_effect effect;          /* compiled init/update kernels */
    hnb_slab slab;              /* particle + indirect buffers */
    uint32_t batch_info_index;  /* row in the uploaded batch-info table */
    uint32_t total_spawn_count; /* BatchSpawnInfo::CpuSpawner.total_spawn_count (mod.rs:7150-7173) */
    hnb_slab parent_slab;       /* 0xFFFFFFFF if none */
    hnb_event_buffer consume_events; /* event buffer read by init (children), 0xFFFFFFFF if none */
    hnb_event_buffer emit_events[4]; /* event buffers appended by update (parents), 0xFFFFFFFF = unused */
} hnb_batch_launch;
/** Initialiser with every optional binding set to "none" (a zero-initialised struct would bind slab / buffer 0). */
#define HNB_BATCH_LAUNCH_INIT(effect_, slab_, batch_info_index_, total_spawn_count_) \
    { (effect_), (slab_), (batch_info_index_), (total_spawn_count_), 0xFFFFFFFFu, 0xFFFFFFFFu, \
      { 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu } }

/**
 * Enqueue one simulation frame: init (per batch with spawns) → indirect + prefix-sum (one fused
 * bookkeeping kernel) → update (per batch) → for HNB_EFFECT_RIBBONS batches the second prefix-sum pass and
 * the ribbon sort. Asynchronous on the context stream.
 */
HNB_API int32_t hnb_simulate(hnb_ctx* ctx, const hnb_batch_launch* batches, uint32_t n);

/**
 * Bounds of one instance's live particles: the axis-aligned box of the `position` attribute. 32 bytes.
 * A component no particle gave a value (an empty instance, or a NaN in every particle) has min = +inf and max = -inf.
 */
typedef struct hnb_instance_bounds {
    float min[3];
    uint32_t count;    /* n = min(alive_count, capacity): the particles the box covers */
    float max[3];
    uint32_t reserved; /* 0 */
} hnb_instance_bounds;

/**
 * Compute the bounds of every instance of one batch on the device: what frustum culling, LOD or a slice allocator asks
 * about an instance each frame, without a read-back of counts and without exporting records.
 *
 * `batch` is the launch descriptor passed to the last hnb_simulate; its `effect`, `slab` and `batch_info_index` are
 * used. Record j of `d_out` receives the bounds of the batch's j-th instance (spawner row spawner_base + j), for every
 * instance of the batch, in one call. `d_out` holds `out_rows` records and is 16-byte-aligned memory the context's device
 * can write: device memory (hnb_device_alloc, for culling on the GPU) or pinned host memory (hnb_host_alloc; the host
 * reads it after hnb_sync or an event of its own on the context stream).
 *
 * Per instance, with W = indirect_write_index, n = min(alive_count, capacity) and list = alive-list column W, all read on
 * the DEVICE from the tables of the last simulated frame (the live set hnb_instance_snapshot defines):
 *   - min[c] / max[c] are the minimum / maximum of component c of `position` AS STORED, over local rows list[first+i],
 *     i < n, each clamped to the slice. Stored means simulation space: an HNB_EFFECT_LOCAL_SPACE effect gives a local
 *     box, to which the caller applies the emitter transform.
 *   - The order is the total order of the key  bits ^ (sign ? 0xFFFFFFFF : 0x80000000)  compared as unsigned: -0 < +0,
 *     and the infinities take part. The result does not depend on scheduling: it is bit-exact. A NaN component is skipped.
 *   - count = n, whatever the components hold.
 *   - Particle extent is NOT included: neither `size` attributes nor render-time size modifiers. The caller inflates
 *     the box by the effect's largest particle size.
 * Nothing of the instance is modified: no record, list, identity claim, lifetime floor, alive bit, metadata word, draw
 * argument or mailbox word. The call reads the slab in whatever column plan it has; it neither fixes the plan of a slab
 * that has none yet nor turns lifetime floors off. Every kind of effect is accepted (emitting parents, ribbons, slot
 * order, relaxed order, sector planes).
 *
 * Call window: between hnb_simulate calls, and BEFORE the next frame's hnb_upload_spawners / hnb_upload_batches. The
 * device keeps the simulated frame's tables until the next hnb_simulate copies new ones; the instance count used to check
 * `out_rows` is the host's batch row. Work is only enqueued on the context stream (two launches), after every launch of
 * the previous hnb_simulate; no synchronisation, and no allocation after the first call (a per-context accumulator of
 * 64 bytes per instance, which grows only when a larger batch is seen).
 *
 * HNB_ERR_INVALID_ARG, with nothing enqueued: `batch` NULL; invalid effect or slab handle; batch_info_index not an
 * uploaded batch row, or the row's instances outside the uploaded spawner table; no metadata row inserted; the effect's
 * stride or HNB_EFFECT_SECTOR_PLANES flag not matching the slab; an effect without a `position` attribute of type
 * HNB_VEC3 at a 4-byte-aligned offset inside the record; `d_out` NULL or not 16-byte aligned; `out_rows` below the
 * batch's instance count. A batch of zero instances is a no-op. Whatever the device tables hold, no access leaves the slab
 * or d_out[0, out_rows): instance count, table rows, slab offset, capacity and list entries are clamped on the device.
 */
HNB_API int32_t hnb_batch_bounds(hnb_ctx* ctx, const hnb_batch_launch* batch, hnb_instance_bounds* d_out, uint32_t out_rows);

/**
 * Sort every instance's live particles back to front on the device, in one call per batch: the draw order that
 * alpha-blended particles need, without a read-back of counts and without exporting records.
 *
 * `batch`, the live set and the call window are those of hnb_batch_bounds. For the batch's j-th instance (spawner row
 * spawner_base + j), with first = its slab offset, n = min(alive_count, capacity), list = alive-list column W
 * (W = indirect_write_index) and the live entries e_i = list[first + i], i < n, each clamped to the slice (entries under
 * the identity claim of column W are i, and are not loaded), all read on the DEVICE from the tables of the last
 * simulated frame:
 *   - Plane j is d_planes[4j .. 4j+3] = (a, b, c, d). The depth of entry e is ((a*x + b*y) + c*z) + d, with (x, y, z) its
 *     `position` AS STORED and every operation one fp32 round-to-nearest step (no contraction). With a camera's forward
 *     axis f and eye p, the plane (f, -f.p) gives view depth; for an HNB_EFFECT_LOCAL_SPACE effect, pass that plane
 *     transformed into the emitter's space.
 *   - d_order[first + r] = e_pi(r) for r < n, where pi sorts by depth DESCENDING (farthest first) in the total order of
 *     the key  bits ^ (sign ? 0xFFFFFFFF : 0x80000000)  (so -0 < +0 and the infinities take part), NaN depths after all
 *     others, and equal depths in ascending i (stable). The result depends on device state alone: it is bit-exact.
 * d_order is indexed by slab row like the alive-list columns: a renderer binds it in place of the column the draw reads
 * (render_indirect_read_index) and keeps the draw-indirect instance_count. Nothing outside d_order[first, first + n) of
 * each instance is written, so one buffer of the slab's capacity per view serves every batch of the slab.
 *
 * Nothing of the instance is modified: no record, list, identity claim, lifetime floor, alive bit, metadata word, draw
 * argument or mailbox word. The call reads the slab in whatever column plan it has; it neither fixes the plan of a slab
 * that has none yet nor turns lifetime floors off. Every effect hnb_batch_bounds accepts is accepted (emitting parents,
 * slot order, relaxed order, sector planes) except an HNB_EFFECT_RIBBONS effect, whose draw follows ribbon order.
 *
 * d_planes and d_order are memory the context's device can read / write: device memory or pinned host memory
 * (hnb_host_alloc). Work is only enqueued on the context stream (HNB_BATCH_DEPTH_ORDER_LAUNCHES = 13 launches, whatever
 * the batch holds); no synchronisation, and no allocation once a context-owned scratch buffer (16 bytes per slab row,
 * 1 KiB per 4096 live rows and about 4 KiB per instance) has grown to the largest call seen.
 *
 * HNB_ERR_INVALID_ARG, with nothing enqueued: every refusal of hnb_batch_bounds; an HNB_EFFECT_RIBBONS effect; `d_planes`
 * NULL or not 16-byte aligned; `plane_rows` below the batch's instance count; `d_order` NULL; `order_rows` below the
 * slab's capacity. A batch of zero instances is a no-op. Whatever the device tables hold, no access leaves the slab,
 * d_planes[0, 4 * plane_rows) or d_order[0, order_rows).
 */
HNB_API int32_t hnb_batch_depth_order(hnb_ctx* ctx, const hnb_batch_launch* batch, const float* d_planes, uint32_t plane_rows,
                                      uint32_t* d_order, uint32_t order_rows);

/**
 * Cull every instance's live particles against a view frustum on the device, in one call per batch, and write each
 * instance's draw arguments: a renderer then sets up quads for the visible particles only, without a read-back of counts.
 *
 * `batch`, the live set and the call window are those of hnb_batch_bounds. For the batch's j-th instance (spawner row
 * spawner_base + j), with first = its slab offset, n = min(alive_count, capacity) and W = indirect_write_index, all read on
 * the DEVICE from the tables of the last simulated frame, the source entries e_i, i < n, each clamped to the slice, are:
 *   - d_src == NULL: alive-list column W at first + i (entries under the identity claim of column W are i, and are not
 *     loaded);
 *   - otherwise: d_src[first + i], for example the d_order of hnb_batch_depth_order, for a culled back-to-front list.
 * Visibility:
 *   - Frustum j is d_frusta[24j .. 24j+23]: HNB_FRUSTUM_PLANES planes (a, b, c, d). Entry e is visible when
 *     ((a*x + b*y) + c*z) + d >= 0 for all six, with (x, y, z) its `position` AS STORED and every operation one fp32
 *     round-to-nearest step (no contraction). A NaN result fails the test; -0 >= 0 passes. No size attribute is read: the
 *     caller adds a particle radius to d of normalised planes. For an HNB_EFFECT_LOCAL_SPACE effect, pass the planes
 *     transformed into the emitter's space.
 *   - d_visible[first + k] receives the k-th visible entry in ascending i, for k < m_j = the number of visible entries. The
 *     result depends on device state alone: it is stable and bit-exact. Nothing else of d_visible is written, so one buffer
 *     of the slab's capacity per view serves every batch of the slab. It is indexed by slab row like the alive-list
 *     columns: a renderer binds it in place of the column the draw reads (render_indirect_read_index).
 *   - d_args[j] receives the instance's device draw-args row (row draw_indirect_index of its spawner row, the row
 *     hnb_read_draw_args reads) with instance_count = m_j: the indirect draw of the visible entries.
 *
 * Nothing of the instance is modified: no record, list, identity claim, lifetime floor, group word, alive bit, metadata
 * word, row of the device draw-args table or mailbox word. The call reads the slab in whatever column plan it has; it
 * neither fixes the plan of a slab that has none yet nor turns lifetime floors off. Every effect hnb_batch_bounds accepts
 * is accepted (emitting parents, slot order, relaxed order, sector planes) except an HNB_EFFECT_RIBBONS effect: dropping a
 * particle from its draw would re-link its ribbon.
 *
 * d_frusta, d_src, d_visible and d_args are memory the context's device can read / write: device memory or pinned host
 * memory (hnb_host_alloc). Work is only enqueued on the context stream (HNB_BATCH_CULL_LAUNCHES = 4 launches, whatever the
 * batch holds); no synchronisation, and no allocation once a context-owned scratch buffer (516 bytes per 4096 live rows and
 * 32 bytes per instance) has grown to the largest call seen.
 *
 * HNB_ERR_INVALID_ARG, with nothing enqueued: every refusal of hnb_batch_bounds; an HNB_EFFECT_RIBBONS effect; `d_frusta`
 * NULL or not 16-byte aligned; `frustum_rows` below the batch's instance count; `d_src` not NULL with `src_rows` below the
 * slab's capacity; `d_visible` NULL; `visible_rows` below the slab's capacity; [d_src, d_src + src_rows) overlapping
 * [d_visible, d_visible + visible_rows); `d_args` NULL or not 4-byte aligned; `args_rows` below the batch's instance count;
 * no draw-args row inserted. A batch of zero instances is a no-op. Whatever the device tables hold, no access leaves the
 * slab, d_frusta[0, 24 * frustum_rows), d_src[0, src_rows), d_visible[0, visible_rows) or d_args[0, args_rows).
 */
#define HNB_FRUSTUM_PLANES 6
HNB_API int32_t hnb_batch_cull(hnb_ctx* ctx, const hnb_batch_launch* batch, const float* d_frusta, uint32_t frustum_rows,
                               const uint32_t* d_src, uint32_t src_rows, uint32_t* d_visible, uint32_t visible_rows,
                               hnb_draw_indexed_indirect_args* d_args, uint32_t args_rows);

/**
 * hnb_batch_cull for `views` cameras at once (split-screen, an editor viewport beside the game view, two eyes, a minimap
 * or a reflection camera), in one call that reads each live particle's source entry and `position` once for all views.
 *
 * Each buffer holds the views stacked view-major. For view v < views and the batch's j-th instance:
 *   - its frustum is d_frusta[24 * (v * frustum_rows + j) .. +23];
 *   - its visible entries go to d_visible + v * visible_rows, indexed by slab row as in hnb_batch_cull;
 *   - its draw-args row goes to d_args[v * args_rows + j].
 * The source entries are shared by every view: the alive list when d_src is NULL, d_src otherwise. View v's output is
 * byte for byte what
 *   hnb_batch_cull(ctx, batch, d_frusta + 24*v*frustum_rows, frustum_rows, d_src, src_rows,
 *                  d_visible + v*visible_rows, visible_rows, d_args + v*args_rows, args_rows)
 * writes: the same live set, clamping, plane test, source order, and every other row left unwritten. A renderer binds view
 * v's slice of d_visible in place of the alive-list column and draws with view v's args rows; it picks visible_rows >= the
 * slab's capacity such that the byte offset 4 * v * visible_rows meets its graphics API's storage-buffer offset alignment.
 *
 * One source serves all views, so a blended effect, which needs its own back-to-front order per view, still takes one
 * hnb_batch_depth_order and one hnb_batch_cull per view.
 *
 * Work is only enqueued on the context stream: HNB_BATCH_CULL_LAUNCHES = 4 launches whatever `views` is, no
 * synchronisation, and no allocation once the context's cull scratch (views * 516 bytes per 4096 live rows and 32 bytes
 * per instance) has grown to the largest call seen. d_frusta, d_src, d_visible and d_args may be device memory or pinned
 * host memory (hnb_host_alloc).
 *
 * HNB_ERR_INVALID_ARG, with nothing enqueued: every refusal of hnb_batch_cull, checked over the whole stacked ranges
 * (HNB_EFFECT_RIBBONS effects included); `views` 0 or above HNB_CULL_MAX_VIEWS; [d_src, d_src + src_rows) overlapping
 * [d_visible, d_visible + views * visible_rows). A batch of zero instances is a no-op. Whatever the device tables hold, no
 * access leaves the slab, d_frusta[0, 24 * views * frustum_rows), d_src[0, src_rows), d_visible[0, views * visible_rows)
 * or d_args[0, views * args_rows).
 */
#define HNB_CULL_MAX_VIEWS 8
HNB_API int32_t hnb_batch_cull_views(hnb_ctx* ctx, const hnb_batch_launch* batch, uint32_t views, const float* d_frusta,
                                     uint32_t frustum_rows, const uint32_t* d_src, uint32_t src_rows, uint32_t* d_visible,
                                     uint32_t visible_rows, hnb_draw_indexed_indirect_args* d_args, uint32_t args_rows);

/* Individual passes, as exercised one by one by the reference's shader contract tests
 * (src/render/shader_contract_tests.rs). They run the un-fused kernels. */
HNB_API int32_t hnb_pass_init(hnb_ctx* ctx, const hnb_batch_launch* batch);
HNB_API int32_t hnb_pass_indirect(hnb_ctx* ctx);                       /* vfx_indirect.wgsl */
HNB_API int32_t hnb_pass_prefix_sum(hnb_ctx* ctx);                     /* vfx_prefix_sum.wgsl */
HNB_API int32_t hnb_pass_update(hnb_ctx* ctx, const hnb_batch_launch* batch); /* vfx_update.wgsl */
/** vfx_sort_fill.wgsl + vfx_sort.wgsl + vfx_sort_copy.wgsl for every instance of the batch (mod.rs:7444-7610):
 *  the alive-list column `indirect_write_index` of each instance is stably sorted by the particle words
 *  (sort_key_offset, sort_key2_offset) of its metadata row — RIBBON_ID, then AGE bits, compared as u32. */
HNB_API int32_t hnb_pass_sort(hnb_ctx* ctx, const hnb_batch_launch* batch);
/** vfx_utils.wgsl::fill_dispatch_args over host-provided arrays (round-trips through the GPU). */
HNB_API int32_t hnb_pass_fill_dispatch_args(hnb_ctx* ctx, const uint32_t* src, uint32_t src_offset,
                                            uint32_t src_stride, uint32_t* dst, uint32_t dst_len,
                                            uint32_t dst_offset, uint32_t dst_stride, uint32_t count);

/* Observability (the reference has no readback; tests and benchmarks need it). */
HNB_API int32_t hnb_read_metadata(hnb_ctx* ctx, uint32_t row, hnb_effect_metadata* out);
HNB_API int32_t hnb_read_draw_args(hnb_ctx* ctx, uint32_t row, hnb_draw_indexed_indirect_args* out);
HNB_API int32_t hnb_read_spawner(hnb_ctx* ctx, uint32_t row, hnb_spawner* out);
HNB_API int32_t hnb_read_batch_info(hnb_ctx* ctx, uint32_t row, hnb_batch_info* out);
HNB_API int32_t hnb_read_prefix_sum(hnb_ctx* ctx, uint32_t first, uint32_t count, uint32_t* out);
HNB_API int32_t hnb_read_dispatch_args(hnb_ctx* ctx, uint32_t row, hnb_dispatch_indirect_args* out);
/** Tile size word of batch `row` as its last update launch used it (0 before the first launch): rows per update tile
 *  (low 16 bits: 32 x K rows per sub-tile x the sub-tile count, see HNB_TILE_CHUNKS) | 0x80000000 for HNB_EFFECT_SLOT_ORDER. */
HNB_API int32_t hnb_read_tile_size(hnb_ctx* ctx, uint32_t row, uint32_t* out);
/** Number of the slab's 32-row groups whose common age is deferred (section 3 of DESIGN.md: the age lives in the group's
 *  word and the age column of its rows is stale), after the context stream's work so far: 0 for a slab that never ran a
 *  deferring update. Waits for the stream; flushes nothing and changes nothing. */
HNB_API int32_t hnb_slab_deferred_groups(hnb_ctx* ctx, hnb_slab slab, uint64_t* out);
/** Enqueue an async copy of draw-args rows [first,first+count) into caller PINNED memory. */
HNB_API int32_t hnb_read_draw_args_async(hnb_ctx* ctx, uint32_t first, uint32_t count,
                                         hnb_draw_indexed_indirect_args* pinned_out);
/** Count mailbox. `pinned_host` (hnb_host_alloc, ring x rows x 8 bytes; NULL detaches) receives one 64-bit word per updated
 *  instance and frame, written by the update pass itself when it publishes `instance_count` (vfx_update.wgsl:164; the draw-indirect
 *  row is written as always): slot [(epoch % ring) * rows + draw_indirect_row] = (epoch << 32) | instance_count, where `epoch` is
 *  the frame's number (hnb_ctx_last_epoch right after the hnb_simulate that enqueued it). The host reads its own memory — no
 *  device-to-host copy and no event sits between two frames of the kernel chain; a slot holds frame `epoch` once its upper half
 *  equals `epoch`. Rows beyond `rows` are not reported. Not available with HNB_EFFECT_RELAXED_ORDER (counts are atomics there). */
HNB_API int32_t hnb_ctx_set_count_mailbox(hnb_ctx* ctx, uint64_t* pinned_host, uint32_t rows, uint32_t ring);
/** Epoch (frame number, 30 bits, never 0) of the frame the last hnb_simulate enqueued. */
HNB_API int32_t hnb_ctx_last_epoch(hnb_ctx* ctx, uint32_t* epoch);
/** Number of times the context zeroed a batch's look-back tile states before an update launch because the batch's use
 *  changed (effect, slab, tile size or instance set of an HNB_EFFECT_SLOT_ORDER batch) or because an HNB_EFFECT_SLOT_ORDER
 *  batch's states were 64 or more frames old (their words keep 6 bits of epoch). Batches of the other orders never add to it. */
HNB_API int32_t hnb_ctx_tile_state_clears(hnb_ctx* ctx, uint64_t* clears);
/** Number of modules the context compiled (or took from its module cache) for an effect bound to a slab whose column plan
 *  is not the effect's own (section 3: a slab keeps the plan of the first effect bound to it). Each (effect, plan) pair counts
 *  once. */
HNB_API int32_t hnb_ctx_plan_compiles(hnb_ctx* ctx, uint64_t* compiles);
/** Pinned host memory helpers for the async paths. */
HNB_API void* hnb_host_alloc(size_t bytes);
HNB_API void hnb_host_free(void* p);

/** Time (ms) spent in the update kernels of the last `n` hnb_simulate calls is measured by CUDA
 *  events recorded around each update launch when enabled (bench roofline leg). */
/** Effective SM clock (MHz) measured on the device over `window_us` microseconds (clock64 vs globaltimer),
 *  enqueued on the context stream; blocks until done. Diagnostic for benchmarks. */
/** Read (and optionally clear) the 16 diagnostic counters written by kernels compiled with HNB_PROFILE=1
 *  (per-phase cycle totals of hnb_update; see hnb_particle_kernels.cuh). */
HNB_API int32_t hnb_ctx_read_debug(hnb_ctx* ctx, uint64_t* out16, int32_t clear);
/** The HNB_PROFILE kernels' per-frame timeline ring: 64 frames x {~earliest CTA residency, ~earliest start after the
 *  dependency wait, ~earliest end of a first sub-tile, latest warp end} in %globaltimer ns, indexed by epoch & 63. */
HNB_API int32_t hnb_ctx_read_debug_ring(hnb_ctx* ctx, uint64_t* out256, int32_t clear);
HNB_API int32_t hnb_ctx_measure_sm_mhz(hnb_ctx* ctx, uint32_t window_us, double* mhz);
HNB_API int32_t hnb_ctx_enable_kernel_timing(hnb_ctx* ctx, int32_t enabled);
HNB_API int32_t hnb_ctx_kernel_time_ms(hnb_ctx* ctx, double* update_ms_total, uint64_t* update_launches);

#ifdef __cplusplus
}
#endif
#endif /* HANABI_B200_H */
