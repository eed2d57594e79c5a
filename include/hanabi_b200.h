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

/**
 * Allocate a slab of `capacity_rows` particles whose reference AoS record is
 * `particle_stride_bytes` (ParticleLayout::min_binding_size, attributes.rs:1837).
 * Storage is SoA: the AoS record is cut into 16-byte planes (float4 columns; an 8- or 4-byte
 * tail gets a float2/u32 column), plus three u32 columns ping/pong/dead. dead[i] = i
 * (effect_cache.rs:309-322); ping/pong = 0.
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
    void* planes[16];          /* column p holds bytes [plane_offset[p], +plane_width[p]) of every record, capacity_rows elements */
    uint32_t plane_offset[16];
    uint32_t plane_width[16];  /* 16, 8 or 4 bytes (32 with HNB_SLAB_SECTOR_PLANES: two 16-byte pieces per element) */
    uint32_t *ping, *pong, *dead; /* the three u32 columns of IndirectEntry */
} hnb_slab_view;
/** A read path for renderers. Writing the index columns (ping / pong) through it is not supported: the update pass may
 * skip alive-list loads and stores where it knows a column to be the identity, and a write through the view does not
 * drop that knowledge. Use hnb_slab_import_indirect_device or hnb_slab_upload_indirect to change the lists. */
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
} hnb_attr_layout;

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
typedef uint32_t hnb_event_buffer;
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
