/*
 * vfx_oracle.c — CPU restatement of the reference's simulation hot path.  TEST INFRASTRUCTURE ONLY.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load
 * this file's library; nothing under bevy_hanabi_b200/ links, imports or executes it.
 *
 * It restates, in plain C on the reference's own data layouts (AoS `Particle` records, interleaved
 * IndirectEntry {particle_index[2], dead_index}, tight EffectMetadata rows):
 *     pcg_hash / to_float01 / frand*          src/render/vfx_common.wgsl:266-335
 *     find_location_from_particle             src/render/vfx_update.wgsl:51-72 (same in vfx_init.wgsl)
 *     vfx_indirect main                       src/render/vfx_indirect.wgsl:31-90
 *     vfx_prefix_sum main                     src/render/vfx_prefix_sum.wgsl:14-43
 *     fill_dispatch_args                      src/render/vfx_utils.wgsl:54-67
 *     ribbon sort: fill / sort / copy         src/render/vfx_sort_fill.wgsl, vfx_sort.wgsl, vfx_sort_copy.wgsl
 *     vfx_init main (structure)               src/render/vfx_init.wgsl:101-196
 *     vfx_update main (structure)             src/render/vfx_update.wgsl:106-167
 *     the generated update body of config C5  src/lib.rs:1223-1281, src/modifier/accel.rs:79-86,
 *                                             src/modifier/force.rs:284-297 (SURVEY.md Appendix E)
 * GPU threads are executed one after the other in ascending global_invocation_id.x: this serial order
 * is the CANONICAL order of the alive / dead lists (the reference's own order depends on atomic
 * scheduling, vfx_update.wgsl:150-151,164-165; only counts and sets are defined there).
 *
 * Parity status: the integer bookkeeping is pinned by the reference's known-answer tests
 * (src/render/shader_contract_tests.rs, headless_batching_tests.rs) replayed in
 * tests/test_oracle_golden.py. Floating-point results of modifiers are "parity unpinned": no
 * reference test executes them (SURVEY.md §8c) and the reference cannot be built here.
 *
 * Build: gcc -O2 -ffp-contract=off -fopenmp -shared -fPIC (see Makefile). No FMA contraction, no
 * fast-math: every float operation is a single correctly rounded IEEE operation.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define ORC_API __attribute__((visibility("default")))

/* ---- table rows (reference src/render/mod.rs:135-622) ------------------------------------- */
typedef struct {
    float delta_time, time, virtual_delta_time, virtual_time, real_delta_time, real_time;
    uint32_t num_effects;
} orc_sim_params;

typedef struct {
    float transform[12];
    float inverse_transform[12];
    int32_t spawn;
    uint32_t seed;
    uint32_t render_indirect_read_index;
    uint32_t effect_metadata_index;
    uint32_t draw_indirect_index;
    uint32_t slab_offset;
    uint32_t parent_slab_offset;
    uint32_t unused;
} orc_spawner;

typedef struct {
    uint32_t total_spawn_count, total_update_count, spawner_base, base_particle, prefix_sum_offset, prefix_sum_count;
} orc_batch_info;

typedef struct {
    uint32_t capacity, alive_count, max_update, max_spawn, indirect_write_index, indirect_render_index,
        init_indirect_dispatch_index, properties_array_index, local_child_index, global_child_index, base_child_index,
        particle_stride, sort_key_offset, sort_key2_offset, particle_counter;
} orc_effect_metadata;

typedef struct {
    uint32_t particle_index[2];
    uint32_t dead_index;
} orc_indirect_entry;

typedef struct {
    uint32_t init_indirect_dispatch_index;
    int32_t event_count;
} orc_child_info;

#define DRAW_INDEXED_INDIRECT_STRIDE 5u

/* ---- PRNG (vfx_common.wgsl:260-335) --------------------------------------------------------- */
ORC_API uint32_t orc_pcg_hash(uint32_t input) {
    uint32_t state = input * 747796405u + 2891336453u;
    uint32_t word = ((state >> ((state >> 28u) + 4u)) ^ state) * 277803737u;
    return (word >> 22u) ^ word;
}
ORC_API float orc_to_float01(uint32_t u) {
    uint32_t bits = (u & 0x007fffffu) | 0x3f800000u;
    float f;
    memcpy(&f, &bits, 4);
    return f - 1.0f;
}
ORC_API float orc_frand(uint32_t* seed) {
    *seed = orc_pcg_hash(*seed);
    return orc_to_float01(orc_pcg_hash(*seed));
}
ORC_API void orc_frand2(uint32_t* seed, float* out) {
    *seed = orc_pcg_hash(*seed); out[0] = orc_to_float01(*seed);
    *seed = orc_pcg_hash(*seed); out[1] = orc_to_float01(*seed);
}
ORC_API void orc_frand3(uint32_t* seed, float* out) {
    *seed = orc_pcg_hash(*seed); out[0] = orc_to_float01(*seed);
    *seed = orc_pcg_hash(*seed); out[1] = orc_to_float01(*seed);
    *seed = orc_pcg_hash(*seed); out[2] = orc_to_float01(*seed);
}
ORC_API void orc_frand4(uint32_t* seed, float* out) {
    uint32_t r0 = orc_pcg_hash(*seed);
    uint32_t r1 = orc_pcg_hash(r0);
    uint32_t r2 = orc_pcg_hash(r1);
    *seed = r2;
    out[0] = orc_to_float01(r0);
    out[1] = orc_to_float01((r0 & 0xff000000u) >> 8u | (r1 & 0x0000ffffu));
    out[2] = orc_to_float01((r1 & 0xffff0000u) >> 8u | (r2 & 0x000000ffu));
    out[3] = orc_to_float01(r2 >> 8u);
}

/* ---- find_location_from_particle (vfx_update.wgsl:51-72) ------------------------------------ */
typedef struct {
    uint32_t effect_index, base_particle, update_index;
} orc_effect_location;

ORC_API orc_effect_location orc_find_location_from_particle(const orc_batch_info* batch_info, const uint32_t* prefix_sum,
                                                            uint32_t update_particle_index) {
    uint32_t lo = batch_info->prefix_sum_offset;
    uint32_t hi = lo + batch_info->prefix_sum_count;
    int num_iter = 0;
    while (lo < hi) {
        uint32_t mid = (hi + lo) >> 1u;
        uint32_t base_particle = prefix_sum[mid];
        if (update_particle_index >= base_particle) {
            lo = mid + 1u;
        } else if (update_particle_index < base_particle) {
            hi = mid;
        }
        num_iter += 1;
        if (num_iter >= 100) {
            orc_effect_location bad = {0xDEADBEEFu, 0xDEADBEEFu, 0xDEADBEEFu};
            return bad;
        }
    }
    orc_effect_location loc;
    loc.base_particle = prefix_sum[lo - 1u];
    loc.effect_index = lo - 1u - batch_info->prefix_sum_offset;
    loc.update_index = update_particle_index - loc.base_particle;
    return loc;
}

/* ---- vfx_indirect main (vfx_indirect.wgsl:31-90), one call = the whole dispatch ------------- */
ORC_API void orc_indirect(const orc_sim_params* sim_params, orc_effect_metadata* effect_metadata_buffer,
                          uint32_t* draw_indirect_buffer, orc_spawner* spawner_buffer, uint32_t* prefix_sum,
                          orc_child_info* child_info_buffer, uint32_t child_info_len) {
    for (uint32_t global_effect_index = 0; global_effect_index < sim_params->num_effects; ++global_effect_index) {
        if (child_info_buffer && global_effect_index < child_info_len) {
            child_info_buffer[global_effect_index].event_count = 0;
        }
        orc_spawner* spawner = &spawner_buffer[global_effect_index];
        orc_effect_metadata* em = &effect_metadata_buffer[spawner->effect_metadata_index];
        uint32_t dri_base = DRAW_INDEXED_INDIRECT_STRIDE * spawner->draw_indirect_index;
        draw_indirect_buffer[dri_base + 1u] = 0u;
        uint32_t capacity = em->capacity;
        uint32_t alive_count = em->alive_count;
        uint32_t dead_count = capacity - alive_count;
        prefix_sum[global_effect_index] = alive_count;
        em->max_update = alive_count;
        em->max_spawn = dead_count;
        uint32_t ping = em->indirect_write_index;
        uint32_t pong = 1u - ping;
        em->indirect_write_index = pong;
        spawner->render_indirect_read_index = pong;
    }
}

/* ---- vfx_prefix_sum main (vfx_prefix_sum.wgsl:14-43) ---------------------------------------- */
ORC_API void orc_prefix_sum(orc_batch_info* batch_infos, uint32_t batch_count, uint32_t* prefix_sum,
                            uint32_t* dispatch_indirect_buffer /* 3 u32 per batch */) {
    for (uint32_t batch_index = 0; batch_index < batch_count; ++batch_index) {
        uint32_t offset = batch_infos[batch_index].prefix_sum_offset;
        uint32_t count = batch_infos[batch_index].prefix_sum_count;
        uint32_t end = offset + count;
        uint32_t sum = 0u;
        for (uint32_t i = offset; i < end; i += 1u) {
            uint32_t c = prefix_sum[i];
            prefix_sum[i] = sum;
            sum = sum + c;
        }
        batch_infos[batch_index].total_update_count = sum;
        dispatch_indirect_buffer[batch_index * 3u + 0u] = (sum + 63u) >> 6u;
        dispatch_indirect_buffer[batch_index * 3u + 1u] = 1u;
        dispatch_indirect_buffer[batch_index * 3u + 2u] = 1u;
    }
}

/* ---- fill_dispatch_args (vfx_utils.wgsl:54-67) ---------------------------------------------- */
ORC_API void orc_fill_dispatch_args(const uint32_t* src_buffer, uint32_t* dst_buffer, uint32_t src_offset,
                                    uint32_t src_stride, uint32_t dst_offset, uint32_t dst_stride, uint32_t count) {
    for (uint32_t thread_index = 0; thread_index < count; ++thread_index) {
        uint32_t src = src_offset + thread_index * src_stride;
        uint32_t dst = dst_offset + thread_index * dst_stride;
        uint32_t thread_count = src_buffer[src];
        dst_buffer[dst] = (thread_count + 63u) >> 6u;
        dst_buffer[dst + 1u] = 1u;
        dst_buffer[dst + 2u] = 1u;
    }
}

/* ---- ribbon sort (vfx_sort_fill.wgsl:38-57, vfx_sort.wgsl:18-55, vfx_sort_copy.wgsl:30-46) --------------
 * Three dispatches per ribbon effect instance, run after the update pass (mod.rs:7444-7610). The sort
 * buffer is `count` followed by {key, key2, value} triples (HAS_DUAL_KEY is always defined, sort.rs:163,:364).
 * Fill threads run in ascending thread index (canonical order; the reference appends with an atomic).
 * "parity unpinned": no reference test executes these shaders. */
typedef struct {
    uint32_t key, key2, value;
} orc_key_value_pair;

ORC_API void orc_sort_fill(int32_t* sort_count, orc_key_value_pair* pairs, const uint32_t* particle_buffer,
                           const uint32_t* indirect_index_buffer, const orc_effect_metadata* effect_metadata,
                           const orc_spawner* spawner, uint32_t thread_count) {
    for (uint32_t thread_index = 0; thread_index < thread_count; ++thread_index) {
        uint32_t count = effect_metadata->alive_count;
        if (thread_index >= count) continue;
        uint32_t base_particle = spawner->slab_offset;
        uint32_t read_index = effect_metadata->indirect_write_index;
        uint32_t particle_index = indirect_index_buffer[(base_particle + thread_index) * 3u + read_index];
        uint32_t particle_offset = (base_particle + particle_index) * effect_metadata->particle_stride;
        uint32_t key_offset = particle_offset + effect_metadata->sort_key_offset;
        uint32_t key2_offset = particle_offset + effect_metadata->sort_key2_offset;
        int32_t pair_index = (*sort_count)++;
        pairs[pair_index].key = particle_buffer[key_offset];
        pairs[pair_index].key2 = particle_buffer[key2_offset];
        pairs[pair_index].value = particle_index;
    }
}

static int compare_greater(orc_key_value_pair kv1, orc_key_value_pair kv2) {
    if (kv1.key > kv2.key) return 1;
    if (kv1.key == kv2.key) return kv1.key2 > kv2.key2;
    return 0;
}

ORC_API void orc_sort(int32_t* sort_count, orc_key_value_pair* pairs) {
    int32_t num_items = *sort_count;
    for (int32_t i = 1; i < num_items; ++i) {
        orc_key_value_pair kv = pairs[i];
        int32_t j = i;
        while (j > 0 && compare_greater(pairs[j - 1], kv)) {
            pairs[j] = pairs[j - 1];
            j -= 1;
        }
        pairs[j] = kv;
    }
    *sort_count = 0;
}

ORC_API void orc_sort_copy(uint32_t* indirect_index_buffer, const orc_key_value_pair* pairs,
                           const orc_effect_metadata* effect_metadata, const orc_spawner* spawner, uint32_t thread_count) {
    for (uint32_t row_index = 0; row_index < thread_count; ++row_index) {
        uint32_t count = effect_metadata->alive_count;
        if (row_index >= count) continue;
        uint32_t base_particle = spawner->slab_offset;
        uint32_t write_index = effect_metadata->indirect_write_index;
        indirect_index_buffer[(base_particle + row_index) * 3u + write_index] = pairs[row_index].value;
    }
}

/* ---- per-effect bodies ------------------------------------------------------------------------
 * A body receives the thread-private copy of the AoS record (`var particle`), like the WGSL templates.
 * update bodies return is_alive. */
typedef struct {
    const orc_sim_params* sim_params;
    const orc_spawner* spawner;
    uint32_t particle_index;
    uint32_t particle_counter;
    uint32_t* seed;
    const void* user;
} orc_thread;

typedef void (*orc_init_body)(uint32_t* particle, orc_thread* t);
typedef int (*orc_update_body)(uint32_t* particle, orc_thread* t);

/* ---- vfx_update main (vfx_update.wgsl:106-167): `thread_count` threads of one dispatch -------- */
ORC_API void orc_update(const orc_sim_params* sim_params, uint32_t* draw_indirect_buffer, uint32_t* particle_buffer,
                        uint32_t stride_words, orc_indirect_entry* indirect_buffer, const orc_spawner* spawners,
                        const uint32_t* prefix_sum, const orc_batch_info* batch_info,
                        orc_effect_metadata* effect_metadatas, uint32_t thread_count, orc_update_body body,
                        const void* user) {
    uint32_t particle[64];
    for (uint32_t update_particle_index = 0; update_particle_index < thread_count; ++update_particle_index) {
        orc_effect_location location = orc_find_location_from_particle(batch_info, prefix_sum, update_particle_index);
        const orc_spawner* spawner = &spawners[batch_info->spawner_base + location.effect_index];
        uint32_t effect_metadata_index = spawner->effect_metadata_index;
        uint32_t base_particle = spawner->slab_offset;
        uint32_t slab_particle_index = base_particle + location.update_index;
        orc_effect_metadata* em = &effect_metadatas[effect_metadata_index];
        if (location.update_index >= em->max_update) continue;
        uint32_t write_index = em->indirect_write_index;
        uint32_t read_index = 1u - write_index;
        uint32_t particle_index = indirect_buffer[slab_particle_index].particle_index[read_index];
        uint32_t seed = orc_pcg_hash(particle_index ^ spawner->seed);
        uint32_t* rec = particle_buffer + (size_t)(base_particle + particle_index) * stride_words;
        memcpy(particle, rec, (size_t)stride_words * 4);
        orc_thread t = {sim_params, spawner, particle_index, 0u, &seed, user};
        int is_alive = body(particle, &t);
        /* WRITEBACK_CODE: every attribute (PREV/NEXT handling is the body's business: it must leave them
         * untouched) */
        memcpy(rec, particle, (size_t)stride_words * 4);
        if (!is_alive) {
            uint32_t alive_index = (em->alive_count--) - 1u; /* atomicSub(...) - 1 */
            indirect_buffer[base_particle + alive_index].dead_index = base_particle + particle_index;
            em->max_spawn += 1u;
        } else {
            uint32_t* instance_count = &draw_indirect_buffer[DRAW_INDEXED_INDIRECT_STRIDE * em->indirect_render_index + 1u];
            uint32_t indirect_index = (*instance_count)++;
            indirect_buffer[base_particle + indirect_index].particle_index[write_index] = particle_index;
        }
    }
}

/* ---- vfx_init main (vfx_init.wgsl:101-196), CPU-spawner variant ------------------------------- */
ORC_API void orc_init(const orc_sim_params* sim_params, uint32_t* particle_buffer, uint32_t stride_words,
                      orc_indirect_entry* indirect_buffer, const orc_spawner* spawners, const uint32_t* prefix_sum,
                      const orc_batch_info* batch_info, orc_effect_metadata* effect_metadatas, uint32_t thread_count,
                      orc_init_body body, const void* user) {
    uint32_t particle[64];
    for (uint32_t update_particle_index = 0; update_particle_index < thread_count; ++update_particle_index) {
        orc_effect_location location = orc_find_location_from_particle(batch_info, prefix_sum, update_particle_index);
        const orc_spawner* spawner = &spawners[batch_info->spawner_base + location.effect_index];
        uint32_t base_particle = spawner->slab_offset;
        orc_effect_metadata* em = &effect_metadatas[spawner->effect_metadata_index];
        uint32_t max_spawn = em->max_spawn;
        if (location.update_index >= max_spawn) continue;
        uint32_t spawn_count = (uint32_t)spawner->spawn;
        if (location.update_index >= spawn_count) continue;
        uint32_t alive_index = em->alive_count++;
        /* the slot of the thread 16 ahead, which spawns too: its dead-stack entry is read and its record written soon */
        if (location.update_index + 16u < max_spawn && location.update_index + 16u < spawn_count)
            __builtin_prefetch(particle_buffer + (size_t)indirect_buffer[base_particle + alive_index + 16u].dead_index * stride_words, 1);
        uint32_t slab_particle_dead_index = indirect_buffer[base_particle + alive_index].dead_index;
        uint32_t particle_index = slab_particle_dead_index - base_particle;
        uint32_t particle_counter = em->particle_counter++;
        uint32_t seed = orc_pcg_hash(particle_index ^ spawner->seed);
        memset(particle, 0, (size_t)stride_words * 4); /* var particle = Particle(); */
        orc_thread t = {sim_params, spawner, particle_index, particle_counter, &seed, user};
        body(particle, &t);
        uint32_t write_index = em->indirect_write_index;
        indirect_buffer[base_particle + alive_index].particle_index[write_index] = particle_index;
        memcpy(particle_buffer + (size_t)(base_particle + particle_index) * stride_words, particle, (size_t)stride_words * 4);
    }
}

/* ---- bodies ------------------------------------------------------------------------------------ */
/* No-op update body for effects without AGE (lib.rs:1250-1254: was_alive = is_alive = true). */
static int body_update_noop(uint32_t* particle, orc_thread* t) {
    (void)particle; (void)t;
    return 1;
}
ORC_API orc_update_body orc_body_update_noop(void) { return body_update_noop; }

/* Config C5 (SURVEY.md Appendix E). Layout {position:vec3@0, age:f32@12, velocity:vec3@16, lifetime:f32@28}.
 * user -> float[4] {accel.x, accel.y, accel.z, drag}. */
static inline int c5_body(float* p, float dt, const float* k) {
    /* AGE_CODE (lib.rs:1229-1247) */
    /* was_alive = age < lifetime; (unused) */
    p[3] = p[3] + dt;
    int is_alive = p[3] < p[7];
    /* REAP_CODE (lib.rs:1256-1264) */
    is_alive = is_alive && (p[3] < p[7]);
    /* AccelModifier (accel.rs:84): velocity += (accel) * dt */
    p[4] = p[4] + k[0] * dt;
    p[5] = p[5] + k[1] * dt;
    p[6] = p[6] + k[2] * dt;
    /* LinearDragModifier (force.rs:284-297): velocity *= max(0., (1.) - ((drag) * (dt))) */
    float f = fmaxf(0.0f, 1.0f - (k[3] * dt));
    p[4] = p[4] * f;
    p[5] = p[5] * f;
    p[6] = p[6] * f;
    /* MotionIntegration::PostUpdate (lib.rs:1109-1121): position += velocity * dt */
    p[0] = p[0] + p[4] * dt;
    p[1] = p[1] + p[5] * dt;
    p[2] = p[2] + p[6] * dt;
    return is_alive;
}
static int body_update_c5(uint32_t* particle, orc_thread* t) {
    return c5_body((float*)particle, t->sim_params->delta_time, (const float*)t->user);
}
ORC_API orc_update_body orc_body_update_c5(void) { return body_update_c5; }

/* Init body writing constants: user -> stride_words u32 words copied into the record. */
typedef struct {
    uint32_t stride_words;
    uint32_t words[64];
} orc_const_init;
static void body_init_const(uint32_t* particle, orc_thread* t) {
    const orc_const_init* ci = (const orc_const_init*)t->user;
    memcpy(particle, ci->words, (size_t)ci->stride_words * 4);
}
ORC_API orc_init_body orc_body_init_const(void) { return body_init_const; }

/* tests/effects.py::drifting_sparks' init, in the generated code's order of PRNG calls: position = frand3() * 2 - 1,
 * velocity = frand3() * 2 - 1, age = 0, lifetime = lo + frand() * (hi - lo), then the Global simulation space's
 * position += the spawner's translation. Same record layout as C5, so its update is body_update_c5 with ACCEL_DRAG.
 * user -> float[2] {lifetime_lo, lifetime_hi}. */
static void body_init_sparks(uint32_t* particle, orc_thread* t) {
    const float* life = (const float*)t->user;
    const float* tr = t->spawner->transform;
    float* p = (float*)particle;
    float r[3];
    orc_frand3(t->seed, r);
    p[0] = r[0] * 2.0f - 1.0f; p[1] = r[1] * 2.0f - 1.0f; p[2] = r[2] * 2.0f - 1.0f;
    orc_frand3(t->seed, r);
    p[4] = r[0] * 2.0f - 1.0f; p[5] = r[1] * 2.0f - 1.0f; p[6] = r[2] * 2.0f - 1.0f;
    p[3] = 0.0f;
    p[7] = life[0] + orc_frand(t->seed) * (life[1] - life[0]);
    p[0] = p[0] + tr[3]; p[1] = p[1] + tr[7]; p[2] = p[2] + tr[11];
}
ORC_API orc_init_body orc_body_init_sparks(void) { return body_init_sparks; }

/* ---- synthetic C5 state, same counter-based generator as hnb_slab_fill_c5 ---------------------- */
/* `logical_first`: row of the LOGICAL instance that slab row `first` holds. A shard of an instance split by index range
 * over several devices (SURVEY.md §8e) stores logical rows [logical_first, logical_first + count) at its own rows
 * [first, first + count): same particle values as the unsharded instance, shard-local indices. */
ORC_API void orc_fill_c5_ex(float* particles_aos /* 8 floats per row */, orc_indirect_entry* indirect, uint32_t first,
                            uint32_t count, uint32_t seed, float lifetime_lo, float lifetime_hi, uint32_t logical_first) {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)count; ++i) {
        uint32_t row = first + (uint32_t)i;
        uint32_t s = orc_pcg_hash((logical_first + (uint32_t)i) ^ seed);
        float v[7];
        for (int k = 0; k < 7; ++k) {
            s = orc_pcg_hash(s);
            v[k] = orc_to_float01(s);
        }
        float* p = particles_aos + (size_t)row * 8;
        p[0] = v[0] * 2.0f - 1.0f; p[1] = v[1] * 2.0f - 1.0f; p[2] = v[2] * 2.0f - 1.0f; p[3] = 0.0f;
        p[4] = v[3] * 2.0f - 1.0f; p[5] = v[4] * 2.0f - 1.0f; p[6] = v[5] * 2.0f - 1.0f;
        p[7] = lifetime_lo + v[6] * (lifetime_hi - lifetime_lo);
        if (indirect) {
            indirect[row].particle_index[0] = (uint32_t)i;
            indirect[row].particle_index[1] = (uint32_t)i;
        }
    }
}

ORC_API void orc_fill_c5(float* particles_aos, orc_indirect_entry* indirect, uint32_t first, uint32_t count, uint32_t seed,
                         float lifetime_lo, float lifetime_hi) {
    orc_fill_c5_ex(particles_aos, indirect, first, count, seed, lifetime_lo, lifetime_hi, first);
}

/* ParticleSlab::new's initial indirect rows (effect_cache.rs:309-322): ping = pong = 0, dead[i] = i. In parallel so that
 * the pages are first touched by the threads that will update them (the CPU baseline of bench.py). */
ORC_API void orc_indirect_reset(orc_indirect_entry* indirect, uint32_t first, uint32_t count) {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)count; ++i) {
        uint32_t row = first + (uint32_t)i;
        indirect[row].particle_index[0] = 0u;
        indirect[row].particle_index[1] = 0u;
        indirect[row].dead_index = row;
    }
}

/* ---- multi-threaded C5 update of ONE effect instance (CPU baseline) ----------------------------
 * Same results as orc_update() with body_update_c5 on a single-instance batch: rows are split into
 * contiguous chunks, one per thread; survivors / dead are counted per chunk, an exclusive scan over the
 * chunks gives each chunk its list offsets, and a second sweep scatters the indices, so both lists come
 * out in serial thread order. Returns the number of survivors. `flags` is a caller-provided scratch of
 * max_update bytes. */
ORC_API uint32_t orc_update_c5_parallel(const orc_sim_params* sim_params, uint32_t* draw_indirect_buffer,
                                        float* particle_buffer, orc_indirect_entry* indirect_buffer,
                                        const orc_spawner* spawner, orc_effect_metadata* em, const float* k,
                                        uint8_t* flags, int num_threads) {
    const uint32_t base_particle = spawner->slab_offset;
    const uint32_t max_update = em->max_update;
    const uint32_t write_index = em->indirect_write_index;
    const uint32_t read_index = 1u - write_index;
    const float dt = sim_params->delta_time;
    if (num_threads < 1) num_threads = 1;
    uint32_t* chunk_alive = (uint32_t*)calloc((size_t)num_threads + 1, sizeof(uint32_t));
#pragma omp parallel num_threads(num_threads)
    {
#ifdef _OPENMP
        int tid = omp_get_thread_num(), nt = omp_get_num_threads();
#else
        int tid = 0, nt = 1;
#endif
        uint64_t lo = (uint64_t)max_update * tid / nt, hi = (uint64_t)max_update * (tid + 1) / nt;
        uint32_t alive = 0;
        for (uint64_t row = lo; row < hi; ++row) {
            if (row + 16 < hi) /* a churned list is a gather: keep later records in flight (speed only) */
                __builtin_prefetch(particle_buffer + (size_t)(base_particle + indirect_buffer[base_particle + row + 16].particle_index[read_index]) * 8, 1);
            uint32_t particle_index = indirect_buffer[base_particle + row].particle_index[read_index];
            float* p = particle_buffer + (size_t)(base_particle + particle_index) * 8;
            float rec[8];
            memcpy(rec, p, 32);
            int is_alive = c5_body(rec, dt, k);
            memcpy(p, rec, 32);
            flags[row] = (uint8_t)is_alive;
            alive += (uint32_t)is_alive;
        }
        chunk_alive[tid + 1] = alive;
#pragma omp barrier
#pragma omp single
        {
            for (int i = 0; i < nt; ++i) chunk_alive[i + 1] += chunk_alive[i];
        }
        uint32_t alive_rank = chunk_alive[tid];
        for (uint64_t row = lo; row < hi; ++row) {
            uint32_t particle_index = indirect_buffer[base_particle + row].particle_index[read_index];
            if (flags[row]) {
                indirect_buffer[base_particle + alive_rank].particle_index[write_index] = particle_index;
                alive_rank++;
            } else {
                uint32_t dead_rank = (uint32_t)row - alive_rank;
                uint32_t alive_index = em->alive_count - 1u - dead_rank;
                indirect_buffer[base_particle + alive_index].dead_index = base_particle + particle_index;
            }
        }
    }
    uint32_t alive_total = chunk_alive[num_threads];
    /* with fewer OpenMP threads than requested the tail entries stay equal to the last real one */
    for (int i = 1; i <= num_threads; ++i) if (chunk_alive[i] > alive_total) alive_total = chunk_alive[i];
    uint32_t dead_total = max_update - alive_total;
    draw_indirect_buffer[DRAW_INDEXED_INDIRECT_STRIDE * em->indirect_render_index + 1u] += alive_total;
    em->alive_count -= dead_total;
    em->max_spawn += dead_total;
    free(chunk_alive);
    return alive_total;
}

/* Order-independent checksum of `count` rows of `stride_words` u32 each: same function as the device-side
 * hnb_slab_checksum (sum over rows of a 64-bit mix of the row's words and its index). */
ORC_API uint64_t orc_checksum_ex(const uint32_t* words, uint32_t first, uint32_t count, uint32_t stride_words, uint64_t index_base) {
    uint64_t acc = 0;
#pragma omp parallel for schedule(static) reduction(+ : acc)
    for (int64_t i = 0; i < (int64_t)count; ++i) {
        uint64_t h = 0xcbf29ce484222325ull ^ (index_base + (uint64_t)i);
        const uint32_t* row = words + (size_t)(first + (uint32_t)i) * stride_words;
        for (uint32_t w = 0; w < stride_words; ++w) h = (h ^ (uint64_t)row[w]) * 0x100000001b3ull;
        h ^= h >> 29; h *= 0xbf58476d1ce4e5b9ull; h ^= h >> 32;
        acc += h;
    }
    return acc;
}

/* The high 32 bits of each row's term of orc_checksum_ex (index_base 0): a digest per row, so that two slabs whose
 * checksums differ can be told apart row by row without keeping either. */
ORC_API void orc_row_digests(const uint32_t* words, uint32_t count, uint32_t stride_words, uint32_t* out) {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)count; ++i) {
        uint64_t h = 0xcbf29ce484222325ull ^ (uint64_t)i;
        const uint32_t* row = words + (size_t)i * stride_words;
        for (uint32_t w = 0; w < stride_words; ++w) h = (h ^ (uint64_t)row[w]) * 0x100000001b3ull;
        h ^= h >> 29; h *= 0xbf58476d1ce4e5b9ull; h ^= h >> 32;
        out[i] = (uint32_t)(h >> 32);
    }
}

ORC_API uint64_t orc_checksum(const uint32_t* words, uint32_t first, uint32_t count, uint32_t stride_words) {
    return orc_checksum_ex(words, first, count, stride_words, 0);
}

/* Thread count of the `parallel for` loops above (fill, reset, checksum); the update takes its own count. A launcher may
 * have exported OMP_NUM_THREADS=1 (torchrun does): the benchmark's CPU arm decides from the CPUs it may actually use. */
ORC_API void orc_set_threads(int n) {
#ifdef _OPENMP
    if (n >= 1) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

ORC_API int orc_max_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
