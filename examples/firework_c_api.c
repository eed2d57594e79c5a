/*
 * firework_c_api.c — the whole path from plain C, no Python: author an effect with the expression module
 * (Level 2, hanabi_b200_graph.h), lower it to CUDA C, compile it (NVRTC), and run frames with
 * EffectSpawner::tick -> Batcher::push -> hnb_simulate (Level 1, hanabi_b200.h).
 *
 * The effect is the "trails" part of the reference's firework example made parent-less
 * (examples/firework.rs:184-251; BASELINE config C2): burst of particles with random directions, linear drag,
 * gravity, age / lifetime.
 *
 *   gcc -O2 -Iinclude examples/firework_c_api.c -Lbevy_hanabi_b200 -lhanabi_b200 -Wl,-rpath,$PWD/bevy_hanabi_b200 -o build/firework_c_api
 *   build/firework_c_api [frames]
 *
 * Exit code 0 on success, 3 when there is no CUDA device (the library has no CPU path; everything up to and
 * including code generation still runs, which is what the CPU test of this example checks).
 */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "hanabi_b200.h"
#include "hanabi_b200_graph.h"

#define CHECK(call)                                                                   \
    do {                                                                              \
        int32_t rc_ = (call);                                                         \
        if (rc_ != HNB_OK) {                                                          \
            fprintf(stderr, "%s -> %d: %s\n", #call, rc_, hnb_last_error());          \
            return rc_ == HNB_ERR_NO_DEVICE ? 3 : 1;                                  \
        }                                                                             \
    } while (0)

static uint32_t bits(float f) {
    uint32_t u;
    memcpy(&u, &f, 4);
    return u;
}
static hnb_expr lit_f(hnb_module* m, float x) {
    uint32_t w[1] = {bits(x)};
    return hnb_module_lit(m, HNB_FLOAT, w);
}
static hnb_expr lit_v3(hnb_module* m, float x, float y, float z) {
    uint32_t w[3] = {bits(x), bits(y), bits(z)};
    return hnb_module_lit(m, HNB_VEC3, w);
}
static uint32_t attribute_index(const char* name) {
    for (uint32_t i = 0; i < hnb_attribute_count(); ++i) {
        const char* n;
        uint32_t vt, def[4];
        hnb_attribute_info(i, &n, &vt, def);
        if (strcmp(n, name) == 0) return i;
    }
    return 0xFFFFFFFFu;
}
static int32_t set_attribute(hnb_asset* a, uint32_t context, const char* attr, hnb_expr value) {
    uint32_t param = attribute_index(attr);
    return hnb_asset_add_modifier(a, context, HNB_MOD_SET_ATTRIBUTE, &value, 1, &param, 1);
}

int main(int argc, char** argv) {
    const int frames = argc > 1 ? atoi(argv[1]) : 120;
    const uint32_t capacity = 32768;
    printf("%s\n", hnb_version());

    /* ---- authoring (CPU only) */
    hnb_module* m = hnb_module_create();
    /* velocity = normalize(rand(vec3) * 2 - 1) * uniform(40, 60) */
    hnb_expr dir = hnb_module_unary(m, HNB_UN_NORMALIZE,
                                    hnb_module_binary(m, HNB_BIN_SUB, hnb_module_binary(m, HNB_BIN_MUL, hnb_module_builtin(m, HNB_BUILTIN_RAND, HNB_VEC3), lit_f(m, 2.f)),
                                                      lit_f(m, 1.f)));
    hnb_expr velocity = hnb_module_binary(m, HNB_BIN_MUL, dir, hnb_module_binary(m, HNB_BIN_UNIFORM_RAND, lit_f(m, 40.f), lit_f(m, 60.f)));
    hnb_expr lifetime = hnb_module_binary(m, HNB_BIN_UNIFORM_RAND, lit_f(m, 0.8f), lit_f(m, 1.2f));
    hnb_expr drag = lit_f(m, 4.f), gravity = lit_v3(m, 0.f, -16.f, 0.f);
    hnb_expr origin = lit_v3(m, 0.f, 0.f, 0.f), zero = lit_f(m, 0.f);
    if (!dir || !velocity || !lifetime) {
        fprintf(stderr, "expression error: %s\n", hnb_last_error());
        return 1;
    }
    hnb_asset* asset = hnb_asset_create("firework_trails", capacity, m);
    CHECK(set_attribute(asset, HNB_CONTEXT_INIT, "position", origin));
    CHECK(set_attribute(asset, HNB_CONTEXT_INIT, "velocity", velocity));
    CHECK(set_attribute(asset, HNB_CONTEXT_INIT, "age", zero));
    CHECK(set_attribute(asset, HNB_CONTEXT_INIT, "lifetime", lifetime));
    CHECK(hnb_asset_add_modifier(asset, HNB_CONTEXT_UPDATE, HNB_MOD_LINEAR_DRAG, &drag, 1, NULL, 0));
    CHECK(hnb_asset_add_modifier(asset, HNB_CONTEXT_UPDATE, HNB_MOD_ACCEL, &gravity, 1, NULL, 0));
    hnb_generated* gen = NULL;
    CHECK(hnb_asset_generate(asset, NULL, 0, &gen));
    hnb_effect_desc desc;
    CHECK(hnb_generated_desc(gen, &desc));
    printf("lowered '%s': %u-byte particle records, %u attributes\n--- update code ---\n%s\n", desc.name, desc.particle_stride, desc.n_attrs,
           desc.update_code);

    /* ---- CPU producers */
    hnb_spawner_settings settings;
    CHECK(hnb_spawner_settings_burst(1000.f, 1.0f, &settings)); /* 1000 particles every second */
    hnb_effect_spawner* spawner = hnb_effect_spawner_create(&settings, 42);
    hnb_batcher* batcher = hnb_batcher_create();

    /* ---- runtime (needs an H100) */
    hnb_ctx* ctx = NULL;
    CHECK(hnb_ctx_create(0, 0, &ctx));
    hnb_effect effect;
    hnb_slab slab;
    CHECK(hnb_effect_compile(ctx, &desc, &effect));
    CHECK(hnb_slab_create(ctx, capacity, desc.particle_stride, &slab));
    hnb_effect_metadata md;
    memset(&md, 0xFF, sizeof md); /* every optional index = invalid */
    md.capacity = capacity;
    md.alive_count = 0;
    md.max_update = 0;
    md.max_spawn = capacity;
    md.indirect_write_index = 0;
    md.indirect_draw_index = 0;
    md.particle_stride = desc.particle_stride / 4;
    md.particle_counter = 0;
    CHECK(hnb_metadata_insert(ctx, 0, &md));
    hnb_draw_indexed_indirect_args draw0 = {6, 0, 0, 0, 0}; /* a quad: index_count 6, instance_count filled by the simulation */
    CHECK(hnb_draw_args_insert(ctx, 0, &draw0));

    /* Time<EffectSimulation> (reference src/time.rs): real frame times in, GpuSimParams out */
    hnb_sim_clock* clock = hnb_sim_clock_create();
    uint32_t peak = 0;
    for (int f = 0; f < frames; ++f) {
        hnb_sim_params sim;
        CHECK(hnb_sim_clock_advance(clock, 16666667ull)); /* a 60 Hz frame */
        CHECK(hnb_sim_clock_sim_params(clock, 1, &sim));
        const float dt = sim.delta_time; /* tick_spawners reads the same clock (spawn.rs:948, :963) */
        uint32_t spawn = 0;
        CHECK(hnb_effect_spawner_tick(spawner, dt, &spawn));
        hnb_spawner row;
        memset(&row, 0, sizeof row);
        row.transform.x_row[0] = row.transform.y_row[1] = row.transform.z_row[2] = 1.f; /* identity */
        row.inverse_transform.x_row[0] = row.inverse_transform.y_row[1] = row.inverse_transform.z_row[2] = 1.f;
        row.spawn = (int32_t)spawn;
        row.seed = 0x1234u + (uint32_t)f;
        row.effect_metadata_index = 0;
        row.draw_indirect_index = 0;
        row.slab_offset = 0;
        row.parent_slab_offset = 0xFFFFFFFFu;
        hnb_batch_key key = {1, slab, effect, 0xFFFFFFFFu, 0xFFFFFFFFu, 0, 1};
        int32_t batch_index = -1;
        hnb_batcher_clear(batcher);
        CHECK(hnb_batcher_push(batcher, &key, 0, 0, spawn, &batch_index));
        const hnb_batch_info* infos;
        const uint32_t* prefix;
        uint32_t n_batches, n_prefix, totals[1];
        CHECK(hnb_batcher_finish(batcher, &infos, &n_batches, &prefix, &n_prefix, totals, 1));

        CHECK(hnb_set_sim_params(ctx, &sim));
        CHECK(hnb_upload_spawners(ctx, &row, 1));
        CHECK(hnb_upload_batches(ctx, infos, n_batches, prefix, n_prefix));
        hnb_batch_launch launch = HNB_BATCH_LAUNCH_INIT(effect, slab, 0, totals[0]);
        CHECK(hnb_simulate(ctx, &launch, 1));
        if (f % 20 == 19 || f == frames - 1) {
            hnb_draw_indexed_indirect_args draw;
            CHECK(hnb_read_draw_args(ctx, 0, &draw)); /* what the indirect draw would consume */
            printf("frame %4d: spawned %4u, alive (instance_count) %u\n", f, spawn, draw.instance_count);
            if (draw.instance_count > peak) peak = draw.instance_count;
        }
    }
    CHECK(hnb_sync(ctx));
    printf("ok: %d frames, peak alive %u, %llu kernel launches\n", frames, peak, (unsigned long long)hnb_ctx_launch_count(ctx));
    hnb_slab_destroy(ctx, slab);
    hnb_effect_destroy(ctx, effect);
    hnb_ctx_destroy(ctx);
    hnb_batcher_destroy(batcher);
    hnb_sim_clock_destroy(clock);
    hnb_effect_spawner_destroy(spawner);
    hnb_generated_destroy(gen);
    hnb_asset_destroy(asset);
    hnb_module_destroy(m);
    return peak > 0 ? 0 : 2;
}
