// hnb_particle_kernels.cuh — hand-written sm_90a kernel templates for the two per-particle passes
// of the hot path. They play the role of the reference's WGSL templates
//   src/render/vfx_init.wgsl   (entry :101-196)   → hnb_init
//   src/render/vfx_update.wgsl (entry :106-167)   → hnb_update
// and are specialised per effect by textual inclusion after a generated section (see
// runtime/effect_source.cpp) which must define, inside namespace hnb:
//
//   HNB_NUM_PLANES, HNB_HAS_PROPERTIES, HNB_CONSUME_EVENTS, HNB_EMIT_EVENTS, HNB_READ_PARENT,
//   HNB_RELAXED_ORDER, HNB_TILE_K
//   struct Particle;  struct Properties;  struct RawParticle;  [struct ParentParticle]
//   hnb_load_raw / hnb_store_raw / hnb_unpack / hnb_pack       (SoA planes <-> Particle)
//   hnb_store_written                          the update's store: only the columns holding a word it may write
//   hnb_init_body(Particle&, Ctx&)            = {{INIT_CODE}} + PREV/NEXT reset + {{SIM_SPACE}}
//   hnb_update_body(Particle&, Ctx&) -> bool  = {{AGE_CODE}} {{REAP_CODE}} {{UPDATE_CODE}}, returns is_alive
//   [HNB_LIFE_FLOOR: hnb_load_raw_but_life / hnb_load_life / hnb_raw_age / hnb_raw_life]  (lifetime floors)
//   [HNB_GROUP_AGE: hnb_load_raw_but_life_age / hnb_load_age / hnb_set_raw_age]  (common ages)
//
// Design (DESIGN.md §kernels):
//   * update is a persistent, single-pass "process + stable compaction" kernel with WARP-AUTONOMOUS
//     tiles: every warp of the persistent grid takes tiles of tile_rows = 32*K*chunks rows of ONE effect
//     instance from a ticket counter. The compaction of a tile (look-back + index writes) is DEFERRED
//     until the warp has streamed its next tile, by which time every predecessor has published its
//     aggregate: nobody waits (see "deferred compaction" below). Rows are read through the alive
//     list (coalesced u32), particles through float4 SoA planes, processed in registers and written
//     back; survivors are compacted into the write list in row order with warp ballots inside the tile
//     and a decoupled look-back chain (one 64-bit state word per tile) across the tiles of the same
//     instance; dead rows are pushed on the dead stack in the same canonical (row) order. There is one
//     block barrier (after the prologue) and — in ordered mode — the only atomic is the tile ticket: the per-particle contended
//     atomics of the reference (vfx_update.wgsl:150,160,164) become exact ranks, which also makes the
//     list ORDER deterministic (= the reference's threads run in ascending global_invocation_id).
//     With HNB_RELAXED_ORDER the chain is replaced by one warp-aggregated atomic per tile (counts and
//     sets identical, order scheduling dependent like the reference).
//   * init pops dead slots by rank as well: thread k of an instance takes dead[alive_count + k]
//     (vfx_init.wgsl:141-143 in serial order); the alive_count / particle_counter increments are
//     applied by the bookkeeping kernel that follows (hnb_static_kernels.cu).
#pragma once

namespace hnb {

#define HNB_BLOCK 256
#define HNB_WARPS (HNB_BLOCK / 32)
// A tile is 1..HNB_MAX_CHUNKS sub-tiles of 32*K rows (BatchParams::tile_rows); at most 16 rows per
// lane, i.e. 512 rows per tile, so that the alive-list entries of TWO tiles (the one being streamed and
// the one whose compaction is deferred) fit a 2 x 2 KB per-warp stash.
#ifndef HNB_ROWS_PER_LANE
#define HNB_ROWS_PER_LANE 16
#endif
#define HNB_MAX_CHUNKS (HNB_ROWS_PER_LANE / HNB_TILE_K)
#if HNB_SLOT_ORDER && HNB_ROWS_PER_LANE > 32
#error "slot order gives each lane one alive-bitmap word of a tile: HNB_ROWS_PER_LANE must be at most 32"
#endif
#ifndef HNB_SMEM_EFFECTS
#define HNB_SMEM_EFFECTS 2047  // tile_prefix entries staged in shared memory (8 KB with the end sentinel)
#endif
#define HNB_SMEM_PREFIX_BYTES ((HNB_SMEM_EFFECTS + 1) * 4)
#ifndef HNB_MIN_BLOCKS
#define HNB_MIN_BLOCKS 3  // H100, C5 at 64 / 8 Mi: 4 CTAs (64 registers) 6 % slower, 2 CTAs within 1 %
#endif
#ifndef HNB_PROFILE
#define HNB_PROFILE 0  // 1: accumulate per-phase cycle counters into BatchParams::debug (diagnostics)
#endif
#ifndef HNB_SLOT_ORDER
#define HNB_SLOT_ORDER 0  // 1 (HNB_EFFECT_SLOT_ORDER): the update pass walks the instance's SLOTS in ascending order, guided by
                          // the slab's alive bitmap, instead of walking the alive list. See "slot order" below.
#endif
#ifndef HNB_LIFE_FLOOR
#define HNB_LIFE_FLOOR 0  // 1 (generated for HNB_ATTR_REAP_ONLY lifetimes in a column of their own): see "lifetime floors" below
#endif
#if HNB_LIFE_FLOOR && (HNB_SLOT_ORDER || HNB_RELAXED_ORDER)
#error "lifetime floors are kept by the ordered update pass only"
#endif
#ifndef HNB_GROUP_AGE
#define HNB_GROUP_AGE 0  // 1 (generated with HNB_LIFE_FLOOR when the age has a column of its own): see "common ages" below
#endif
#if HNB_GROUP_AGE && !HNB_LIFE_FLOOR
#error "common ages are kept with lifetime floors only"
#endif

// --- tile state word of the decoupled look-back ---
//   default:    [63:34] epoch | [33:32] flag | [31:0] survivors
//   slot order: [63:62] flag | [61:56] epoch & 63 | [55:28] survivors | [27:0] valid rows   (two running counts: the dead
//               stack position of a dead row needs the number of ALIVE-BEFORE-THE-PASS rows in front of it, which in
//               alive-list order is simply the row number; instances are limited to 2^28 slots)
#define HNB_FLAG_AGGREGATE 1ull
#define HNB_FLAG_PREFIX 2ull
#if HNB_SLOT_ORDER
HNB_DI u64 hnb_pack_state(u32 epoch, u64 flag, u32 survivors, u32 valid) {
    return (flag << 62) | (u64(epoch & 63u) << 56) | (u64(survivors) << 28) | u64(valid);
}
HNB_DI u32 hnb_state_flag(u64 s, u32 epoch) { return ((u32(s >> 56) & 63u) == (epoch & 63u)) ? u32(s >> 62) : 0u; }
HNB_DI u64 hnb_state_value(u64 s) { return s & 0x00ffffffffffffffull; }
#else
HNB_DI u64 hnb_pack_state(u32 epoch, u64 flag, u32 value) { return (u64(epoch) << 34) | (flag << 32) | u64(value); }
HNB_DI u32 hnb_state_flag(u64 s, u32 epoch) { return (u32(s >> 34) == epoch) ? (u32(s >> 32) & 3u) : 0u; }
HNB_DI u64 hnb_state_value(u64 s) { return s & 0xffffffffull; }
#endif
HNB_DI void hnb_st_state(u64* p, u64 v) { asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }
HNB_DI u64 hnb_ld_state(const u64* p) {
    u64 v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}

// one 64-bit word into the host's count mailbox (system scope: the reader is the CPU)
HNB_DI void hnb_post_count(const BatchParams& P, u32 epoch, u32 render_index, u32 count) {
    if (!P.mailbox || render_index >= P.mailbox_rows) return;
    unsigned long long* slot = P.mailbox + size_t(epoch % P.mailbox_ring) * P.mailbox_rows + render_index;
    const unsigned long long word = (u64(epoch) << 32) | u64(count);
#if defined(__CUDA_ARCH__)
    asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(slot), "l"(word) : "memory");
#else
    *(volatile unsigned long long*)slot = word;
#endif
}

HNB_DI u32 hnb_lanemask_lt() {
    u32 m;
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
    return m;
}

// find_location_from_particle (vfx_update.wgsl:51-72 / vfx_init.wgsl:51-72): upper bound of `x` in
// prefix[lo,hi), minus one. `prefix[lo]` is 0 by construction so the result is always >= lo.
template <typename Ptr> HNB_DI u32 hnb_find_effect(Ptr prefix, u32 lo, u32 hi, u32 x) {
    while (lo < hi) {
        const u32 mid = (hi + lo) >> 1u;
        if (x >= prefix[mid]) lo = mid + 1u; else hi = mid;
    }
    return lo - 1u;
}

// ---------------------------------------------------------------------------------------------
// init  ≙ vfx_init.wgsl main()
// ---------------------------------------------------------------------------------------------
// Each CUDA thread runs HNB_INIT_ITEMS of the reference's init threads (logical thread index = CTA base +
// k*HNB_BLOCK + threadIdx, so every k is a coalesced row of the dead stack / alive list). One spawn per thread is
// latency-bound: the work is a chain broadcast loads -> dead-slot load -> PRNG -> stores, so a thread lives long
// for 40 bytes of traffic; with the items' chains issued together the launch is bandwidth-bound instead.
#ifndef HNB_INIT_ITEMS
#define HNB_INIT_ITEMS 4
#endif
// CPU prefix sums of a batch's spawn counts staged in shared memory (batches of up to this many instances; 4 KB of dynamic
// shared memory, mirrored by hnb_rt::kInitSmemBytes on the host)
#define HNB_INIT_SMEM_EFFECTS 1024
// Dynamic shared memory of both kernels (hnb_init: the staged spawn prefix; hnb_update: see its carve-up)
extern __shared__ __align__(16) unsigned char hnb_smem[];
extern "C" __global__ void __launch_bounds__(HNB_BLOCK) hnb_init(const BatchParams P) {
    // The words only the HOST writes — the batch info and the CPU prefix sums of the spawn counts (batch.rs:358-383), staged in
    // shared memory so that the per-thread location search (vfx_init.wgsl:51-72; ten dependent steps for a batch of 1024
    // instances) runs on shared memory instead of on ten L2 round trips — are read BEFORE the dependency wait when they came
    // with a stream-ordered copy, and after it when the kernel just ahead of this one is the one that stores them
    // (`late_tables`: the frame block travelled as a kernel parameter, k_frame_block).
    BatchInfo bi;
    u32* const sh_spawn_prefix = (u32*)hnb_smem;
    bool staged = false;
#pragma unroll
    for (int phase = 0; phase < 2; ++phase) {
        if ((phase == 1) == (P.late_tables != 0u)) {
            bi.spawner_base = P.bi_spawner_base;  // (kernel parameters: the host knows its batch info when it launches)
            bi.prefix_sum_offset = P.bi_prefix_sum_offset;
            bi.prefix_sum_count = P.bi_prefix_sum_count;
            staged = bi.prefix_sum_count <= HNB_INIT_SMEM_EFFECTS;
            if (staged) {
                for (u32 i = threadIdx.x; i < bi.prefix_sum_count; i += HNB_BLOCK) sh_spawn_prefix[i] = P.spawn_prefix[bi.prefix_sum_offset + i];
                __syncthreads();
            }
        }
        if (phase == 0) {
            hnb_pdl_wait();  // the previous frame's update wrote the dead stack and the counters read below
            // Dependents are signalled AFTER the wait: a successor (this frame's bookkeeping) reads host-written arena words before
            // its own wait, and the arena may be (re)written by the predecessor of THIS grid when a frame block travels as a
            // kernel parameter — a successor must therefore never become resident before this grid's predecessors are complete.
            hnb_pdl_launch_dependents();
        }
    }
    struct Item {
        const Spawner* spawner;
        const EffectMetadata* md;
        u32 update_index, alive_index, dead;
        bool ok;
    } items[HNB_INIT_ITEMS];

    // ---- locate, apply the caps, pop the dead slot. The chain location -> spawner row -> metadata row -> dead slot is four
    // DEPENDENT round trips; it is walked phase by phase over ALL items, so that the items' loads of a phase are in flight
    // together whatever instances they belong to (a batch of 1024 instances spawning one particle each gives every item of a
    // thread a different instance: item after item would be sixteen round trips, phase after phase is four).
    u32 md_index[HNB_INIT_ITEMS], max_spawn[HNB_INIT_ITEMS], alive_count[HNB_INIT_ITEMS], requested[HNB_INIT_ITEMS], slab_offset[HNB_INIT_ITEMS];
    // phase A: location in the packed init space of this batch (CPU prefix sums of spawn counts, batch.rs:358-383); the
    // spawner row's CPU words
#pragma unroll
    for (int k = 0; k < HNB_INIT_ITEMS; ++k) {
        Item& it = items[k];
        const u32 thread_index = (blockIdx.x * HNB_INIT_ITEMS + k) * HNB_BLOCK + threadIdx.x;  // global_invocation_id.x
        it.ok = thread_index < P.init_thread_count;
        it.dead = 0u; it.update_index = 0u; it.alive_index = 0u;
        it.spawner = P.spawners; it.md = P.metadata;
        md_index[k] = 0u; requested[k] = 0u; slab_offset[k] = 0u;
        if (it.ok) {
            u32 effect_index;
            if (staged) {
                effect_index = hnb_find_effect(sh_spawn_prefix, 0u, bi.prefix_sum_count, thread_index);
                it.update_index = thread_index - sh_spawn_prefix[effect_index];
            } else {
                const u32 slot = hnb_find_effect(P.spawn_prefix, bi.prefix_sum_offset, bi.prefix_sum_offset + bi.prefix_sum_count, thread_index);
                effect_index = slot - bi.prefix_sum_offset;
                it.update_index = thread_index - P.spawn_prefix[slot];
            }
            it.spawner = &P.spawners[bi.spawner_base + effect_index];
            md_index[k] = it.spawner->effect_metadata_index;
            slab_offset[k] = it.spawner->slab_offset;
#if !HNB_CONSUME_EVENTS
            requested[k] = u32(it.spawner->spawn);
#endif
        }
    }
    // phase B: the metadata row
#pragma unroll
    for (int k = 0; k < HNB_INIT_ITEMS; ++k) {
        Item& it = items[k];
        max_spawn[k] = 0u; alive_count[k] = 0u;
        if (it.ok) {
            it.md = &P.metadata[md_index[k]];
            max_spawn[k] = it.md->max_spawn;
            alive_count[k] = it.md->alive_count;
#if HNB_CONSUME_EVENTS
            requested[k] = it.md->global_child_index;  // (index of the child info; its event count is loaded in phase B2)
#endif
        }
    }
#if HNB_CONSUME_EVENTS
    // phase B2: GPU-event driven instance: requested = event_count (vfx_init.wgsl:123-129), event_index = update_index
#pragma unroll
    for (int k = 0; k < HNB_INIT_ITEMS; ++k)
        if (items[k].ok) requested[k] = u32(P.child_infos[requested[k]].event_count);
#endif
    // phase C: cap to the number of dead particles and to the request (vfx_init.wgsl:115-137), recycle a dead slot.
    // Serial-order equivalent of `atomicAdd(alive_count, 1)` (:141): every thread with a smaller update_index also passed
    // the caps, so this thread's rank IS update_index.
#pragma unroll
    for (int k = 0; k < HNB_INIT_ITEMS; ++k) {
        Item& it = items[k];
        it.ok = it.ok && it.update_index < max_spawn[k] && it.update_index < requested[k];
        if (it.ok) {
            it.alive_index = alive_count[k] + it.update_index;
            it.dead = P.slab.dead_index[slab_offset[k] + it.alive_index];
        }
    }

    // ---- initialise and store
#pragma unroll
    for (int k = 0; k < HNB_INIT_ITEMS; ++k) {
        const Item& it = items[k];
        if (!it.ok) continue;
        const Spawner* spawner = it.spawner;
        const EffectMetadata* md = it.md;
        const u32 base_particle = spawner->slab_offset;
        const u32 particle_index = it.dead - base_particle;

        Ctx hnb_ctx;
        hnb_ctx.particle_index = particle_index;
        hnb_ctx.particle_counter = md->particle_counter + it.update_index;  // atomicAdd(particle_counter, 1) (:151)
        hnb_ctx.seed = pcg_hash(particle_index ^ spawner->seed);            // :154
        hnb_ctx.sim = &P.frame->sim;
        hnb_ctx.spawner = spawner;
        hnb_ctx.transform = hnb_transform_from_rows(spawner->transform, spawner->transform + 4, spawner->transform + 8);
        hnb_ctx.inverse_transform = hnb_transform_from_rows(spawner->inverse_transform, spawner->inverse_transform + 4,
                                                            spawner->inverse_transform + 8);
        hnb_ctx.is_alive = true;
#if HNB_HAS_PROPERTIES
        hnb_ctx.props = (const Properties*)((const char*)P.properties + size_t(md->properties_array_index) * P.properties_stride);
#else
        hnb_ctx.props = nullptr;
#endif
#if HNB_READ_PARENT
        {
            const u32 parent_base_particle = spawner->parent_slab_offset;
            hnb_ctx.parent_particle_index = P.consume_events[it.update_index];
            ParentRawParticle praw;
            hnb_parent_load_raw(praw, P.parent_slab, parent_base_particle + hnb_ctx.parent_particle_index);
            hnb_parent_unpack(praw, hnb_ctx.parent_particle);
        }
#endif

        Particle particle = Particle();
        hnb_init_body(particle, hnb_ctx);

        // Append to the alive list (:191-192) and write the particle back (:195). The instance's first appended row ends what an
        // identity claim on the column can cover.
        if (it.update_index == 0u && P.slab.ident_claim) {
            u64* const claim = &P.slab.ident_claim[md->indirect_write_index];
            if (hnb_claim_len(hnb_claim_load(claim), base_particle) > it.alive_index) hnb_claim_store(claim, hnb_claim_pack(base_particle, it.alive_index));
        }
        P.slab.particle_index[md->indirect_write_index][base_particle + it.alive_index] = particle_index;
#if HNB_SLOT_ORDER
        atomicOr(&P.slab.alive_bits[(base_particle + particle_index) >> 5u], 1u << ((base_particle + particle_index) & 31u));
#endif
        RawParticle raw;
        hnb_raw_zero(raw);
        hnb_pack<true>(particle, raw);  // init also stores PREV/NEXT (vfx_init.wgsl:175-181)
        hnb_store_raw(raw, P.slab, base_particle + particle_index);
#if HNB_LIFE_FLOOR
        // the slot's lifetime changed: its group's floor proves nothing until an update stores a new one
        if (P.life_floor) P.life_floor[(base_particle + particle_index) >> 5u] = __uint_as_float(HNB_LIFE_FLOOR_NONE);
#endif
#if HNB_GROUP_AGE
        // ... and so did its age: the group's common age is unknown
        if (P.group_age) P.group_age[(base_particle + particle_index) >> 5u] = HNB_GROUP_AGE_NONE;
#endif
    }
}

// ---------------------------------------------------------------------------------------------
// update  ≙ vfx_update.wgsl main()
// ---------------------------------------------------------------------------------------------
// A tile whose rows have been simulated (pass 1) and whose compaction is still to be done. Lives in
// shared memory (one per warp) so that it costs no registers while the next tile is being streamed.
struct PendingTile {
    u32 tile, row0, tile_alive;
    u32 base_particle, max_update, write_index, render_index;
    u32 inst_first_tile, inst_end_tile, metadata_index, buffer;
    u32 tile_valid;  // slot order: rows of the tile that were alive before the pass
    // identity claims as read when the instance was bound (a parked tile may be compacted after the instance's last tile has
    // rewritten the claim): read-column rows known to be the identity, length of the write column's claim for this instance
    u32 trust_r, claim_w;
    // not a field of the parked tile: lane 0's running count, over the tile being streamed, of the common-age words it made
    // deferred less those it found deferred (HNB_GROUP_AGE; kept here rather than in a register, which hnb_update lacks)
    u32 defer_delta;
    u32 _pad;
};
static_assert(sizeof(PendingTile) == 64, "update_smem_bytes on the host reserves 64 bytes per warp for the parked tile");

// Compaction of one tile: exclusive prefix of survivors over the previous tiles of the instance
// (decoupled look-back), then survivors -> write list, dead -> dead stack (vfx_update.wgsl:148-166).
HNB_DI void hnb_compact_tile(const BatchParams& P, const PendingTile& pt, const u32* survivors, const u32* valids, const u32 (*pidx_stash)[32],
                             u32 chunks, u32 epoch, u32 lane, long long& prof_polls) {
    u64* const states = P.tile_state;
    const u32 tile = pt.tile, row0 = pt.row0, tile_alive = pt.tile_alive, max_update = pt.max_update;
    const u32 base_particle = pt.base_particle, inst_first_tile = pt.inst_first_tile;
    EffectMetadata* const md = &P.metadata[pt.metadata_index];
    u32* __restrict__ write_col = P.slab.particle_index[pt.write_index] + base_particle;
    (void)prof_polls;

    u32 alive_before = 0u;
#if HNB_SLOT_ORDER
    u32 valid_before = 0u;
    u64 sum_before = 0ull;  // both counts, packed like the state word's value
#else
    (void)valids;
#endif
#if HNB_RELAXED_ORDER
    // Reference-style order (vfx_update.wgsl:164) with one warp-aggregated atomic per tile.
    if (lane == 0) alive_before = atomicAdd(&P.draw_args[HNB_DRAW_INDEXED_INDIRECT_STRIDE * pt.render_index + 1u], tile_alive);
    alive_before = __shfl_sync(0xffffffffu, alive_before, 0);
#else
    if (tile != inst_first_tile) {
        // Walk back over the predecessors' states, 32 of them per round trip (lane l examines tile pos - l), summing
        // AGGREGATEs until the first PREFIX. Tiles before the instance's first tile count as a PREFIX of 0. With deferred
        // compaction the first window almost always holds a PREFIX (128 predecessors per round trip measured 2.7 % slower).
        u32 pos = tile - 1u;  // newest predecessor not yet accounted for
        for (;;) {
#if HNB_SLOT_ORDER
            const u64 s = (pos >= inst_first_tile + lane) ? hnb_ld_state(&states[pos - lane]) : hnb_pack_state(epoch, HNB_FLAG_PREFIX, 0u, 0u);
#else
            const u64 s = (pos >= inst_first_tile + lane) ? hnb_ld_state(&states[pos - lane]) : hnb_pack_state(epoch, HNB_FLAG_PREFIX, 0u);
#endif
            const u32 flag = hnb_state_flag(s, epoch);
            const u32 ready_mask = __ballot_sync(0xffffffffu, flag != 0u);
            const u32 prefix_mask = __ballot_sync(0xffffffffu, flag == u32(HNB_FLAG_PREFIX));
            const u32 first_p = prefix_mask ? (u32)(__ffs(prefix_mask) - 1) : 32u;
            const u32 need = first_p >= 31u ? 0xffffffffu : ((2u << first_p) - 1u);
            if ((ready_mask & need) != need) {  // a needed predecessor has not published yet: poll again from here
#if HNB_PROFILE
                prof_polls++;
#endif
                continue;
            }
#if HNB_SLOT_ORDER
            u64 contrib = lane <= first_p ? hnb_state_value(s) : 0ull;
#pragma unroll
            for (int d = 16; d > 0; d >>= 1) contrib += __shfl_xor_sync(0xffffffffu, contrib, d);
            sum_before += contrib;
#else
            u32 contrib = lane <= first_p ? u32(s) : 0u;
#pragma unroll
            for (int d = 16; d > 0; d >>= 1) contrib += __shfl_xor_sync(0xffffffffu, contrib, d);
            alive_before += contrib;
#endif
            if (prefix_mask) break;
            pos -= 32u;
        }
#if HNB_SLOT_ORDER
        alive_before = u32(sum_before >> 28) & 0x0fffffffu;
        valid_before = u32(sum_before) & 0x0fffffffu;
        if (lane == 0) hnb_st_state(&states[tile], hnb_pack_state(epoch, HNB_FLAG_PREFIX, alive_before + tile_alive, valid_before + pt.tile_valid));
#else
        if (lane == 0) hnb_st_state(&states[tile], hnb_pack_state(epoch, HNB_FLAG_PREFIX, alive_before + tile_alive));
#endif
    }
#endif

    // survivors into the write list, the dead onto the dead stack, indices from the shared-memory stash
    u32 alive_rank_base = alive_before;
#if HNB_SLOT_ORDER
    // slot order: a row IS its slot; rows that were alive before the pass are the set bits of `valids`
    (void)pidx_stash;
    u32 valid_rank_base = valid_before;
#pragma unroll 4
    for (u32 jk = 0; jk < chunks * HNB_TILE_K; ++jk) {
        const u32 row = row0 + jk * 32u + lane;
        const u32 ballot = survivors[jk], vmask = valids[jk];
        if ((vmask >> lane) & 1u) {
            const u32 alive_rank = alive_rank_base + __popc(ballot & hnb_lanemask_lt());
            if ((ballot >> lane) & 1u) {
                write_col[alive_rank] = row;
            } else {
                // serial-order value of atomicSub(alive_count,1)-1 when the threads run in ascending slot order
                const u32 dead_rank = valid_rank_base + __popc(vmask & hnb_lanemask_lt()) - alive_rank;
                P.slab.dead_index[base_particle + (max_update - 1u - dead_rank)] = base_particle + row;
            }
        }
        alive_rank_base += __popc(ballot);
        valid_rank_base += __popc(vmask);
    }
    if (lane == 0 && tile + 1u == pt.inst_end_tile) {
        const u32 alive_total = alive_before + tile_alive;
        const u32 dead_total = max_update - alive_total;
        P.draw_args[HNB_DRAW_INDEXED_INDIRECT_STRIDE * pt.render_index + 1u] = alive_total;
        hnb_post_count(P, epoch, pt.render_index, alive_total);
        md->alive_count = md->alive_count - dead_total;
        md->max_spawn = md->max_spawn + dead_total;
        // the bitmap and the counters must describe the same population (debug word 15 counts instances where they do not)
        if (valid_before + pt.tile_valid != max_update && P.debug) atomicAdd(&P.debug[15], 1ull);
    }
#else
    const u32 claim_w = pt.claim_w;
#pragma unroll 4
    for (u32 jk = 0; jk < chunks * HNB_TILE_K; ++jk) {
        const u32 row = row0 + jk * 32u + lane;
        const u32 ballot = survivors[jk];
        if (row < max_update) {
            const u32 pidx = pidx_stash[jk][lane];
            const u32 alive_rank = alive_rank_base + __popc(ballot & hnb_lanemask_lt());  // surviving rows before `row`
            if ((ballot >> lane) & 1u) {
                if (pidx != alive_rank || alive_rank >= claim_w) write_col[alive_rank] = pidx;  // (else: the claim says it is there)
            } else {
#if HNB_RELAXED_ORDER
                const u32 alive_index = atomicSub(&md->alive_count, 1u) - 1u;
                P.slab.dead_index[base_particle + alive_index] = base_particle + pidx;
                atomicAdd(&md->max_spawn, 1u);
#else
                // `row - alive_rank` dead rows precede this one: serial-order value of
                // atomicSub(alive_count,1)-1 given alive_count == max_update at pass start.
                const u32 alive_index = max_update - 1u - (row - alive_rank);
                P.slab.dead_index[base_particle + alive_index] = base_particle + pidx;
#endif
            }
        }
        alive_rank_base += __popc(ballot);
    }
#if !HNB_RELAXED_ORDER
    // the last tile of the instance publishes the totals (replaces the per-particle atomics on
    // instance_count / alive_count / max_spawn)
    if (lane == 0 && tile + 1u == pt.inst_end_tile) {
        const u32 alive_total = alive_before + tile_alive;
        const u32 dead_total = max_update - alive_total;
        P.draw_args[HNB_DRAW_INDEXED_INDIRECT_STRIDE * pt.render_index + 1u] = alive_total;
        hnb_post_count(P, epoch, pt.render_index, alive_total);
        md->alive_count = md->alive_count - dead_total;
        md->max_spawn = md->max_spawn + dead_total;
        // The next claim on the write column: with an identity read list and no death, rows [0, max_update) now hold their own
        // index (rows beyond were not written, so a longer claim still holds there); otherwise drop the instance's claim.
        if (P.slab.ident_claim) {
            u64* const claim = &P.slab.ident_claim[pt.write_index];
            if (pt.trust_r >= max_update && alive_total == max_update) hnb_claim_store(claim, hnb_claim_pack(base_particle, claim_w > max_update ? claim_w : max_update));
            else if (claim_w != 0u) hnb_claim_store(claim, 0ull);
        }
    }
#endif
#endif  // HNB_SLOT_ORDER
}

extern "C" __global__ void __launch_bounds__(HNB_BLOCK, HNB_MIN_BLOCKS) hnb_update(const BatchParams P) {
    // Dynamic shared memory (size = hnb_update_smem_bytes, computed identically on the host):
    //   tile-prefix table | per warp, 2 buffers (streamed tile, parked tile): alive-list entries [2][R][32], survivor ballots
    //   [2][R], valid masks [2][R] | per warp: one PendingTile record | per warp: Properties staging slot
    u32* const sh_tile_prefix = (u32*)hnb_smem;
    typedef u32 PidxBuf[HNB_ROWS_PER_LANE][32];
    typedef u32 SurvBuf[HNB_ROWS_PER_LANE];
    enum : size_t { kStash = (sizeof(PidxBuf) + 2 * sizeof(SurvBuf)) * 2 * HNB_WARPS };
    PidxBuf(*const sh_pidx)[2] = (PidxBuf(*)[2])(hnb_smem + HNB_SMEM_PREFIX_BYTES);
    SurvBuf(*const sh_survivors)[2] = (SurvBuf(*)[2])(hnb_smem + HNB_SMEM_PREFIX_BYTES + sizeof(PidxBuf) * 2 * HNB_WARPS);
    SurvBuf(*const sh_valids)[2] = (SurvBuf(*)[2])(hnb_smem + HNB_SMEM_PREFIX_BYTES + (sizeof(PidxBuf) + sizeof(SurvBuf)) * 2 * HNB_WARPS);  // slot order
    PendingTile* const sh_pending = (PendingTile*)(hnb_smem + HNB_SMEM_PREFIX_BYTES + kStash);
#if HNB_HAS_PROPERTIES
    typedef unsigned char PropsBuf[(sizeof(Properties) + 15) / 16 * 16];
    PropsBuf* const sh_props = (PropsBuf*)(hnb_smem + HNB_SMEM_PREFIX_BYTES + kStash + sizeof(PendingTile) * HNB_WARPS);
#endif
    const u32 tid = threadIdx.x;
    const u32 lane = tid & 31u;
    const u32 warp = tid >> 5u;
    // Programmatic dependent launch: this grid may have become resident while the bookkeeping kernel (and, behind it,
    // the previous frame's update) was still running — its launch latency and CTA start skew are hidden. Nothing
    // those kernels write has been read yet; from here on it is all visible. The next kernel in the stream (the next
    // frame's bookkeeping) is signalled AFTER the wait below: it reads host-written arena words before ITS wait, and this
    // frame's bookkeeping may be the one that writes them (frame block as a kernel parameter), so it must be complete first.
#if HNB_PROFILE
    // per-frame timeline ring (diagnostics, tools/diag_frame_chain.py): 4 words per frame at debug[16 + 4 * (epoch & 63)]:
    // ~(earliest CTA residency), ~(earliest start after the dependency wait), ~(earliest end of a first sub-tile), latest warp end
    unsigned long long prof_resident;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(prof_resident));
#endif
    hnb_pdl_wait();
    hnb_pdl_launch_dependents();
#if HNB_PROFILE
    if (lane == 0 && P.debug) { unsigned long long _g; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(_g)); atomicMax(&P.debug[8], ~_g); }
    unsigned long long* const prof_ring = P.debug ? P.debug + 16 + 4 * (P.frame->epoch & 63u) : nullptr;
    if (lane == 0 && prof_ring) {
        unsigned long long _g; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(_g));
        atomicMax(&prof_ring[0], ~prof_resident);
        atomicMax(&prof_ring[1], ~_g);
    }
#endif

    // (Reading the host-written batch info / first spawner row before the wait was tried: it gains a little on an overlapped
    // chain and loses more on a launch that is NOT overlapped with its predecessor, because the wait then separates two groups
    // of dependent loads that used to be issued together. The bookkeeping kernel keeps its variant.)
    const u32 bi_spawner_base = P.bi_spawner_base, bi_prefix_sum_offset = P.bi_prefix_sum_offset, n_effects = P.bi_prefix_sum_count;  // (kernel parameters: no load)
    const u32* g_tile_prefix = P.tile_prefix + bi_prefix_sum_offset;
    const u32 total_tiles = *P.batch_tiles;
    const u32 epoch = P.frame->epoch;
    const bool staged = n_effects <= HNB_SMEM_EFFECTS;
    if (staged) {
        for (u32 i = tid; i < n_effects; i += HNB_BLOCK) sh_tile_prefix[i] = g_tile_prefix[i];
        if (tid == 0) sh_tile_prefix[n_effects] = total_tiles;
    }
    u64* const states = P.tile_state;
    // rows per tile = 32 lanes * K rows per lane * chunks; the chunk count is chosen per launch by the
    // host (and used by the bookkeeping kernel for the tile prefix), so it is a run-time value here
    const u32 tile_rows = hnb_tile_rows(P.tile_rows);
    const u32 chunks = tile_rows / (32u * HNB_TILE_K);
    PendingTile* const parked = &sh_pending[warp];  // this warp's parked tile
    // Tiles this warp has streamed so far (ordered builds): the next one uses stash buffer streamed & 1, the parked tile, if
    // any (streamed != 0), the other one. One counter rather than a buffer index and a has-parked flag: the extra live
    // register made the slot-order and force-field builds of hnb_update spill.
    u32 streamed = 0u;
#if HNB_GROUP_AGE
    if (lane == 0) parked->defer_delta = 0u;
#endif

    // cached descriptor of the instance the current tile belongs to (reloaded when a tile leaves
    // [inst_first_tile, inst_end_tile))
    u32 inst_first_tile = 1u, inst_end_tile = 0u;  // empty range
    Spawner* spawner = nullptr;
    u32 metadata_index = 0u;
    u32 base_particle = 0u, spawner_seed = 0u, max_update = 0u, write_index = 0u, render_index = 0u;
    u32 trust_r = 0u, claim_w = 0u;  // identity claims of the instance (see PendingTile)
#if HNB_SLOT_ORDER
    u32 inst_capacity = 0u;  // slots of the cached instance
#endif
    const u32* __restrict__ read_col = nullptr;

    Ctx hnb_ctx;
    hnb_ctx.sim = &P.frame->sim;
    hnb_ctx.particle_counter = 0u;
    hnb_ctx.props = nullptr;
#if HNB_EMIT_EVENTS
    hnb_ctx.child_infos = P.child_infos;
    for (int i = 0; i < HNB_MAX_EVENT_BINDINGS; ++i) {
        hnb_ctx.emit_events[i] = P.emit_events[i];
        hnb_ctx.emit_events_capacity[i] = P.emit_events_capacity[i];
    }
#endif

    // Binds the cached descriptor of one instance of the batch. `md_known`: the metadata row index is already known (kernel
    // parameter), so the metadata loads do not wait for the spawner row.
    auto bind_instance = [&](u32 effect_index, bool md_known, u32 md_hint) {
        spawner = &P.spawners[bi_spawner_base + effect_index];
        metadata_index = md_known ? md_hint : spawner->effect_metadata_index;
        const EffectMetadata* md = &P.metadata[metadata_index];
        base_particle = spawner->slab_offset;
        spawner_seed = spawner->seed;
        max_update = md->max_update;  // :119
#if HNB_SLOT_ORDER
        inst_capacity = md->capacity;
#endif
        write_index = md->indirect_write_index;
        render_index = md->indirect_render_index;
        read_col = P.slab.particle_index[1u - write_index] + base_particle;
#if HNB_RELAXED_ORDER || HNB_SLOT_ORDER
        // these orders trust no identity claim, and the list they write ends the instance's claim on the write column
        if (lane == 0 && P.slab.ident_claim && hnb_claim_len(hnb_claim_load(&P.slab.ident_claim[write_index]), base_particle) != 0u)
            hnb_claim_store(&P.slab.ident_claim[write_index], 0ull);
#else
        if (P.slab.ident_claim) {
            const u32 claim_r = hnb_claim_len(hnb_claim_load(&P.slab.ident_claim[1u - write_index]), base_particle);
            trust_r = claim_r < max_update ? claim_r : max_update;
            claim_w = hnb_claim_len(hnb_claim_load(&P.slab.ident_claim[write_index]), base_particle);
        }
#endif
        hnb_ctx.spawner = spawner;
        hnb_ctx.transform = hnb_transform_from_rows(spawner->transform, spawner->transform + 4, spawner->transform + 8);
        hnb_ctx.inverse_transform = hnb_transform_from_rows(spawner->inverse_transform, spawner->inverse_transform + 4,
                                                            spawner->inverse_transform + 8);
#if HNB_HAS_PROPERTIES
        {
            const u32* src = (const u32*)((const char*)P.properties + size_t(md->properties_array_index) * P.properties_stride);
            __syncwarp();
            for (u32 i = lane; i < sizeof(Properties) / 4u; i += 32u) ((u32*)sh_props[warp])[i] = src[i];
            __syncwarp();
            hnb_ctx.props = (const Properties*)sh_props[warp];
        }
#endif
#if HNB_EMIT_EVENTS
        hnb_ctx.base_child_index = md->base_child_index;
#endif
    };
    // A batch of ONE instance (BASELINE's C2, C3, C5): which instance the first tile belongs to needs no ticket and no search, and
    // its metadata row index came as a kernel parameter — its spawner row and metadata row are requested now, together with the
    // tile-prefix / ticket round trip instead of two dependent round trips behind it.
    if (n_effects == 1u) {
        bind_instance(0u, true, P.first_md_index);
        inst_first_tile = 0u;
        inst_end_tile = total_tiles;
    }
    // First tiles: one ticket request per CTA for its eight warps (all warps of the grid start within a few
    // microseconds of each other; this keeps 7/8 of those same-address atomics off the start of the kernel).
    __shared__ u32 sh_first_ticket;
    if (tid == 0) sh_first_ticket = atomicAdd(P.ticket, HNB_WARPS);
    __syncthreads();  // the only block barrier of the kernel

    // Tiles are handed out by a ticket counter, so every tile's predecessors in the look-back chain have
    // been taken by a running warp before it.
    u32 tile = sh_first_ticket + warp;
    long long prof_polls = 0;
#if HNB_PROFILE
    // per-warp cycle accounting of the phases (diagnostics only)
    long long prof_t0 = clock64(), prof_pass1 = 0, prof_compact = 0, prof_tiles = 0;
    const long long prof_start = prof_t0;
#define HNB_PROF_MARK(acc) { const long long _t = clock64(); acc += _t - prof_t0; prof_t0 = _t; }
    // timeline (ns, %globaltimer): [8] = ~(earliest warp start) [9] latest first ticket [10] latest end of a warp's
    // first pass 1 [11] latest warp end [12] = ~(earliest end of a first pass 1) [13] = ~(earliest warp end)
#define HNB_PROF_TIME(slot, invert) if (lane == 0 && P.debug) { unsigned long long _g; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(_g)); atomicMax(&P.debug[slot], (invert) ? ~_g : _g); }
    bool prof_first = true;
    HNB_PROF_TIME(9, false)
#else
#define HNB_PROF_MARK(acc)
#endif

    while (tile < total_tiles) {
        if (tile < inst_first_tile || tile >= inst_end_tile) {
            // Which instance does this tile belong to? (per-warp replacement of the per-thread binary
            // search of vfx_update.wgsl:51-72; all lanes read the same words: broadcast)
            u32 effect_index;
            if (staged) {
                effect_index = hnb_find_effect(sh_tile_prefix, 0u, n_effects, tile);
                inst_first_tile = sh_tile_prefix[effect_index];
                inst_end_tile = sh_tile_prefix[effect_index + 1u];
            } else {
                effect_index = hnb_find_effect(g_tile_prefix, 0u, n_effects, tile);
                inst_first_tile = g_tile_prefix[effect_index];
                inst_end_tile = effect_index + 1u < n_effects ? g_tile_prefix[effect_index + 1u] : total_tiles;
            }
            bind_instance(effect_index, false, 0u);
        }
        const u32 row0 = (tile - inst_first_tile) * tile_rows;
        u32* const survivors = sh_survivors[warp][streamed & 1u];
        u32(*const pidx_stash)[32] = sh_pidx[warp][streamed & 1u];

        // ---- pass 1: stream the tile's rows in `chunks` sub-tiles of 32*K rows:
        //      alive-list entry -> particle record -> simulate -> write back; remember who survived.
        u32 tile_alive = 0u;
#if HNB_SLOT_ORDER
        // Slot order: row r of the tile IS slot row0 + r of the instance; the slab's alive bitmap says which slots hold a
        // particle. Instances start on multiples of 32 slab rows (checked on the host), so word row0/32 + jk of the
        // bitmap belongs to this warp alone: lane jk loads it now and stores the survivors' ballot back after the pass —
        // 4 bytes per 32 slots instead of 4 bytes per particle of alive-list reads, and every record access of a warp
        // falls into one contiguous span of each plane, however the population was recycled.
        u32* const valids = sh_valids[warp][streamed & 1u];
        u32* const tile_bits = P.slab.alive_bits + ((base_particle + row0) >> 5u);
        const bool owns_word = lane < chunks * HNB_TILE_K && row0 + lane * 32u < inst_capacity;
        u32 my_bits = owns_word ? tile_bits[lane] : 0u;
        if (owns_word && inst_capacity - (row0 + lane * 32u) < 32u) my_bits &= (1u << (inst_capacity - (row0 + lane * 32u))) - 1u;
        u32 my_new_bits = 0u, tile_valid = 0u;
        (void)read_col;
#else
        // Rows below trust_r hold their own index (identity claim): their alive-list entries are not loaded. When that covers
        // the whole tile (warp-uniform), neither are the next sub-tiles' entries prefetched.
        const bool tile_known = row0 + tile_rows <= trust_r;
        u32 pidx_next[HNB_TILE_K];
#pragma unroll
        for (int k = 0; k < HNB_TILE_K; ++k) {
            const u32 row = row0 + k * 32u + lane;
            pidx_next[k] = row < trust_r ? row : (row < max_update ? read_col[row] : 0u);
        }
#endif
#if HNB_LIFE_FLOOR
        // Lifetime floors (DESIGN.md §3). In a tile wholly below trust_r every row holds its own index, so when the instance
        // starts on a 32-row group, row group k of a sub-tile is one slab group, and it lies wholly inside the instance's
        // slice (its rows are below max_update <= capacity): a group shared by two instances is neither read nor stored.
        // P.life_floor is NULL when the slab uses no floors. Any other tile loads whole records, as without floors.
        const bool tile_floors = P.life_floor != nullptr && tile_known && (base_particle & 31u) == 0u;  // warp-uniform
#endif
#if HNB_GROUP_AGE
        // Common ages (DESIGN.md §3) are read and stored in the same tiles as the floors. P.group_age is NULL when the slab
        // keeps none. A word counts only when the previous frame's update stored it: rows of a group that frame updated
        // outside a floor tile (a tile size or claim that changed, a batch that sat out) leave the word an older epoch.
        const bool tile_ages = tile_floors && P.group_age != nullptr;  // warp-uniform
        // With P.defer_ages a floor tile may leave a group's word deferred: the word then holds the age of all 32 rows and
        // their age column is stale. Such a group can also reach a tile that is not a floor tile (a tile size or claim that
        // changed, deaths elsewhere that made the list a gather): there each row reads its group's word next to its record
        // loads, takes the deferred age, stores its age as usual, and counts itself in the word (below).
        // Reading every row's word made the churned update 3.4 % slower on the H100 where nothing was deferred: the slab's
        // count of deferred words (hnb_deferred_groups) gates it. Other warps change the count while this one reads it, so
        // lanes may read different values: the ballot makes the gate warp-uniform (the ballots under it need every lane),
        // and a lane that read 0 still reads its group's word when another lane of the warp saw a deferred one.
        const bool tile_defer_rows = !tile_ages && P.defer_ages != 0u && P.group_age != nullptr &&
                                     __ballot_sync(0xffffffffu, *hnb_deferred_groups(P.group_age, P.slab.capacity_rows) != 0ull) != 0u;
#endif
#if HNB_GROUP_AGE
        // Two copies of the sub-tile loop: copy 0 for floor tiles that keep common ages (`ages` true, `defer_rows` false),
        // copy 1 for every other tile. With one copy, the code only other tiles run (reading each row's word, counting
        // rows into deferred words) made the floor tiles 7 % slower on the H100 without running.
#pragma unroll
        for (int copy = 0; copy < 2; ++copy) {
        const bool ages = copy == 0;
        if (ages != tile_ages) continue;
        const bool floors = ages || tile_floors, defer_rows = !ages && tile_defer_rows;
#elif HNB_LIFE_FLOOR
        {
        const bool floors = tile_floors;
#endif
#pragma unroll 1
        for (u32 j = 0; j < chunks; ++j) {
            u32 pidx[HNB_TILE_K];
            bool valid[HNB_TILE_K];
            RawParticle raw[HNB_TILE_K];
#if HNB_GROUP_AGE
            u32 deferred_rows = 0u;  // bit k: row k of this lane took its age from a deferred word outside a floor tile
#endif
#if HNB_LIFE_FLOOR
            // lane k < HNB_TILE_K holds the floor of the sub-tile's row group k: one coalesced load
            const u32 g_first = ((base_particle + row0) >> 5u) + j * HNB_TILE_K;  // slab group of row group 0
            const u32 my_floor = floors && lane < HNB_TILE_K ? __float_as_uint(P.life_floor[g_first + lane]) : HNB_LIFE_FLOOR_NONE;
#endif
            // gather the particle records (all loads in flight before any use)
#if HNB_SLOT_ORDER
#pragma unroll
            for (int k = 0; k < HNB_TILE_K; ++k) {
                const u32 vmask = __shfl_sync(0xffffffffu, my_bits, int(j * HNB_TILE_K + k));
                pidx[k] = row0 + (j * HNB_TILE_K + k) * 32u + lane;
                valid[k] = (vmask >> lane) & 1u;
                if (lane == 0) valids[j * HNB_TILE_K + k] = vmask;
                tile_valid += __popc(vmask);
                if (valid[k]) hnb_load_raw(raw[k], P.slab, base_particle + pidx[k]);
                else hnb_raw_zero(raw[k]);
            }
#else
#pragma unroll
            for (int k = 0; k < HNB_TILE_K; ++k) {
                const u32 row = row0 + (j * HNB_TILE_K + k) * 32u + lane;
                pidx[k] = pidx_next[k];
                pidx_stash[j * HNB_TILE_K + k][lane] = pidx[k];
                valid[k] = row < max_update;
#if HNB_LIFE_FLOOR
#if HNB_GROUP_AGE
                // A known common age A: every row of the group holds A in its age column, which is then not loaded. Every lane
                // reads the group's word (one broadcast access) right before the row's record loads. Kept across the
                // sub-tile in one register, as the floors are, the K words spill at 80 registers; read together ahead of the
                // record loads, they made the pass 1.7 % slower on the H100. A deferred word is known whatever its epoch: no
                // update but the one that consumes it advances its group's ages.
                u64 word = HNB_GROUP_AGE_NONE;
                if (ages) word = P.group_age[g_first + k];
                else if (defer_rows && valid[k]) word = P.group_age[(base_particle + pidx[k]) >> 5u];
                const bool deferred = hnb_group_age_deferred(word);
                const u32 A = deferred || u32(word >> 32) == epoch - 1u ? u32(word) : HNB_LIFE_FLOOR_NONE;
                if (defer_rows && deferred) deferred_rows |= 1u << k;
                if (ages && deferred && lane == 0) parked->defer_delta -= 1u;
#endif
                if (valid[k]) {
#if HNB_GROUP_AGE
                    hnb_load_raw_but_life_age(raw[k], P.slab, base_particle + pidx[k]);
                    if (A != HNB_LIFE_FLOOR_NONE) hnb_set_raw_age(raw[k], __uint_as_float(A));
                    else hnb_load_age(raw[k], P.slab, base_particle + pidx[k]);
#else
                    hnb_load_raw_but_life(raw[k], P.slab, base_particle + pidx[k]);
#endif
                    if (!floors) hnb_load_life(raw[k], P.slab, base_particle + pidx[k]);  // (with floors: below)
                }
#else
                if (valid[k]) hnb_load_raw(raw[k], P.slab, base_particle + pidx[k]);
#endif
                else hnb_raw_zero(raw[k]);
            }
            // prefetch the alive-list entries of the next sub-tile (coalesced u32)
            if (j + 1 < chunks) {
                if (tile_known) {
#pragma unroll
                    for (int k = 0; k < HNB_TILE_K; ++k) pidx_next[k] = row0 + ((j + 1) * HNB_TILE_K + k) * 32u + lane;
                } else {
#pragma unroll
                    for (int k = 0; k < HNB_TILE_K; ++k) {
                        const u32 row = row0 + ((j + 1) * HNB_TILE_K + k) * 32u + lane;
                        pidx_next[k] = row < trust_r ? row : (row < max_update ? read_col[row] : 0u);
                    }
                }
            }
#endif
            // simulate + write back (WRITEBACK_CODE: every attribute except PREV/NEXT, lib.rs:1270-1281)
#pragma unroll
            for (int k = 0; k < HNB_TILE_K; ++k) {
                bool alive = false;
#if HNB_LIFE_FLOOR
                if (floors) {
                    // The floor F of a group is at most the lifetime of each of its particles, so `age < F && age + dt < F`
                    // (the fp32 sums the age code computes) proves `age < lifetime` both times the body compares them. A proven
                    // row takes F as its lifetime: every use of it is one of those comparisons (HNB_ATTR_REAP_ONLY), and the
                    // lifetime column is never stored. Any other row loads its lifetime here. A NaN on either side proves
                    // nothing. (Deciding every row of the sub-tile before the first body, to issue these loads together,
                    // costs registers that hnb_update does not have at 3 CTAs per SM.)
                    const f32 F = __uint_as_float(__shfl_sync(0xffffffffu, my_floor, k));
                    bool proven = false;
                    if (valid[k]) {
                        const f32 age = hnb_raw_age(raw[k]);
                        proven = age < F && age + hnb_ctx.sim->delta_time < F;
                        if (proven) hnb_raw_life(raw[k]) = F;
                        else hnb_load_life(raw[k], P.slab, base_particle + pidx[k]);
                    }
                    // Every row (all are valid below trust_r) loaded its lifetime: store their minimum as the group's floor,
                    // a NaN anywhere making it NaN (fminf would drop it).
                    if (__ballot_sync(0xffffffffu, proven) == 0u) {
                        f32 m = valid[k] ? hnb_raw_life(raw[k]) : __uint_as_float(0x7f800000u);
#pragma unroll
                        for (int d = 16; d > 0; d >>= 1) {
                            const f32 o = __shfl_xor_sync(0xffffffffu, m, d);
                            m = (m != m || m < o) ? m : o;
                        }
                        if (lane == 0) P.life_floor[g_first + k] = m;
                    }
                }
#endif
                if (valid[k]) {
                    Particle particle;
                    hnb_unpack(raw[k], particle);
                    hnb_ctx.particle_index = pidx[k];
                    hnb_ctx.seed = pcg_hash(pidx[k] ^ spawner_seed);  // :138
                    hnb_ctx.is_alive = true;
#if HNB_EMIT_EVENTS && HNB_ORDERED_EVENTS
#pragma unroll
                    for (int b = 0; b < HNB_MAX_EVENT_BINDINGS; ++b) hnb_ctx.event_request[b] = 0u;
#endif
                    alive = hnb_update_body(particle, hnb_ctx);
#if HNB_EMIT_EVENTS && HNB_ORDERED_EVENTS
                    {
                        const u32 row = row0 + (j * HNB_TILE_K + k) * 32u + lane;  // update thread index within the (single) instance
#pragma unroll
                        for (int b = 0; b < HNB_MAX_EVENT_BINDINGS; ++b)
                            if (P.event_counts[b]) P.event_counts[b][row] = hnb_ctx.event_request[b];
                    }
#endif
                    // hnb_pack<false> leaves the PREV/NEXT words of raw[k] as they were LOADED, and the store below writes whole
                    // columns: a column that also holds a word the update writes gets its links written back unchanged.
                    // That equals the reference's WRITEBACK_CODE (which never stores them) only because no kernel of this
                    // path maintains links while an update is in flight; a link-maintaining pass added later must not
                    // overlap hnb_update, or PREV/NEXT must be declared HNB_ATTR_UPDATE_READ_ONLY (the graph lowering does),
                    // which gives them columns of their own that hnb_store_written never stores.
                    hnb_pack<false>(particle, raw[k]);
#if HNB_GROUP_AGE
                    // In a floor tile the age column is stored below, once the warp knows whether the group is deferred; the
                    // other columns are stored here, as soon as they are packed.
                    if (ages) hnb_store_written_but_age(raw[k], P.slab, base_particle + pidx[k]);
                    else
#endif
                    hnb_store_written(raw[k], P.slab, base_particle + pidx[k]);
                }
                const u32 ballot = __ballot_sync(0xffffffffu, alive);
#if HNB_GROUP_AGE
                if (ages) {
                    // Every row of the group is valid and stores its record, dead or alive, so the new ages are what its age
                    // column holds after the store: when all 32 are bit-equal (and not the sentinel's bits) they are the
                    // group's common age as of this epoch. With P.defer_ages, a group whose 32 rows all survive is left
                    // deferred instead, and its age column is not stored: none of its rows reaches the dead stack, so the
                    // next update of the instance walks all of them again. Any other group leaves a word that is not
                    // deferred: known, or (with P.defer_ages, which may have found it deferred) the sentinel. Without
                    // P.defer_ages a group of differing ages stores nothing, and its word's epoch is stale next frame.
                    const u32 a = __float_as_uint(hnb_raw_age(raw[k]));
                    const u32 a0 = __shfl_sync(0xffffffffu, a, 0);
                    const bool same = __ballot_sync(0xffffffffu, a == a0) == 0xffffffffu && a0 != HNB_LIFE_FLOOR_NONE;
                    const bool defer = P.defer_ages && same && ballot == 0xffffffffu;
                    if (!defer) hnb_store_age(raw[k], P.slab, base_particle + pidx[k]);
                    if (lane == 0) {
                        if (defer) P.group_age[g_first + k] = HNB_GROUP_AGE_DEFERRED | a0, parked->defer_delta += 1u;
                        else if (same) P.group_age[g_first + k] = (u64(epoch) << 32) | a0;
                        else if (P.defer_ages) P.group_age[g_first + k] = HNB_GROUP_AGE_NONE;
                    }
                }
#endif
                if (lane == 0) survivors[j * HNB_TILE_K + k] = ballot;
                tile_alive += __popc(ballot);
#if HNB_SLOT_ORDER
                if (lane == j * HNB_TILE_K + k) my_new_bits = ballot;
#endif
            }
#if HNB_GROUP_AGE
            if (defer_rows && __ballot_sync(0xffffffffu, deferred_rows != 0u) != 0u) {
                // Rows that took a deferred age count themselves into its word, one atomic per group and warp. Each of a
                // deferred group's 32 rows is walked exactly once in the launch, and read the word before it counts, so
                // the add that makes 32 ends the deferral: the ages are all in the column now. (Outside the loop above,
                // which the floor tiles' copy of this loop runs without any of it.)
#pragma unroll
                for (int k = 0; k < HNB_TILE_K; ++k) {
                    const bool mine = (deferred_rows >> k) & 1u;
                    const u32 g = (base_particle + pidx[k]) >> 5u;
                    for (u32 pending = __ballot_sync(0xffffffffu, mine); pending;) {
                        const u32 leader = u32(__ffs(pending) - 1);
                        const u32 lg = __shfl_sync(0xffffffffu, g, int(leader));
                        const u32 peers = __ballot_sync(0xffffffffu, mine && g == lg);
                        if (lane == leader) {
                            const u32 n = u32(__popc(peers));
                            const u64 old = atomicAdd((unsigned long long*)&P.group_age[lg], (unsigned long long)n << 32);
                            if (u32(old >> 32) - u32(HNB_GROUP_AGE_DEFERRED >> 32) + n == 32u) {
                                P.group_age[lg] = HNB_GROUP_AGE_NONE;
                                atomicAdd((unsigned long long*)hnb_deferred_groups(P.group_age, P.slab.capacity_rows), ~0ull);  // -1
                            }
                        }
                        pending &= ~peers;
                    }
                }
            }
#endif
#if HNB_PROFILE
            if (prof_first && j == 0u && lane == 0 && prof_ring) { unsigned long long _g; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(_g)); atomicMax(&prof_ring[2], ~_g); }
#endif
        }
#if HNB_LIFE_FLOOR
        }
#endif
#if HNB_GROUP_AGE
        // (a group this tile made deferred is counted late, but no other walker of this launch meets it)
        if (lane == 0 && parked->defer_delta != 0u) {
            atomicAdd((unsigned long long*)hnb_deferred_groups(P.group_age, P.slab.capacity_rows), (unsigned long long)(long long)int(parked->defer_delta));
            parked->defer_delta = 0u;
        }
#endif
        // Publish this tile's survivor count right away: the first tile of an instance knows its prefix (0),
        // the others publish an AGGREGATE that successors can sum over while this tile's own prefix is
        // still unknown.
#if HNB_SLOT_ORDER
        if (owns_word) tile_bits[lane] = my_new_bits;  // the survivors are the next frame's population of these slots
        if (lane == 0) hnb_st_state(&states[tile], hnb_pack_state(epoch, tile == inst_first_tile ? HNB_FLAG_PREFIX : HNB_FLAG_AGGREGATE, tile_alive, tile_valid));
#elif !HNB_RELAXED_ORDER
        if (lane == 0) hnb_st_state(&states[tile], hnb_pack_state(epoch, tile == inst_first_tile ? HNB_FLAG_PREFIX : HNB_FLAG_AGGREGATE, tile_alive));
#endif
        HNB_PROF_MARK(prof_pass1)
#if HNB_PROFILE
        if (prof_first) { HNB_PROF_TIME(10, false) HNB_PROF_TIME(12, true) prof_first = false; }
#endif

#if !HNB_RELAXED_ORDER
        ++streamed;  // this tile is parked below; if it is not the warp's first, the previous one is resolved first
#endif
        // Request the next tile now; the atomic's round trip hides behind the compaction below.
        u32 next_tile = 0u;
        if (lane == 0) next_tile = atomicAdd(P.ticket, 1u);

        // ---- deferred compaction. Resolving THIS tile now would mean waiting for every in-flight predecessor
        // to finish its pass 1 (they started at about the same time, and pass-1 durations vary). Instead the
        // tile is parked and the PREVIOUS tile of this warp is resolved: its predecessors published their
        // aggregates a whole pass 1 ago, so the look-back finds them immediately.
#if !HNB_RELAXED_ORDER
        __syncwarp();
        if (streamed != 1u) {  // resolve the parked tile: its stash buffer is the one the next tile will reuse
            const PendingTile pt = *parked;
            hnb_compact_tile(P, pt, sh_survivors[warp][pt.buffer], sh_valids[warp][pt.buffer], sh_pidx[warp][pt.buffer], chunks, epoch, lane, prof_polls);
        }
        __syncwarp();
        if (lane == 0) {
            parked->tile = tile; parked->row0 = row0; parked->tile_alive = tile_alive;
            parked->base_particle = base_particle; parked->max_update = max_update; parked->write_index = write_index;
            parked->render_index = render_index; parked->inst_first_tile = inst_first_tile; parked->inst_end_tile = inst_end_tile;
            parked->metadata_index = metadata_index;
            parked->buffer = ~streamed & 1u;
            parked->trust_r = trust_r; parked->claim_w = claim_w;
#if HNB_SLOT_ORDER
            parked->tile_valid = tile_valid;
#endif
        }
        __syncwarp();
#else
        {
            __syncwarp();
            PendingTile pt;
            pt.tile = tile; pt.row0 = row0; pt.tile_alive = tile_alive; pt.base_particle = base_particle;
            pt.max_update = max_update; pt.write_index = write_index; pt.render_index = render_index;
            pt.inst_first_tile = inst_first_tile; pt.inst_end_tile = inst_end_tile; pt.metadata_index = metadata_index;
            pt.trust_r = trust_r; pt.claim_w = claim_w;
#if HNB_SLOT_ORDER
            pt.tile_valid = tile_valid;
            hnb_compact_tile(P, pt, survivors, valids, pidx_stash, chunks, epoch, lane, prof_polls);
#else
            hnb_compact_tile(P, pt, survivors, nullptr, pidx_stash, chunks, epoch, lane, prof_polls);
#endif
            __syncwarp();
        }
#endif
        HNB_PROF_MARK(prof_compact)
        tile = __shfl_sync(0xffffffffu, next_tile, 0);
#if HNB_PROFILE
        prof_tiles++;
#endif
    }
#if !HNB_RELAXED_ORDER
    __syncwarp();
    if (streamed != 0u) {  // no more tiles: resolve the parked one
        const PendingTile pt = *parked;
        hnb_compact_tile(P, pt, sh_survivors[warp][pt.buffer], sh_valids[warp][pt.buffer], sh_pidx[warp][pt.buffer], chunks, epoch, lane, prof_polls);
    }
#endif
#if HNB_PROFILE
    HNB_PROF_MARK(prof_compact)
    if (lane == 0 && P.debug) {
        atomicAdd(&P.debug[0], (unsigned long long)prof_pass1);
        atomicAdd(&P.debug[1], (unsigned long long)prof_compact);
        atomicAdd(&P.debug[3], (unsigned long long)prof_polls);
        atomicAdd(&P.debug[4], (unsigned long long)prof_tiles);
        atomicAdd(&P.debug[5], 1ull);  // warps
        atomicMax(&P.debug[6], (unsigned long long)(clock64() - prof_start));  // longest-lived warp (cycles)
    }
    HNB_PROF_TIME(11, false) HNB_PROF_TIME(13, true)
    if (lane == 0 && prof_ring) { unsigned long long _g; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(_g)); atomicMax(&prof_ring[3], _g); }
#endif
}

}  // namespace hnb
