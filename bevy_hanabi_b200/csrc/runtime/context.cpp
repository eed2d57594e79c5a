// context.cpp — Level-1 runtime behind include/hanabi_b200.h: context, slabs, compiled effects,
// per-frame tables and the simulate() driver.
//
// Mirrors, on the host side, what the reference keeps in EffectCache / EffectsMeta / Batcher /
// PropertyCache (src/render/{effect_cache,batch,property}.rs, mod.rs) and the pass recording of
// simulate() (src/render/mod.rs:6942-7613) — flattened into plain device arrays, one CUDA stream,
// and one host->device copy per frame.
#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>  // header-only NVTX v3: a no-op unless a tool (nsys, ncu --nvtx) injects itself

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../kernels/hnb_static_kernels.h"
#include "cuda_owned.h"
#include "driver.h"
#include "effect_source.h"
#include "hanabi_b200.h"
#include "nvrtc_compile.h"
#include "tile_state_rule.h"

using namespace hnb_rt;

static_assert(sizeof(hnb_spawner) == 128 && sizeof(hnb::Spawner) == 128, "GpuSpawnerParams is 128 bytes");
static_assert(sizeof(hnb_effect_metadata) == 60 && sizeof(hnb::EffectMetadata) == 60, "GpuEffectMetadata is 60 bytes");
static_assert(sizeof(hnb_batch_info) == 24 && sizeof(hnb::BatchInfo) == 24, "GpuBatchInfo is 24 bytes");
static_assert(sizeof(hnb_sim_params) == 28 && sizeof(hnb::SimParams) == 28, "GpuSimParams is 28 bytes");
static_assert(sizeof(hnb_draw_indexed_indirect_args) == 20, "GpuDrawIndexedIndirectArgs is 20 bytes");
static_assert(sizeof(hnb_indirect_index) == 12, "GpuIndirectIndex is 12 bytes");
static_assert(sizeof(hnb_child_info) == 8 && sizeof(hnb::ChildInfo) == 8, "GpuChildInfo is 8 bytes");
static_assert(sizeof(hnb::FrameHeader) == 64, "frame header is 64 bytes");

// ---------------------------------------------------------------------------------------------
// Errors
// ---------------------------------------------------------------------------------------------
namespace {
thread_local std::string g_last_error;

struct HnbError : std::runtime_error {
    int32_t code;
    HnbError(int32_t c, const std::string& m) : std::runtime_error(m), code(c) {}
};
[[noreturn]] void fail(int32_t code, const std::string& msg) { throw HnbError(code, msg); }

#define CUDA_CHECK(expr)                                                                                     \
    do {                                                                                                     \
        cudaError_t _e = (expr);                                                                             \
        if (_e != cudaSuccess) fail(HNB_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));        \
    } while (0)

template <typename F> int32_t guarded(F&& f) {
    try {
        f();
        return HNB_OK;
    } catch (const HnbError& e) {
        g_last_error = e.what();
        return e.code;
    } catch (const std::invalid_argument& e) {
        g_last_error = e.what();
        return HNB_ERR_INVALID_ARG;
    } catch (const std::exception& e) {
        g_last_error = e.what();
        return HNB_ERR_CUDA;
    }
}

uint32_t ceil_div(uint32_t a, uint32_t b) { return (a + b - 1) / b; }
size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }
}  // namespace

// ---------------------------------------------------------------------------------------------
// Objects
// ---------------------------------------------------------------------------------------------
namespace {

struct Slab {
    bool live = false;
    uint32_t capacity = 0, stride = 0;
    bool sector_planes = false;  // HNB_SLAB_SECTOR_PLANES
    std::vector<Plane> planes;   // physical columns
    DeviceArray<char> d_planes[HNB_RT_MAX_PLANES];
    DeviceArray<uint32_t> ping, pong, dead;
    DeviceArray<uint32_t> alive_bits;  // one bit per row (HNB_EFFECT_SLOT_ORDER effects keep it current)
    DeviceArray<unsigned long long> ident_claim;  // [2]: identity claims of ping / pong (hnb_claim_pack)
    // HNB_EFFECT_ORDERED_EVENTS scratch, allocated on first use: per channel the per-row event counts and their block sums
    DeviceArray<uint32_t> event_counts[HNB_MAX_EVENT_BINDINGS];
    DeviceArray<uint32_t> event_block_sums[HNB_MAX_EVENT_BINDINGS];
};

struct KernelModule {
    CUmodule mod = nullptr;
    CUfunction init = nullptr, update = nullptr;
    int update_blocks_per_sm = 1;
    std::string log;
};

struct Effect {
    bool live = false;
    uint64_t hash = 0;
    KernelModule* km = nullptr;
    uint32_t tile_k = 4, flags = 0, particle_stride = 0, parent_stride = 0, rows_per_lane = 16, update_smem = 0;
    int update_blocks_per_sm = 1;
    uint32_t props_size = 0, props_stride = 0;
    DeviceArray<char> d_props;  // rows of props_stride bytes
    std::string name;
};

// Pinned staging slot of the per-frame upload (see flush_arena).
constexpr size_t kDebugWords = 16 + 4 * 64;
constexpr int kStageSlots = 32;  // frames the host may queue ahead of the GPU before blocking
struct StageSlot {
    PinnedBlock h;
    Event done;
    bool used = false;
};

struct SideStream {
    Stream stream;
    Event done;
};

struct ArenaLayout {
    size_t off_batch_infos, off_tile_size, off_spawners, off_range, off_spawn_prefix, off_prefix_sum, total;
    static ArenaLayout make(uint32_t E, uint32_t B) {
        ArenaLayout l;
        size_t o = sizeof(hnb::FrameHeader);
        l.off_batch_infos = o; o += size_t(B) * sizeof(hnb_batch_info);
        l.off_tile_size = o; o += size_t(B) * 4;
        o = align_up(o, 16);
        l.off_spawners = o; o += size_t(E) * sizeof(hnb_spawner);
        l.off_range = o; o += size_t(E) * 4;
        l.off_spawn_prefix = o; o += size_t(E) * 4;
        l.off_prefix_sum = o; o += size_t(E) * 4;
        l.total = o;
        return l;
    }
};

}  // namespace

namespace {
struct LaunchPlan;
}

struct hnb_ctx {
    // Members are destroyed in reverse order: every buffer and event below goes first, then the side streams, and the
    // context stream last.
    Stream stream;  // created with the context, or the caller's external stream (borrowed, never destroyed)
    // side streams: the update (and independent init) launches of a multi-batch frame run concurrently
    std::vector<SideStream> side_streams;
    Event fork_event;

    int device = 0;
    int sm_count = 132;
    std::vector<uint8_t> init_pending;   // per batch: a stand-alone hnb_pass_init whose accounting hnb_pass_indirect has not applied yet
    std::vector<LaunchPlan> frame_plans;  // hnb_simulate's per-frame launch plans (kept to avoid a heap allocation per frame)
    DriverApi drv;
    uint64_t launches = 0;

    // per-frame arena (host pinned + device mirror), exact-size layout for (E, B)
    uint32_t E = 0, B = 0;
    ArenaLayout lay = ArenaLayout::make(0, 0);
    PinnedBlock h_arena;
    DeviceArray<char> d_arena;
    bool dirty_tables = true;  // spawners / batch infos / prefix sums changed since last flush
    StageSlot stage[kStageSlots];  // pinned snapshots of the frame block, one per in-flight frame
    uint32_t stage_next = 0;
    uint32_t epoch = 0;

    // persistent device tables
    DeviceArray<hnb::EffectMetadata> d_metadata;
    DeviceArray<hnb_draw_indexed_indirect_args> d_draw_args;
    DeviceArray<hnb::ChildInfo> d_child_infos;  // its size is the logical array length the kernels read (num_child_infos)
    // per-instance / per-batch scratch
    DeviceArray<uint32_t> d_tile_prefix;
    // per batch slot: the dispatch args (3 words), then the tile counts, then the tickets. One block, so that growing
    // it takes one synchronisation.
    DeviceArray<uint32_t> d_batch_scratch;
    std::vector<DeviceArray<unsigned long long>> d_tile_state;  // per batch
    std::vector<hnb_rt::TileStateSlot> tile_state_slot;  // when the batch's states were last zeroed (tile_state_rule.h)
    uint64_t tile_state_clears = 0;  // zeroings tile_state_needs_clear asked for (hnb_ctx_tile_state_clears)
    uint64_t md_generation = 1;            // bumped by hnb_metadata_insert

    std::vector<Slab> slabs;
    std::vector<Effect> effects;
    std::vector<DeviceArray<uint32_t>> event_buffers;
    std::unordered_map<uint64_t, std::unique_ptr<KernelModule>> modules;  // ≙ ShaderCache

    // kernel timing
    bool timing = false;
    std::vector<std::pair<Event, Event>> ev_pending, ev_free;
    double update_ms = 0.0;
    uint64_t update_launches = 0;
    // ribbon sort scratch (large path), sized to the largest ribbon slab seen so far: keys[2] (8 bytes per row), then
    // vals[2] (4 bytes per row), so three 8-byte words per row in one block that grows with one synchronisation
    DeviceArray<uint64_t> d_sort_scratch;
    DeviceArray<uint32_t> d_sort_hist;
    uint32_t tile_chunks_override = 0;  // HNB_TILE_CHUNKS env: fixed sub-tile count per tile (tuning)
    bool param_upload = true; // HNB_PARAM_UPLOAD=0: always copy the frame block with the copy engine (never as a kernel parameter)
    unsigned long long* mailbox = nullptr;  // device alias of the caller's pinned count mailbox (hnb_ctx_set_count_mailbox)
    uint32_t mailbox_rows = 0, mailbox_ring = 0;
    bool plan_dirty = false;  // plan_batch changed a tile-size or range word of the host frame block since the last upload
    uint64_t frame_copies = 0, frames = 0;  // hnb_simulate calls that needed the host->device copy of the frame block / all calls
    DeviceArray<unsigned long long> d_debug;  // 16 diagnostic counters + a 64-frame timeline ring of 4 words (HNB_PROFILE kernels)

    hnb::FrameHeader* header() { return reinterpret_cast<hnb::FrameHeader*>(h_arena.get()); }
    template <typename T> T* h_at(size_t off) { return reinterpret_cast<T*>(h_arena.get() + off); }
    template <typename T> T* d_at(size_t off) { return reinterpret_cast<T*>(d_arena.get() + off); }
    uint32_t scratch_B() const { return uint32_t(d_batch_scratch.size() / 5); }
    uint32_t* dispatch_args() const { return d_batch_scratch.get(); }
    uint32_t* batch_tiles() const { return d_batch_scratch.get() + 3 * size_t(scratch_B()); }
    uint32_t* tickets() const { return d_batch_scratch.get() + 4 * size_t(scratch_B()); }
    uint32_t* draw_args() const { return reinterpret_cast<uint32_t*>(d_draw_args.get()); }  // as the kernels index it: 5 words per row
};

namespace {

// Moves the tables of the frame block from layout `ol` (E = oE, B = oB) to layout `nl`, keeping the rows both have.
void relocate_tables(char* dst, const ArenaLayout& nl, uint32_t E, uint32_t B, const char* src, const ArenaLayout& ol, uint32_t oE, uint32_t oB) {
    const uint32_t mB = std::min(oB, B), mE = std::min(oE, E);
    memcpy(dst, src, sizeof(hnb::FrameHeader));
    memcpy(dst + nl.off_batch_infos, src + ol.off_batch_infos, size_t(mB) * sizeof(hnb_batch_info));
    memcpy(dst + nl.off_tile_size, src + ol.off_tile_size, size_t(mB) * 4);
    memcpy(dst + nl.off_spawners, src + ol.off_spawners, size_t(mE) * sizeof(hnb_spawner));
    memcpy(dst + nl.off_range, src + ol.off_range, size_t(mE) * 4);
    memcpy(dst + nl.off_spawn_prefix, src + ol.off_spawn_prefix, size_t(mE) * 4);
    memcpy(dst + nl.off_prefix_sum, src + ol.off_prefix_sum, size_t(mE) * 4);
}

void ensure_arena(hnb_ctx* c, uint32_t E, uint32_t B) {
    if (E == c->E && B == c->B && c->h_arena) return;
    ArenaLayout nl = ArenaLayout::make(E, B);
    size_t need = std::max<size_t>(nl.total, 256);
    // the tables move to their new offsets through a copy of the old host block
    std::vector<char> old(c->h_arena.get(), c->h_arena.get() + (c->h_arena ? c->lay.total : 0));
    if (need > c->h_arena.size()) {
        size_t cap = std::max(need * 2, size_t(4096));
        PinnedBlock nh;
        CUDA_CHECK(nh.alloc(cap));
        memset(nh.get(), 0, cap);
        CUDA_CHECK(grow(c->d_arena, cap, 0, c->stream));
        c->h_arena = std::move(nh);
    } else if (c->h_arena) {
        memset(c->h_arena.get() + sizeof(hnb::FrameHeader), 0, nl.total - sizeof(hnb::FrameHeader));
    }
    if (!old.empty()) relocate_tables(c->h_arena.get(), nl, E, B, old.data(), c->lay, c->E, c->B);
    c->lay = nl;
    c->E = E;
    c->B = B;
    c->dirty_tables = true;
}

void ensure_scratch(hnb_ctx* c) {
    if (c->E > c->d_tile_prefix.size()) CUDA_CHECK(grow(c->d_tile_prefix, std::max<uint32_t>(c->E * 2, 64), 0, c->stream));
    if (c->B > c->scratch_B()) {
        uint32_t cap = std::max<uint32_t>(c->B * 2, 16);
        CUDA_CHECK(grow(c->d_batch_scratch, size_t(cap) * 5, 0, c->stream));
        c->d_tile_state.resize(cap);
        c->tile_state_slot.resize(cap);
    }
}

hnb::StaticTables static_tables(hnb_ctx* c) {
    hnb::StaticTables T{};
    T.frame = c->d_at<hnb::FrameHeader>(0);
    T.spawners = c->d_at<hnb::Spawner>(c->lay.off_spawners);
    T.spawn_range = c->d_at<uint32_t>(c->lay.off_range);
    T.prefix_sum = c->d_at<uint32_t>(c->lay.off_prefix_sum);
    T.tile_prefix = c->d_tile_prefix.get();
    T.batch_infos = c->d_at<hnb::BatchInfo>(c->lay.off_batch_infos);
    T.batch_tile_size = c->d_at<uint32_t>(c->lay.off_tile_size);
    T.dispatch_args = c->dispatch_args();
    T.batch_tiles = c->batch_tiles();
    T.tickets = c->tickets();
    T.metadata = c->d_metadata.get();
    T.draw_args = c->draw_args();
    T.child_infos = c->d_child_infos.get();
    T.num_child_infos = uint32_t(c->d_child_infos.size());
    return T;
}

// One host->device copy of the frame block: everything when the tables changed, else the header + per-frame
// ranges (`with_ranges`), else only the 64-byte header.
void flush_arena(hnb_ctx* c, bool with_ranges) {
    if (!c->h_arena) ensure_arena(c, c->E, c->B);
    size_t bytes;
    if (c->dirty_tables) bytes = c->lay.total;
    else if (with_ranges) bytes = c->lay.off_prefix_sum;  // everything but the GPU-rewritten prefix sums
    else bytes = sizeof(hnb::FrameHeader);
    // The copy executes when the stream reaches it, not now: the host arena (epoch, ranges, tables) will be
    // rewritten for the NEXT frame long before that if the caller queues frames ahead. Snapshot the bytes into
    // a pinned staging slot that is not reused until its copy has completed.
    StageSlot& slot = c->stage[c->stage_next++ % kStageSlots];
    if (slot.used) CUDA_CHECK(cudaEventSynchronize(slot.done));
    if (slot.h.size() < bytes) CUDA_CHECK(slot.h.alloc(std::max(bytes * 2, size_t(4096))));
    if (!slot.done) CUDA_CHECK(slot.done.create(cudaEventDisableTiming));
    memcpy(slot.h.get(), c->h_arena.get(), bytes);
    CUDA_CHECK(cudaMemcpyAsync(c->d_arena.get(), slot.h.get(), bytes, cudaMemcpyHostToDevice, c->stream));
    CUDA_CHECK(cudaEventRecord(slot.done, c->stream));
    slot.used = true;
    c->dirty_tables = false;
    if (bytes >= c->lay.off_prefix_sum) c->plan_dirty = false;
}

void next_epoch(hnb_ctx* c) {
    c->epoch = (c->epoch + 1u) & 0x3fffffffu;
    if (c->epoch == 0) {
        // 30-bit wrap (207 days at 60 frames/s): a tile state left untouched since the same epoch of the previous
        // cycle would look current, so drop them all. 0 = "never written".
        c->epoch = 1;
        for (const auto& ts : c->d_tile_state)
            if (ts) CUDA_CHECK(cudaMemsetAsync(ts.get(), 0, ts.size() * 8, c->stream));
    }
    c->header()->epoch = c->epoch;
    c->header()->num_batches = c->B;
}

Slab& get_slab(hnb_ctx* c, hnb_slab s) {
    if (s >= c->slabs.size() || !c->slabs[s].live) fail(HNB_ERR_INVALID_ARG, "invalid slab handle");
    return c->slabs[s];
}
Effect& get_effect(hnb_ctx* c, hnb_effect e) {
    if (e >= c->effects.size() || !c->effects[e].live) fail(HNB_ERR_INVALID_ARG, "invalid effect handle");
    return c->effects[e];
}

hnb::PlaneSet plane_set(const Slab& s) {
    hnb::PlaneSet ps{};
    for (size_t p = 0; p < s.planes.size(); ++p) {
        ps.ptr[p] = s.d_planes[p].get();
        ps.words[p] = s.planes[p].width / 4;
        ps.word_off[p] = s.planes[p].offset / 4;
        for (uint32_t w = 0; w < s.planes[p].width / 4; ++w) ps.word_to_plane[s.planes[p].offset / 4 + w] = (unsigned char)p;
    }
    return ps;
}

hnb::SlabView slab_view(const Slab& s) {
    hnb::SlabView v{};
    for (size_t p = 0; p < s.planes.size(); ++p) v.planes[p] = s.d_planes[p].get();
    v.particle_index[0] = s.ping.get();
    v.particle_index[1] = s.pong.get();
    v.dead_index = s.dead.get();
    v.alive_bits = s.alive_bits.get();
    v.ident_claim = s.ident_claim.get();
    v.capacity_rows = s.capacity;
    return v;
}

// Drops both identity claims of the slab, in stream order: for writers of the index columns that do not keep them true.
void clear_ident_claims(hnb_ctx* c, const Slab& s) {
    CUDA_CHECK(cudaMemsetAsync(s.ident_claim.get(), 0, 2 * sizeof(unsigned long long), c->stream));
}

// Copies `bytes` from the device to the host in stream order (and then zeroes the source when `clear`), and waits.
void read_back(hnb_ctx* c, void* out, void* d_src, size_t bytes, bool clear = false) {
    CUDA_CHECK(cudaMemcpyAsync(out, d_src, bytes, cudaMemcpyDeviceToHost, c->stream));
    if (clear) CUDA_CHECK(cudaMemsetAsync(d_src, 0, bytes, c->stream));
    CUDA_CHECK(cudaStreamSynchronize(c->stream));
}

void check_rows(const Slab& s, uint32_t first, uint32_t count) {
    if (uint64_t(first) + count > s.capacity) fail(HNB_ERR_OUT_OF_RANGE, "row range exceeds slab capacity");
}

// Staging through a device buffer in chunks (AoS <-> planes transposes run on the device).
constexpr size_t kChunkBytes = size_t(64) << 20;

// `precompiled`: a cubin already built for exactly this source (hnb_compile_job), or NULL to compile here.
KernelModule* get_module(hnb_ctx* c, const std::string& source, const std::string& name, uint64_t hash, bool fast_math,
                         const std::string* precompiled = nullptr) {
    auto it = c->modules.find(hash);
    if (it != c->modules.end()) return it->second.get();
    std::string cubin, log;
    if (precompiled) cubin = *precompiled;
    else if (!nvrtc_compile_sm90a(source, name + ".cu", cubin, log, fast_math)) fail(HNB_ERR_NVRTC, log);
    auto km = std::make_unique<KernelModule>();
    km->log = log;
    CUresult r = c->drv.ModuleLoadData(&km->mod, cubin.data());
    if (r != CUDA_SUCCESS) fail(HNB_ERR_CUDA, "cuModuleLoadData: " + cu_error_string(c->drv, r));
    r = c->drv.ModuleGetFunction(&km->init, km->mod, "hnb_init");
    if (r != CUDA_SUCCESS) fail(HNB_ERR_CUDA, "cuModuleGetFunction(hnb_init): " + cu_error_string(c->drv, r));
    r = c->drv.ModuleGetFunction(&km->update, km->mod, "hnb_update");
    if (r != CUDA_SUCCESS) fail(HNB_ERR_CUDA, "cuModuleGetFunction(hnb_update): " + cu_error_string(c->drv, r));
    km->update_blocks_per_sm = 1;  // per effect: depends on its dynamic shared memory (see hnb_effect_compile)
    KernelModule* out = km.get();
    c->modules.emplace(hash, std::move(km));
    return out;
}

struct LaunchPlan {
    Effect* fx;
    Slab* slab;
    uint32_t batch;
    uint32_t total_spawn;
    hnb::BatchParams params;
    uint32_t init_blocks;
    uint32_t update_blocks;
};

void ensure_tile_state(hnb_ctx* c, uint32_t batch, uint32_t tiles) {
    if (c->d_tile_state[batch].size() >= tiles) return;
    CUDA_CHECK(grow(c->d_tile_state[batch], tiles + tiles / 2 + 64, 0, c->stream));
    c->tile_state_slot[batch] = hnb_rt::TileStateSlot{};
}

// Build the kernel parameters of one batch and write its per-instance init thread ranges and tile
// size into the host arena.
LaunchPlan plan_batch(hnb_ctx* c, const hnb_batch_launch& bl, bool set_ranges) {
    LaunchPlan lp{};
    lp.fx = &get_effect(c, bl.effect);
    lp.slab = &get_slab(c, bl.slab);
    if (lp.fx->particle_stride != lp.slab->stride) fail(HNB_ERR_LAYOUT, "effect particle stride does not match the slab");
    if (((lp.fx->flags & HNB_EFFECT_SECTOR_PLANES) != 0) != lp.slab->sector_planes)
        fail(HNB_ERR_LAYOUT, "effect and slab disagree on HNB_EFFECT_SECTOR_PLANES / HNB_SLAB_SECTOR_PLANES");
    if (bl.batch_info_index >= c->B) fail(HNB_ERR_OUT_OF_RANGE, "batch_info_index out of range");
    lp.batch = bl.batch_info_index;
    lp.total_spawn = bl.total_spawn_count;
    const hnb_batch_info& bi = c->h_at<hnb_batch_info>(c->lay.off_batch_infos)[lp.batch];
    if (uint64_t(bi.prefix_sum_offset) + bi.prefix_sum_count > c->E || uint64_t(bi.spawner_base) + bi.prefix_sum_count > c->E)
        fail(HNB_ERR_OUT_OF_RANGE, "batch references instances outside the uploaded spawner table");
    // Rows per warp tile: 32 lanes x K rows per lane x chunks. Larger tiles shorten the look-back chain and
    // amortise the per-tile work (ticket, state word, instance lookup); smaller tiles spread a small slab over more
    // warps. With W = one sub-tile per resident warp (C5 on an H100: 3168 warps x 128 rows = 396 Ki rows):
    //  * from 8 W up the launch streams at the HBM rate and the largest tile wins at every size;
    //  * below, the launch is latency-bound and runs in ROUNDS: every resident warp takes one tile per round, and a tile
    //    costs a fixed part (ticket, first alive-list entries, look-back, compaction) plus a part per sub-tile: pick the
    //    chunk count that minimises rounds x (3.6 + chunks), preferring larger tiles on a tie. The constant was fitted on
    //    an earlier GPU. On an H100 (tools/sweep_small.py, C5) the rule is within 3 % of the best forced chunk count from
    //    1 Mi rows up; at 256-512 Ki rows forcing 3-4 chunks shortens the frame by 15-20 % (not retuned).
    const uint32_t sub_tile = 32u * lp.fx->tile_k;
    const uint32_t total_warps = uint32_t(lp.fx->update_blocks_per_sm) * uint32_t(c->sm_count) * 8u;
    const uint32_t max_chunks = std::max(1u, lp.fx->rows_per_lane / lp.fx->tile_k);
    uint32_t chunks = c->tile_chunks_override;
    if (chunks == 0) {
        const uint64_t wave = uint64_t(total_warps) * sub_tile;
        const uint64_t rows = lp.slab->capacity;
        if (rows >= 8 * wave) {
            chunks = max_chunks;
        } else {
            double best = 0.0;
            for (uint32_t ch = 1; ch <= max_chunks; ++ch) {
                const uint64_t tiles = (rows + uint64_t(sub_tile) * ch - 1) / (uint64_t(sub_tile) * ch) + bi.prefix_sum_count - 1;
                const uint64_t rounds = std::max<uint64_t>(1, (tiles + total_warps - 1) / total_warps);
                const double cost = double(rounds) * (3.6 + double(ch));
                if (chunks == 0 || cost <= best) { best = cost; chunks = ch; }
            }
        }
    }
    chunks = std::max(1u, std::min(chunks, max_chunks));
    const uint32_t tile = sub_tile * chunks;
    // Tile size word shared with the bookkeeping kernels (hnb_tile_rows + flags)
    const bool slot_order = (lp.fx->flags & HNB_EFFECT_SLOT_ORDER) != 0;
    const uint32_t tile_word = tile | (slot_order ? HNB_TILE_SLOT_ORDER : 0u), small_tile = tile;
    if (slot_order) {
        // bitmap words must belong to one instance (and one warp) each
        const hnb_spawner* sp = c->h_at<hnb_spawner>(c->lay.off_spawners);
        for (uint32_t i = 0; i < bi.prefix_sum_count; ++i)
            if (sp[bi.spawner_base + i].slab_offset & 31u) fail(HNB_ERR_LAYOUT, "HNB_EFFECT_SLOT_ORDER needs every instance to start on a multiple of 32 slab rows");
        // a slot-order state word packs each running count into 28 bits
        if (lp.slab->capacity >= (1u << 28)) fail(HNB_ERR_LAYOUT, "HNB_EFFECT_SLOT_ORDER needs a slab of fewer than 2^28 rows");
    }
    if (c->h_at<uint32_t>(c->lay.off_tile_size)[lp.batch] != tile_word) {
        c->h_at<uint32_t>(c->lay.off_tile_size)[lp.batch] = tile_word;
        c->plan_dirty = true;
    }

    const bool consume = (lp.fx->flags & HNB_EFFECT_CONSUME_GPU_SPAWN_EVENTS) != 0;
    uint32_t init_threads = 0;
    if (consume) {
        if (bl.consume_events >= c->event_buffers.size()) fail(HNB_ERR_INVALID_ARG, "event-driven effect needs a consume_events buffer");
        // One logical init thread per event-buffer ENTRY, not per 64-thread workgroup of the reference's dispatch: the
        // threads of the last partial workgroup would read past the buffer when a parent over-emits (event_count is
        // unclamped, lib.rs:976-993), which WGSL's robust buffer access forgives and raw CUDA does not. The init
        // accounting in the bookkeeping kernel uses the same bound (range = capacity).
        init_threads = uint32_t(c->event_buffers[bl.consume_events].size());
    } else {
        init_threads = ceil_div(lp.total_spawn, 64) * 64;  // dispatch_workgroups(ceil(n/64)), mod.rs:7157-7173
    }
    if (set_ranges) {
        uint32_t* range = c->h_at<uint32_t>(c->lay.off_range);
        const uint32_t* sp = c->h_at<uint32_t>(c->lay.off_spawn_prefix);
        for (uint32_t i = 0; i < bi.prefix_sum_count; ++i) {
            uint32_t g = bi.prefix_sum_offset + i;
            uint32_t r = 0;
            if (init_threads) {
                uint32_t end = (i + 1 < bi.prefix_sum_count) ? sp[g + 1] : init_threads;
                r = end > sp[g] ? end - sp[g] : 0;
                if (consume && r) r |= 0x80000000u;
            }
            if (range[g] != r) {
                range[g] = r;
                c->plan_dirty = true;
            }
            // a non-zero range must reach the device every frame: the bookkeeping kernel zeroes it after use
            if (r) c->plan_dirty = true;
        }
    }
    ensure_tile_state(c, lp.batch, lp.slab->capacity / small_tile + bi.prefix_sum_count + 1);  // ceil(rows_i / tile) summed over the instances
    {
        // Slot-order state words carry only 6 bits of epoch: the array is zeroed when the slot's use changes (signature)
        // and at least every 64 frames of the slot (tile_state_rule.h). The signature alone is not enough: a batch slot
        // that sits out for 64 frames, or serves another instance of the same effect and slab with fewer tiles, leaves
        // words whose tag matches a later frame's.
        uint64_t sig = 0;
        if (slot_order) {
            sig = 0xcbf29ce484222325ull;
            for (uint64_t v : {uint64_t(bl.effect), uint64_t(bl.slab), uint64_t(tile_word), uint64_t(bi.prefix_sum_count), uint64_t(bi.spawner_base), c->md_generation})
                sig = (sig ^ v) * 0x100000001b3ull;
            sig |= 1;
        }
        if (hnb_rt::tile_state_needs_clear(c->tile_state_slot[lp.batch], sig, hnb_rt::tile_state_run_epoch(c->epoch))) {
            CUDA_CHECK(cudaMemsetAsync(c->d_tile_state[lp.batch].get(), 0, c->d_tile_state[lp.batch].size() * 8, c->stream));
            c->tile_state_clears++;
        }
    }

    hnb::BatchParams& P = lp.params;
    P.frame = c->d_at<hnb::FrameHeader>(0);
    P.spawners = c->d_at<hnb::Spawner>(c->lay.off_spawners);
    P.spawn_prefix = c->d_at<uint32_t>(c->lay.off_spawn_prefix);
    P.prefix_sum = c->d_at<uint32_t>(c->lay.off_prefix_sum);
    P.tile_prefix = c->d_tile_prefix.get();
    P.batch_info = c->d_at<hnb::BatchInfo>(c->lay.off_batch_infos) + lp.batch;
    P.batch_tiles = c->batch_tiles() + lp.batch;
    P.ticket = c->tickets() + lp.batch;
    P.tile_state = c->d_tile_state[lp.batch].get();
    P.metadata = c->d_metadata.get();
    P.draw_args = c->draw_args();
    P.child_infos = c->d_child_infos.get();
    P.properties = lp.fx->d_props.get();
    P.properties_stride = lp.fx->props_stride;
    P.slab = slab_view(*lp.slab);
    if (bl.parent_slab != 0xFFFFFFFFu) {
        const Slab& parent = get_slab(c, bl.parent_slab);
        if (parent.sector_planes) fail(HNB_ERR_LAYOUT, "a parent slab read by a child effect must use the default plane layout");
        P.parent_slab = slab_view(parent);
    }
    if (consume) P.consume_events = c->event_buffers[bl.consume_events].get();
    for (int i = 0; i < HNB_MAX_EVENT_BINDINGS; ++i) {
        if (bl.emit_events[i] != 0xFFFFFFFFu) {
            if (bl.emit_events[i] >= c->event_buffers.size()) fail(HNB_ERR_INVALID_ARG, "invalid emit event buffer");
            P.emit_events[i] = c->event_buffers[bl.emit_events[i]].get();
            P.emit_events_capacity[i] = uint32_t(c->event_buffers[bl.emit_events[i]].size());
        }
    }
    if ((lp.fx->flags & HNB_EFFECT_ORDERED_EVENTS) && (lp.fx->flags & HNB_EFFECT_EMIT_GPU_SPAWN_EVENTS)) {
        if (bi.prefix_sum_count != 1) fail(HNB_ERR_INVALID_ARG, "HNB_EFFECT_ORDERED_EVENTS needs a batch of exactly one instance");
        for (int i = 0; i < HNB_MAX_EVENT_BINDINGS; ++i) {
            if (!P.emit_events[i]) continue;
            // each allocated when missing: a frame that failed between the two allocations is completed by the next
            if (!lp.slab->event_counts[i]) CUDA_CHECK(lp.slab->event_counts[i].alloc(lp.slab->capacity));
            if (!lp.slab->event_block_sums[i]) CUDA_CHECK(lp.slab->event_block_sums[i].alloc(hnb::ordered_event_blocks(lp.slab->capacity) + 1));
            P.event_counts[i] = lp.slab->event_counts[i].get();
        }
    }
    P.init_thread_count = init_threads;
    P.debug = c->d_debug.get();
    P.bi_spawner_base = bi.spawner_base;
    P.bi_prefix_sum_offset = bi.prefix_sum_offset;
    P.bi_prefix_sum_count = bi.prefix_sum_count;
    P.first_md_index = bi.prefix_sum_count ? c->h_at<hnb_spawner>(c->lay.off_spawners)[bi.spawner_base].effect_metadata_index : 0u;
    P.mailbox = c->mailbox;
    P.mailbox_rows = c->mailbox_rows;
    P.mailbox_ring = c->mailbox_ring;
    P.tile_rows = tile_word;
    lp.init_blocks = ceil_div(init_threads, 256 * hnb_rt::kInitItems);  // HNB_INIT_ITEMS logical init threads per CUDA thread
    uint32_t max_tiles = lp.slab->capacity / small_tile + bi.prefix_sum_count + 1;
    lp.update_blocks = std::min<uint32_t>(ceil_div(max_tiles, 8), uint32_t(lp.fx->update_blocks_per_sm) * uint32_t(c->sm_count));
    if (lp.update_blocks == 0) lp.update_blocks = 1;
    if (lp.fx->props_size && !lp.fx->d_props) fail(HNB_ERR_NOT_READY, "effect uses properties but none were uploaded");
    return lp;
}

// hnb_init / hnb_update start with griddepcontrol.wait, so they may always be launched with programmatic stream
// serialization: behind a kernel they become resident early (launch latency hidden), behind anything else the attribute
// has no effect.
void launch_kernel(hnb_ctx* c, CUfunction f, uint32_t blocks, hnb::BatchParams& P, uint32_t smem_bytes = 0, cudaStream_t st = nullptr) {
    void* args[] = {&P};
    CUlaunchConfig cfg{};
    cfg.gridDimX = blocks; cfg.gridDimY = 1; cfg.gridDimZ = 1;
    cfg.blockDimX = 256; cfg.blockDimY = 1; cfg.blockDimZ = 1;
    cfg.sharedMemBytes = smem_bytes;
    cfg.hStream = (CUstream)(st ? st : c->stream);
    CUlaunchAttribute attr{};
    attr.id = CU_LAUNCH_ATTRIBUTE_PROGRAMMATIC_STREAM_SERIALIZATION;
    attr.value.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    CUresult r = c->drv.LaunchKernelEx(&cfg, f, args, nullptr);
    if (r != CUDA_SUCCESS) fail(HNB_ERR_CUDA, "cuLaunchKernelEx: " + cu_error_string(c->drv, r));
    c->launches++;
}

void launch_update(hnb_ctx* c, LaunchPlan& lp, cudaStream_t st = nullptr) {
    if (!st) st = c->stream;
    std::pair<Event, Event> ev;
    if (c->timing) {
        if (!c->ev_free.empty()) { ev = std::move(c->ev_free.back()); c->ev_free.pop_back(); }
        else { CUDA_CHECK(ev.first.create(cudaEventDefault)); CUDA_CHECK(ev.second.create(cudaEventDefault)); }
        CUDA_CHECK(cudaEventRecord(ev.first, st));
    }
    launch_kernel(c, lp.fx->km->update, lp.update_blocks, lp.params, lp.fx->update_smem, st);
    if (c->timing) {
        CUDA_CHECK(cudaEventRecord(ev.second, st));
        c->ev_pending.push_back(std::move(ev));
    }
}

// Fork / join of the context stream for the independent launches of one pass. The reference records one
// dispatch per batch into a single compute pass (mod.rs:7280-7370) and leaves the overlap to the driver; here
// launch k goes to lane k % lanes (lane 0 = the context stream itself). Small batches are latency-bound
// (a few microseconds of work behind ~10 of launch and pipeline ramp), so concurrency is what fills the GPU.
constexpr uint32_t kMaxSideStreams = 7;
struct Fork {
    hnb_ctx* c;
    uint32_t lanes = 1;
    Fork(hnb_ctx* ctx, uint32_t launches) : c(ctx) {
        if (launches < 2) return;
        lanes = std::min<uint32_t>(launches, kMaxSideStreams + 1);
        while (c->side_streams.size() < lanes - 1) {
            SideStream s;
            CUDA_CHECK(s.stream.create(cudaStreamNonBlocking));
            CUDA_CHECK(s.done.create(cudaEventDisableTiming));
            c->side_streams.push_back(std::move(s));
        }
        if (!c->fork_event) CUDA_CHECK(c->fork_event.create(cudaEventDisableTiming));
        CUDA_CHECK(cudaEventRecord(c->fork_event, c->stream));
        for (uint32_t i = 0; i + 1 < lanes; ++i) CUDA_CHECK(cudaStreamWaitEvent(c->side_streams[i].stream, c->fork_event, 0));
    }
    cudaStream_t lane(uint32_t k) const {
        const uint32_t l = k % lanes;
        return l == 0 ? c->stream : c->side_streams[l - 1].stream;
    }
    void join() {
        for (uint32_t i = 0; i + 1 < lanes; ++i) {
            CUDA_CHECK(cudaEventRecord(c->side_streams[i].done, c->side_streams[i].stream));
            CUDA_CHECK(cudaStreamWaitEvent(c->stream, c->side_streams[i].done, 0));
        }
        lanes = 1;
    }
};

// Ribbon sort of one batch ("hanabi:sort" fill / sort / copy, mod.rs:7444-7610): every instance of the batch gets
// the alive-list column the update pass just wrote stably sorted by (RIBBON_ID, AGE bits).
void launch_ribbon_sort(hnb_ctx* c, const LaunchPlan& lp) {
    const hnb_batch_info& bi = c->h_at<hnb_batch_info>(c->lay.off_batch_infos)[lp.batch];
    const bool any_large = lp.slab->capacity > HNB_RIBBON_SORT_SMALL_MAX;
    if (any_large && c->d_sort_scratch.size() < size_t(lp.slab->capacity) * 3) {
        CUDA_CHECK(grow(c->d_sort_scratch, size_t(lp.slab->capacity) * 3, 0, c->stream));
        if (!c->d_sort_hist) CUDA_CHECK(c->d_sort_hist.alloc(hnb::ribbon_sort_hist_words(uint32_t(c->sm_count))));
    }
    const size_t sort_rows = c->d_sort_scratch.size() / 3;
    uint64_t* keys = c->d_sort_scratch.get();
    uint32_t* vals = reinterpret_cast<uint32_t*>(keys + 2 * sort_rows);
    hnb::RibbonSortArgs a{};
    a.planes = plane_set(*lp.slab);
    a.ping = lp.slab->ping.get();
    a.pong = lp.slab->pong.get();
    a.spawners = c->d_at<hnb::Spawner>(c->lay.off_spawners);
    a.metadata = c->d_metadata.get();
    a.spawner_base = bi.spawner_base;
    a.instance_count = bi.prefix_sum_count;
    for (int i = 0; i < 2; ++i) { a.scratch_keys[i] = (u64*)(keys + i * sort_rows); a.scratch_vals[i] = vals + i * sort_rows; }
    a.scratch_hist = c->d_sort_hist.get();
    a.scratch_rows = uint32_t(sort_rows);
    a.scratch_grid = uint32_t(c->sm_count);
    if (any_large) CUDA_CHECK(cudaMemsetAsync(c->d_sort_hist.get(), 0, size_t(2 * 8 * 256) * 4, c->stream));
    clear_ident_claims(c, *lp.slab);  // the sort permutes the column the update just wrote
    uint32_t launched = 0;
    CUDA_CHECK(hnb::launch_ribbon_sort(a, any_large, uint32_t(c->sm_count), c->stream, &launched));
    c->launches += launched;
}

// NVTX ranges named like the reference's compute passes (mod.rs:7029 "hanabi:init", :7186 "hanabi:indirect_dispatch",
// :7283 "hanabi:update"), so that an nsys timeline of this backend lines up with a wgpu capture of the reference.
struct PassRange {
    explicit PassRange(const char* name) { nvtxRangePushA(name); }
    ~PassRange() { nvtxRangePop(); }
    PassRange(const PassRange&) = delete;
    PassRange& operator=(const PassRange&) = delete;
};

void check_coverage(hnb_ctx* c, const std::vector<LaunchPlan>& plans) {
    // the fused bookkeeping kernel visits instances batch by batch: the launched batches must tile
    // [0, num_effects) exactly (Batcher::push allocates spawners and prefix entries in sync)
    std::vector<std::pair<uint32_t, uint32_t>> ranges;
    const hnb_batch_info* bis = c->h_at<hnb_batch_info>(c->lay.off_batch_infos);
    for (uint32_t b = 0; b < c->B; ++b) ranges.push_back({bis[b].prefix_sum_offset, bis[b].prefix_sum_count});
    std::sort(ranges.begin(), ranges.end());
    uint32_t pos = 0;
    for (auto& r : ranges) {
        if (r.first != pos) fail(HNB_ERR_BATCH_COVERAGE, "batches do not tile the spawner table");
        pos += r.second;
    }
    if (pos != c->header()->sim.num_effects) fail(HNB_ERR_BATCH_COVERAGE, "batches do not cover sim_params.num_effects instances");
    for (uint32_t b = 0; b < c->B; ++b)
        if (bis[b].spawner_base != bis[b].prefix_sum_offset) fail(HNB_ERR_BATCH_COVERAGE, "spawner_base must equal prefix_sum_offset");
    // Row indices the kernels dereference without a bounds check (wgpu would clamp them): validated whenever the
    // caller uploaded new rows.
    if (c->dirty_tables) {
        const hnb_spawner* sp = c->h_at<hnb_spawner>(c->lay.off_spawners);
        for (uint32_t i = 0; i < c->header()->sim.num_effects; ++i) {
            if (sp[i].effect_metadata_index >= c->d_metadata.size()) fail(HNB_ERR_OUT_OF_RANGE, "spawner row " + std::to_string(i) + ": effect_metadata_index outside the metadata table");
            if (sp[i].draw_indirect_index >= c->d_draw_args.size()) fail(HNB_ERR_OUT_OF_RANGE, "spawner row " + std::to_string(i) + ": draw_indirect_index outside the draw-args table");
        }
    }
    std::vector<bool> seen(c->B, false);
    for (auto& p : plans) {
        if (seen[p.batch]) fail(HNB_ERR_INVALID_ARG, "batch launched twice");
        seen[p.batch] = true;
    }
    for (uint32_t b = 0; b < c->B; ++b)
        if (!seen[b]) fail(HNB_ERR_NOT_READY, "every uploaded batch must be launched by hnb_simulate");
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------
extern "C" {

const char* hnb_last_error(void) { return g_last_error.c_str(); }
// shared with graph/graph_cabi.cpp (not part of the public ABI: hidden visibility)
__attribute__((visibility("hidden"))) void hnb_set_last_error_(const char* msg) { g_last_error = msg ? msg : ""; }
const char* hnb_version(void) { return "hanabi_b200 0.1.0 (sm_90a)"; }

int32_t hnb_ctx_create(int32_t cuda_device, uintptr_t external_stream, hnb_ctx** out) {
    return guarded([&] {
        if (!out) fail(HNB_ERR_INVALID_ARG, "out is NULL");
        *out = nullptr;
        int n = 0;
        cudaError_t e = cudaGetDeviceCount(&n);
        if (e != cudaSuccess || n == 0) {
            (void)cudaGetLastError();
            fail(HNB_ERR_NO_DEVICE, std::string("no CUDA device available (") + (e != cudaSuccess ? cudaGetErrorString(e) : "0 devices") +
                                        "): hanabi_b200 has no CPU fallback");
        }
        if (cuda_device < 0 || cuda_device >= n) fail(HNB_ERR_INVALID_ARG, "cuda_device out of range");
        CUDA_CHECK(cudaSetDevice(cuda_device));
        CUDA_CHECK(cudaFree(0));
        auto c = std::make_unique<hnb_ctx>();
        c->device = cuda_device;
        std::string err;
        if (!load_driver_api(c->drv, err)) fail(HNB_ERR_NO_DEVICE, err);
        cudaDeviceProp prop;
        CUDA_CHECK(cudaGetDeviceProperties(&prop, cuda_device));
        c->sm_count = prop.multiProcessorCount;
        if (prop.major != 9 || prop.minor != 0) fail(HNB_ERR_NO_DEVICE, "hanabi_b200 kernels are built for sm_90a only; device is sm_" + std::to_string(prop.major * 10 + prop.minor));
        if (external_stream) c->stream.borrow((cudaStream_t)external_stream);
        else CUDA_CHECK(c->stream.create(cudaStreamNonBlocking));
        if (const char* env = getenv("HNB_TILE_CHUNKS")) c->tile_chunks_override = (uint32_t)atoi(env);
        if (const char* env = getenv("HNB_EPOCH_START")) c->epoch = uint32_t(strtoul(env, nullptr, 0)) & 0x3fffffffu;  // tests: start near the wrap
        if (const char* env = getenv("HNB_PARAM_UPLOAD")) c->param_upload = atoi(env) != 0;
        ensure_arena(c.get(), 0, 0);
        CUDA_CHECK(grow(c->d_debug, kDebugWords, 0, c->stream));
        *out = c.release();
    });
}

void hnb_ctx_destroy(hnb_ctx* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    for (auto& m : c->modules) if (m.second->mod) c->drv.ModuleUnload(m.second->mod);
    delete c;
}

int32_t hnb_sync(hnb_ctx* c) {
    return guarded([&] { CUDA_CHECK(cudaStreamSynchronize(c->stream)); });
}
uintptr_t hnb_ctx_stream(hnb_ctx* c) { return (uintptr_t)c->stream.get(); }
uint64_t hnb_ctx_launch_count(hnb_ctx* c) { return c->launches; }
void hnb_ctx_frame_count(hnb_ctx* c, uint64_t* frames, uint64_t* frame_block_copies) {
    if (frames) *frames = c->frames;
    if (frame_block_copies) *frame_block_copies = c->frame_copies;
}

// ---- slabs ----------------------------------------------------------------------------------
int32_t hnb_slab_create(hnb_ctx* c, uint32_t capacity_rows, uint32_t stride, hnb_slab* out) { return hnb_slab_create_ex(c, capacity_rows, stride, 0u, out); }

int32_t hnb_slab_create_ex(hnb_ctx* c, uint32_t capacity_rows, uint32_t stride, uint32_t flags, hnb_slab* out) {
    return guarded([&] {
        if (!out || capacity_rows == 0) fail(HNB_ERR_INVALID_ARG, "bad slab arguments");
        if (flags & ~uint32_t(HNB_SLAB_SECTOR_PLANES)) fail(HNB_ERR_INVALID_ARG, "unknown slab flags");
        CUDA_CHECK(cudaSetDevice(c->device));
        Slab s;
        s.capacity = capacity_rows;
        s.stride = stride;
        s.sector_planes = (flags & HNB_SLAB_SECTOR_PLANES) != 0;
        s.planes = physical_planes(stride, s.sector_planes);
        // planes zero-filled (debug builds of the reference poison the particle buffer instead, effect_cache.rs:284-296)
        for (size_t p = 0; p < s.planes.size(); ++p) CUDA_CHECK(grow(s.d_planes[p], size_t(capacity_rows) * s.planes[p].width, 0, c->stream));
        CUDA_CHECK(s.ping.alloc(capacity_rows));
        CUDA_CHECK(s.pong.alloc(capacity_rows));
        CUDA_CHECK(s.dead.alloc(capacity_rows));
        CUDA_CHECK(grow(s.alive_bits, size_t(capacity_rows) / 32 + 2, 0, c->stream));
        CUDA_CHECK(s.ident_claim.alloc(2));
        clear_ident_claims(c, s);
        CUDA_CHECK(hnb::launch_slab_reset(s.ping.get(), s.pong.get(), s.dead.get(), 0, capacity_rows, c->stream));
        c->launches++;
        s.live = true;
        c->slabs.push_back(std::move(s));
        *out = (hnb_slab)(c->slabs.size() - 1);
    });
}

int32_t hnb_slab_destroy(hnb_ctx* c, hnb_slab h) {
    return guarded([&] {
        Slab& s = get_slab(c, h);
        CUDA_CHECK(cudaStreamSynchronize(c->stream));
        s = Slab{};  // releases its buffers; live = false, and the handle is never reused
    });
}

int32_t hnb_slab_reset_rows(hnb_ctx* c, hnb_slab h, uint32_t first, uint32_t count) {
    return guarded([&] {
        Slab& s = get_slab(c, h);
        check_rows(s, first, count);
        clear_ident_claims(c, s);
        CUDA_CHECK(hnb::launch_slab_reset(s.ping.get(), s.pong.get(), s.dead.get(), first, count, c->stream));
        CUDA_CHECK(hnb::launch_bits_range(s.alive_bits.get(), first, count, false, c->stream));
        c->launches += 2;
    });
}

int32_t hnb_slab_rebuild_alive_bits(hnb_ctx* c, hnb_slab h, uint32_t first, uint32_t rows, uint32_t column, uint32_t alive_count) {
    return guarded([&] {
        Slab& s = get_slab(c, h);
        check_rows(s, first, rows);
        if (column > 1 || alive_count > rows) fail(HNB_ERR_INVALID_ARG, "bad alive-list column or count");
        CUDA_CHECK(hnb::launch_bits_range(s.alive_bits.get(), first, rows, false, c->stream));
        CUDA_CHECK(hnb::launch_bits_from_list(s.alive_bits.get(), (column ? s.pong : s.ping).get() + first, first, alive_count, c->stream));
        c->launches += rows ? 1 + (alive_count ? 1 : 0) : 0;
    });
}

namespace {
// AoS records <-> the slab's planes through a device staging buffer, chunk by chunk: on upload the host records are
// copied up (and only read) and transposed into the planes, on download the planes are transposed and copied down.
void transfer_aos(hnb_ctx* c, hnb_slab h, uint32_t first, uint32_t count, void* host, bool upload) {
    Slab& s = get_slab(c, h);
    check_rows(s, first, count);
    if (count == 0) return;
    const uint32_t rows_per_chunk = (uint32_t)std::max<size_t>(1, kChunkBytes / s.stride);
    DeviceArray<char> staging;
    CUDA_CHECK(staging.alloc(size_t(std::min(rows_per_chunk, count)) * s.stride));
    uint32_t* stage = reinterpret_cast<uint32_t*>(staging.get());
    hnb::PlaneSet ps = plane_set(s);
    for (uint32_t done = 0; done < count; done += rows_per_chunk) {
        uint32_t n = std::min(rows_per_chunk, count - done);
        const size_t at = size_t(done) * s.stride, bytes = size_t(n) * s.stride;
        if (upload) {
            CUDA_CHECK(cudaMemcpyAsync(stage, (const char*)host + at, bytes, cudaMemcpyHostToDevice, c->stream));
            CUDA_CHECK(hnb::launch_aos_to_planes(stage, ps, first + done, n, s.stride / 4, c->stream));
            c->launches++;
        } else {
            CUDA_CHECK(hnb::launch_planes_to_aos(stage, ps, first + done, n, s.stride / 4, c->stream));
            c->launches++;
            CUDA_CHECK(cudaMemcpyAsync((char*)host + at, stage, bytes, cudaMemcpyDeviceToHost, c->stream));
        }
        CUDA_CHECK(cudaStreamSynchronize(c->stream));
    }
}
}  // namespace

int32_t hnb_slab_upload_aos(hnb_ctx* c, hnb_slab h, uint32_t first, uint32_t count, const void* aos) {
    return guarded([&] { transfer_aos(c, h, first, count, const_cast<void*>(aos), true); });
}

int32_t hnb_slab_download_aos(hnb_ctx* c, hnb_slab h, uint32_t first, uint32_t count, void* aos) {
    return guarded([&] { transfer_aos(c, h, first, count, aos, false); });
}

int32_t hnb_slab_upload_indirect(hnb_ctx* c, hnb_slab h, uint32_t first, uint32_t count, const hnb_indirect_index* rows) {
    return guarded([&] {
        Slab& s = get_slab(c, h);
        check_rows(s, first, count);
        if (count == 0) return;
        DeviceArray<uint32_t> stage;
        CUDA_CHECK(stage.alloc(size_t(count) * 3));
        CUDA_CHECK(cudaMemcpyAsync(stage.get(), rows, size_t(count) * 12, cudaMemcpyHostToDevice, c->stream));
        clear_ident_claims(c, s);
        CUDA_CHECK(hnb::launch_indirect_deinterleave(stage.get(), s.ping.get(), s.pong.get(), s.dead.get(), first, count, c->stream));
        c->launches++;
        CUDA_CHECK(cudaStreamSynchronize(c->stream));
    });
}

int32_t hnb_slab_download_indirect(hnb_ctx* c, hnb_slab h, uint32_t first, uint32_t count, hnb_indirect_index* rows) {
    return guarded([&] {
        Slab& s = get_slab(c, h);
        check_rows(s, first, count);
        if (count == 0) return;
        DeviceArray<uint32_t> stage;
        CUDA_CHECK(stage.alloc(size_t(count) * 3));
        CUDA_CHECK(hnb::launch_indirect_interleave(stage.get(), s.ping.get(), s.pong.get(), s.dead.get(), first, count, c->stream));
        c->launches++;
        CUDA_CHECK(cudaMemcpyAsync(rows, stage.get(), size_t(count) * 12, cudaMemcpyDeviceToHost, c->stream));
        CUDA_CHECK(cudaStreamSynchronize(c->stream));
    });
}

// ---- device-resident interop (§8 f-2): the consumer of the hot path is the render pass, which binds the particle
// buffer as AoS records and the indirect buffer as interleaved rows ON THE DEVICE (vfx_render.wgsl:228-231,
// mod.rs:139-146). These run asynchronously on the context stream; no host copy is involved.
int32_t hnb_slab_export_aos_device(hnb_ctx* c, hnb_slab h, uint32_t first, uint32_t count, void* d_dst) {
    return guarded([&] {
        Slab& s = get_slab(c, h);
        check_rows(s, first, count);
        if (count && !d_dst) fail(HNB_ERR_INVALID_ARG, "d_dst is NULL");
        if ((uintptr_t)d_dst & 3u) fail(HNB_ERR_INVALID_ARG, "d_dst must be 4-byte aligned (16-byte aligned for full speed)");
        CUDA_CHECK(hnb::launch_planes_to_aos((uint32_t*)d_dst, plane_set(s), first, count, s.stride / 4, c->stream));
        c->launches += count ? 1 : 0;
    });
}
int32_t hnb_slab_import_aos_device(hnb_ctx* c, hnb_slab h, uint32_t first, uint32_t count, const void* d_src) {
    return guarded([&] {
        Slab& s = get_slab(c, h);
        check_rows(s, first, count);
        if (count && !d_src) fail(HNB_ERR_INVALID_ARG, "d_src is NULL");
        if ((uintptr_t)d_src & 3u) fail(HNB_ERR_INVALID_ARG, "d_src must be 4-byte aligned (16-byte aligned for full speed)");
        CUDA_CHECK(hnb::launch_aos_to_planes((const uint32_t*)d_src, plane_set(s), first, count, s.stride / 4, c->stream));
        c->launches += count ? 1 : 0;
    });
}
int32_t hnb_slab_export_indirect_device(hnb_ctx* c, hnb_slab h, uint32_t first, uint32_t count, hnb_indirect_index* d_dst) {
    return guarded([&] {
        Slab& s = get_slab(c, h);
        check_rows(s, first, count);
        if (count && !d_dst) fail(HNB_ERR_INVALID_ARG, "d_dst is NULL");
        CUDA_CHECK(hnb::launch_indirect_interleave((uint32_t*)d_dst, s.ping.get(), s.pong.get(), s.dead.get(), first, count, c->stream));
        c->launches += count ? 1 : 0;
    });
}
int32_t hnb_slab_import_indirect_device(hnb_ctx* c, hnb_slab h, uint32_t first, uint32_t count, const hnb_indirect_index* d_src) {
    return guarded([&] {
        Slab& s = get_slab(c, h);
        check_rows(s, first, count);
        if (count && !d_src) fail(HNB_ERR_INVALID_ARG, "d_src is NULL");
        clear_ident_claims(c, s);
        CUDA_CHECK(hnb::launch_indirect_deinterleave((const uint32_t*)d_src, s.ping.get(), s.pong.get(), s.dead.get(), first, count, c->stream));
        c->launches += count ? 1 : 0;
    });
}
int32_t hnb_slab_device_view(hnb_ctx* c, hnb_slab h, hnb_slab_view* out) {
    return guarded([&] {
        Slab& s = get_slab(c, h);
        if (!out) fail(HNB_ERR_INVALID_ARG, "out is NULL");
        memset(out, 0, sizeof(*out));
        out->capacity_rows = s.capacity;
        out->particle_stride = s.stride;
        out->num_planes = (uint32_t)s.planes.size();
        for (size_t p = 0; p < s.planes.size(); ++p) {
            out->planes[p] = s.d_planes[p].get();
            out->plane_offset[p] = s.planes[p].offset;
            out->plane_width[p] = s.planes[p].width;
        }
        out->ping = s.ping.get();
        out->pong = s.pong.get();
        out->dead = s.dead.get();
    });
}
void* hnb_device_alloc(hnb_ctx* c, size_t bytes) {
    void* p = nullptr;
    if (cudaSetDevice(c->device) != cudaSuccess || cudaMalloc(&p, bytes) != cudaSuccess) {
        (void)cudaGetLastError();
        return nullptr;
    }
    return p;
}
void hnb_device_free(hnb_ctx* c, void* p) {
    if (!p) return;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    cudaFree(p);
}
int32_t hnb_device_download(hnb_ctx* c, void* host_dst, const void* d_src, size_t bytes) {
    return guarded([&] {
        CUDA_CHECK(cudaMemcpyAsync(host_dst, d_src, bytes, cudaMemcpyDeviceToHost, c->stream));
        CUDA_CHECK(cudaStreamSynchronize(c->stream));
    });
}
int32_t hnb_device_upload(hnb_ctx* c, void* d_dst, const void* host_src, size_t bytes) {
    return guarded([&] {
        CUDA_CHECK(cudaMemcpyAsync(d_dst, host_src, bytes, cudaMemcpyHostToDevice, c->stream));
        CUDA_CHECK(cudaStreamSynchronize(c->stream));
    });
}

int32_t hnb_slab_fill_c5(hnb_ctx* c, hnb_slab h, uint32_t first, uint32_t count, uint32_t seed, float lo, float hi) {
    return hnb_slab_fill_c5_ex(c, h, first, count, seed, lo, hi, first);
}

int32_t hnb_slab_fill_c5_ex(hnb_ctx* c, hnb_slab h, uint32_t first, uint32_t count, uint32_t seed, float lo, float hi, uint32_t logical_first) {
    return guarded([&] {
        Slab& s = get_slab(c, h);
        check_rows(s, first, count);
        if (s.stride != 32) fail(HNB_ERR_LAYOUT, "hnb_slab_fill_c5 needs the 32-byte {position,age,velocity,lifetime} layout");
        if (s.sector_planes) fail(HNB_ERR_LAYOUT, "hnb_slab_fill_c5 writes the default plane layout; spawn through the init pass or use hnb_slab_upload_aos");
        CUDA_CHECK(hnb::launch_fill_c5(s.d_planes[0].get(), s.d_planes[1].get(), s.ping.get(), s.pong.get(), s.ident_claim.get(), first, count, seed, lo, hi,
                                       logical_first, c->stream));
        CUDA_CHECK(hnb::launch_bits_range(s.alive_bits.get(), first, count, true, c->stream));
        c->launches += 2;
    });
}

// The scratch (rows x the widest column) is taken with cudaMallocAsync and given back with cudaFreeAsync on the context
// stream: the call stays asynchronous (no synchronisation to grow or free a buffer the stream may still use), and a
// context does not keep up to 2 GiB between repacks that may be seconds apart.
namespace {
// The checks every call that rewrites or reads one instance's slice through its lists makes (`what`: the call's name).
void check_instance_slice(hnb_ctx* c, const Slab& s, const Effect& fx, uint32_t metadata_row, uint32_t first, uint32_t rows,
                          const char* what) {
    const std::string w = what;
    if (uint64_t(first) + rows > s.capacity) fail(HNB_ERR_INVALID_ARG, w + ": rows outside the slab");
    if (metadata_row >= c->d_metadata.size()) fail(HNB_ERR_INVALID_ARG, w + ": metadata row out of range");
    if (fx.particle_stride != s.stride) fail(HNB_ERR_INVALID_ARG, w + ": effect particle stride does not match the slab");
    if (((fx.flags & HNB_EFFECT_SECTOR_PLANES) != 0) != s.sector_planes)
        fail(HNB_ERR_INVALID_ARG, w + ": effect and slab disagree on HNB_EFFECT_SECTOR_PLANES / HNB_SLAB_SECTOR_PLANES");
    if (fx.flags & HNB_EFFECT_EMIT_GPU_SPAWN_EVENTS)
        fail(HNB_ERR_INVALID_ARG, w + ": pending GPU spawn events name parent slots; an emitting effect cannot be " +
                                      (w == "hnb_slab_repack" ? "repacked" : "snapshot or restored"));
}

hnb::RepackArgs repack_args(hnb_ctx* c, const Slab& s, uint32_t metadata_row, uint32_t first, uint32_t rows) {
    hnb::RepackArgs a{};
    a.metadata = c->d_metadata.get() + metadata_row;
    a.ping = s.ping.get();
    a.pong = s.pong.get();
    a.dead = s.dead.get();
    a.alive_bits = s.alive_bits.get();
    a.claim = s.ident_claim.get();
    a.first = first;
    a.rows = rows;
    return a;
}

hnb::SnapshotArgs snapshot_args(hnb_ctx* c, const Slab& s, uint32_t metadata_row, uint32_t first, uint32_t rows) {
    hnb::SnapshotArgs a{};
    a.metadata = c->d_metadata.get() + metadata_row;
    a.ping = s.ping.get();
    a.pong = s.pong.get();
    a.planes = plane_set(s);
    a.num_planes = (uint32_t)s.planes.size();
    a.stride_words = s.stride / 4;
    a.first = first;
    a.rows = rows;
    return a;
}
}  // namespace

int32_t hnb_slab_repack(hnb_ctx* c, hnb_slab h, hnb_effect e, uint32_t metadata_row, uint32_t first, uint32_t rows) {
    return guarded([&] {
        Slab& s = get_slab(c, h);
        const Effect& fx = get_effect(c, e);
        check_instance_slice(c, s, fx, metadata_row, first, rows, "hnb_slab_repack");
        if (rows == 0) return;
        CUDA_CHECK(cudaSetDevice(c->device));
        const hnb::RepackArgs a = repack_args(c, s, metadata_row, first, rows);
        uint32_t widest = 0;
        for (const Plane& p : s.planes) widest = std::max(widest, p.width);
        void* scratch = nullptr;
        CUDA_CHECK(cudaMallocAsync(&scratch, size_t(rows) * widest, c->stream));
        cudaError_t err = cudaSuccess;
        for (size_t p = 0; p < s.planes.size() && err == cudaSuccess; ++p) {
            const uint32_t width = s.planes[p].width;
            err = hnb::launch_repack_gather(a, s.d_planes[p].get(), scratch, width, c->stream);
            if (err == cudaSuccess)
                err = cudaMemcpyAsync(s.d_planes[p].get() + size_t(first) * width, scratch, size_t(rows) * width, cudaMemcpyDeviceToDevice, c->stream);
            c->launches++;
        }
        // the lists last: every gather reads them
        if (err == cudaSuccess) err = hnb::launch_repack_lists(a, c->stream);
        c->launches++;
        const cudaError_t freed = cudaFreeAsync(scratch, c->stream);
        CUDA_CHECK(err);
        CUDA_CHECK(freed);
    });
}

static_assert(HNB_SNAPSHOT_MAGIC == HNB_SNAPSHOT_MAGIC_WORD && HNB_SNAPSHOT_VERSION == HNB_SNAPSHOT_VERSION_WORD &&
                  sizeof(hnb_instance_snapshot_header) == HNB_SNAPSHOT_HEADER_WORDS * 4,
              "snapshot header of include/hanabi_b200.h and of the kernels");

size_t hnb_instance_snapshot_bytes(uint32_t particle_stride, uint32_t rows) {
    return sizeof(hnb_instance_snapshot_header) + size_t(rows) * particle_stride;
}

// One launch: the kernel reads n, W and particle_counter on the device, so the host never waits for them.
int32_t hnb_instance_snapshot(hnb_ctx* c, hnb_slab h, hnb_effect e, uint32_t metadata_row, uint32_t first, uint32_t rows,
                              void* d_dst, size_t dst_bytes) {
    return guarded([&] {
        Slab& s = get_slab(c, h);
        const Effect& fx = get_effect(c, e);
        check_instance_slice(c, s, fx, metadata_row, first, rows, "hnb_instance_snapshot");
        if (!d_dst || ((uintptr_t)d_dst & 15u)) fail(HNB_ERR_INVALID_ARG, "hnb_instance_snapshot: d_dst is NULL or not 16-byte aligned");
        if (dst_bytes < hnb_instance_snapshot_bytes(s.stride, rows))
            fail(HNB_ERR_INVALID_ARG, "hnb_instance_snapshot: dst_bytes is below hnb_instance_snapshot_bytes(stride, rows)");
        if (rows == 0) return;
        CUDA_CHECK(cudaSetDevice(c->device));
        CUDA_CHECK(hnb::launch_snapshot_gather(snapshot_args(c, s, metadata_row, first, rows), (uint32_t*)d_dst, c->stream));
        c->launches++;
    });
}

// Two launches: the records and the metadata words, then hnb_slab_repack's list writer, which reads m back from
// alive_count.
int32_t hnb_instance_restore(hnb_ctx* c, hnb_slab h, hnb_effect e, uint32_t metadata_row, uint32_t first, uint32_t rows,
                             const void* d_src, size_t src_bytes) {
    return guarded([&] {
        Slab& s = get_slab(c, h);
        const Effect& fx = get_effect(c, e);
        check_instance_slice(c, s, fx, metadata_row, first, rows, "hnb_instance_restore");
        if (!d_src || ((uintptr_t)d_src & 15u)) fail(HNB_ERR_INVALID_ARG, "hnb_instance_restore: d_src is NULL or not 16-byte aligned");
        if (src_bytes < sizeof(hnb_instance_snapshot_header)) fail(HNB_ERR_INVALID_ARG, "hnb_instance_restore: src_bytes is below the 64-byte header");
        if (rows == 0) return;
        CUDA_CHECK(cudaSetDevice(c->device));
        hnb::SnapshotArgs a = snapshot_args(c, s, metadata_row, first, rows);
        a.src_bytes = src_bytes;
        CUDA_CHECK(hnb::launch_restore_scatter(a, (const uint32_t*)d_src, c->stream));
        c->launches++;
        CUDA_CHECK(hnb::launch_repack_lists(repack_args(c, s, metadata_row, first, rows), c->stream));
        c->launches++;
    });
}

int32_t hnb_slab_checksum(hnb_ctx* c, hnb_slab h, uint32_t first, uint32_t count, uint64_t* out) {
    return hnb_slab_checksum_ex(c, h, first, count, 0, out);
}

namespace {
// Hashes rows [first, first + count) of the columns `ps` (`words` per row) on the device into `out`, and waits.
void checksum(hnb_ctx* c, const hnb::PlaneSet& ps, uint32_t first, uint32_t count, uint32_t words, uint64_t index_base, uint64_t* out) {
    DeviceArray<unsigned long long> d;
    CUDA_CHECK(d.alloc(1));
    CUDA_CHECK(cudaMemsetAsync(d.get(), 0, 8, c->stream));
    CUDA_CHECK(hnb::launch_checksum(ps, first, count, words, index_base, d.get(), c->stream));
    c->launches++;
    read_back(c, out, d.get(), 8);
}
}  // namespace

int32_t hnb_slab_checksum_ex(hnb_ctx* c, hnb_slab h, uint32_t first, uint32_t count, uint64_t index_base, uint64_t* out) {
    return guarded([&] {
        Slab& s = get_slab(c, h);
        check_rows(s, first, count);
        checksum(c, plane_set(s), first, count, s.stride / 4, index_base, out);
    });
}

int32_t hnb_slab_checksum_indirect(hnb_ctx* c, hnb_slab h, uint32_t first, uint32_t count, uint64_t* out) {
    return guarded([&] {
        Slab& s = get_slab(c, h);
        check_rows(s, first, count);
        // hash the rows as the reference's interleaved IndirectEntry {ping, pong, dead}
        hnb::PlaneSet ps{};
        uint32_t* cols[3] = {s.ping.get(), s.pong.get(), s.dead.get()};
        for (int p = 0; p < 3; ++p) {
            ps.ptr[p] = cols[p];
            ps.words[p] = 1;
            ps.word_off[p] = (uint32_t)p;
            ps.word_to_plane[p] = (unsigned char)p;
        }
        checksum(c, ps, first, count, 3, 0, out);
    });
}

// ---- effects --------------------------------------------------------------------------------
int32_t hnb_effect_generate_source(const hnb_effect_desc* desc, char* out, size_t cap, size_t* len) {
    return guarded([&] {
        if (!desc) fail(HNB_ERR_INVALID_ARG, "desc is NULL");
        std::string src = generate_effect_source(*desc);
        if (len) *len = src.size();
        if (out && cap) {
            size_t n = std::min(cap - 1, src.size());
            memcpy(out, src.data(), n);
            out[n] = 0;
        }
    });
}

int32_t hnb_nvrtc_check(const char* source, size_t* cubin_size) {
    return guarded([&] {
        std::string cubin, log;
        // generated sources state their own compile mode (effect_source.cpp)
        const bool fast_math = std::string(source).find("#define HNB_FAST_MATH 1") != std::string::npos;
        if (!nvrtc_compile_sm90a(source, "check.cu", cubin, log, fast_math)) fail(HNB_ERR_NVRTC, log);
        g_last_error = log;  // compiler log (ptxas -v) available to the caller even on success
        if (cubin_size) *cubin_size = cubin.size();
    });
}

// Everything hnb_effect_compile derives from the descriptor before it touches the GPU (the descriptor's strings need
// not outlive the call that builds this).
struct EffectBlueprint {
    std::string source, name;
    uint64_t hash = 0;
    bool fast_math = false;
    uint32_t tile_k = 4, rows_per_lane = 16, update_smem = 0, flags = 0, particle_stride = 0, parent_stride = 0, props_size = 0;
};
static EffectBlueprint make_blueprint(const hnb_effect_desc& desc) {
    EffectBlueprint bp;
    bp.source = generate_effect_source(desc);
    bp.hash = fnv1a64(bp.source);
    bp.name = desc.name ? desc.name : "effect";
    bp.fast_math = (desc.flags & HNB_EFFECT_FAST_MATH) != 0;  // the flag is part of the source (hash)
    bp.tile_k = choose_tile_k(desc);
    bp.rows_per_lane = rows_per_lane();
    bp.update_smem = update_smem_bytes(desc);
    bp.flags = desc.flags;
    bp.particle_stride = desc.particle_stride;
    bp.parent_stride = desc.parent_particle_stride;
    bp.props_size = desc.properties_size;
    return bp;
}
// Load (or find in the cache) the module of `bp` and register an effect for it.
static hnb_effect install_effect(hnb_ctx* c, const EffectBlueprint& bp, const std::string* precompiled_cubin) {
    CUDA_CHECK(cudaSetDevice(c->device));
    Effect fx;
    fx.hash = bp.hash;
    fx.name = bp.name;
    fx.km = get_module(c, bp.source, fx.name, fx.hash, bp.fast_math, precompiled_cubin);
    fx.tile_k = bp.tile_k;
    fx.rows_per_lane = bp.rows_per_lane;
    fx.update_smem = bp.update_smem;
    {
        CUresult r = c->drv.FuncSetAttribute(fx.km->update, CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES, (int)fx.update_smem);
        if (r != CUDA_SUCCESS) fail(HNB_ERR_CUDA, "cuFuncSetAttribute(max dynamic smem " + std::to_string(fx.update_smem) + "): " + cu_error_string(c->drv, r));
        int bps = 0;
        r = c->drv.OccupancyMaxActiveBlocksPerMultiprocessor(&bps, fx.km->update, 256, fx.update_smem);
        if (r != CUDA_SUCCESS || bps < 1) bps = 1;
        fx.update_blocks_per_sm = bps;
    }
    fx.flags = bp.flags;
    fx.particle_stride = bp.particle_stride;
    fx.parent_stride = bp.parent_stride;
    fx.props_size = bp.props_size;
    fx.props_stride = (uint32_t)align_up(bp.props_size, 16);
    fx.live = true;
    c->effects.push_back(std::move(fx));
    return (hnb_effect)(c->effects.size() - 1);
}

int32_t hnb_effect_compile(hnb_ctx* c, const hnb_effect_desc* desc, hnb_effect* out) {
    return guarded([&] {
        if (!desc || !out) fail(HNB_ERR_INVALID_ARG, "NULL argument");
        *out = install_effect(c, make_blueprint(*desc), nullptr);
    });
}

// ---- background compilation ------------------------------------------------------------------
// The reference compiles pipelines asynchronously and neither ticks nor batches an effect until both are ready
// (spawn.rs:968-973, mod.rs:3853-3894). A compile job runs the NVRTC step (the 0.3-1 s part) on its own thread and
// needs no context; hnb_effect_create_from_job() then only loads the finished cubin.
struct hnb_compile_job {
    EffectBlueprint bp;
    std::string cubin, log;
    std::atomic<int> state{0};  // 0 running, 1 ready, -1 failed
    std::thread worker;
};

hnb_compile_job* hnb_compile_job_start(const hnb_effect_desc* desc) {
    hnb_compile_job* job = nullptr;
    int32_t rc = guarded([&] {
        if (!desc) fail(HNB_ERR_INVALID_ARG, "desc is NULL");
        auto j = std::make_unique<hnb_compile_job>();
        j->bp = make_blueprint(*desc);  // copies every string of the descriptor
        hnb_compile_job* raw = j.get();
        raw->worker = std::thread([raw] {
            const bool ok = nvrtc_compile_sm90a(raw->bp.source, raw->bp.name + ".cu", raw->cubin, raw->log, raw->bp.fast_math);
            raw->state.store(ok ? 1 : -1, std::memory_order_release);
        });
        job = j.release();
    });
    return rc == HNB_OK ? job : nullptr;
}

int32_t hnb_compile_job_poll(hnb_compile_job* job) {
    if (!job) return HNB_ERR_INVALID_ARG;
    const int st = job->state.load(std::memory_order_acquire);
    if (st == 0) return 0;
    if (st == 1) return 1;
    g_last_error = job->log;
    return HNB_ERR_NVRTC;
}

int32_t hnb_compile_job_wait(hnb_compile_job* job) {
    if (!job) return HNB_ERR_INVALID_ARG;
    if (job->worker.joinable()) job->worker.join();
    return hnb_compile_job_poll(job);
}

void hnb_compile_job_destroy(hnb_compile_job* job) {
    if (!job) return;
    if (job->worker.joinable()) job->worker.join();
    delete job;
}

int32_t hnb_effect_create_from_job(hnb_ctx* c, hnb_compile_job* job, hnb_effect* out) {
    return guarded([&] {
        if (!job || !out) fail(HNB_ERR_INVALID_ARG, "NULL argument");
        const int st = job->state.load(std::memory_order_acquire);
        if (st == 0) fail(HNB_ERR_NOT_READY, "the compile job is still running");
        if (st < 0) fail(HNB_ERR_NVRTC, job->log);
        *out = install_effect(c, job->bp, &job->cubin);
    });
}

int32_t hnb_effect_destroy(hnb_ctx* c, hnb_effect h) {
    return guarded([&] {
        Effect& fx = get_effect(c, h);
        CUDA_CHECK(cudaStreamSynchronize(c->stream));
        fx.d_props.reset();
        fx.live = false;  // the compiled module stays in the cache (ShaderCache never evicts either)
    });
}

int32_t hnb_upload_properties(hnb_ctx* c, hnb_effect h, uint32_t array_index, const void* blob, uint32_t bytes) {
    return guarded([&] {
        Effect& fx = get_effect(c, h);
        if (fx.props_size == 0) fail(HNB_ERR_INVALID_ARG, "effect has no properties");
        if (bytes != fx.props_size) fail(HNB_ERR_LAYOUT, "property blob size does not match the effect's PropertyLayout");
        const uint32_t rows = uint32_t(fx.d_props.size() / fx.props_stride);
        if (array_index >= rows) {
            uint32_t cap = std::max<uint32_t>(array_index + 1, std::max<uint32_t>(rows * 2, 4));
            CUDA_CHECK(grow(fx.d_props, size_t(cap) * fx.props_stride, fx.d_props.size(), c->stream));
        }
        CUDA_CHECK(cudaMemcpyAsync(fx.d_props.get() + size_t(array_index) * fx.props_stride, blob, bytes, cudaMemcpyHostToDevice, c->stream));
        CUDA_CHECK(cudaStreamSynchronize(c->stream));  // blob is pageable caller memory
    });
}

// ---- per-frame tables -------------------------------------------------------------------------
int32_t hnb_set_sim_params(hnb_ctx* c, const hnb_sim_params* p) {
    return guarded([&] {
        if (!p) fail(HNB_ERR_INVALID_ARG, "params is NULL");
        memcpy(&c->header()->sim, p, sizeof(*p));
    });
}

int32_t hnb_upload_spawners(hnb_ctx* c, const hnb_spawner* rows, uint32_t n) {
    return guarded([&] {
        if (n && !rows) fail(HNB_ERR_INVALID_ARG, "rows is NULL");
        const uint32_t old_e = c->E, old_b = c->B;
        const char* const old_arena = c->h_arena.get();
        ensure_arena(c, n, c->B);
        // A host that uploads its tables every frame whether they changed or not (the reference does: mod.rs:4679-4705) should not
        // pay for it: identical rows over an unchanged layout leave the frame a header-only frame.
        if (old_arena == c->h_arena.get() && old_e == c->E && old_b == c->B && n &&
            memcmp(c->h_arena.get() + c->lay.off_spawners, rows, size_t(n) * sizeof(hnb_spawner)) == 0)
            return;
        memcpy(c->h_arena.get() + c->lay.off_spawners, rows, size_t(n) * sizeof(hnb_spawner));
        c->dirty_tables = true;
    });
}

int32_t hnb_upload_batches(hnb_ctx* c, const hnb_batch_info* rows, uint32_t nb, const uint32_t* prefix, uint32_t np) {
    return guarded([&] {
        if ((nb && !rows) || (np && !prefix)) fail(HNB_ERR_INVALID_ARG, "NULL table");
        const uint32_t old_e = c->E, old_b = c->B;
        const char* const old_arena = c->h_arena.get();
        ensure_arena(c, std::max(c->E, np), nb);
        if (np > c->E) fail(HNB_ERR_OUT_OF_RANGE, "more prefix entries than instances");
        if (old_arena == c->h_arena.get() && old_e == c->E && old_b == c->B && nb &&
            memcmp(c->h_arena.get() + c->lay.off_batch_infos, rows, size_t(nb) * sizeof(hnb_batch_info)) == 0 &&
            (np == 0 || memcmp(c->h_arena.get() + c->lay.off_spawn_prefix, prefix, size_t(np) * 4) == 0))
            return;  // unchanged (see hnb_upload_spawners); the per-frame spawn ranges are recomputed by every launch plan
        memcpy(c->h_arena.get() + c->lay.off_batch_infos, rows, size_t(nb) * sizeof(hnb_batch_info));
        memcpy(c->h_arena.get() + c->lay.off_spawn_prefix, prefix, size_t(np) * 4);
        memcpy(c->h_arena.get() + c->lay.off_prefix_sum, prefix, size_t(np) * 4);  // same buffer in the reference (batch.rs:194-216)
        memset(c->h_arena.get() + c->lay.off_range, 0, size_t(c->E) * 4);
        c->dirty_tables = true;
    });
}

int32_t hnb_metadata_insert(hnb_ctx* c, uint32_t row, const hnb_effect_metadata* md) {
    return guarded([&] {
        if (!md) fail(HNB_ERR_INVALID_ARG, "md is NULL");
        c->md_generation++;
        const uint32_t rows = uint32_t(c->d_metadata.size());
        if (row + 1 > rows) CUDA_CHECK(grow(c->d_metadata, std::max<uint32_t>(row + 1, std::max<uint32_t>(rows * 2, 16)), rows, c->stream));
        CUDA_CHECK(cudaMemcpyAsync(c->d_metadata.get() + row, md, sizeof(*md), cudaMemcpyHostToDevice, c->stream));
        CUDA_CHECK(cudaStreamSynchronize(c->stream));
    });
}

int32_t hnb_draw_args_insert(hnb_ctx* c, uint32_t row, const hnb_draw_indexed_indirect_args* a) {
    return guarded([&] {
        if (!a) fail(HNB_ERR_INVALID_ARG, "args is NULL");
        const uint32_t rows = uint32_t(c->d_draw_args.size());
        if (row >= rows) CUDA_CHECK(grow(c->d_draw_args, std::max<uint32_t>(row + 1, std::max<uint32_t>(rows * 2, 16)), rows, c->stream));
        CUDA_CHECK(cudaMemcpyAsync(c->d_draw_args.get() + row, a, sizeof(*a), cudaMemcpyHostToDevice, c->stream));
        CUDA_CHECK(cudaStreamSynchronize(c->stream));
    });
}

int32_t hnb_event_buffer_create(hnb_ctx* c, uint32_t capacity, hnb_event_buffer* out) {
    return guarded([&] {
        if (!out || !capacity) fail(HNB_ERR_INVALID_ARG, "bad event buffer arguments");
        DeviceArray<uint32_t> b;
        CUDA_CHECK(grow(b, capacity, 0, c->stream));
        c->event_buffers.push_back(std::move(b));
        *out = (hnb_event_buffer)(c->event_buffers.size() - 1);
    });
}

int32_t hnb_child_info_insert(hnb_ctx* c, uint32_t row, const hnb_child_info* info) {
    return guarded([&] {
        if (!info) fail(HNB_ERR_INVALID_ARG, "info is NULL");
        // the table is exactly as long as the logical array (arrayLength() in vfx_indirect.wgsl:43)
        const uint32_t rows = uint32_t(c->d_child_infos.size());
        if (row >= rows) CUDA_CHECK(grow(c->d_child_infos, row + 1, rows, c->stream));
        CUDA_CHECK(cudaMemcpyAsync(c->d_child_infos.get() + row, info, sizeof(*info), cudaMemcpyHostToDevice, c->stream));
        CUDA_CHECK(cudaStreamSynchronize(c->stream));
    });
}

int32_t hnb_read_child_info(hnb_ctx* c, uint32_t row, hnb_child_info* out) {
    return guarded([&] {
        if (row >= c->d_child_infos.size()) fail(HNB_ERR_OUT_OF_RANGE, "child info row out of range");
        read_back(c, out, c->d_child_infos.get() + row, sizeof(*out));
    });
}

int32_t hnb_event_buffer_download(hnb_ctx* c, hnb_event_buffer h, uint32_t first, uint32_t count, uint32_t* out) {
    return guarded([&] {
        if (h >= c->event_buffers.size()) fail(HNB_ERR_INVALID_ARG, "invalid event buffer");
        auto& b = c->event_buffers[h];
        if (uint64_t(first) + count > b.size()) fail(HNB_ERR_OUT_OF_RANGE, "event range out of bounds");
        read_back(c, out, b.get() + first, size_t(count) * 4);
    });
}

// ---- the hot path -----------------------------------------------------------------------------
int32_t hnb_simulate(hnb_ctx* c, const hnb_batch_launch* batches, uint32_t n) {
    return guarded([&] {
        if (n && !batches) fail(HNB_ERR_INVALID_ARG, "batches is NULL");
        CUDA_CHECK(cudaSetDevice(c->device));
        if (c->header()->sim.num_effects > c->E) fail(HNB_ERR_NOT_READY, "sim_params.num_effects exceeds the uploaded spawner table");
        ensure_scratch(c);
        std::vector<LaunchPlan>& plans = c->frame_plans;  // reused from frame to frame: no allocation in steady state
        plans.clear();
        plans.reserve(n);
        for (uint32_t i = 0; i < n; ++i) plans.push_back(plan_batch(c, batches[i], true));
        check_coverage(c, plans);  // nothing has been enqueued yet: a bad frame is skipped as a whole
        next_epoch(c);
        // The frame block reaches the device with ONE copy — or with none: when no table row, tile size or init range
        // changed since the last upload (a steady-state frame without spawns), the only new bytes are the 64-byte
        // header (sim params, epoch), and those ride in the bookkeeping kernel's parameter space. The frame is then
        // a pure kernel chain, which programmatic dependent launch pipelines against the previous frame.
        // ... or, third way, with the bookkeeping LAUNCH: when the frame has no init pass (nothing reads the tables before the
        // bookkeeping kernel) and the host-written part of the arena fits the kernel parameter space, it travels there and CTA 0
        // stores it into the device arena. A copy-engine operation between two kernels of the chain costs its own latency and
        // the programmatic overlap of the kernel behind it, every frame of a host that rewrites its tables every frame.
        const bool copy_block = c->dirty_tables || c->plan_dirty;
        bool any_init = false;
        for (auto& lp : plans) any_init |= lp.init_blocks != 0;
        const bool param_block = copy_block && c->param_upload && c->B > 0 && c->lay.off_prefix_sum <= HNB_FRAME_BLOCK_MAX_BYTES;
        // with an init pass the block needs a (one-CTA) kernel of its own at the head of the frame: init reads the tables first
        const bool block_kernel = param_block && any_init;
        if (block_kernel) {
            CUDA_CHECK(hnb::launch_frame_block(c->d_arena.get(), c->h_arena.get(), uint32_t(c->lay.off_prefix_sum), c->stream));
            c->launches++;
            for (auto& lp : plans) lp.params.late_tables = 1u;
        }
        if (copy_block && !param_block) flush_arena(c, true);
        if (block_kernel) { c->dirty_tables = false; c->plan_dirty = false; }  // (stored by k_frame_block, enqueued above)
        c->frames++;
        c->frame_copies += (copy_block && !param_block) ? 1 : 0;
        // pass "hanabi:init" (mod.rs:7025-7179). Batches write disjoint slab rows and table rows; the only
        // cross-batch access is a child reading its parent's records, so frames with event-driven children keep
        // the reference's serial order.
        {
            PassRange range("hanabi:init");
            uint32_t inits = 0;
            bool reads_parent = false;
            for (auto& lp : plans) {
                inits += lp.init_blocks ? 1 : 0;
                reads_parent |= (lp.fx->flags & (HNB_EFFECT_READ_PARENT_PARTICLE | HNB_EFFECT_CONSUME_GPU_SPAWN_EVENTS)) != 0;
            }
            Fork fork(c, reads_parent ? 1 : inits);
            uint32_t k = 0;
            for (auto& lp : plans)
                if (lp.init_blocks) launch_kernel(c, lp.fx->km->init, lp.init_blocks, lp.params, hnb_rt::kInitSmemBytes, fork.lane(k++));
            fork.join();
        }
        // passes "hanabi:indirect_dispatch" + "hanabi:update_prefix_sum" (mod.rs:7182-7275), fused
        {
            PassRange range("hanabi:indirect_dispatch");  // + "hanabi:update_prefix_sum"
            const void* block = nullptr;   // what rides in the kernel's parameter space: nothing / the 64-byte header / header + tables
            uint32_t block_bytes = 0;
            if (param_block && !block_kernel) { block = c->h_arena.get(); block_bytes = uint32_t(c->lay.off_prefix_sum); }
            else if (block_kernel) { /* already stored by k_frame_block, header included */ }
            else if (!copy_block) { block = c->header(); block_bytes = uint32_t(sizeof(hnb::FrameHeader)); }
            CUDA_CHECK(hnb::launch_bookkeeping(static_tables(c), c->header()->sim.num_effects, c->B, block, block_bytes, c->stream));
            if (param_block && !block_kernel) { c->dirty_tables = false; c->plan_dirty = false; }  // the tables went with this launch
            c->launches += 1 + (c->d_child_infos.size() ? 1 : 0);
            std::fill(c->init_pending.begin(), c->init_pending.end(), 0);
        }
        // pass "hanabi:update" (mod.rs:7280-7370): batches are independent (event appends are atomic)
        {
            PassRange range("hanabi:update");
            Fork fork(c, uint32_t(plans.size()));
            uint32_t k = 0;
            for (auto& lp : plans) launch_update(c, lp, fork.lane(k++));
            fork.join();
        }
        // HNB_EFFECT_ORDERED_EVENTS: append the events the update rows asked for, in row order (three small launches
        // per channel; the default is the reference's per-particle atomics inside the update kernel)
        for (auto& lp : plans) {
            if (!(lp.fx->flags & HNB_EFFECT_ORDERED_EVENTS) || !(lp.fx->flags & HNB_EFFECT_EMIT_GPU_SPAWN_EVENTS)) continue;
            const hnb_batch_info& bi = c->h_at<hnb_batch_info>(c->lay.off_batch_infos)[lp.batch];
            const hnb_spawner& sp = c->h_at<hnb_spawner>(c->lay.off_spawners)[bi.spawner_base];
            if (sp.effect_metadata_index >= c->d_metadata.size()) fail(HNB_ERR_OUT_OF_RANGE, "spawner row points outside the metadata table");
            for (int i = 0; i < HNB_MAX_EVENT_BINDINGS; ++i) {
                if (!lp.params.event_counts[i]) continue;
                hnb::EventAppendArgs a{};
                a.counts = lp.params.event_counts[i];
                a.ping = lp.slab->ping.get();
                a.pong = lp.slab->pong.get();
                a.spawner = c->d_at<hnb::Spawner>(c->lay.off_spawners) + bi.spawner_base;
                a.metadata = c->d_metadata.get() + sp.effect_metadata_index;
                a.block_sums = lp.slab->event_block_sums[i].get();
                a.child_infos = c->d_child_infos.get();
                a.binding = uint32_t(i);
                a.buffer = lp.params.emit_events[i];
                a.capacity = lp.params.emit_events_capacity[i];
                CUDA_CHECK(hnb::launch_ordered_event_append(a, lp.slab->capacity, c->stream));
                c->launches += 3;
            }
        }
        // ribbons: passes "hanabi:sort_prefix_sum" (the reference re-runs vfx_prefix_sum over every batch,
        // mod.rs:7393-7428) and "hanabi:sort" (mod.rs:7444-7610)
        bool needs_sort = false;
        for (auto& lp : plans) needs_sort |= (lp.fx->flags & HNB_EFFECT_RIBBONS) != 0;
        if (needs_sort) {
            PassRange range("hanabi:sort");
            CUDA_CHECK(hnb::launch_prefix_sum(static_tables(c), c->B, c->stream));
            c->launches += c->B ? 1 : 0;
            for (auto& lp : plans)
                if (lp.fx->flags & HNB_EFFECT_RIBBONS) launch_ribbon_sort(c, lp);
        }
    });
}

int32_t hnb_pass_sort(hnb_ctx* c, const hnb_batch_launch* b) {
    return guarded([&] {
        if (!b) fail(HNB_ERR_INVALID_ARG, "batch is NULL");
        ensure_scratch(c);
        LaunchPlan lp = plan_batch(c, *b, false);
        flush_arena(c, false);
        launch_ribbon_sort(c, lp);
    });
}

int32_t hnb_pass_init(hnb_ctx* c, const hnb_batch_launch* b) {
    return guarded([&] {
        if (!b) fail(HNB_ERR_INVALID_ARG, "batch is NULL");
        ensure_scratch(c);
        // The init kernel pops dead slots by rank from the counters as they stood at the START of the pass, and its
        // alive_count / particle_counter increments are applied by the indirect pass that follows (spawn_range[]): a
        // second stand-alone init of the same batch before that pass would pop the same slots and lose the first
        // launch's increments (the reference's atomics accumulate, vfx_init.wgsl:141-151). Refuse it.
        if (b->batch_info_index < c->init_pending.size() && c->init_pending[b->batch_info_index])
            fail(HNB_ERR_INVALID_ARG, "hnb_pass_init: this batch already has an init pass pending; run hnb_pass_indirect first");
        LaunchPlan lp = plan_batch(c, *b, true);
        c->header()->num_batches = c->B;
        if (c->header()->epoch == 0) next_epoch(c);
        flush_arena(c, true);
        if (lp.init_blocks) {
            launch_kernel(c, lp.fx->km->init, lp.init_blocks, lp.params, hnb_rt::kInitSmemBytes);
            if (c->init_pending.size() <= b->batch_info_index) c->init_pending.resize(size_t(b->batch_info_index) + 1, 0);
            c->init_pending[b->batch_info_index] = 1;
        }
    });
}

int32_t hnb_pass_indirect(hnb_ctx* c) {
    return guarded([&] {
        ensure_scratch(c);
        c->header()->num_batches = c->B;
        flush_arena(c, false);
        uint32_t ne = c->header()->sim.num_effects;
        if (ne > c->E) fail(HNB_ERR_NOT_READY, "sim_params.num_effects exceeds the uploaded spawner table");
        CUDA_CHECK(hnb::launch_indirect(static_tables(c), ne, c->stream));
        c->launches += ne ? (1 + (c->d_child_infos.size() ? 1 : 0)) : 0;
        std::fill(c->init_pending.begin(), c->init_pending.end(), 0);  // the deferred init accounting has been applied
    });
}

int32_t hnb_pass_prefix_sum(hnb_ctx* c) {
    return guarded([&] {
        ensure_scratch(c);
        c->header()->num_batches = c->B;
        // The tile prefix written by this stand-alone pass uses a nominal tile size; hnb_pass_update() rebuilds
        // it for its own launch geometry (k_tile_prefix), so only the reference outputs matter here.
        uint32_t* ts = c->h_at<uint32_t>(c->lay.off_tile_size);
        for (uint32_t b = 0; b < c->B; ++b) if (ts[b] == 0) ts[b] = 128;
        flush_arena(c, false);
        if (c->B) CUDA_CHECK(cudaMemcpyAsync(c->d_arena.get() + c->lay.off_tile_size, ts, size_t(c->B) * 4, cudaMemcpyHostToDevice, c->stream));
        CUDA_CHECK(hnb::launch_prefix_sum(static_tables(c), c->B, c->stream));
        c->launches += c->B ? 1 : 0;
    });
}

int32_t hnb_pass_update(hnb_ctx* c, const hnb_batch_launch* b) {
    return guarded([&] {
        if (!b) fail(HNB_ERR_INVALID_ARG, "batch is NULL");
        ensure_scratch(c);
        LaunchPlan lp = plan_batch(c, *b, false);
        next_epoch(c);
        flush_arena(c, false);
        CUDA_CHECK(hnb::launch_tile_prefix(static_tables(c), lp.batch, lp.params.tile_rows, c->stream));
        c->launches++;
        launch_update(c, lp);
    });
}

int32_t hnb_pass_fill_dispatch_args(hnb_ctx* c, const uint32_t* src, uint32_t src_offset, uint32_t src_stride, uint32_t* dst,
                                    uint32_t dst_len, uint32_t dst_offset, uint32_t dst_stride, uint32_t count) {
    return guarded([&] {
        if (count == 0) return;
        uint32_t src_len = src_offset + (count - 1) * src_stride + 1;
        if (dst_offset + (count - 1) * dst_stride + 3 > dst_len) fail(HNB_ERR_OUT_OF_RANGE, "dst too small");
        DeviceArray<uint32_t> ds, dd;
        CUDA_CHECK(ds.alloc(src_len));
        CUDA_CHECK(dd.alloc(dst_len));
        CUDA_CHECK(cudaMemcpyAsync(ds.get(), src, size_t(src_len) * 4, cudaMemcpyHostToDevice, c->stream));
        CUDA_CHECK(cudaMemcpyAsync(dd.get(), dst, size_t(dst_len) * 4, cudaMemcpyHostToDevice, c->stream));
        CUDA_CHECK(hnb::launch_fill_dispatch_args(ds.get(), dd.get(), src_offset, src_stride, dst_offset, dst_stride, count, c->stream));
        c->launches++;
        CUDA_CHECK(cudaMemcpyAsync(dst, dd.get(), size_t(dst_len) * 4, cudaMemcpyDeviceToHost, c->stream));
        CUDA_CHECK(cudaStreamSynchronize(c->stream));
    });
}

// ---- readback ---------------------------------------------------------------------------------
int32_t hnb_read_metadata(hnb_ctx* c, uint32_t row, hnb_effect_metadata* out) {
    return guarded([&] {
        if (row >= c->d_metadata.size()) fail(HNB_ERR_OUT_OF_RANGE, "metadata row out of range");
        read_back(c, out, c->d_metadata.get() + row, sizeof(*out));
    });
}
int32_t hnb_read_draw_args(hnb_ctx* c, uint32_t row, hnb_draw_indexed_indirect_args* out) {
    return guarded([&] {
        if (row >= c->d_draw_args.size()) fail(HNB_ERR_OUT_OF_RANGE, "draw args row out of range");
        read_back(c, out, c->d_draw_args.get() + row, sizeof(*out));
    });
}
int32_t hnb_read_draw_args_async(hnb_ctx* c, uint32_t first, uint32_t count, hnb_draw_indexed_indirect_args* pinned_out) {
    return guarded([&] {
        if (uint64_t(first) + count > c->d_draw_args.size()) fail(HNB_ERR_OUT_OF_RANGE, "draw args rows out of range");
        CUDA_CHECK(cudaMemcpyAsync(pinned_out, c->d_draw_args.get() + first, size_t(count) * 20, cudaMemcpyDeviceToHost, c->stream));
    });
}
int32_t hnb_read_spawner(hnb_ctx* c, uint32_t row, hnb_spawner* out) {
    return guarded([&] {
        if (row >= c->E) fail(HNB_ERR_OUT_OF_RANGE, "spawner row out of range");
        read_back(c, out, c->d_arena.get() + c->lay.off_spawners + size_t(row) * 128, 128);
    });
}
int32_t hnb_read_batch_info(hnb_ctx* c, uint32_t row, hnb_batch_info* out) {
    return guarded([&] {
        if (row >= c->B) fail(HNB_ERR_OUT_OF_RANGE, "batch row out of range");
        read_back(c, out, c->d_arena.get() + c->lay.off_batch_infos + size_t(row) * 24, 24);
    });
}
int32_t hnb_read_prefix_sum(hnb_ctx* c, uint32_t first, uint32_t count, uint32_t* out) {
    return guarded([&] {
        if (uint64_t(first) + count > c->E) fail(HNB_ERR_OUT_OF_RANGE, "prefix range out of bounds");
        read_back(c, out, c->d_arena.get() + c->lay.off_prefix_sum + size_t(first) * 4, size_t(count) * 4);
    });
}
int32_t hnb_read_dispatch_args(hnb_ctx* c, uint32_t row, hnb_dispatch_indirect_args* out) {
    return guarded([&] {
        if (row >= c->scratch_B()) fail(HNB_ERR_OUT_OF_RANGE, "dispatch args row out of range");
        read_back(c, out, c->dispatch_args() + size_t(row) * 3, 12);
    });
}
int32_t hnb_read_tile_size(hnb_ctx* c, uint32_t row, uint32_t* out) {
    return guarded([&] {
        if (!out) fail(HNB_ERR_INVALID_ARG, "NULL argument");
        if (row >= c->B) fail(HNB_ERR_OUT_OF_RANGE, "batch row out of range");
        *out = c->h_at<uint32_t>(c->lay.off_tile_size)[row];  // host copy of the word plan_batch passed to the batch's last launch
    });
}

int32_t hnb_ctx_set_count_mailbox(hnb_ctx* c, uint64_t* pinned_host, uint32_t rows, uint32_t ring) {
    return guarded([&] {
        if (!c) fail(HNB_ERR_INVALID_ARG, "ctx is NULL");
        if (!pinned_host) { c->mailbox = nullptr; c->mailbox_rows = c->mailbox_ring = 0; return; }
        if (rows == 0 || ring == 0) fail(HNB_ERR_INVALID_ARG, "count mailbox needs rows >= 1 and ring >= 1");
        CUDA_CHECK(cudaSetDevice(c->device));
        void* dev = nullptr;
        if (cudaHostGetDevicePointer(&dev, pinned_host, 0) != cudaSuccess) {
            (void)cudaGetLastError();
            fail(HNB_ERR_INVALID_ARG, "count mailbox must be pinned host memory (hnb_host_alloc)");
        }
        memset(pinned_host, 0, size_t(rows) * ring * 8);
        c->mailbox = (unsigned long long*)dev;
        c->mailbox_rows = rows;
        c->mailbox_ring = ring;
    });
}
int32_t hnb_ctx_last_epoch(hnb_ctx* c, uint32_t* epoch) {
    return guarded([&] {
        if (!c || !epoch) fail(HNB_ERR_INVALID_ARG, "NULL argument");
        *epoch = c->epoch;
    });
}
int32_t hnb_ctx_tile_state_clears(hnb_ctx* c, uint64_t* clears) {
    return guarded([&] {
        if (!c || !clears) fail(HNB_ERR_INVALID_ARG, "NULL argument");
        *clears = c->tile_state_clears;
    });
}

void* hnb_host_alloc(size_t bytes) {
    void* p = nullptr;
    if (cudaMallocHost(&p, bytes) != cudaSuccess) {
        (void)cudaGetLastError();
        return nullptr;
    }
    return p;
}
void hnb_host_free(void* p) {
    if (p) cudaFreeHost(p);
}

int32_t hnb_ctx_read_debug(hnb_ctx* c, uint64_t* out16, int32_t clear) {
    return guarded([&] {
        read_back(c, out16, c->d_debug.get(), 16 * 8, clear != 0);
    });
}

int32_t hnb_ctx_read_debug_ring(hnb_ctx* c, uint64_t* out256, int32_t clear) {
    return guarded([&] {
        read_back(c, out256, c->d_debug.get() + 16, 256 * 8, clear != 0);
    });
}

int32_t hnb_ctx_measure_sm_mhz(hnb_ctx* c, uint32_t window_us, double* mhz) {
    return guarded([&] {
        DeviceArray<unsigned long long> d;
        CUDA_CHECK(d.alloc(2));
        CUDA_CHECK(hnb::launch_measure_sm_clock(d.get(), (unsigned long long)window_us * 1000ull, c->stream));
        c->launches++;
        unsigned long long h[2] = {0, 0};
        read_back(c, h, d.get(), 16);
        if (mhz) *mhz = h[1] ? double(h[0]) / (double(h[1]) * 1e-3) : 0.0;
    });
}

int32_t hnb_ctx_enable_kernel_timing(hnb_ctx* c, int32_t enabled) {
    c->timing = enabled != 0;
    return HNB_OK;
}
int32_t hnb_ctx_kernel_time_ms(hnb_ctx* c, double* update_ms_total, uint64_t* update_launches) {
    return guarded([&] {
        CUDA_CHECK(cudaStreamSynchronize(c->stream));
        for (auto& ev : c->ev_pending) {
            float ms = 0.f;
            CUDA_CHECK(cudaEventElapsedTime(&ms, ev.first, ev.second));
            c->update_ms += ms;
            c->update_launches++;
        }
        for (auto& ev : c->ev_pending) c->ev_free.push_back(std::move(ev));
        c->ev_pending.clear();
        if (update_ms_total) *update_ms_total = c->update_ms;
        if (update_launches) *update_launches = c->update_launches;
        c->update_ms = 0.0;
        c->update_launches = 0;
    });
}

}  // extern "C"
