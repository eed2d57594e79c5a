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
#include <utility>
#include <vector>

#include "../kernels/hnb_static_kernels.h"
#include "cuda_owned.h"
#include "driver.h"
#include "effect_source.h"
#include "hanabi_b200.h"
#include "nvrtc_compile.h"
#include "slab_access_rule.h"
#include "tile_state_rule.h"

using namespace hnb_rt;

static_assert(sizeof(hnb_spawner) == 128 && sizeof(hnb::Spawner) == 128, "GpuSpawnerParams is 128 bytes");
static_assert(sizeof(hnb_effect_metadata) == 60 && sizeof(hnb::EffectMetadata) == 60, "GpuEffectMetadata is 60 bytes");
static_assert(sizeof(hnb_batch_info) == 24 && sizeof(hnb::BatchInfo) == 24, "GpuBatchInfo is 24 bytes");
static_assert(sizeof(hnb_sim_params) == 28 && sizeof(hnb::SimParams) == 28, "GpuSimParams is 28 bytes");
static_assert(sizeof(hnb_draw_indexed_indirect_args) == 20, "GpuDrawIndexedIndirectArgs is 20 bytes");
static_assert(HNB_BATCH_CULL_MAX_VIEWS == HNB_CULL_MAX_VIEWS, "the multi-view cull kernels hold every view the C API accepts");
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
    // Physical columns, carved from one zero-filled block of capacity x stride bytes: column p starts at capacity x
    // planes[p].offset.
    std::vector<Plane> planes;
    DeviceArray<char> d_block;
    char* column(size_t p) const { return d_block.get() + size_t(capacity) * planes[p].offset; }
    DeviceArray<uint32_t> ping, pong, dead;
    DeviceArray<uint32_t> alive_bits;  // one bit per row (HNB_EFFECT_SLOT_ORDER effects keep it current)
    DeviceArray<unsigned long long> ident_claim;  // [2]: identity claims of ping / pong (hnb_claim_pack)
    DeviceArray<uint32_t> life_floor;             // one f32 per 32 rows
    DeviceArray<unsigned long long> group_age;    // one word per 32 rows, then hnb_deferred_groups
    hnb_rt::SlabState state;  // what the claims, group words and plan may be trusted for (slab_access_rule.h)
    // HNB_EFFECT_ORDERED_EVENTS scratch, allocated on first use: per channel the per-row event counts and their block sums
    DeviceArray<uint32_t> event_counts[HNB_MAX_EVENT_BINDINGS];
    DeviceArray<uint32_t> event_block_sums[HNB_MAX_EVENT_BINDINGS];
};

struct KernelModule {
    CUmodule mod = nullptr;
    CUfunction init = nullptr, update = nullptr;
    int update_blocks_per_sm = 1;
    hnb_rt::ModuleWords words;  // what it keeps of the slab's group words
    std::string log;
};

// A deep copy of an effect descriptor: what a context needs to compile the effect again for another column plan.
struct OwnedDesc {
    hnb_effect_desc d{};
    std::vector<std::string> names, parent_names;
    std::vector<hnb_attr_layout> attrs, parent_attrs;
    std::string name, properties_struct, init_code, init_extra, sim_space_code, age_code, reap_code, update_code, update_extra;
    explicit OwnedDesc(const hnb_effect_desc& src) {
        auto s = [](const char* p) { return std::string(p ? p : ""); };
        name = s(src.name); properties_struct = s(src.properties_struct); init_code = s(src.init_code);
        init_extra = s(src.init_extra); sim_space_code = s(src.sim_space_code); age_code = s(src.age_code);
        reap_code = s(src.reap_code); update_code = s(src.update_code); update_extra = s(src.update_extra);
        auto copy = [&](const hnb_attr_layout* a, uint32_t n, std::vector<std::string>& ns, std::vector<hnb_attr_layout>& out) {
            for (uint32_t i = 0; a && i < n; ++i) ns.push_back(s(a[i].name));
            for (uint32_t i = 0; a && i < n; ++i) out.push_back({ns[i].c_str(), a[i].value_type, a[i].offset, a[i].flags});
        };
        copy(src.attrs, src.n_attrs, names, attrs);
        copy(src.parent_attrs, src.n_parent_attrs, parent_names, parent_attrs);
        d = src;
        d.name = name.c_str(); d.properties_struct = src.properties_struct ? properties_struct.c_str() : nullptr;
        d.init_code = init_code.c_str(); d.init_extra = init_extra.c_str(); d.sim_space_code = sim_space_code.c_str();
        d.age_code = age_code.c_str(); d.reap_code = reap_code.c_str(); d.update_code = update_code.c_str();
        d.update_extra = update_extra.c_str();
        d.attrs = attrs.empty() ? nullptr : attrs.data();
        d.parent_attrs = parent_attrs.empty() ? nullptr : parent_attrs.data();
    }
    OwnedDesc(const OwnedDesc&) = delete;
    OwnedDesc& operator=(const OwnedDesc&) = delete;
};

struct Effect {
    bool live = false;
    uint64_t hash = 0;
    KernelModule* km = nullptr;        // the module of the effect's own column plan
    std::vector<Plane> plan;           // column_plan of the descriptor
    std::shared_ptr<const OwnedDesc> desc;
    struct PlanModule {
        std::vector<Plane> plan, parent_plan;  // parent_plan empty: a parent slab in the default cut
        KernelModule* km;
    };
    std::vector<PlanModule> plan_modules;  // modules for slabs (or parent slabs) of other plans
    bool fast_math = false;
    uint32_t tile_k = 4, flags = 0, particle_stride = 0, parent_stride = 0, rows_per_lane = 16, update_smem = 0;
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
    uint64_t plan_compiles = 0;      // (effect, other column plan) modules made by module_for_plan (hnb_ctx_plan_compiles)
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
    bool defer_ages = true;   // HNB_DEFER_AGES=0: no update leaves common ages deferred (DESIGN.md §3; A/B measurements)
    unsigned long long* mailbox = nullptr;  // device alias of the caller's pinned count mailbox (hnb_ctx_set_count_mailbox)
    uint32_t mailbox_rows = 0, mailbox_ring = 0;
    bool plan_dirty = false;  // bind_launch changed a tile-size or range word of the host frame block since the last upload
    uint64_t frame_copies = 0, frames = 0;  // hnb_simulate calls that needed the host->device copy of the frame block / all calls
    DeviceArray<unsigned long long> d_bounds_acc;  // hnb_batch_bounds: 8 slots per instance of the largest batch seen, zero between calls
    DeviceArray<uint32_t> d_depth_scratch;  // hnb_batch_depth_order: pass buffers, histograms and instance plan of the largest call seen
    DeviceArray<uint32_t> d_cull_scratch;  // hnb_batch_cull: tile masks, tile prefixes and instance plan of the largest call seen
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

void prepare_slab(hnb_ctx* c, Slab& s, hnb_rt::SlabAccess access, uint32_t first = 0, uint32_t count = 0,
                  const hnb_rt::ModuleWords& m = {});

void next_epoch(hnb_ctx* c) {
    c->epoch = (c->epoch + 1u) & 0x3fffffffu;
    if (c->epoch == 0) {
        // 30-bit wrap (207 days at 60 frames/s): a tile state left untouched since the same epoch of the previous
        // cycle would look current, so drop them all. 0 = "never written".
        c->epoch = 1;
        for (const auto& ts : c->d_tile_state)
            if (ts) CUDA_CHECK(cudaMemsetAsync(ts.get(), 0, ts.size() * 8, c->stream));
        // the same for a common age stored a whole cycle ago (DESIGN.md §3)
        for (Slab& s : c->slabs)
            if (s.live) prepare_slab(c, s, hnb_rt::SlabAccess::Invalidate);
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

hnb::PlaneSet plane_set(const std::vector<Plane>& planes, char* block, uint32_t capacity) {
    hnb::PlaneSet ps{};
    for (size_t p = 0; p < planes.size(); ++p) {
        ps.ptr[p] = block + size_t(capacity) * planes[p].offset;
        ps.words[p] = planes[p].width / 4;
        ps.word_off[p] = planes[p].word[0];
        if (!planes[p].contiguous()) {
            ps.word_off[p] = HNB_PLANE_WORD_LIST;
            for (uint32_t l = 0; l < planes[p].width / 4; ++l) ps.word_off[p] |= uint32_t(planes[p].word[l]) << (6 * l);
        }
        for (uint32_t l = 0; l < planes[p].width / 4; ++l) ps.word_to_plane[planes[p].word[l]] = (unsigned char)p;
    }
    return ps;
}
hnb::PlaneSet plane_set(const Slab& s) { return plane_set(s.planes, s.d_block.get(), s.capacity); }

// Enqueues, in stream order, what `access` to rows [first, first + count) of the slab must do first (slab_access_rule.h):
// drops the identity claims, then writes the deferred ages of the rows' 32-row groups back to their rows (k_flush_group_ages)
// and, for writers, sets every word and lifetime floor of those groups to the sentinel. A deferred word a reader flushes
// becomes the word known at the context's epoch, which the next frame's update reads as known.
void prepare_slab(hnb_ctx* c, Slab& s, hnb_rt::SlabAccess access, uint32_t first, uint32_t count, const hnb_rt::ModuleWords& m) {
    const hnb_rt::SlabWork w = hnb_rt::slab_access(s.state, access, first, count, s.capacity, m);
    if (w.drop_claims) CUDA_CHECK(cudaMemsetAsync(s.ident_claim.get(), 0, 2 * sizeof(unsigned long long), c->stream));
    if (w.flush) {
        CUDA_CHECK(hnb::launch_flush_group_ages(plane_set(s), s.state.age_word, s.group_age.get(), s.life_floor.get(), w.first, w.count,
                                                s.capacity, w.clear, c->epoch, c->stream));
        c->launches++;
    } else if (w.clear) {
        const size_t g0 = w.first / 32u, g1 = (size_t(w.first) + w.count + 31u) / 32u;
        CUDA_CHECK(cudaMemsetAsync(s.life_floor.get() + g0, 0xff, (g1 - g0) * sizeof(uint32_t), c->stream));
        CUDA_CHECK(cudaMemsetAsync(s.group_age.get() + g0, 0xff, (g1 - g0) * sizeof(unsigned long long), c->stream));
    }
}

// AoS records <-> columns go through a device staging buffer in chunks of this size.
constexpr size_t kChunkBytes = size_t(64) << 20;

// The first effect bound to a slab (a launch, hnb_slab_repack, hnb_instance_restore) gives it that effect's column plan;
// later binds keep it, and so does a slab whose columns were handed out (hnb_slab_device_view pins the plan it shows).
// Records written before (in the default cut) move to the new columns once, through a second block of capacity x stride
// bytes and one synchronisation; when that block cannot be allocated the slab keeps its default cut (the effect then runs
// a module generated for it). Callers validate everything else first: a failure here leaves the slab as it was.
void fix_plan(hnb_ctx* c, Slab& s, const std::vector<Plane>& plan) {
    if (s.state.plan_fixed) return;
    if (plan != s.planes && s.state.written) {
        DeviceArray<char> next, staging;
        const uint32_t rows_per_chunk = (uint32_t)std::min<size_t>(s.capacity, std::max<size_t>(1, kChunkBytes / s.stride));
        if (next.alloc(size_t(s.capacity) * s.stride) != cudaSuccess || staging.alloc(size_t(rows_per_chunk) * s.stride) != cudaSuccess) {
            (void)cudaGetLastError();
            s.state.plan_fixed = true;
            return;
        }
        // before the records move: a deferred age goes back to the columns it is moved from
        prepare_slab(c, s, hnb_rt::SlabAccess::Invalidate);
        const hnb::PlaneSet from = plane_set(s), to = plane_set(plan, next.get(), s.capacity);
        uint32_t* stage = reinterpret_cast<uint32_t*>(staging.get());
        for (uint32_t done = 0; done < s.capacity; done += rows_per_chunk) {
            const uint32_t n = std::min(rows_per_chunk, s.capacity - done);
            CUDA_CHECK(hnb::launch_planes_to_aos(stage, from, done, n, s.stride / 4, c->stream));
            CUDA_CHECK(hnb::launch_aos_to_planes(stage, to, done, n, s.stride / 4, c->stream));
            c->launches += 2;
        }
        CUDA_CHECK(cudaStreamSynchronize(c->stream));  // the old block and the staging buffer are released below
        s.d_block.swap(next);
    }
    s.planes = plan;
    s.state.plan_fixed = true;
}
void fix_default_plan(hnb_ctx* c, Slab& s) { fix_plan(c, s, physical_planes(s.stride, s.sector_planes)); }

hnb::SlabView slab_view(const Slab& s) {
    hnb::SlabView v{};
    for (size_t p = 0; p < s.planes.size(); ++p) v.planes[p] = s.column(p);
    v.particle_index[0] = s.ping.get();
    v.particle_index[1] = s.pong.get();
    v.dead_index = s.dead.get();
    v.alive_bits = s.alive_bits.get();
    v.ident_claim = s.ident_claim.get();
    v.capacity_rows = s.capacity;
    return v;
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
    km->update_blocks_per_sm = 1;  // depends on the effect's dynamic shared memory (set_update_smem)
    km->words.life_floor = source.find("\n#define HNB_LIFE_FLOOR 1\n") != std::string::npos;
    km->words.group_age = source.find("\n#define HNB_GROUP_AGE 1\n") != std::string::npos;
    if (const size_t at = source.find("\n#define HNB_GROUP_AGE_WORD "); at != std::string::npos)
        km->words.age_word = uint32_t(strtoul(source.c_str() + at + 27, nullptr, 10));
    KernelModule* out = km.get();
    c->modules.emplace(hash, std::move(km));
    return out;
}

// Lets hnb_update of `km` take `smem` bytes of dynamic shared memory and records how many of its CTAs fit on an SM.
void set_update_smem(hnb_ctx* c, KernelModule* km, uint32_t smem) {
    CUresult r = c->drv.FuncSetAttribute(km->update, CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES, (int)smem);
    if (r != CUDA_SUCCESS) fail(HNB_ERR_CUDA, "cuFuncSetAttribute(max dynamic smem " + std::to_string(smem) + "): " + cu_error_string(c->drv, r));
    int bps = 0;
    r = c->drv.OccupancyMaxActiveBlocksPerMultiprocessor(&bps, km->update, 256, smem);
    km->update_blocks_per_sm = (r != CUDA_SUCCESS || bps < 1) ? 1 : bps;
}

// The module that runs `fx` on a slab of column plan `plan`, reading a parent slab of plan `parent` (NULL: none, or the
// default cut): the effect's own, or one compiled for these plans on first use.
KernelModule* module_for_plan(hnb_ctx* c, Effect& fx, const std::vector<Plane>& plan, const std::vector<Plane>* parent) {
    static const std::vector<Plane> kDefault;
    const std::vector<Plane>& pp = parent ? *parent : kDefault;
    if (plan == fx.plan && pp.empty()) return fx.km;
    for (const auto& pm : fx.plan_modules)
        if (pm.plan == plan && pm.parent_plan == pp) return pm.km;
    const std::string source = generate_effect_source(fx.desc->d, &plan, parent);
    KernelModule* km = get_module(c, source, fx.name, fnv1a64(source), fx.fast_math);
    set_update_smem(c, km, fx.update_smem);
    fx.plan_modules.push_back({plan, pp, km});
    c->plan_compiles++;
    return km;
}

struct LaunchPlan {
    Effect* fx;
    Slab* slab;
    Slab* parent;      // the parent slab a child reads, or NULL
    KernelModule* km;  // fx compiled for the slab's plan and the parent slab's (bind_launch)
    uint32_t batch;
    uint32_t init_threads;
    hnb::BatchParams params;
    uint32_t init_blocks;
    uint32_t update_blocks;
};

// Every check of one launch; writes nothing, so a call can refuse a bad launch without side effects. Fills in what needs
// no module: the effect, the slabs, the batch and the init threads.
LaunchPlan check_launch(hnb_ctx* c, const hnb_batch_launch& bl) {
    LaunchPlan lp{};
    lp.fx = &get_effect(c, bl.effect);
    lp.slab = &get_slab(c, bl.slab);
    const Effect& fx = *lp.fx;
    if (fx.particle_stride != lp.slab->stride) fail(HNB_ERR_LAYOUT, "effect particle stride does not match the slab");
    if (((fx.flags & HNB_EFFECT_SECTOR_PLANES) != 0) != lp.slab->sector_planes)
        fail(HNB_ERR_LAYOUT, "effect and slab disagree on HNB_EFFECT_SECTOR_PLANES / HNB_SLAB_SECTOR_PLANES");
    if (bl.parent_slab != 0xFFFFFFFFu) {
        lp.parent = &get_slab(c, bl.parent_slab);
        if (lp.parent->sector_planes) fail(HNB_ERR_LAYOUT, "a parent slab read by a child effect must not use sector planes");
    }
    if (bl.batch_info_index >= c->B) fail(HNB_ERR_OUT_OF_RANGE, "batch_info_index out of range");
    lp.batch = bl.batch_info_index;
    const hnb_batch_info& bi = c->h_at<hnb_batch_info>(c->lay.off_batch_infos)[lp.batch];
    if (uint64_t(bi.prefix_sum_offset) + bi.prefix_sum_count > c->E || uint64_t(bi.spawner_base) + bi.prefix_sum_count > c->E)
        fail(HNB_ERR_OUT_OF_RANGE, "batch references instances outside the uploaded spawner table");
    if (fx.flags & HNB_EFFECT_SLOT_ORDER) {
        // bitmap words must belong to one instance (and one warp) each
        const hnb_spawner* sp = c->h_at<hnb_spawner>(c->lay.off_spawners);
        for (uint32_t i = 0; i < bi.prefix_sum_count; ++i)
            if (sp[bi.spawner_base + i].slab_offset & 31u) fail(HNB_ERR_LAYOUT, "HNB_EFFECT_SLOT_ORDER needs every instance to start on a multiple of 32 slab rows");
        // a slot-order state word packs each running count into 28 bits
        if (lp.slab->capacity >= (1u << 28)) fail(HNB_ERR_LAYOUT, "HNB_EFFECT_SLOT_ORDER needs a slab of fewer than 2^28 rows");
    }
    if (fx.flags & HNB_EFFECT_CONSUME_GPU_SPAWN_EVENTS) {
        if (bl.consume_events >= c->event_buffers.size()) fail(HNB_ERR_INVALID_ARG, "event-driven effect needs a consume_events buffer");
        // One logical init thread per event-buffer ENTRY, not per 64-thread workgroup of the reference's dispatch: the
        // threads of the last partial workgroup would read past the buffer when a parent over-emits (event_count is
        // unclamped, lib.rs:976-993), which WGSL's robust buffer access forgives and raw CUDA does not. The init
        // accounting in the bookkeeping kernel uses the same bound (range = capacity).
        lp.init_threads = uint32_t(c->event_buffers[bl.consume_events].size());
    } else {
        lp.init_threads = ceil_div(bl.total_spawn_count, 64) * 64;  // dispatch_workgroups(ceil(n/64)), mod.rs:7157-7173
    }
    for (int i = 0; i < HNB_MAX_EVENT_BINDINGS; ++i)
        if (bl.emit_events[i] != 0xFFFFFFFFu && bl.emit_events[i] >= c->event_buffers.size()) fail(HNB_ERR_INVALID_ARG, "invalid emit event buffer");
    if ((fx.flags & HNB_EFFECT_ORDERED_EVENTS) && (fx.flags & HNB_EFFECT_EMIT_GPU_SPAWN_EVENTS) && bi.prefix_sum_count != 1)
        fail(HNB_ERR_INVALID_ARG, "HNB_EFFECT_ORDERED_EVENTS needs a batch of exactly one instance");
    if (fx.props_size && !fx.d_props) fail(HNB_ERR_NOT_READY, "effect uses properties but none were uploaded");
    lp.init_blocks = ceil_div(lp.init_threads, 256 * hnb_rt::kInitItems);  // HNB_INIT_ITEMS logical init threads per CUDA thread
    return lp;
}

// The first bind of a slab fixes its plan (fix_plan) to the launch's effect's own; an unbound parent slab read by a child
// keeps the default cut. Launch order decides when two effects of different plans bind one fresh slab in one call.
void fix_launch_plans(hnb_ctx* c, const LaunchPlan& lp) {
    fix_plan(c, *lp.slab, lp.fx->plan);
    if (lp.parent) fix_default_plan(c, *lp.parent);
}

// Sub-tiles per update tile (`forced`: HNB_TILE_CHUNKS, 0 = by slab size) for `rows` slab rows in `instances` instances.
// Rows per warp tile: 32 lanes x K rows per lane x chunks. Larger tiles shorten the look-back chain and amortise the
// per-tile work (ticket, state word, instance lookup); smaller tiles spread a small slab over more warps. With W = one
// sub-tile per resident warp (C5 on an H100: 3168 warps x 128 rows = 396 Ki rows):
//  * from 8 W up the launch streams at the HBM rate and the largest tile wins at every size;
//  * below, the launch is latency-bound and runs in ROUNDS: every resident warp takes one tile per round, and a tile
//    costs a fixed part (ticket, first alive-list entries, look-back, compaction) plus a part per sub-tile: pick the
//    chunk count that minimises rounds x (3.6 + chunks), preferring larger tiles on a tie. The constant was fitted on
//    an earlier GPU. On an H100 (tools/sweep_small.py, C5) the rule is within 3 % of the best forced chunk count from
//    1 Mi rows up; at 256-512 Ki rows forcing 3-4 chunks shortens the frame by 15-20 % (not retuned).
uint32_t tile_chunks(uint32_t forced, uint64_t rows, uint32_t instances, uint32_t sub_tile, uint32_t total_warps, uint32_t max_chunks) {
    uint32_t chunks = forced;
    if (chunks == 0) {
        const uint64_t wave = uint64_t(total_warps) * sub_tile;
        if (rows >= 8 * wave) {
            chunks = max_chunks;
        } else {
            double best = 0.0;
            for (uint32_t ch = 1; ch <= max_chunks; ++ch) {
                const uint64_t tiles = (rows + uint64_t(sub_tile) * ch - 1) / (uint64_t(sub_tile) * ch) + instances - 1;
                const uint64_t rounds = std::max<uint64_t>(1, (tiles + total_warps - 1) / total_warps);
                const double cost = double(rounds) * (3.6 + double(ch));
                if (chunks == 0 || cost <= best) { best = cost; chunks = ch; }
            }
        }
    }
    return std::max(1u, std::min(chunks, max_chunks));
}

void ensure_tile_state(hnb_ctx* c, uint32_t batch, uint32_t tiles) {
    if (c->d_tile_state[batch].size() >= tiles) return;
    CUDA_CHECK(grow(c->d_tile_state[batch], tiles + tiles / 2 + 64, 0, c->stream));
    c->tile_state_slot[batch] = hnb_rt::TileStateSlot{};
}

// Binds a checked launch once the plans of its slabs are fixed (fix_launch_plans): picks the module for those plans and the
// tile size, writes the tile size and (`set_ranges`) the per-instance init thread ranges into the host frame block,
// readies the batch's tile states and ordered-event scratch, and builds the kernel parameters.
void bind_launch(hnb_ctx* c, LaunchPlan& lp, const hnb_batch_launch& bl, bool set_ranges) {
    const Effect& fx = *lp.fx;
    Slab& slab = *lp.slab;
    const hnb_batch_info& bi = c->h_at<hnb_batch_info>(c->lay.off_batch_infos)[lp.batch];
    const std::vector<Plane>* parent_plan = nullptr;  // a parent slab in the default cut needs no module of its own
    if (lp.parent && !is_default_cut(lp.parent->planes, lp.parent->stride)) parent_plan = &lp.parent->planes;
    lp.km = module_for_plan(c, *lp.fx, slab.planes, parent_plan);

    const uint32_t sub_tile = 32u * fx.tile_k;
    const uint32_t total_warps = uint32_t(lp.km->update_blocks_per_sm) * uint32_t(c->sm_count) * 8u;
    const uint32_t tile = sub_tile * tile_chunks(c->tile_chunks_override, slab.capacity, bi.prefix_sum_count, sub_tile, total_warps,
                                                 std::max(1u, fx.rows_per_lane / fx.tile_k));
    // Tile size word shared with the bookkeeping kernels (hnb_tile_rows + flags)
    const bool slot_order = (fx.flags & HNB_EFFECT_SLOT_ORDER) != 0;
    const uint32_t tile_word = tile | (slot_order ? HNB_TILE_SLOT_ORDER : 0u);
    if (c->h_at<uint32_t>(c->lay.off_tile_size)[lp.batch] != tile_word) {
        c->h_at<uint32_t>(c->lay.off_tile_size)[lp.batch] = tile_word;
        c->plan_dirty = true;
    }
    const bool consume = (fx.flags & HNB_EFFECT_CONSUME_GPU_SPAWN_EVENTS) != 0;
    if (set_ranges) {
        uint32_t* range = c->h_at<uint32_t>(c->lay.off_range);
        const uint32_t* sp = c->h_at<uint32_t>(c->lay.off_spawn_prefix);
        for (uint32_t i = 0; i < bi.prefix_sum_count; ++i) {
            uint32_t g = bi.prefix_sum_offset + i;
            uint32_t r = 0;
            if (lp.init_threads) {
                uint32_t end = (i + 1 < bi.prefix_sum_count) ? sp[g + 1] : lp.init_threads;
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
    const uint32_t max_tiles = slab.capacity / tile + bi.prefix_sum_count + 1;  // ceil(rows_i / tile) summed over the instances
    ensure_tile_state(c, lp.batch, max_tiles);
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
    P.properties = fx.d_props.get();
    P.properties_stride = fx.props_stride;
    P.slab = slab_view(slab);
    if (lp.parent) P.parent_slab = slab_view(*lp.parent);
    // An update that keeps the common ages may defer them (launch_update decides, once every launch of the frame is bound).
    prepare_slab(c, slab, hnb_rt::SlabAccess::Bind, 0, 0, lp.km->words);
    P.life_floor = slab.state.floors_off ? nullptr : reinterpret_cast<float*>(slab.life_floor.get());
    P.group_age = hnb_rt::keeps_group_ages(slab.state) ? slab.group_age.get() : nullptr;
    P.defer_ages = P.group_age && c->defer_ages ? 1u : 0u;
    if (consume) P.consume_events = c->event_buffers[bl.consume_events].get();
    for (int i = 0; i < HNB_MAX_EVENT_BINDINGS; ++i) {
        if (bl.emit_events[i] == 0xFFFFFFFFu) continue;
        P.emit_events[i] = c->event_buffers[bl.emit_events[i]].get();
        P.emit_events_capacity[i] = uint32_t(c->event_buffers[bl.emit_events[i]].size());
    }
    if ((fx.flags & HNB_EFFECT_ORDERED_EVENTS) && (fx.flags & HNB_EFFECT_EMIT_GPU_SPAWN_EVENTS)) {
        for (int i = 0; i < HNB_MAX_EVENT_BINDINGS; ++i) {
            if (!P.emit_events[i]) continue;
            // each allocated when missing: a frame that failed between the two allocations is completed by the next
            if (!slab.event_counts[i]) CUDA_CHECK(slab.event_counts[i].alloc(slab.capacity));
            if (!slab.event_block_sums[i]) CUDA_CHECK(slab.event_block_sums[i].alloc(hnb::ordered_event_blocks(slab.capacity) + 1));
            P.event_counts[i] = slab.event_counts[i].get();
        }
    }
    P.init_thread_count = lp.init_threads;
    P.debug = c->d_debug.get();
    P.bi_spawner_base = bi.spawner_base;
    P.bi_prefix_sum_offset = bi.prefix_sum_offset;
    P.bi_prefix_sum_count = bi.prefix_sum_count;
    P.first_md_index = bi.prefix_sum_count ? c->h_at<hnb_spawner>(c->lay.off_spawners)[bi.spawner_base].effect_metadata_index : 0u;
    P.mailbox = c->mailbox;
    P.mailbox_rows = c->mailbox_rows;
    P.mailbox_ring = c->mailbox_ring;
    P.tile_rows = tile_word;
    lp.update_blocks = std::max(1u, std::min<uint32_t>(ceil_div(max_tiles, 8), uint32_t(lp.km->update_blocks_per_sm) * uint32_t(c->sm_count)));
}

// A stand-alone pass's one launch: checked, then bound.
LaunchPlan check_and_bind(hnb_ctx* c, const hnb_batch_launch& bl, bool set_ranges) {
    LaunchPlan lp = check_launch(c, bl);
    ensure_scratch(c);
    fix_launch_plans(c, lp);
    bind_launch(c, lp, bl, set_ranges);
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
    // A launch bound after this one may have switched the slab's common ages off (bind_launch): then nothing is deferred.
    Slab& slab = *lp.slab;
    if (!hnb_rt::keeps_group_ages(slab.state)) lp.params.defer_ages = 0u;
    if (lp.params.defer_ages) prepare_slab(c, slab, hnb_rt::SlabAccess::DeferringUpdate, 0, 0, lp.km->words);
    std::pair<Event, Event> ev;
    if (c->timing) {
        if (!c->ev_free.empty()) { ev = std::move(c->ev_free.back()); c->ev_free.pop_back(); }
        else { CUDA_CHECK(ev.first.create(cudaEventDefault)); CUDA_CHECK(ev.second.create(cudaEventDefault)); }
        CUDA_CHECK(cudaEventRecord(ev.first, st));
    }
    launch_kernel(c, lp.km->update, lp.update_blocks, lp.params, lp.fx->update_smem, st);
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
    // the sort permutes the column the update just wrote, and its second key is the age
    prepare_slab(c, *lp.slab, hnb_rt::SlabAccess::ListSort);
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

// The frame block reaches the device with ONE copy — or with none: when no table row, tile size or init range changed
// since the last upload (a steady-state frame without spawns), the only new bytes are the 64-byte header (sim params,
// epoch), and those ride in the bookkeeping kernel's parameter space. The frame is then a pure kernel chain, which
// programmatic dependent launch pipelines against the previous frame.
// ... or, third way, with the bookkeeping LAUNCH: when the frame has no init pass (nothing reads the tables before the
// bookkeeping kernel) and the host-written part of the arena fits the kernel parameter space, it travels there and CTA 0
// stores it into the device arena. A copy-engine operation between two kernels of the chain costs its own latency and the
// programmatic overlap of the kernel behind it, every frame of a host that rewrites its tables every frame. With an init
// pass the block needs a (one-CTA) kernel of its own at the head of the frame: init reads the tables first.
// Returns what the bookkeeping launch carries in its parameter space: the header alone, header + tables, or nothing.
std::pair<const void*, uint32_t> send_frame_block(hnb_ctx* c, std::vector<LaunchPlan>& plans) {
    std::pair<const void*, uint32_t> carried{c->header(), uint32_t(sizeof(hnb::FrameHeader))};
    if (c->dirty_tables || c->plan_dirty) {
        const uint32_t bytes = uint32_t(c->lay.off_prefix_sum);
        if (!c->param_upload || c->B == 0 || bytes > HNB_FRAME_BLOCK_MAX_BYTES) {
            flush_arena(c, true);
            c->frame_copies++;
            carried = {nullptr, 0};
        } else if (std::none_of(plans.begin(), plans.end(), [](const LaunchPlan& lp) { return lp.init_blocks != 0; })) {
            carried = {c->h_arena.get(), bytes};
        } else {
            CUDA_CHECK(hnb::launch_frame_block(c->d_arena.get(), c->h_arena.get(), bytes, c->stream));
            c->launches++;
            for (auto& lp : plans) lp.params.late_tables = 1u;
            carried = {nullptr, 0};
        }
        c->dirty_tables = false;
        c->plan_dirty = false;
    }
    c->frames++;
    return carried;
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
        if (const char* env = getenv("HNB_DEFER_AGES")) c->defer_ages = atoi(env) != 0;
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
        s.state.plan_fixed = s.sector_planes;  // sector-plane effects address the sector cut only
        // zero-filled (debug builds of the reference poison the particle buffer instead, effect_cache.rs:284-296)
        CUDA_CHECK(grow(s.d_block, size_t(capacity_rows) * stride, 0, c->stream));
        CUDA_CHECK(s.ping.alloc(capacity_rows));
        CUDA_CHECK(s.pong.alloc(capacity_rows));
        CUDA_CHECK(s.dead.alloc(capacity_rows));
        CUDA_CHECK(grow(s.alive_bits, size_t(capacity_rows) / 32 + 2, 0, c->stream));
        CUDA_CHECK(s.ident_claim.alloc(2));
        CUDA_CHECK(s.life_floor.alloc(size_t(capacity_rows) / 32 + 1));
        CUDA_CHECK(s.group_age.alloc(size_t(capacity_rows) / 32 + 2));  // the groups' words, then hnb_deferred_groups
        prepare_slab(c, s, hnb_rt::SlabAccess::RowReset, 0, capacity_rows);
        CUDA_CHECK(cudaMemsetAsync(hnb::hnb_deferred_groups(s.group_age.get(), capacity_rows), 0, sizeof(unsigned long long), c->stream));
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
        prepare_slab(c, s, hnb_rt::SlabAccess::RowReset, first, count);
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
        prepare_slab(c, s, hnb_rt::SlabAccess::AliveBitsWrite, first, rows);  // slots may become alive whose lifetimes no floor covers
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
    prepare_slab(c, s, upload ? hnb_rt::SlabAccess::RecordWrite : hnb_rt::SlabAccess::RecordRead, first, count);
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
        prepare_slab(c, s, hnb_rt::SlabAccess::ListWrite, first, count);
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
        prepare_slab(c, s, hnb_rt::SlabAccess::RecordRead, first, count);
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
        prepare_slab(c, s, hnb_rt::SlabAccess::RecordWrite, first, count);
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
        prepare_slab(c, s, hnb_rt::SlabAccess::ListWrite, first, count);
        CUDA_CHECK(hnb::launch_indirect_deinterleave((const uint32_t*)d_src, s.ping.get(), s.pong.get(), s.dead.get(), first, count, c->stream));
        c->launches += count ? 1 : 0;
    });
}
int32_t hnb_slab_device_view(hnb_ctx* c, hnb_slab h, hnb_slab_view* out) {
    return guarded([&] {
        Slab& s = get_slab(c, h);
        if (!out) fail(HNB_ERR_INVALID_ARG, "out is NULL");
        fix_default_plan(c, s);  // handed-out columns never move: an unbound slab keeps the default cut from now on
        prepare_slab(c, s, hnb_rt::SlabAccess::ViewOut);
        memset(out, 0, sizeof(*out));
        out->capacity_rows = s.capacity;
        out->particle_stride = s.stride;
        out->num_planes = (uint32_t)s.planes.size();
        for (size_t p = 0; p < s.planes.size(); ++p) {
            out->planes[p] = s.column(p);
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
        if (s.sector_planes) fail(HNB_ERR_LAYOUT, "hnb_slab_fill_c5 writes the default or a column plan; spawn through the init pass or use hnb_slab_upload_aos");
        prepare_slab(c, s, hnb_rt::SlabAccess::RecordWrite, first, count);
        CUDA_CHECK(hnb::launch_fill_c5(plane_set(s), s.ping.get(), s.pong.get(), s.ident_claim.get(), first, count, seed, lo, hi,
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
// `emit` NULL: a call that takes no event buffers, which refuses emitting effects. Otherwise the instance's event buffers
// (hnb_batch_launch.emit_events): the effect must emit, with one distinct buffer per channel and UINT32_MAX past them.
void check_instance_slice(hnb_ctx* c, const Slab& s, const Effect& fx, uint32_t metadata_row, uint32_t first, uint32_t rows,
                          const char* what, const hnb_event_buffer* emit = nullptr) {
    const std::string w = what;
    if (uint64_t(first) + rows > s.capacity) fail(HNB_ERR_INVALID_ARG, w + ": rows outside the slab");
    if (metadata_row >= c->d_metadata.size()) fail(HNB_ERR_INVALID_ARG, w + ": metadata row out of range");
    if (fx.particle_stride != s.stride) fail(HNB_ERR_INVALID_ARG, w + ": effect particle stride does not match the slab");
    if (((fx.flags & HNB_EFFECT_SECTOR_PLANES) != 0) != s.sector_planes)
        fail(HNB_ERR_INVALID_ARG, w + ": effect and slab disagree on HNB_EFFECT_SECTOR_PLANES / HNB_SLAB_SECTOR_PLANES");
    const bool emits = (fx.flags & HNB_EFFECT_EMIT_GPU_SPAWN_EVENTS) != 0;
    if (!emit) {
        if (emits)
            fail(HNB_ERR_INVALID_ARG, w + ": pending GPU spawn events name parent slots; an emitting effect cannot be " +
                                          (w == "hnb_slab_repack"       ? "repacked"
                                           : w == "hnb_instance_append" ? "appended to"
                                                                        : "snapshot or restored") +
                                          " without its event buffers");
        return;
    }
    if (!emits) fail(HNB_ERR_INVALID_ARG, w + ": the effect does not have HNB_EFFECT_EMIT_GPU_SPAWN_EVENTS");
    const uint32_t channels = fx.desc->d.num_event_bindings;
    if (channels > HNB_MAX_EVENT_BINDINGS) fail(HNB_ERR_INVALID_ARG, w + ": the effect has more event channels than emit_events holds");
    for (uint32_t b = 0; b < HNB_MAX_EVENT_BINDINGS; ++b) {
        if (b >= channels) {
            if (emit[b] != 0xFFFFFFFFu) fail(HNB_ERR_INVALID_ARG, w + ": an event buffer is given for a channel the effect does not have");
            continue;
        }
        if (emit[b] >= c->event_buffers.size()) fail(HNB_ERR_INVALID_ARG, w + ": a channel of the effect has no valid event buffer");
        for (uint32_t o = 0; o < b; ++o)
            if (emit[o] == emit[b]) fail(HNB_ERR_INVALID_ARG, w + ": the same event buffer is given for two channels");
    }
}

// The checked event buffers of an emitting instance and the context's child-info rows their counts live in.
hnb::EventChannels event_channels(hnb_ctx* c, const Effect& fx, const hnb_event_buffer* emit) {
    hnb::EventChannels ev{};
    ev.count = fx.desc->d.num_event_bindings;
    for (uint32_t b = 0; b < ev.count; ++b) {
        ev.buffer[b] = c->event_buffers[emit[b]].get();
        ev.capacity[b] = uint32_t(c->event_buffers[emit[b]].size());
    }
    ev.child_infos = c->d_child_infos.get();
    ev.num_child_infos = uint32_t(c->d_child_infos.size());
    return ev;
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

namespace {
// hnb_slab_repack and, with `emit`, hnb_slab_repack_events: the inverse permutation (for the events) and every column
// gather read the lists, so the list writer goes last.
int32_t slab_repack(hnb_ctx* c, hnb_slab h, hnb_effect e, uint32_t metadata_row, uint32_t first, uint32_t rows,
                    const hnb_event_buffer* emit, const char* what) {
    return guarded([&] {
        Slab& s = get_slab(c, h);
        const Effect& fx = get_effect(c, e);
        check_instance_slice(c, s, fx, metadata_row, first, rows, what, emit);
        if (rows == 0) return;
        fix_plan(c, s, fx.plan);
        CUDA_CHECK(cudaSetDevice(c->device));
        const hnb::RepackArgs a = repack_args(c, s, metadata_row, first, rows);
        prepare_slab(c, s, hnb_rt::SlabAccess::InstanceRewrite, first, rows);
        uint32_t widest = 0;
        for (const Plane& p : s.planes) widest = std::max(widest, p.width);
        void* scratch = nullptr;
        CUDA_CHECK(cudaMallocAsync(&scratch, size_t(rows) * (widest + (emit ? 4 : 0)), c->stream));
        uint32_t* inv = (uint32_t*)((char*)scratch + size_t(rows) * widest);
        cudaError_t err = cudaSuccess;
        if (emit) {
            err = hnb::launch_repack_inverse(a, inv, c->stream);
            c->launches++;
        }
        for (size_t p = 0; p < s.planes.size() && err == cudaSuccess; ++p) {
            const uint32_t width = s.planes[p].width;
            err = hnb::launch_repack_gather(a, s.column(p), scratch, width, c->stream);
            if (err == cudaSuccess)
                err = cudaMemcpyAsync(s.column(p) + size_t(first) * width, scratch, size_t(rows) * width, cudaMemcpyDeviceToDevice, c->stream);
            c->launches++;
        }
        if (emit && err == cudaSuccess) {
            err = hnb::launch_events_translate(a, inv, event_channels(c, fx, emit), 0, nullptr, c->stream);
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

// hnb_instance_snapshot (one launch: the kernel reads n, W and particle_counter on the device, so the host never waits for
// them) and, with `emit`, hnb_instance_snapshot_events (the records, then the inverse permutation in a stream-ordered
// scratch of rows words, then the header's event words and the events).
int32_t instance_snapshot(hnb_ctx* c, hnb_slab h, hnb_effect e, uint32_t metadata_row, uint32_t first, uint32_t rows,
                          const hnb_event_buffer* emit, void* d_dst, size_t dst_bytes, const char* what) {
    return guarded([&] {
        Slab& s = get_slab(c, h);
        const Effect& fx = get_effect(c, e);
        const std::string w = what;
        check_instance_slice(c, s, fx, metadata_row, first, rows, what, emit);
        if (!d_dst || ((uintptr_t)d_dst & 15u)) fail(HNB_ERR_INVALID_ARG, w + ": d_dst is NULL or not 16-byte aligned");
        hnb::EventChannels ev{};
        if (emit) {
            ev = event_channels(c, fx, emit);
            uint32_t capacity[HNB_MAX_EVENT_BINDINGS] = {};
            for (uint32_t b = 0; b < ev.count; ++b) capacity[b] = ev.capacity[b];
            if (dst_bytes < hnb_instance_snapshot_events_bytes(s.stride, rows, capacity))
                fail(HNB_ERR_INVALID_ARG, w + ": dst_bytes is below hnb_instance_snapshot_events_bytes(stride, rows, capacities)");
        } else if (dst_bytes < hnb_instance_snapshot_bytes(s.stride, rows)) {
            fail(HNB_ERR_INVALID_ARG, w + ": dst_bytes is below hnb_instance_snapshot_bytes(stride, rows)");
        }
        if (rows == 0) return;
        CUDA_CHECK(cudaSetDevice(c->device));
        prepare_slab(c, s, hnb_rt::SlabAccess::RecordRead, first, rows);
        CUDA_CHECK(hnb::launch_snapshot_gather(snapshot_args(c, s, metadata_row, first, rows), (uint32_t*)d_dst, c->stream,
                                               emit ? s.dead.get() : nullptr));
        c->launches++;
        if (!emit) return;
        const hnb::RepackArgs a = repack_args(c, s, metadata_row, first, rows);
        void* inv = nullptr;
        CUDA_CHECK(cudaMallocAsync(&inv, size_t(rows) * 4, c->stream));
        cudaError_t err = hnb::launch_repack_inverse(a, (uint32_t*)inv, c->stream);
        if (err == cudaSuccess) err = hnb::launch_events_translate(a, (const uint32_t*)inv, ev, s.stride / 4, (uint32_t*)d_dst, c->stream);
        c->launches += 2;
        const cudaError_t freed = cudaFreeAsync(inv, c->stream);
        CUDA_CHECK(err);
        CUDA_CHECK(freed);
    });
}

// hnb_instance_restore (two launches: the records and the metadata words, then hnb_slab_repack's list writer, which reads
// m back from alive_count) and, with `emit`, hnb_instance_restore_events (then one CTA per channel for the events).
int32_t instance_restore(hnb_ctx* c, hnb_slab h, hnb_effect e, uint32_t metadata_row, uint32_t first, uint32_t rows,
                         const hnb_event_buffer* emit, const void* d_src, size_t src_bytes, const char* what) {
    return guarded([&] {
        Slab& s = get_slab(c, h);
        const Effect& fx = get_effect(c, e);
        const std::string w = what;
        check_instance_slice(c, s, fx, metadata_row, first, rows, what, emit);
        if (!d_src || ((uintptr_t)d_src & 15u)) fail(HNB_ERR_INVALID_ARG, w + ": d_src is NULL or not 16-byte aligned");
        if (src_bytes < sizeof(hnb_instance_snapshot_header)) fail(HNB_ERR_INVALID_ARG, w + ": src_bytes is below the 64-byte header");
        if (rows == 0) return;
        CUDA_CHECK(cudaSetDevice(c->device));
        fix_plan(c, s, fx.plan);
        prepare_slab(c, s, hnb_rt::SlabAccess::InstanceRewrite, first, rows);
        hnb::SnapshotArgs a = snapshot_args(c, s, metadata_row, first, rows);
        a.src_bytes = src_bytes;
        const hnb::EventChannels ev = emit ? event_channels(c, fx, emit) : hnb::EventChannels{};
        CUDA_CHECK(hnb::launch_restore_scatter(a, (const uint32_t*)d_src, c->stream, emit ? &ev.count : nullptr));
        c->launches++;
        CUDA_CHECK(hnb::launch_repack_lists(repack_args(c, s, metadata_row, first, rows), c->stream));
        c->launches++;
        if (!emit) return;
        CUDA_CHECK(hnb::launch_restore_events(a, (const uint32_t*)d_src, ev, c->stream));
        c->launches++;
    });
}

// hnb_instance_append (two launches: the records, list entries, bits and group words, then the metadata words and the claim
// cut, which the first reads).
int32_t instance_append(hnb_ctx* c, hnb_slab h, hnb_effect e, uint32_t metadata_row, uint32_t first, uint32_t rows,
                        const void* d_src, size_t src_bytes) {
    return guarded([&] {
        Slab& s = get_slab(c, h);
        const Effect& fx = get_effect(c, e);
        const char* what = "hnb_instance_append";
        const std::string w = what;
        check_instance_slice(c, s, fx, metadata_row, first, rows, what);
        if (!d_src || ((uintptr_t)d_src & 15u)) fail(HNB_ERR_INVALID_ARG, w + ": d_src is NULL or not 16-byte aligned");
        if (src_bytes < sizeof(hnb_instance_snapshot_header)) fail(HNB_ERR_INVALID_ARG, w + ": src_bytes is below the 64-byte header");
        if (rows == 0) return;
        CUDA_CHECK(cudaSetDevice(c->device));
        fix_plan(c, s, fx.plan);
        prepare_slab(c, s, hnb_rt::SlabAccess::Append, first, rows);
        hnb::AppendArgs a{};
        a.s = snapshot_args(c, s, metadata_row, first, rows);
        a.s.src_bytes = src_bytes;
        a.ping = s.ping.get();
        a.pong = s.pong.get();
        a.dead = s.dead.get();
        a.alive_bits = (fx.flags & HNB_EFFECT_SLOT_ORDER) ? s.alive_bits.get() : nullptr;
        a.life_floor = s.life_floor.get();
        a.group_age = s.group_age.get();
        a.claim = s.ident_claim.get();
        uint32_t launches = 0;
        const cudaError_t err = hnb::launch_append(a, (const uint32_t*)d_src, c->stream, &launches);
        c->launches += launches;
        CUDA_CHECK(err);
    });
}
}  // namespace

int32_t hnb_slab_repack(hnb_ctx* c, hnb_slab h, hnb_effect e, uint32_t metadata_row, uint32_t first, uint32_t rows) {
    return slab_repack(c, h, e, metadata_row, first, rows, nullptr, "hnb_slab_repack");
}
int32_t hnb_slab_repack_events(hnb_ctx* c, hnb_slab h, hnb_effect e, uint32_t metadata_row, uint32_t first, uint32_t rows,
                               const hnb_event_buffer emit_events[HNB_MAX_EVENT_BINDINGS]) {
    if (!emit_events) return guarded([] { fail(HNB_ERR_INVALID_ARG, "hnb_slab_repack_events: emit_events is NULL"); });
    return slab_repack(c, h, e, metadata_row, first, rows, emit_events, "hnb_slab_repack_events");
}

static_assert(HNB_SNAPSHOT_MAGIC == HNB_SNAPSHOT_MAGIC_WORD && HNB_SNAPSHOT_VERSION == HNB_SNAPSHOT_VERSION_WORD &&
                  HNB_SNAPSHOT_EVENTS_VERSION == HNB_SNAPSHOT_EVENTS_VERSION_WORD &&
                  sizeof(hnb_instance_snapshot_header) == HNB_SNAPSHOT_HEADER_WORDS * 4,
              "snapshot header of include/hanabi_b200.h and of the kernels");

size_t hnb_instance_snapshot_bytes(uint32_t particle_stride, uint32_t rows) {
    return sizeof(hnb_instance_snapshot_header) + size_t(rows) * particle_stride;
}
size_t hnb_instance_snapshot_events_bytes(uint32_t particle_stride, uint32_t rows, const uint32_t event_capacity[HNB_MAX_EVENT_BINDINGS]) {
    size_t bytes = hnb_instance_snapshot_bytes(particle_stride, rows);
    for (int b = 0; event_capacity && b < HNB_MAX_EVENT_BINDINGS; ++b) bytes += size_t(event_capacity[b]) * 4;
    return bytes;
}

int32_t hnb_instance_snapshot(hnb_ctx* c, hnb_slab h, hnb_effect e, uint32_t metadata_row, uint32_t first, uint32_t rows,
                              void* d_dst, size_t dst_bytes) {
    return instance_snapshot(c, h, e, metadata_row, first, rows, nullptr, d_dst, dst_bytes, "hnb_instance_snapshot");
}
int32_t hnb_instance_snapshot_events(hnb_ctx* c, hnb_slab h, hnb_effect e, uint32_t metadata_row, uint32_t first, uint32_t rows,
                                     const hnb_event_buffer emit_events[HNB_MAX_EVENT_BINDINGS], void* d_dst, size_t dst_bytes) {
    if (!emit_events) return guarded([] { fail(HNB_ERR_INVALID_ARG, "hnb_instance_snapshot_events: emit_events is NULL"); });
    return instance_snapshot(c, h, e, metadata_row, first, rows, emit_events, d_dst, dst_bytes, "hnb_instance_snapshot_events");
}

int32_t hnb_instance_restore(hnb_ctx* c, hnb_slab h, hnb_effect e, uint32_t metadata_row, uint32_t first, uint32_t rows,
                             const void* d_src, size_t src_bytes) {
    return instance_restore(c, h, e, metadata_row, first, rows, nullptr, d_src, src_bytes, "hnb_instance_restore");
}
int32_t hnb_instance_restore_events(hnb_ctx* c, hnb_slab h, hnb_effect e, uint32_t metadata_row, uint32_t first, uint32_t rows,
                                    const hnb_event_buffer emit_events[HNB_MAX_EVENT_BINDINGS], const void* d_src, size_t src_bytes) {
    if (!emit_events) return guarded([] { fail(HNB_ERR_INVALID_ARG, "hnb_instance_restore_events: emit_events is NULL"); });
    return instance_restore(c, h, e, metadata_row, first, rows, emit_events, d_src, src_bytes, "hnb_instance_restore_events");
}
int32_t hnb_instance_append(hnb_ctx* c, hnb_slab h, hnb_effect e, uint32_t metadata_row, uint32_t first, uint32_t rows,
                            const void* d_src, size_t src_bytes) {
    return instance_append(c, h, e, metadata_row, first, rows, d_src, src_bytes);
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
        prepare_slab(c, s, hnb_rt::SlabAccess::RecordRead, first, count);
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
namespace {
void copy_source(const std::string& src, char* out, size_t cap, size_t* len) {
    if (len) *len = src.size();
    if (out && cap) {
        size_t n = std::min(cap - 1, src.size());
        memcpy(out, src.data(), n);
        out[n] = 0;
    }
}
}  // namespace

int32_t hnb_effect_generate_source(const hnb_effect_desc* desc, char* out, size_t cap, size_t* len) {
    return guarded([&] {
        if (!desc) fail(HNB_ERR_INVALID_ARG, "desc is NULL");
        copy_source(generate_effect_source(*desc), out, cap, len);
    });
}

int32_t hnb_effect_generate_source_for_plan(const hnb_effect_desc* desc, uint32_t n_planes, const uint32_t* offsets, const uint32_t* widths,
                                            char* out, size_t cap, size_t* len) {
    return guarded([&] {
        if (!desc || !offsets || !widths) fail(HNB_ERR_INVALID_ARG, "NULL argument");
        if (n_planes > HNB_RT_MAX_PLANES) fail(HNB_ERR_INVALID_ARG, "more than 16 columns");
        std::vector<Plane> plan;
        for (uint32_t p = 0; p < n_planes; ++p) plan.push_back({offsets[p], widths[p]});
        copy_source(generate_effect_source(*desc, &plan), out, cap, len);
    });
}

int32_t hnb_effect_column_plan(const hnb_effect_desc* desc, uint32_t* offsets, uint32_t* widths, uint32_t* n) {
    return guarded([&] {
        if (!desc || !n) fail(HNB_ERR_INVALID_ARG, "NULL argument");
        const std::vector<Plane> plan = column_plan(desc->particle_stride, desc->attrs, desc->attrs ? desc->n_attrs : 0, desc->flags);
        *n = (uint32_t)plan.size();
        for (size_t p = 0; p < plan.size(); ++p) {
            if (offsets) offsets[p] = plan[p].offset;
            if (widths) widths[p] = plan[p].width;
        }
    });
}

int32_t hnb_effect_column_words(const hnb_effect_desc* desc, uint32_t* words, uint32_t* n) {
    return guarded([&] {
        if (!desc || !n) fail(HNB_ERR_INVALID_ARG, "NULL argument");
        const std::vector<Plane> plan = column_plan(desc->particle_stride, desc->attrs, desc->attrs ? desc->n_attrs : 0, desc->flags);
        uint32_t k = 0;
        for (const Plane& p : plan)
            for (uint32_t l = 0; l < p.width / 4; ++l, ++k)
                if (words) words[k] = p.word[l];
        *n = k;
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
    std::vector<Plane> plan;
    std::shared_ptr<const OwnedDesc> desc;
};
static EffectBlueprint make_blueprint(const hnb_effect_desc& desc) {
    EffectBlueprint bp;
    bp.source = generate_effect_source(desc);
    bp.plan = column_plan(desc.particle_stride, desc.attrs, desc.n_attrs, desc.flags);
    bp.desc = std::make_shared<const OwnedDesc>(desc);
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
    set_update_smem(c, fx.km, fx.update_smem);
    fx.plan = bp.plan;
    fx.desc = bp.desc;
    fx.fast_math = bp.fast_math;
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
        // A new metadata row may end an instance without any writer of its rows: the slice's next owner would not walk every
        // row of a deferred group. So every age goes back to its column first (DESIGN.md §3).
        for (Slab& s : c->slabs)
            if (s.live) prepare_slab(c, s, hnb_rt::SlabAccess::MetadataWrite);
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
        // Every launch is checked before anything is written or enqueued: a bad frame is skipped as a whole.
        std::vector<LaunchPlan>& plans = c->frame_plans;  // reused from frame to frame: no allocation in steady state
        plans.clear();
        plans.reserve(n);
        for (uint32_t i = 0; i < n; ++i) plans.push_back(check_launch(c, batches[i]));
        check_coverage(c, plans);
        ensure_scratch(c);
        for (const auto& lp : plans) fix_launch_plans(c, lp);
        for (uint32_t i = 0; i < n; ++i) bind_launch(c, plans[i], batches[i], true);
        next_epoch(c);
        const auto [block, block_bytes] = send_frame_block(c, plans);
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
                if (lp.init_blocks) launch_kernel(c, lp.km->init, lp.init_blocks, lp.params, hnb_rt::kInitSmemBytes, fork.lane(k++));
            fork.join();
        }
        // passes "hanabi:indirect_dispatch" + "hanabi:update_prefix_sum" (mod.rs:7182-7275), fused
        {
            PassRange range("hanabi:indirect_dispatch");  // + "hanabi:update_prefix_sum"
            CUDA_CHECK(hnb::launch_bookkeeping(static_tables(c), c->header()->sim.num_effects, c->B, block, block_bytes, c->stream));
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
            const hnb_spawner& sp = c->h_at<hnb_spawner>(c->lay.off_spawners)[bi.spawner_base];  // row checked by check_coverage
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

static_assert(sizeof(hnb_instance_bounds) == 32, "hnb_instance_bounds is two 16-byte stores");

// The checks hnb_batch_bounds and hnb_batch_depth_order share, and where `position` sits in the slab's current columns.
// Everything is checked on the host before anything is enqueued; what the instances look like (counts, W, slab offsets,
// metadata rows) is read by the kernels from the device tables of the last simulated frame, clamped there.
struct BatchPosition {
    const Slab* slab;
    const Effect* effect;
    const hnb_batch_info* batch;  // the host's row: its prefix_sum_count sizes the call
    const hnb_attr_layout* position;
};
static BatchPosition check_batch_position(hnb_ctx* c, const hnb_batch_launch* b, const std::string& w) {
    if (!b) fail(HNB_ERR_INVALID_ARG, w + ": batch is NULL");
    const Slab& s = get_slab(c, b->slab);
    const Effect& fx = get_effect(c, b->effect);
    if (b->batch_info_index >= c->B) fail(HNB_ERR_INVALID_ARG, w + ": batch_info_index is not an uploaded batch row");
    const hnb_batch_info& bi = c->h_at<hnb_batch_info>(c->lay.off_batch_infos)[b->batch_info_index];
    if (uint64_t(bi.spawner_base) + bi.prefix_sum_count > c->E)
        fail(HNB_ERR_INVALID_ARG, w + ": the batch references instances outside the uploaded spawner table");
    if (fx.particle_stride != s.stride) fail(HNB_ERR_INVALID_ARG, w + ": effect particle stride does not match the slab");
    if (((fx.flags & HNB_EFFECT_SECTOR_PLANES) != 0) != s.sector_planes)
        fail(HNB_ERR_INVALID_ARG, w + ": effect and slab disagree on HNB_EFFECT_SECTOR_PLANES / HNB_SLAB_SECTOR_PLANES");
    const hnb_attr_layout* position = nullptr;
    for (const hnb_attr_layout& a : fx.desc->attrs)
        if (a.name && std::string(a.name) == "position") position = &a;
    if (!position || position->value_type != HNB_VEC3 || (position->offset & 3u) || uint64_t(position->offset) + 12 > s.stride)
        fail(HNB_ERR_INVALID_ARG, w + ": the effect has no `position` attribute of type HNB_VEC3 inside its record");
    return BatchPosition{&s, &fx, &bi, position};
}
// The device side of a checked batch with at least one instance. `fast`: position's three words share one 16-byte quad.
static hnb::BoundsArgs batch_position_args(hnb_ctx* c, const hnb_batch_launch* b, const BatchPosition& bp, bool* fast) {
    const Slab& s = *bp.slab;
    hnb::BoundsArgs a{};
    a.batch_info = c->d_at<hnb::BatchInfo>(c->lay.off_batch_infos) + b->batch_info_index;
    a.spawners = c->d_at<hnb::Spawner>(c->lay.off_spawners);
    a.metadata = c->d_metadata.get();
    a.num_spawners = c->E;
    a.num_metadata = uint32_t(c->d_metadata.size());
    a.ping = s.ping.get();
    a.pong = s.pong.get();
    a.claim = s.ident_claim.get();
    a.capacity_rows = s.capacity;
    a.max_instances = bp.batch->prefix_sum_count;
    // position in the slab's CURRENT columns: a plan may cut its three words apart
    const hnb::PlaneSet ps = plane_set(s);
    for (uint32_t k = 0; k < 3; ++k) {
        const uint32_t word = bp.position->offset / 4 + k, p = ps.word_to_plane[word];
        a.col[k] = static_cast<const uint32_t*>(ps.ptr[p]);
        a.col_words[k] = ps.words[p];
        a.col_lane[k] = hnb::hnb_word_lane(ps, word);
    }
    *fast = a.col[2] == a.col[0] && (a.col_lane[0] & 3u) == 0 && (a.col_words[0] & 3u) == 0 && a.col_lane[1] == a.col_lane[0] + 1 &&
            a.col_lane[2] == a.col_lane[0] + 2;
    return a;
}

int32_t hnb_batch_bounds(hnb_ctx* c, const hnb_batch_launch* b, hnb_instance_bounds* d_out, uint32_t out_rows) {
    return guarded([&] {
        const std::string w = "hnb_batch_bounds";
        const BatchPosition bp = check_batch_position(c, b, w);
        const hnb_batch_info& bi = *bp.batch;
        if (!d_out || ((uintptr_t)d_out & 15u)) fail(HNB_ERR_INVALID_ARG, w + ": d_out is NULL or not 16-byte aligned");
        if (out_rows < bi.prefix_sum_count) fail(HNB_ERR_INVALID_ARG, w + ": out_rows is below the batch's instance count");
        if (bi.prefix_sum_count == 0) return;
        if (c->d_metadata.size() == 0) fail(HNB_ERR_INVALID_ARG, w + ": no metadata row was inserted");
        CUDA_CHECK(cudaSetDevice(c->device));
        if (c->d_bounds_acc.size() < size_t(bi.prefix_sum_count) * 8)
            CUDA_CHECK(grow(c->d_bounds_acc, std::max<size_t>(bi.prefix_sum_count, c->d_metadata.size()) * 8, 0, c->stream));

        bool fast = false;
        hnb::BoundsArgs a = batch_position_args(c, b, bp, &fast);
        a.acc = c->d_bounds_acc.get();
        a.out = d_out;
        CUDA_CHECK(hnb::launch_batch_bounds(a, fast, uint32_t(c->sm_count), c->stream));
        c->launches += HNB_BATCH_BOUNDS_LAUNCHES;
    });
}

int32_t hnb_batch_depth_order(hnb_ctx* c, const hnb_batch_launch* b, const float* d_planes, uint32_t plane_rows, uint32_t* d_order,
                              uint32_t order_rows) {
    return guarded([&] {
        const std::string w = "hnb_batch_depth_order";
        // a ribbon effect is refused before anything else about it is checked
        if (b && (get_effect(c, b->effect).flags & HNB_EFFECT_RIBBONS))
            fail(HNB_ERR_INVALID_ARG, w + ": a ribbon effect is drawn in ribbon order, not in depth order");
        const BatchPosition bp = check_batch_position(c, b, w);
        const hnb_batch_info& bi = *bp.batch;
        if (!d_planes || ((uintptr_t)d_planes & 15u)) fail(HNB_ERR_INVALID_ARG, w + ": d_planes is NULL or not 16-byte aligned");
        if (plane_rows < bi.prefix_sum_count) fail(HNB_ERR_INVALID_ARG, w + ": plane_rows is below the batch's instance count");
        if (!d_order) fail(HNB_ERR_INVALID_ARG, w + ": d_order is NULL");
        if (order_rows < bp.slab->capacity) fail(HNB_ERR_INVALID_ARG, w + ": order_rows is below the slab's capacity");
        if (bi.prefix_sum_count == 0) return;
        if (c->d_metadata.size() == 0) fail(HNB_ERR_INVALID_ARG, w + ": no metadata row was inserted");
        CUDA_CHECK(cudaSetDevice(c->device));
        // scratch: four words per slab row, 256 per tile, 1024 + 8 per instance, the tile count
        const size_t rows = bp.slab->capacity, inst = bi.prefix_sum_count;
        const size_t max_tiles = hnb::depth_order_max_tiles(bp.slab->capacity, bi.prefix_sum_count);
        const size_t words = 4 * rows + 256 * max_tiles + 1032 * inst + 1;
        if (c->d_depth_scratch.size() < words) CUDA_CHECK(grow(c->d_depth_scratch, words, 0, c->stream));

        bool fast = false;
        hnb::DepthOrderArgs a{};
        a.src = batch_position_args(c, b, bp, &fast);
        a.planes = d_planes;
        a.order = d_order;
        uint32_t* p = c->d_depth_scratch.get();
        for (int k = 0; k < 2; ++k) {
            a.keys[k] = p + (2 * k) * rows;
            a.vals[k] = p + (2 * k + 1) * rows;
        }
        a.hist = p + 4 * rows;
        a.totals = a.hist + 256 * max_tiles;
        a.info = a.totals + 1024 * inst;
        a.total_tiles = a.info + 8 * inst;
        a.max_tiles = uint32_t(max_tiles);
        CUDA_CHECK(hnb::launch_batch_depth_order(a, fast, uint32_t(c->sm_count), c->stream));
        c->launches += HNB_BATCH_DEPTH_ORDER_LAUNCHES;
    });
}

// hnb_batch_cull (views = 1) and hnb_batch_cull_views: `views` views stacked view-major in d_frusta, d_visible and
// d_args, with one source. Refusals name the entry point `w`.
static void batch_cull(hnb_ctx* c, const hnb_batch_launch* b, const std::string& w, uint32_t views, const float* d_frusta,
                       uint32_t frustum_rows, const uint32_t* d_src, uint32_t src_rows, uint32_t* d_visible, uint32_t visible_rows,
                       hnb_draw_indexed_indirect_args* d_args, uint32_t args_rows) {
    // a ribbon effect is refused before anything else about it is checked
    if (b && (get_effect(c, b->effect).flags & HNB_EFFECT_RIBBONS))
        fail(HNB_ERR_INVALID_ARG, w + ": a ribbon effect cannot be culled per particle, its ribbons would be re-linked");
    if (views == 0 || views > HNB_CULL_MAX_VIEWS) fail(HNB_ERR_INVALID_ARG, w + ": views is 0 or above HNB_CULL_MAX_VIEWS");
    const BatchPosition bp = check_batch_position(c, b, w);
    const hnb_batch_info& bi = *bp.batch;
    const size_t rows = bp.slab->capacity, inst = bi.prefix_sum_count;
    if (!d_frusta || ((uintptr_t)d_frusta & 15u)) fail(HNB_ERR_INVALID_ARG, w + ": d_frusta is NULL or not 16-byte aligned");
    if (frustum_rows < inst) fail(HNB_ERR_INVALID_ARG, w + ": frustum_rows is below the batch's instance count");
    if (d_src && src_rows < rows) fail(HNB_ERR_INVALID_ARG, w + ": src_rows is below the slab's capacity");
    if (!d_visible) fail(HNB_ERR_INVALID_ARG, w + ": d_visible is NULL");
    if (visible_rows < rows) fail(HNB_ERR_INVALID_ARG, w + ": visible_rows is below the slab's capacity");
    // d_src against every view's entries
    if (d_src && (uintptr_t)d_src < (uintptr_t)(d_visible + size_t(views) * visible_rows) && (uintptr_t)d_visible < (uintptr_t)(d_src + src_rows))
        fail(HNB_ERR_INVALID_ARG, w + ": d_src and d_visible overlap");
    if (!d_args || ((uintptr_t)d_args & 3u)) fail(HNB_ERR_INVALID_ARG, w + ": d_args is NULL or not 4-byte aligned");
    if (args_rows < inst) fail(HNB_ERR_INVALID_ARG, w + ": args_rows is below the batch's instance count");
    if (inst == 0) return;
    if (c->d_metadata.size() == 0) fail(HNB_ERR_INVALID_ARG, w + ": no metadata row was inserted");
    if (c->d_draw_args.size() == 0) fail(HNB_ERR_INVALID_ARG, w + ": no draw-args row was inserted");
    CUDA_CHECK(cudaSetDevice(c->device));
    // scratch: per view a mask and a prefix word per tile; 8 words per instance, the tile count
    const size_t max_tiles = hnb::depth_order_max_tiles(bp.slab->capacity, bi.prefix_sum_count);
    const size_t words = views * (HNB_BATCH_CULL_MASK_WORDS + 1) * max_tiles + 8 * inst + 1;
    if (c->d_cull_scratch.size() < words) CUDA_CHECK(grow(c->d_cull_scratch, words, 0, c->stream));

    bool fast = false;
    hnb::CullViewsArgs v{};
    hnb::CullArgs& a = v.c;
    a.src = batch_position_args(c, b, bp, &fast);
    a.frusta = d_frusta;
    a.src_list = d_src;
    a.visible = d_visible;
    a.args = reinterpret_cast<uint32_t*>(d_args);
    a.draw_args = c->draw_args();
    a.num_draw_args = uint32_t(c->d_draw_args.size());
    a.mask = c->d_cull_scratch.get();
    a.prefix = a.mask + views * HNB_BATCH_CULL_MASK_WORDS * max_tiles;
    a.info = a.prefix + views * max_tiles;
    a.total_tiles = a.info + 8 * inst;
    a.max_tiles = uint32_t(max_tiles);
    v.views = views;
    v.frustum_rows = frustum_rows;
    v.visible_rows = visible_rows;
    v.args_rows = args_rows;
    // one view runs the single-view kernels
    if (views == 1) CUDA_CHECK(hnb::launch_batch_cull(a, fast, uint32_t(c->sm_count), c->stream));
    else CUDA_CHECK(hnb::launch_batch_cull_views(v, fast, uint32_t(c->sm_count), c->stream));
    c->launches += HNB_BATCH_CULL_LAUNCHES;
}

int32_t hnb_batch_cull(hnb_ctx* c, const hnb_batch_launch* b, const float* d_frusta, uint32_t frustum_rows, const uint32_t* d_src,
                       uint32_t src_rows, uint32_t* d_visible, uint32_t visible_rows, hnb_draw_indexed_indirect_args* d_args,
                       uint32_t args_rows) {
    return guarded([&] {
        batch_cull(c, b, "hnb_batch_cull", 1, d_frusta, frustum_rows, d_src, src_rows, d_visible, visible_rows, d_args, args_rows);
    });
}

int32_t hnb_batch_cull_views(hnb_ctx* c, const hnb_batch_launch* b, uint32_t views, const float* d_frusta, uint32_t frustum_rows,
                             const uint32_t* d_src, uint32_t src_rows, uint32_t* d_visible, uint32_t visible_rows,
                             hnb_draw_indexed_indirect_args* d_args, uint32_t args_rows) {
    return guarded([&] {
        batch_cull(c, b, "hnb_batch_cull_views", views, d_frusta, frustum_rows, d_src, src_rows, d_visible, visible_rows, d_args,
                   args_rows);
    });
}

int32_t hnb_pass_sort(hnb_ctx* c, const hnb_batch_launch* b) {
    return guarded([&] {
        if (!b) fail(HNB_ERR_INVALID_ARG, "batch is NULL");
        LaunchPlan lp = check_and_bind(c, *b, false);
        flush_arena(c, false);
        launch_ribbon_sort(c, lp);
    });
}

int32_t hnb_pass_init(hnb_ctx* c, const hnb_batch_launch* b) {
    return guarded([&] {
        if (!b) fail(HNB_ERR_INVALID_ARG, "batch is NULL");
        // The init kernel pops dead slots by rank from the counters as they stood at the START of the pass, and its
        // alive_count / particle_counter increments are applied by the indirect pass that follows (spawn_range[]): a
        // second stand-alone init of the same batch before that pass would pop the same slots and lose the first
        // launch's increments (the reference's atomics accumulate, vfx_init.wgsl:141-151). Refuse it.
        if (b->batch_info_index < c->init_pending.size() && c->init_pending[b->batch_info_index])
            fail(HNB_ERR_INVALID_ARG, "hnb_pass_init: this batch already has an init pass pending; run hnb_pass_indirect first");
        LaunchPlan lp = check_and_bind(c, *b, true);
        c->header()->num_batches = c->B;
        if (c->header()->epoch == 0) next_epoch(c);
        flush_arena(c, true);
        if (lp.init_blocks) {
            launch_kernel(c, lp.km->init, lp.init_blocks, lp.params, hnb_rt::kInitSmemBytes);
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
        LaunchPlan lp = check_and_bind(c, *b, false);
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
        *out = c->h_at<uint32_t>(c->lay.off_tile_size)[row];  // host copy of the word bind_launch passed to the batch's last launch
    });
}
int32_t hnb_slab_deferred_groups(hnb_ctx* c, hnb_slab h, uint64_t* out) {
    return guarded([&] {
        if (!out) fail(HNB_ERR_INVALID_ARG, "NULL argument");
        const Slab& s = get_slab(c, h);
        // a plain read of the count word after the stream's work: nothing is flushed, so the words stay as the updates left them
        read_back(c, out, hnb::hnb_deferred_groups(s.group_age.get(), s.capacity), sizeof(uint64_t));
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
int32_t hnb_ctx_plan_compiles(hnb_ctx* c, uint64_t* compiles) {
    return guarded([&] {
        if (!c || !compiles) fail(HNB_ERR_INVALID_ARG, "NULL argument");
        *compiles = c->plan_compiles;
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
