// slab_access_rule.h — what each access to a slab first does to the state derived from its records and lists.
//
// A slab carries, beside its records and index columns:
//  * Identity claims (DESIGN.md §3): one word per index column, `{base, len}` with `col[base + i] == i`. A writer of the index
//    columns that does not keep them true drops both.
//  * Lifetime floors: one f32 per 32 rows, HNB_LIFE_FLOOR_NONE (all bits set) until an update of an effect with floors
//    stores one. Invariant: a floor is at most the lifetime of every particle of its group.
//  * Common ages: one word per 32 rows, (epoch << 32) | the age bits of every row of the group, or all bits set. Invariant:
//    the update that stored the word left those bits in the age column of all 32 rows.
//  * Deferred common ages: an update may leave a word deferred (BatchParams::defer_ages). Its group's age is then in the
//    word, not in record word `age_word` of the rows. Invariant: every row of a deferred group is alive, none is on the
//    dead stack, and the next update of the instance walks all 32 rows, so that update is the only one to advance them.
//  * The column plan: until an effect is bound, the slab is in the default cut. The first bind fixes the plan (fix_plan)
//    and moves the records written before (`written`) to the effect's columns.
//
// Every access other than the update pass keeps these true in stream order, before any later update:
//  * a reader of records first writes deferred ages back to the rows it reads (flush; the words stay known);
//  * a writer of records first writes them back and sets the floors and words of every 32-row group it touches to the
//    sentinel (clear: by the flush on a slab that may defer, by two memsets on one that never did);
//  * a writer of alive lists or dead stacks at positions [first, first + count): its entries name rows anywhere in an
//    instance's slice, not the rows at those positions. A row of a deferred group that such a write moves to the dead
//    stack breaks the deferral invariant, and no later update would walk all 32 rows of it. So a slab that may hold
//    deferred words is cleared whole.
// `floors_off` / `ages_off` are permanent: once records may be written that no writer here sees (a view), or a module
// that neither keeps nor clears the words ran (it may write lifetimes or ages), no update gets them again. A slab stops
// deferring (`defers`) only when the whole slab is cleared, and starts only with a deferring update launch.
//
// Plain C++ without CUDA: context.cpp includes it (prepare_slab runs the work), and the CPU tests compile it with g++.
#pragma once

#include <stdint.h>

namespace hnb_rt {

struct SlabState {
    bool plan_fixed = false;  // the column plan is fixed (fix_plan); sector-plane slabs are created fixed
    bool written = false;     // records were written in the default cut before the plan was fixed
    bool floors_off = false;  // no update gets the lifetime floors any more
    bool ages_off = false;    // no update gets the common ages any more
    bool defers = false;      // an update may have left words deferred since the last whole-slab clear
    uint32_t age_word = 0;    // with `defers`: the record word the deferred ages belong in
};

// What a module keeps of the group words (read from its generated source).
struct ModuleWords {
    bool life_floor = false;  // HNB_LIFE_FLOOR: keeps the slab's lifetime floors (and clears them on init)
    bool group_age = false;   // HNB_GROUP_AGE: keeps the slab's common ages too
    uint32_t age_word = 0;    // with group_age: the record word of the age (HNB_GROUP_AGE_WORD)
};

// One kind per writer / reader of the DESIGN.md §3 tables. The rows [first, first + count) are the call's.
enum class SlabAccess : int {
    RecordRead,      // download / export AoS, snapshot, checksum: flush the rows' groups
    RecordWrite,     // fill, upload / import AoS: clear the rows' groups; before the plan is fixed, the records move with it
    RowReset,        // slab create (all rows), reset_rows: identity lists over the rows, no claims, the rows' groups cleared
    ListWrite,       // upload / import indirect: no claims; the list rule
    AliveBitsWrite,  // rebuild_alive_bits: the list rule (slots it marks alive may lie in any group); the claims stay
    InstanceRewrite, // repack, restore (called after fix_plan): clear the slice's groups; the kernels set the claims
    Append,          // instance_append: nothing first (see slab_access)
    Invalidate,      // 30-bit epoch wrap, plan migration (before the records move): clear the whole slab
    MetadataWrite,   // metadata_insert: clear the whole slab when it may defer
    ViewOut,         // device_view (called after the plan is pinned): clear the whole slab when it may defer; floors off
    Bind,            // a launch binds module `m` to the slab
    DeferringUpdate, // an update launch of module `m` that may leave words deferred (keeps_group_ages)
    ListSort,        // ribbon sort: no claims (it permutes the alive list), then flush the whole slab (its key is the age)
};

// The work to enqueue before the access, in this order: the claims, then the group words of rows [first, first + count).
struct SlabWork {
    bool drop_claims = false;  // zero both identity claims
    bool flush = false;        // write deferred ages back (k_flush_group_ages); the sentinel too when `clear`
    bool clear = false;        // set every floor and word of the groups to the sentinel (memsets when not `flush`)
    uint32_t first = 0, count = 0;
};

// Whether updates on the slab get the common ages (and so may defer them).
inline bool keeps_group_ages(const SlabState& s) { return !s.floors_off && !s.ages_off; }

// Returns what `a` on rows [first, first + count) of a slab of `capacity` rows must enqueue first, and updates `s`.
// Where the code does more or less than the tables ask, it is noted here and kept:
//  * RowReset and RecordWrite (the fill writes identity lists too) take the range rule: the entries they write name the
//    rows at their own positions; rows that the entries they overwrite named elsewhere are not flushed.
//  * AliveBitsWrite writes no index column, yet takes the list rule (without dropping the claims).
//  * MetadataWrite and ViewOut enqueue nothing on a slab that never deferred, where Invalidate still clears.
//  * Append clears nothing: the written slots come from the dead stack, so under the deferral invariant none lies in a
//    deferred group, and its kernel sets the sentinel on the group of each slot it writes, as init does (DESIGN.md §4.12).
//    It is called after fix_plan, as InstanceRewrite is, so neither needs `written`.
inline SlabWork slab_access(SlabState& s, SlabAccess a, uint32_t first, uint32_t count, uint32_t capacity,
                            const ModuleWords& m = {}) {
    SlabWork w;
    bool clear = false, read = false, whole = false;
    switch (a) {
    case SlabAccess::RecordRead: read = true; break;
    case SlabAccess::RecordWrite: s.written = true; clear = true; break;
    case SlabAccess::RowReset: w.drop_claims = true; clear = true; break;
    case SlabAccess::ListWrite: w.drop_claims = true; clear = true; whole = s.defers && count != 0; break;
    case SlabAccess::AliveBitsWrite: clear = true; whole = s.defers && count != 0; break;
    case SlabAccess::InstanceRewrite: clear = true; break;
    case SlabAccess::Append: break;
    case SlabAccess::Invalidate: clear = whole = true; break;
    case SlabAccess::MetadataWrite: clear = whole = s.defers; break;
    case SlabAccess::ViewOut:
        s.floors_off = true;  // records written through the view would not clear the floors
        clear = whole = s.defers;
        break;
    case SlabAccess::Bind:
        // A module that keeps no floors (no common ages) may write lifetimes (ages) without keeping the words true; a module
        // that keeps the age in another record word would read the deferred words wrongly. Relaxed-order and slot-order
        // modules keep no floors.
        if (!m.life_floor) s.floors_off = true;
        if (!m.group_age) s.ages_off = true;
        clear = whole = s.defers && (!keeps_group_ages(s) || m.age_word != s.age_word);
        break;
    case SlabAccess::DeferringUpdate:
        s.defers = true;
        s.age_word = m.age_word;
        break;
    case SlabAccess::ListSort: w.drop_claims = true; read = whole = true; break;
    }
    if (whole) first = 0, count = capacity;
    if (count == 0) return w;
    w.flush = s.defers && (clear || read);
    w.clear = clear;
    if (w.flush || w.clear) w.first = first, w.count = count;
    if (w.flush && w.clear && first == 0 && count == capacity) s.defers = false;  // no word is deferred any more
    return w;
}

}  // namespace hnb_rt
