// tile_state_rule.h — when a batch slot's look-back tile states must be zeroed before an update launch.
//
// The update pass publishes one state word per tile and reads its predecessors' words back; a word counts as published
// when its epoch tag equals the current frame's. Default and relaxed order words carry the full 30-bit epoch (next_epoch
// zeroes every array when it wraps). Slot-order words carry only `epoch & 63`, so a word left in the array 64 frames (or
// any multiple) earlier looks current. That happens whenever a tile is not rewritten every frame: a batch slot that sits
// out, or one that is pointed at another instance with a different tile count. The host therefore remembers, per batch
// slot, the epoch of the first run since the array was last zeroed, and zeroes it again before a run 64 or more frames
// later: every word then left in the array was written at most 63 frames before the run, and none can carry its tag.
//
// Plain C++ without CUDA: context.cpp includes it, and the CPU tests compile it with g++ to run the same decision.
#pragma once

#include <stdint.h>

namespace hnb_rt {

constexpr uint32_t kSlotOrderEpochPeriod = 64;  // 6 bits of epoch in a slot-order state word (hnb_pack_state)

struct TileStateSlot {
    uint64_t sig = 0;          // what the array was last written for (0: default / relaxed order, or nothing yet)
    uint32_t first_epoch = 0;  // epoch of the first run since the array was last zeroed (0: no run yet)
};

// The epoch next_epoch() stores after `epoch`: 30 bits, 0 skipped. hnb_simulate and hnb_pass_update plan their batches
// before they advance the epoch, so this is the epoch of the run being planned.
inline uint32_t tile_state_run_epoch(uint32_t epoch) {
    const uint32_t e = (epoch + 1u) & 0x3fffffffu;
    return e ? e : 1u;
}

// Called for every planned run of a batch slot. `sig` describes what the run uses the slot for (nonzero for slot order,
// see bind_launch; 0 for the other orders) and `run_epoch` is the run's epoch. Returns true when the slot's array must be
// zeroed before the run, and updates `s`.
//  * A change of signature zeroes the array (another effect, slab, tile size or instance set).
//  * Slot order zeroes it when the run is 64 or more epochs after the first run since the last zeroing.
//  * A run epoch below the recorded one means the 30-bit epoch wrapped since, and next_epoch zeroed every array when it
//    did (before this run, if the wrap is this run's): the array holds nothing older than this run.
inline bool tile_state_needs_clear(TileStateSlot& s, uint64_t sig, uint32_t run_epoch) {
    if (sig != s.sig) {
        s.sig = sig;
        s.first_epoch = run_epoch;
        return true;
    }
    if (sig == 0) return false;
    if (s.first_epoch == 0 || run_epoch < s.first_epoch) {
        s.first_epoch = run_epoch;
        return false;
    }
    if (run_epoch - s.first_epoch < kSlotOrderEpochPeriod) return false;
    s.first_epoch = run_epoch;
    return true;
}

}  // namespace hnb_rt
