// effect_source.h — generation of the per-effect CUDA C translation unit.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "hanabi_b200.h"

#define HNB_RT_MAX_PLANES 16

namespace hnb_rt {

struct ValueTypeInfo {
    const char* cuda;  // type name in generated code, e.g. "vec3<f32>"
    const char* elem;  // element type name
    int count;         // number of 32-bit components
    char kind;         // 'f','i','u','b'
};
ValueTypeInfo value_type_info(uint32_t value_type);

// One SoA plane: `width` bytes (16, 8 or 4; 32 for a sector-plane column) per row, at capacity x `offset` bytes of the slab
// block, holding record words word[0 .. width/4) in lane order. Plane{offset, width} is the piece [offset, offset + width)
// of the reference AoS record; a word map (column_plan) may give a column words that are not consecutive.
struct Plane {
    uint32_t offset = 0, width = 0;
    uint8_t word[8] = {};
    Plane() = default;
    Plane(uint32_t off, uint32_t w) : offset(off), width(w) {
        for (uint32_t l = 0; l < w / 4 && l < 8; ++l) word[l] = uint8_t(off / 4 + l);
    }
    bool contiguous() const {
        for (uint32_t l = 0; l < width / 4; ++l)
            if (word[l] != offset / 4 + l) return false;
        return true;
    }
    bool operator==(const Plane& o) const {
        if (offset != o.offset || width != o.width) return false;
        for (uint32_t l = 0; l < width / 4; ++l)
            if (word[l] != o.word[l]) return false;
        return true;
    }
    bool operator!=(const Plane& o) const { return !(*this == o); }
};
// Cut an AoS record of `stride_bytes` into planes: as many 16-byte planes as fit, then an 8- and/or
// 4-byte tail. Because the reference layout keeps vec3/vec4 16-byte aligned and vec2 8-byte aligned
// (attributes.rs:1516-1670) no attribute straddles two planes.
std::vector<Plane> cut_planes(uint32_t stride_bytes);
// Physical columns of a slab: the pieces themselves, or (sector planes) pairs of 16-byte pieces in 32-byte-wide columns.
std::vector<Plane> physical_planes(uint32_t stride_bytes, bool sector_planes);
// The effect's column plan (hnb_effect_column_plan): the default cut unless some attribute is HNB_ATTR_UPDATE_READ_ONLY;
// then runs of written / unwritten words get columns of their own, so the update stores only columns it writes. An effect
// that keeps lifetime floors gets a word map instead (DESIGN.md §4.1): the age and the lifetime in f32 columns of their own,
// the other words packed, unless that takes more columns than the runs do.
std::vector<Plane> column_plan(uint32_t stride_bytes, const hnb_attr_layout* attrs, uint32_t n_attrs, uint32_t effect_flags);
bool is_default_cut(const std::vector<Plane>& plan, uint32_t stride_bytes);
// Throws std::invalid_argument unless `plan` is 4/8/16-byte columns laid out back to back in the slab block, each aligned to
// its width, whose words are every record word once.
void check_plan(const std::vector<Plane>& plan, uint32_t stride_bytes);

// Update tiles are walked by one warp each: tile_rows = 32 lanes * k rows per lane * chunks. k is
// chosen from the record size (register footprint) at compile time, the chunk count per launch.
// logical init threads (vfx_init.wgsl invocations) per CUDA thread of hnb_init == HNB_INIT_ITEMS of the generated kernels
constexpr uint32_t kInitItems = 4;
constexpr uint32_t kInitSmemBytes = 1024 * 4;  // HNB_INIT_SMEM_EFFECTS spawn-prefix entries staged by hnb_init
uint32_t rows_per_lane();  // == HNB_ROWS_PER_LANE of the generated kernels: tile_rows <= 32 * rows_per_lane()
uint32_t choose_tile_k(const hnb_effect_desc& d);
// Dynamic shared memory of hnb_update for this effect (tile-prefix table + per-warp double-buffered stash +
// parked-tile record + Properties staging).
uint32_t update_smem_bytes(const hnb_effect_desc& d);

// The complete translation unit (throws std::invalid_argument on a bad description), for the effect's own column plan or
// for `plan` (a slab's plan other than the effect's), reading a parent slab in the default cut or in `parent_plan`.
std::string generate_effect_source(const hnb_effect_desc& d, const std::vector<Plane>* plan = nullptr,
                                   const std::vector<Plane>* parent_plan = nullptr);

}  // namespace hnb_rt
