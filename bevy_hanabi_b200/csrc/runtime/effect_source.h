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

// One SoA plane: bytes [offset, offset+width) of the reference AoS record; width is 16, 8 or 4.
struct Plane {
    uint32_t offset;
    uint32_t width;
};
// Cut an AoS record of `stride_bytes` into planes: as many 16-byte planes as fit, then an 8- and/or
// 4-byte tail. Because the reference layout keeps vec3/vec4 16-byte aligned and vec2 8-byte aligned
// (attributes.rs:1516-1670) no attribute straddles two planes.
std::vector<Plane> cut_planes(uint32_t stride_bytes);
// Physical columns of a slab: the pieces themselves, or (sector planes) pairs of 16-byte pieces in 32-byte-wide columns.
std::vector<Plane> physical_planes(uint32_t stride_bytes, bool sector_planes);

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

// The complete translation unit (throws std::invalid_argument on a bad description).
std::string generate_effect_source(const hnb_effect_desc& d);

}  // namespace hnb_rt
