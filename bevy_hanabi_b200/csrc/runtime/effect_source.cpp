// effect_source.cpp — assembles the CUDA C translation unit of one effect: the analogue of the
// template substitution at the end of EffectShaderSources::generate (reference src/lib.rs:1026-1069 for
// init, :1283-1302 for update) plus ParticleLayout::generate_code (src/attributes.rs:1883-1913).
//
// TU = hnb_wgsl.cuh + hnb_tables.cuh + [generated types] + hnb_effect_ctx.cuh + [generated functions]
//      + hnb_particle_kernels.cuh, everything inside namespace hnb.
#include "effect_source.h"

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <sstream>
#include <stdexcept>

namespace hnb_rt {

extern const char* const kSrcWgsl;
extern const char* const kSrcTables;
extern const char* const kSrcEffectCtx;
extern const char* const kSrcParticleKernels;

ValueTypeInfo value_type_info(uint32_t vt) {
    switch (vt) {
        case HNB_BOOL: return {"bool", "bool", 1, 'b'};
        case HNB_FLOAT: return {"f32", "f32", 1, 'f'};
        case HNB_INT: return {"i32", "i32", 1, 'i'};
        case HNB_UINT: return {"u32", "u32", 1, 'u'};
        case HNB_BVEC2: return {"vec2<bool>", "bool", 2, 'b'};
        case HNB_BVEC3: return {"vec3<bool>", "bool", 3, 'b'};
        case HNB_BVEC4: return {"vec4<bool>", "bool", 4, 'b'};
        case HNB_VEC2: return {"vec2<f32>", "f32", 2, 'f'};
        case HNB_VEC3: return {"vec3<f32>", "f32", 3, 'f'};
        case HNB_VEC4: return {"vec4<f32>", "f32", 4, 'f'};
        case HNB_IVEC2: return {"vec2<i32>", "i32", 2, 'i'};
        case HNB_IVEC3: return {"vec3<i32>", "i32", 3, 'i'};
        case HNB_IVEC4: return {"vec4<i32>", "i32", 4, 'i'};
        case HNB_UVEC2: return {"vec2<u32>", "u32", 2, 'u'};
        case HNB_UVEC3: return {"vec3<u32>", "u32", 3, 'u'};
        case HNB_UVEC4: return {"vec4<u32>", "u32", 4, 'u'};
        default: throw std::invalid_argument("unsupported value type in particle layout");
    }
}

std::vector<Plane> cut_planes(uint32_t stride_bytes) {
    if (stride_bytes == 0 || (stride_bytes & 3u)) throw std::invalid_argument("particle stride must be a non-zero multiple of 4");
    std::vector<Plane> planes;
    uint32_t off = 0;
    while (off < stride_bytes) {
        uint32_t rem = stride_bytes - off;
        uint32_t w = rem >= 16 ? 16 : (rem >= 8 ? 8 : 4);
        planes.push_back({off, w});
        off += w;
    }
    if (planes.size() > HNB_RT_MAX_PLANES) throw std::invalid_argument("particle layout too large (more than 16 planes)");
    return planes;
}

// Physical columns of a slab. Default: one column per piece of cut_planes(). Sector planes (HNB_SLAB_SECTOR_PLANES): two
// consecutive 16-byte pieces share one 32-byte-wide column, so that a gathered record piece pair is one full DRAM sector.
std::vector<Plane> physical_planes(uint32_t stride_bytes, bool sector_planes) {
    std::vector<Plane> pieces = cut_planes(stride_bytes);
    if (!sector_planes) return pieces;
    std::vector<Plane> out;
    for (size_t p = 0; p < pieces.size();) {
        if (p + 1 < pieces.size() && pieces[p].width == 16 && pieces[p + 1].width == 16) {
            out.push_back({pieces[p].offset, 32});
            p += 2;
        } else {
            out.push_back(pieces[p]);
            p += 1;
        }
    }
    return out;
}

namespace {

const char* comp_name(int c) {
    static const char* n[] = {"x", "y", "z", "w"};
    return n[c];
}

// lvalue of word `word_in_plane` of plane p inside RawParticle
std::string raw_word(const Plane& pl, size_t p, uint32_t word_in_plane) {
    std::ostringstream s;
    s << "r.q" << p;
    if (pl.width > 4) s << "." << comp_name((int)word_in_plane);
    return s.str();
}

struct FieldRef {
    std::string expr;  // e.g. p.position.x
    char kind;         // f,i,u
};

// physical column and element index of piece p of row `row` ("row" is the generated variable name)
static std::string piece_address(const std::vector<Plane>& pieces, size_t p, bool sector) {
    if (!sector) return "s.planes[" + std::to_string(p) + "], row";
    size_t column = 0;
    for (size_t q = 0; q < pieces.size();) {
        const bool pair = q + 1 < pieces.size() && pieces[q].width == 16 && pieces[q + 1].width == 16;
        if (pair && (p == q || p == q + 1)) return "s.planes[" + std::to_string(column) + "], 2u * row + " + std::to_string(p - q) + "u";
        if (!pair && p == q) return "s.planes[" + std::to_string(column) + "], row";
        q += pair ? 2 : 1;
        ++column;
    }
    throw std::logic_error("piece_address");
}

void gen_layout_code(std::ostringstream& o, const char* prefix, const char* struct_name, const hnb_attr_layout* attrs,
                     uint32_t n_attrs, uint32_t stride, bool with_store, bool sector = false) {
    auto planes = cut_planes(stride);
    // map AoS word -> field component
    std::vector<FieldRef> words(stride / 4);
    std::vector<bool> skip_pack(stride / 4, false);
    o << "struct " << struct_name << " {\n";
    for (uint32_t i = 0; i < n_attrs; ++i) {
        const auto& a = attrs[i];
        auto ti = value_type_info(a.value_type);
        if (ti.kind == 'b') throw std::invalid_argument("bool attributes are not supported in particle layouts");
        if (a.offset & 3u || a.offset + 4u * ti.count > stride) throw std::invalid_argument("attribute offset out of the particle record");
        o << "    " << ti.cuda << " " << a.name << ";\n";
        const bool is_link = !strcmp(a.name, "prev") || !strcmp(a.name, "next");
        for (int c = 0; c < ti.count; ++c) {
            uint32_t w = a.offset / 4 + c;
            if (!words[w].expr.empty()) throw std::invalid_argument("overlapping attributes in particle layout");
            std::string e = std::string("p.") + a.name;
            if (ti.count > 1) e += std::string(".") + comp_name(c);
            words[w] = {e, ti.kind};
            skip_pack[w] = is_link;  // WRITEBACK_CODE excludes PREV/NEXT (lib.rs:1270-1281)
        }
    }
    o << "};\n";
    o << "struct " << prefix << "RawParticle {\n";
    for (size_t p = 0; p < planes.size(); ++p)
        o << "    " << (planes[p].width == 16 ? "float4" : planes[p].width == 8 ? "float2" : "f32") << " q" << p << ";\n";
    o << "};\n";
    const std::string raw_t = std::string(prefix) + "RawParticle";
    std::string fn_prefix = std::string("hnb_") + (strlen(prefix) ? "parent_" : "");
    // zero
    o << "HNB_DI void " << fn_prefix << "raw_zero(" << raw_t << "& r) {\n";
    for (size_t p = 0; p < planes.size(); ++p) {
        if (planes[p].width == 16) o << "    r.q" << p << " = make_float4(0.f, 0.f, 0.f, 0.f);\n";
        else if (planes[p].width == 8) o << "    r.q" << p << " = make_float2(0.f, 0.f);\n";
        else o << "    r.q" << p << " = 0.f;\n";
    }
    o << "}\n";
    // load
    o << "HNB_DI void " << fn_prefix << "load_raw(" << raw_t << "& r, const SlabView& s, u32 row) {\n";
    for (size_t p = 0; p < planes.size(); ++p) {
        const char* t = planes[p].width == 16 ? "float4" : planes[p].width == 8 ? "float2" : "f32";
        o << "    r.q" << p << " = HNB_LOAD_PLANE(" << t << ", " << piece_address(planes, p, sector) << ");\n";
    }
    o << "}\n";
    if (with_store) {
        o << "HNB_DI void " << fn_prefix << "store_raw(const " << raw_t << "& r, const SlabView& s, u32 row) {\n";
        for (size_t p = 0; p < planes.size(); ++p) {
            const char* t = planes[p].width == 16 ? "float4" : planes[p].width == 8 ? "float2" : "f32";
            o << "    HNB_STORE_PLANE(" << t << ", " << piece_address(planes, p, sector) << ", r.q" << p << ");\n";
        }
        o << "}\n";
    }
    // unpack
    o << "HNB_DI void " << fn_prefix << "unpack(const " << raw_t << "& r, " << struct_name << "& p) {\n";
    for (size_t p = 0; p < planes.size(); ++p) {
        for (uint32_t w = 0; w < planes[p].width / 4; ++w) {
            const auto& f = words[planes[p].offset / 4 + w];
            if (f.expr.empty()) continue;  // padding word
            std::string src = raw_word(planes[p], p, w);
            if (f.kind == 'f') o << "    " << f.expr << " = " << src << ";\n";
            else if (f.kind == 'u') o << "    " << f.expr << " = __float_as_uint(" << src << ");\n";
            else o << "    " << f.expr << " = __float_as_int(" << src << ");\n";
        }
    }
    o << "}\n";
    if (with_store) {
        o << "template <bool HNB_LINKS> HNB_DI void " << fn_prefix << "pack(const " << struct_name << "& p, " << raw_t << "& r) {\n";
        for (size_t p = 0; p < planes.size(); ++p) {
            for (uint32_t w = 0; w < planes[p].width / 4; ++w) {
                uint32_t aw = planes[p].offset / 4 + w;
                const auto& f = words[aw];
                if (f.expr.empty()) continue;
                std::string dst = raw_word(planes[p], p, w);
                if (skip_pack[aw]) {
                    o << "    if (HNB_LINKS) ";
                } else {
                    o << "    ";
                }
                if (f.kind == 'f') o << dst << " = " << f.expr << ";\n";
                else if (f.kind == 'u') o << dst << " = __uint_as_float(" << f.expr << ");\n";
                else o << dst << " = __int_as_float(" << f.expr << ");\n";
            }
        }
        o << "}\n";
    }
}

bool has_attr(const hnb_effect_desc& d, const char* name) {
    for (uint32_t i = 0; i < d.n_attrs; ++i)
        if (!strcmp(d.attrs[i].name, name)) return true;
    return false;
}

const char* nz(const char* s) { return s ? s : ""; }

}  // namespace

uint32_t rows_per_lane() {
    // rows of a tile handled by one lane (tile <= 32 * rows_per_lane rows); HNB_ROWS_PER_LANE env for tuning, 4-32.
    // Larger values are clamped to 32: slot order gives each lane one alive-bitmap word of the tile, so a tile may span at
    // most 32 words (32 x 32 rows).
    if (const char* e = getenv("HNB_ROWS_PER_LANE")) {
        int v = atoi(e);
        if (v >= 4) return (uint32_t)std::min(v, 32);
    }
    return 16;
}

uint32_t update_smem_bytes(const hnb_effect_desc& d) {
    // must mirror the carve-up at the top of hnb_update (hnb_particle_kernels.cuh)
    const uint32_t R = rows_per_lane(), warps = 8;
    uint32_t bytes = (2047 + 1) * 4;
    bytes += (R * 32 * 4 + 2 * R * 4) * 2 * warps;  // alive-list entries, survivor ballots, valid masks: streamed and parked tile
    bytes += 64 * warps;                            // PendingTile record of the parked tile
    if (d.properties_size) bytes += ((d.properties_size + 15) / 16 * 16) * warps;
    return bytes;
}

uint32_t choose_tile_k(const hnb_effect_desc& d) {
    // HNB_TILE_K env for tuning experiments (rows a lane keeps in flight per sub-tile; must divide HNB_ROWS_PER_LANE)
    if (const char* e = getenv("HNB_TILE_K")) {
        int v = atoi(e);
        if ((v == 1 || v == 2 || v == 4 || v == 8) && rows_per_lane() % uint32_t(v) == 0) return (uint32_t)v;
    }
    // rows per thread: keep (index + record) register footprint around 40 words
    uint32_t words = d.particle_stride / 4 + 1;
    uint32_t k = 40 / words;
    if (k >= 4) return 4;
    if (k >= 2) return 2;
    return 1;
}

std::string generate_effect_source(const hnb_effect_desc& d) {
    if (!d.attrs || d.n_attrs == 0) throw std::invalid_argument("effect has an empty particle layout");
    const auto planes = cut_planes(d.particle_stride);
    const bool read_parent = (d.flags & HNB_EFFECT_READ_PARENT_PARTICLE) != 0;
    const bool consume = (d.flags & HNB_EFFECT_CONSUME_GPU_SPAWN_EVENTS) != 0;
    const bool emit = (d.flags & HNB_EFFECT_EMIT_GPU_SPAWN_EVENTS) != 0;
    if (read_parent && (!d.parent_attrs || d.n_parent_attrs == 0)) throw std::invalid_argument("READ_PARENT_PARTICLE without parent layout");
    if ((d.flags & HNB_EFFECT_SLOT_ORDER) && (d.flags & (HNB_EFFECT_RELAXED_ORDER | HNB_EFFECT_ORDERED_EVENTS | HNB_EFFECT_SECTOR_PLANES)))
        throw std::invalid_argument("HNB_EFFECT_SLOT_ORDER cannot be combined with RELAXED_ORDER, ORDERED_EVENTS or SECTOR_PLANES");

    std::ostringstream o;
    o << "// ---- generated by hanabi_b200 for effect '" << nz(d.name) << "' ----\n";
    o << kSrcWgsl << "\n" << kSrcTables << "\n";
    o << "namespace hnb {\n";
    // Tuning hook for experiments: HNB_DEFINES="NAME=VALUE;NAME2=VALUE2" prepends #defines that the
    // kernel templates honour through #ifndef guards (tile shape, cache hints).
    if (const char* env = getenv("HNB_DEFINES")) {
        std::string e(env);
        size_t pos = 0;
        while (pos < e.size()) {
            size_t end = e.find(';', pos);
            if (end == std::string::npos) end = e.size();
            std::string item = e.substr(pos, end - pos);
            size_t eq = item.find('=');
            // The host sizes the dynamic shared memory and the grid from its own copy of these (update_smem_bytes,
            // plan_batch): overriding them here would make the kernel's carve-up disagree with the launch. Ignored, loudly.
            static const char* const kHostMirrored[] = {"HNB_SMEM_EFFECTS", "HNB_BLOCK", "HNB_WARPS", "HNB_ROWS_PER_LANE", "HNB_TILE_K",
                                                        "HNB_NUM_PLANES", "HNB_INIT_ITEMS", "HNB_MAX_CHUNKS", "HNB_INIT_SMEM_EFFECTS"};
            const std::string name = item.substr(0, eq);
            bool mirrored = false;
            for (const char* m : kHostMirrored) mirrored |= name == m;
            if (mirrored) {
                fprintf(stderr, "hanabi_b200: HNB_DEFINES entry '%s' ignored (the host mirrors this constant)\n", name.c_str());
            } else if (!item.empty()) {
                o << "#define " << name << " " << (eq == std::string::npos ? "1" : item.substr(eq + 1)) << "\n";
            }
            pos = end + 1;
        }
    }
    o << "#define HNB_NUM_PLANES " << planes.size() << "\n";
    o << "#define HNB_TILE_K " << choose_tile_k(d) << "\n";
    o << "#define HNB_ROWS_PER_LANE " << rows_per_lane() << "\n";
    o << "#define HNB_INIT_ITEMS " << kInitItems << "\n";
    o << "#define HNB_HAS_PROPERTIES " << (d.properties_size ? 1 : 0) << "\n";
    o << "#define HNB_CONSUME_EVENTS " << (consume ? 1 : 0) << "\n";
    o << "#define HNB_EMIT_EVENTS " << (emit ? 1 : 0) << "\n";
    o << "#define HNB_READ_PARENT " << (read_parent ? 1 : 0) << "\n";
    o << "#define HNB_RELAXED_ORDER " << ((d.flags & HNB_EFFECT_RELAXED_ORDER) ? 1 : 0) << "\n";
    o << "#define HNB_SLOT_ORDER " << ((d.flags & HNB_EFFECT_SLOT_ORDER) ? 1 : 0) << "\n";
    o << "#define HNB_ORDERED_EVENTS " << ((emit && (d.flags & HNB_EFFECT_ORDERED_EVENTS)) ? 1 : 0) << "\n";
    o << "#define HNB_FAST_MATH " << ((d.flags & HNB_EFFECT_FAST_MATH) ? 1 : 0) << "\n";  // compiled with contraction + approximate div/sqrt
    o << "#ifndef HNB_LOAD_PLANE\n"
         "#define HNB_LOAD_PLANE(T, base, row) (((const T*)(base))[row])\n"
         "#define HNB_STORE_PLANE(T, base, row, v) (((T*)(base))[row] = (v))\n"
         "#endif\n";
    // {{ATTRIBUTES}} / {{PROPERTIES}} / {{PARENT_ATTRIBUTES}}
    gen_layout_code(o, "", "Particle", d.attrs, d.n_attrs, d.particle_stride, true, (d.flags & HNB_EFFECT_SECTOR_PLANES) != 0);
    if (read_parent) gen_layout_code(o, "Parent", "ParentParticle", d.parent_attrs, d.n_parent_attrs, d.parent_particle_stride, false);
    if (d.properties_size) {
        o << "struct Properties {\n" << nz(d.properties_struct) << "\n};\n";
        o << "static_assert(sizeof(Properties) == " << d.properties_size << ", \"Properties layout mismatch\");\n";
    } else {
        o << "struct Properties { u32 _unused; };\n";
    }
    o << "}  // namespace hnb\n";
    o << kSrcEffectCtx << "\n";
    o << "namespace hnb {\n";
    // {{INIT_EXTRA}} / {{UPDATE_EXTRA}}
    o << "// ---- INIT_EXTRA ----\n" << nz(d.init_extra) << "\n";
    o << "// ---- UPDATE_EXTRA ----\n" << nz(d.update_extra) << "\n";
    // init body: {{INIT_CODE}}, PREV/NEXT reset (vfx_init.wgsl:175-181), {{SIMULATION_SPACE_TRANSFORM_PARTICLE}}
    o << "HNB_DI void hnb_init_body(Particle& particle, Ctx& hnb_ctx) {\n    HNB_CTX_PROLOGUE\n";
    o << nz(d.init_code) << "\n";
    if (has_attr(d, "prev")) o << "    particle.prev = 0xffffffffu;\n";
    if (has_attr(d, "next")) o << "    particle.next = 0xffffffffu;\n";
    if (!consume) o << nz(d.sim_space_code) << "\n";
    o << "}\n";
    // update body: {{AGE_CODE}} {{REAP_CODE}} {{UPDATE_CODE}}
    o << "HNB_DI bool hnb_update_body(Particle& particle, Ctx& hnb_ctx) {\n    HNB_CTX_PROLOGUE\n";
    o << nz(d.age_code) << "\n" << nz(d.reap_code) << "\n" << nz(d.update_code) << "\n";
    o << "    return is_alive;\n}\n";
    o << "}  // namespace hnb\n";
    o << kSrcParticleKernels << "\n";
    return o.str();
}

}  // namespace hnb_rt
