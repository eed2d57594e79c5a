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

// Per AoS word: does some attribute the update may write cover it (attributes without HNB_ATTR_UPDATE_READ_ONLY)?
std::vector<bool> written_words(uint32_t stride, const hnb_attr_layout* attrs, uint32_t n_attrs) {
    std::vector<bool> written(stride / 4, false);
    for (uint32_t i = 0; i < n_attrs; ++i) {
        const auto ti = value_type_info(attrs[i].value_type);
        if (attrs[i].offset & 3u || attrs[i].offset + 4u * ti.count > stride) throw std::invalid_argument("attribute offset out of the particle record");
        if (attrs[i].flags & HNB_ATTR_UPDATE_READ_ONLY) continue;
        for (int c = 0; c < ti.count; ++c) written[attrs[i].offset / 4 + c] = true;
    }
    return written;
}

bool any_read_only(const hnb_attr_layout* attrs, uint32_t n_attrs) {
    for (uint32_t i = 0; i < n_attrs; ++i)
        if (attrs[i].flags & HNB_ATTR_UPDATE_READ_ONLY) return true;
    return false;
}

const hnb_attr_layout* find_attr(const hnb_attr_layout* attrs, uint32_t n_attrs, const char* name) {
    for (uint32_t i = 0; i < n_attrs; ++i)
        if (!strcmp(attrs[i].name, name)) return &attrs[i];
    return nullptr;
}

// Lifetime floors (DESIGN.md §3) need an f32 lifetime flagged HNB_ATTR_REAP_ONLY and read-only (so the column is never
// stored and only the standard age / reap code compares it), an f32 age, and the ordered pass (the floor is kept per 32
// rows of an identity-claimed tile). Slot order keeps none: there inits clear the floors of many groups every frame, and
// the lifetime loads those groups then need, issued behind the age, cost more than the floors save. The lifetime also
// needs a 4-byte column of its own in the slab's plan (life_floor_plane).
bool keeps_floors(const hnb_attr_layout* attrs, uint32_t n_attrs, uint32_t effect_flags) {
    if (effect_flags & (HNB_EFFECT_SECTOR_PLANES | HNB_EFFECT_RELAXED_ORDER | HNB_EFFECT_SLOT_ORDER)) return false;
    const hnb_attr_layout* life = find_attr(attrs, n_attrs, "lifetime");
    const hnb_attr_layout* age = find_attr(attrs, n_attrs, "age");
    const uint32_t need = HNB_ATTR_UPDATE_READ_ONLY | HNB_ATTR_REAP_ONLY;
    return life && age && life->value_type == HNB_FLOAT && age->value_type == HNB_FLOAT && (life->flags & need) == need;
}

// The word map of an effect with floors: the age and the lifetime in f32 columns of their own (the update may then skip
// either load), the other written words packed in record order into 16-, 8- and 4-byte columns, then the other unwritten
// words the same way. Columns are laid out widest first, so each sits at a multiple of its width in the slab block.
std::vector<Plane> word_map_plan(uint32_t stride, const hnb_attr_layout* attrs, uint32_t n_attrs, const std::vector<bool>& written) {
    const uint32_t age = find_attr(attrs, n_attrs, "age")->offset / 4, life = find_attr(attrs, n_attrs, "lifetime")->offset / 4;
    std::vector<Plane> cols;
    auto pack = [&](const std::vector<uint32_t>& words) {
        for (size_t i = 0; i < words.size();) {
            const size_t left = words.size() - i, n = left >= 4 ? 4 : left >= 2 ? 2 : 1;
            Plane p;
            p.width = uint32_t(4 * n);
            for (size_t l = 0; l < n; ++l) p.word[l] = uint8_t(words[i + l]);
            cols.push_back(p);
            i += n;
        }
    };
    std::vector<uint32_t> w_words, r_words;
    for (uint32_t w = 0; w < stride / 4; ++w)
        if (w != age && w != life) (written[w] ? w_words : r_words).push_back(w);
    pack(w_words);
    pack({age});
    pack({life});
    pack(r_words);
    std::stable_sort(cols.begin(), cols.end(), [](const Plane& a, const Plane& b) { return a.width > b.width; });
    uint32_t off = 0;
    for (Plane& p : cols) {
        p.offset = off;
        off += p.width;
    }
    return cols;
}

// Runs of written / unwritten words, each cut into aligned columns.
std::vector<Plane> column_plan_runs(uint32_t stride, const std::vector<bool>& written) {
    std::vector<Plane> out;
    for (uint32_t w = 0; w < stride / 4;) {
        uint32_t end = w;
        while (end < stride / 4 && written[end] == written[w]) ++end;
        // a column of width W starts at a multiple of W: a slab block carves it at capacity * offset bytes, aligned for
        // W-byte loads whatever the capacity
        for (uint32_t off = 4 * w; off < 4 * end;) {
            uint32_t width = 16;
            while (width > 4 && (off % width || off + width > 4 * end)) width /= 2;
            out.push_back({off, width});
            off += width;
        }
        w = end;
    }
    return out;
}

}  // namespace

std::vector<Plane> column_plan(uint32_t stride, const hnb_attr_layout* attrs, uint32_t n_attrs, uint32_t effect_flags) {
    if (effect_flags & HNB_EFFECT_SECTOR_PLANES) return physical_planes(stride, true);
    std::vector<Plane> cut = cut_planes(stride);
    if ((effect_flags & HNB_EFFECT_EMIT_GPU_SPAWN_EVENTS) || !any_read_only(attrs, n_attrs)) return cut;
    const std::vector<bool> written = written_words(stride, attrs, n_attrs);
    std::vector<Plane> out = column_plan_runs(stride, written);
    if (out.size() > HNB_RT_MAX_PLANES) return cut;
    // An effect whose lifetime the runs already give a 4-byte column (so that it keeps floors) gets the word map, unless that
    // takes more columns: a gathered record would then touch more sectors.
    if (!keeps_floors(attrs, n_attrs, effect_flags)) return out;
    const uint32_t life = find_attr(attrs, n_attrs, "lifetime")->offset;
    if (std::none_of(out.begin(), out.end(), [&](const Plane& p) { return p.offset == life && p.width == 4; })) return out;
    std::vector<Plane> map = word_map_plan(stride, attrs, n_attrs, written);
    return map.size() <= out.size() ? map : out;
}

bool is_default_cut(const std::vector<Plane>& plan, uint32_t stride) { return plan == cut_planes(stride); }

namespace {

const char* comp_name(int c) {
    static const char* n[] = {"x", "y", "z", "w"};
    return n[c];
}

// A plan with a column whose words are not consecutive: its RawParticle holds the record words in record order (w0, w1,
// ...), so that it is the AoS record, and each column load or store moves its words to or from their places.
bool is_word_map(const std::vector<Plane>& planes) {
    return std::any_of(planes.begin(), planes.end(), [](const Plane& p) { return !p.contiguous(); });
}

// lvalue of word `word_in_plane` of plane p inside RawParticle
std::string raw_word(const Plane& pl, size_t p, uint32_t word_in_plane, bool mapped = false) {
    std::ostringstream s;
    if (mapped) {
        s << "r.w" << unsigned(pl.word[word_in_plane]);
        return s.str();
    }
    s << "r.q" << p;
    if (pl.width > 4) s << "." << comp_name((int)word_in_plane);
    return s.str();
}

const char* plane_type(const Plane& pl) { return pl.width == 16 ? "float4" : pl.width == 8 ? "float2" : "f32"; }

// Statements loading column p of row `row` into RawParticle r, of a word map (the other plans load r.qP directly).
std::string mapped_load(const Plane& pl, size_t p, const std::string& address) {
    std::ostringstream s;
    if (pl.width == 4) {
        s << "    " << raw_word(pl, p, 0, true) << " = HNB_LOAD_PLANE(f32, " << address << ");\n";
        return s.str();
    }
    s << "    { const " << plane_type(pl) << " v = HNB_LOAD_PLANE(" << plane_type(pl) << ", " << address << ");";
    for (uint32_t l = 0; l < pl.width / 4; ++l) s << " " << raw_word(pl, p, l, true) << " = v." << comp_name(int(l)) << ";";
    s << " }\n";
    return s.str();
}

// The value of column p a store of a word map writes.
std::string mapped_value(const Plane& pl, size_t p) {
    if (pl.width == 4) return raw_word(pl, p, 0, true);
    std::string s = std::string("make_") + plane_type(pl) + "(";
    for (uint32_t l = 0; l < pl.width / 4; ++l) s += (l ? ", " : "") + raw_word(pl, p, l, true);
    return s + ")";
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

// `planes`: the record pieces the generated code addresses (the column plan; with sector planes the default cut, whose
// 16-byte pieces pair up into 32-byte columns).
void gen_layout_code(std::ostringstream& o, const char* prefix, const char* struct_name, const hnb_attr_layout* attrs,
                     uint32_t n_attrs, uint32_t stride, const std::vector<Plane>& planes, bool with_store, bool sector = false) {
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
    const bool mapped = is_word_map(planes);
    o << "struct " << prefix << "RawParticle {\n";
    if (mapped) {
        for (uint32_t w = 0; w < stride / 4; ++w) o << "    f32 w" << w << ";\n";
    } else {
        for (size_t p = 0; p < planes.size(); ++p)
            o << "    " << (planes[p].width == 16 ? "float4" : planes[p].width == 8 ? "float2" : "f32") << " q" << p << ";\n";
    }
    o << "};\n";
    const std::string raw_t = std::string(prefix) + "RawParticle";
    std::string fn_prefix = std::string("hnb_") + (strlen(prefix) ? "parent_" : "");
    // zero
    o << "HNB_DI void " << fn_prefix << "raw_zero(" << raw_t << "& r) {\n";
    for (size_t p = 0; p < planes.size(); ++p) {
        if (mapped) {
            for (uint32_t l = 0; l < planes[p].width / 4; ++l) o << "    " << raw_word(planes[p], p, l, true) << " = 0.f;\n";
        } else if (planes[p].width == 16) o << "    r.q" << p << " = make_float4(0.f, 0.f, 0.f, 0.f);\n";
        else if (planes[p].width == 8) o << "    r.q" << p << " = make_float2(0.f, 0.f);\n";
        else o << "    r.q" << p << " = 0.f;\n";
    }
    o << "}\n";
    // load
    o << "HNB_DI void " << fn_prefix << "load_raw(" << raw_t << "& r, const SlabView& s, u32 row) {\n";
    for (size_t p = 0; p < planes.size(); ++p) {
        const char* t = planes[p].width == 16 ? "float4" : planes[p].width == 8 ? "float2" : "f32";
        if (mapped) o << mapped_load(planes[p], p, piece_address(planes, p, sector));
        else o << "    r.q" << p << " = HNB_LOAD_PLANE(" << t << ", " << piece_address(planes, p, sector) << ");\n";
    }
    o << "}\n";
    if (with_store) {
        const auto value = [&](size_t p) { return mapped ? mapped_value(planes[p], p) : "r.q" + std::to_string(p); };
        o << "HNB_DI void " << fn_prefix << "store_raw(const " << raw_t << "& r, const SlabView& s, u32 row) {\n";
        for (size_t p = 0; p < planes.size(); ++p) {
            const char* t = planes[p].width == 16 ? "float4" : planes[p].width == 8 ? "float2" : "f32";
            o << "    HNB_STORE_PLANE(" << t << ", " << piece_address(planes, p, sector) << ", " << value(p) << ");\n";
        }
        o << "}\n";
        // The update's store: the pieces holding a word the update may write. With no read-only attribute, every piece
        // (the same stores as store_raw).
        const bool all = !any_read_only(attrs, n_attrs);
        const std::vector<bool> written = written_words(stride, attrs, n_attrs);
        o << "HNB_DI void " << fn_prefix << "store_written(const " << raw_t << "& r, const SlabView& s, u32 row) {\n";
        for (size_t p = 0; p < planes.size(); ++p) {
            bool store = all;
            for (uint32_t w = 0; w < planes[p].width / 4; ++w) store = store || written[planes[p].word[w]];
            if (!store) continue;
            const char* t = planes[p].width == 16 ? "float4" : planes[p].width == 8 ? "float2" : "f32";
            o << "    HNB_STORE_PLANE(" << t << ", " << piece_address(planes, p, sector) << ", " << value(p) << ");\n";
        }
        o << "}\n";
    }
    // unpack
    o << "HNB_DI void " << fn_prefix << "unpack(const " << raw_t << "& r, " << struct_name << "& p) {\n";
    for (size_t p = 0; p < planes.size(); ++p) {
        for (uint32_t w = 0; w < planes[p].width / 4; ++w) {
            const auto& f = words[planes[p].word[w]];
            if (f.expr.empty()) continue;  // padding word
            std::string src = raw_word(planes[p], p, w, mapped);
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
                uint32_t aw = planes[p].word[w];
                const auto& f = words[aw];
                if (f.expr.empty()) continue;
                std::string dst = raw_word(planes[p], p, w, mapped);
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

const hnb_attr_layout* find_attr(const hnb_effect_desc& d, const char* name) {
    for (uint32_t i = 0; i < d.n_attrs; ++i)
        if (!strcmp(d.attrs[i].name, name)) return &d.attrs[i];
    return nullptr;
}

// Lifetime floors (DESIGN.md §3): the column of `planes` that holds the lifetime and nothing else, when the update pass of
// this effect may prove particles alive from a floor instead of loading it (keeps_floors); -1 otherwise.
int life_floor_plane(const hnb_effect_desc& d, const std::vector<Plane>& planes, bool sector) {
    if (sector || !keeps_floors(d.attrs, d.n_attrs, d.flags)) return -1;
    const uint32_t life = find_attr(d, "lifetime")->offset / 4;
    for (size_t p = 0; p < planes.size(); ++p)
        if (planes[p].word[0] == life && planes[p].width == 4) return int(p);
    return -1;
}

// The accessors hnb_update uses with HNB_LIFE_FLOOR: every column load but the lifetime's, the lifetime load, the age word
// and the lifetime word of a RawParticle. In a word map whose age has a column of its own, HNB_GROUP_AGE too (common ages,
// DESIGN.md §3): every column load but the lifetime's and the age's, the age load, and a store of the age word. Other
// plans generate what they generated before word maps.
void gen_life_floor_code(std::ostringstream& o, const hnb_effect_desc& d, const std::vector<Plane>& planes, int life_plane) {
    const uint32_t age_word = find_attr(d, "age")->offset / 4;
    size_t age_plane = 0;
    uint32_t age_lane = 0;
    for (size_t p = 0; p < planes.size(); ++p)
        for (uint32_t l = 0; l < planes[p].width / 4; ++l)
            if (planes[p].word[l] == age_word) age_plane = p, age_lane = l;
    const bool mapped = is_word_map(planes);
    const auto load = [&](size_t p) {
        const std::string address = "s.planes[" + std::to_string(p) + "], row";
        if (mapped) return mapped_load(planes[p], p, address);
        return "    r.q" + std::to_string(p) + " = HNB_LOAD_PLANE(" + plane_type(planes[p]) + ", " + address + ");\n";
    };
    const std::string life = raw_word(planes[life_plane], life_plane, 0, mapped), age = raw_word(planes[age_plane], age_plane, age_lane, mapped);
    o << "#define HNB_LIFE_FLOOR 1\n";
    o << "HNB_DI void hnb_load_raw_but_life(RawParticle& r, const SlabView& s, u32 row) {\n";
    for (size_t p = 0; p < planes.size(); ++p)
        if (int(p) != life_plane) o << load(p);
    o << "}\n";
    o << "HNB_DI void hnb_load_life(RawParticle& r, const SlabView& s, u32 row) { " << life << " = HNB_LOAD_PLANE(f32, s.planes["
      << life_plane << "], row); }\n";
    o << "HNB_DI f32 hnb_raw_age(const RawParticle& r) { return " << age << "; }\n";
    o << "HNB_DI f32& hnb_raw_life(RawParticle& r) { return " << life << "; }\n";
    if (!mapped || planes[age_plane].width != 4) return;  // common ages come with word maps only
    o << "#define HNB_GROUP_AGE 1\n";
    o << "HNB_DI void hnb_load_raw_but_life_age(RawParticle& r, const SlabView& s, u32 row) {\n";
    for (size_t p = 0; p < planes.size(); ++p)
        if (int(p) != life_plane && p != age_plane) o << load(p);
    o << "}\n";
    o << "HNB_DI void hnb_load_age(RawParticle& r, const SlabView& s, u32 row) { " << age << " = HNB_LOAD_PLANE(f32, s.planes["
      << age_plane << "], row); }\n";
    o << "HNB_DI void hnb_set_raw_age(RawParticle& r, f32 age) { " << age << " = age; }\n";
    // The record word of the age (the runtime writes deferred ages back to it); the update's store in a floor tile,
    // hnb_store_written without the age column, and the store of the age column, which a group left deferred skips.
    o << "#define HNB_GROUP_AGE_WORD " << age_word << "\n";
    o << "HNB_DI void hnb_store_age(const RawParticle& r, const SlabView& s, u32 row) { HNB_STORE_PLANE(f32, s.planes[" << age_plane
      << "], row, " << age << "); }\n";
    const bool all = !any_read_only(d.attrs, d.n_attrs);
    const std::vector<bool> written = written_words(d.particle_stride, d.attrs, d.n_attrs);
    o << "HNB_DI void hnb_store_written_but_age(const RawParticle& r, const SlabView& s, u32 row) {\n";
    for (size_t p = 0; p < planes.size(); ++p) {
        bool store = all;
        for (uint32_t w = 0; w < planes[p].width / 4; ++w) store = store || written[planes[p].word[w]];
        if (!store || p == age_plane) continue;
        o << "    HNB_STORE_PLANE(" << plane_type(planes[p]) << ", s.planes[" << p << "], row, " << mapped_value(planes[p], p) << ");\n";
    }
    o << "}\n";
}

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

void check_plan(const std::vector<Plane>& plan, uint32_t stride) {
    uint32_t off = 0;
    std::vector<bool> seen(stride / 4, false);
    for (const Plane& p : plan) {
        if (p.offset != off || (p.width != 4 && p.width != 8 && p.width != 16) || p.offset % p.width)
            throw std::invalid_argument("column plan: columns must be contiguous, 4, 8 or 16 bytes wide and aligned to their width");
        for (uint32_t l = 0; l < p.width / 4; ++l) {
            if (p.word[l] >= seen.size() || seen[p.word[l]]) throw std::invalid_argument("column plan: every record word must be in one column");
            seen[p.word[l]] = true;
        }
        off += p.width;
    }
    if (off != stride || plan.empty() || plan.size() > HNB_RT_MAX_PLANES) throw std::invalid_argument("column plan does not cover the particle record");
}

std::string generate_effect_source(const hnb_effect_desc& d, const std::vector<Plane>* plan, const std::vector<Plane>* parent_plan) {
    if (!d.attrs || d.n_attrs == 0) throw std::invalid_argument("effect has an empty particle layout");
    const bool sector = (d.flags & HNB_EFFECT_SECTOR_PLANES) != 0;
    if (plan && sector) throw std::invalid_argument("a sector-plane effect has no other column plan");
    if (plan) check_plan(*plan, d.particle_stride);
    if (parent_plan) check_plan(*parent_plan, d.parent_particle_stride);
    const auto planes = sector ? cut_planes(d.particle_stride) : plan ? *plan : column_plan(d.particle_stride, d.attrs, d.n_attrs, d.flags);
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
            // bind_launch): overriding them here would make the kernel's carve-up disagree with the launch. Ignored, loudly.
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
    gen_layout_code(o, "", "Particle", d.attrs, d.n_attrs, d.particle_stride, planes, true, sector);
    if (const int life_plane = life_floor_plane(d, planes, sector); life_plane >= 0) gen_life_floor_code(o, d, planes, life_plane);
    // a parent slab is read in the default cut (emitting effects keep it: column_plan), or in the plan its first bound
    // effect gave it
    if (read_parent)
        gen_layout_code(o, "Parent", "ParentParticle", d.parent_attrs, d.n_parent_attrs, d.parent_particle_stride,
                        parent_plan ? *parent_plan : cut_planes(d.parent_particle_stride), false);
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
