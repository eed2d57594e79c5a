// graph_cabi.cpp — extern "C" surface of the authoring layer (include/hanabi_b200_graph.h).
#include <set>
#include <algorithm>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "hanabi_b200_graph.h"
#include "hanabi_graph.h"

using namespace hnb_graph;

extern "C" void hnb_set_last_error_(const char* msg);  // defined in runtime/context.cpp

struct hnb_asset {
    EffectAsset a;
};
struct hnb_generated {
    EffectShaderSource src;
    std::string name;
    std::vector<hnb_attr_layout> attrs, parent_attrs;
    std::vector<std::string> names, parent_names;
};

namespace {

int32_t code_of(const ExprError& e) { return e.kind == ExprError::Validate ? HNB_ERR_LAYOUT : HNB_ERR_EXPR; }

template <typename F> int32_t guarded(F&& f) {
    try {
        f();
        return HNB_OK;
    } catch (const ExprError& e) {
        hnb_set_last_error_(e.what());
        return code_of(e);
    } catch (const std::exception& e) {
        hnb_set_last_error_(e.what());
        return HNB_ERR_INVALID_ARG;
    }
}
template <typename F> uint32_t handle_or_zero(F&& f) {
    try {
        return f();
    } catch (const std::exception& e) {
        hnb_set_last_error_(e.what());
        return 0;
    }
}
void copy_out(const std::string& s, char* out, size_t cap) {
    if (!out || !cap) return;
    size_t n = std::min(cap - 1, s.size());
    memcpy(out, s.data(), n);
    out[n] = 0;
}
Attribute attr_or_throw(const char* name) {
    Attribute a = name ? attribute_by_name(name) : -1;
    if (a < 0) throw ExprError(ExprError::GraphEvalError, std::string("unknown attribute '") + (name ? name : "(null)") + "'");
    return a;
}
Value value_from(uint32_t vt, const uint32_t* words) {
    ValueType t(vt);
    if (vt > HNB_MAT4X3) throw ExprError(ExprError::TypeError, "invalid value type");
    if (!words) throw ExprError(ExprError::TypeError, "NULL literal data");
    Value v = Value::from_words(t, words);
    if (t.elem() == ScalarType::Bool)
        for (int i = 0; i < t.count(); ++i) v.bits[i] = v.bits[i] ? 0xFFFFFFFFu : 0u;
    return v;
}
// static storage for names handed out through hnb_attr_layout (attribute names are static, pads too)
const char* static_name(const std::string& s) {
    static const char* pads[] = {"pad0", "pad1", "pad2", "pad3", "pad4"};
    for (auto p : pads)
        if (s == p) return p;
    Attribute a = attribute_by_name(s);
    return a >= 0 ? attribute_info(a).name : "?";
}
void fill_layout(const ParticleLayout& pl, hnb_attr_layout* out, uint32_t cap, uint32_t* n, uint32_t* size, uint32_t* align) {
    if (n) *n = (uint32_t)pl.layout.size();
    if (size) *size = pl.size();
    if (align) *align = pl.align;
    for (size_t i = 0; i < pl.layout.size() && i < cap && out; ++i) {
        out[i].name = static_name(pl.layout[i].name);
        out[i].value_type = pl.layout[i].type.code;
        out[i].offset = pl.layout[i].offset;
        out[i].flags = 0;
    }
}

}  // namespace

extern "C" {

hnb_module* hnb_module_create(void) { return new hnb_module(); }
void hnb_module_destroy(hnb_module* m) { delete m; }

hnb_expr hnb_module_lit(hnb_module* m, uint32_t value_type, const uint32_t* words) {
    return handle_or_zero([&] { return m->m.lit(value_from(value_type, words)); });
}
// Module::get (expr.rs:607-612) flattened: read back one stored expression
uint32_t hnb_module_len(const hnb_module* m) { return m ? (uint32_t)m->m.size() : 0; }
int32_t hnb_module_get(const hnb_module* m, hnb_expr e, hnb_expr_info* out) {
    return guarded([&] {
        if (!m || !out) throw ExprError(ExprError::GraphEvalError, "NULL argument");
        const Expr& x = m->m.try_get(e);
        memset(out, 0, sizeof(*out));
        out->kind = (uint32_t)x.kind;
        out->value_type = x.kind == Expr::Literal ? x.literal.type.code : x.type.code;
        switch (x.kind) {
            case Expr::BuiltIn: out->op = (uint32_t)x.builtin; break;
            case Expr::Literal: memcpy(out->literal_words, x.literal.bits, sizeof(out->literal_words)); break;
            case Expr::Property: out->property = x.property; break;
            case Expr::Attribute:
            case Expr::ParentAttribute: out->attribute = attribute_info(x.attribute).name; break;
            case Expr::Unary: out->op = x.op; out->operands[0] = x.a; break;
            case Expr::Binary: out->op = x.op; out->operands[0] = x.a; out->operands[1] = x.b; break;
            case Expr::Ternary: out->op = x.op; out->operands[0] = x.a; out->operands[1] = x.b; out->operands[2] = x.c; break;
            case Expr::Cast: out->operands[0] = x.a; break;
        }
    });
}
hnb_expr hnb_module_attr(hnb_module* m, const char* name) {
    return handle_or_zero([&] { return m->m.attr(attr_or_throw(name)); });
}
hnb_expr hnb_module_parent_attr(hnb_module* m, const char* name) {
    return handle_or_zero([&] { return m->m.parent_attr(attr_or_throw(name)); });
}
hnb_prop hnb_module_add_property(hnb_module* m, const char* name, uint32_t value_type, const uint32_t* words) {
    return handle_or_zero([&] {
        if (!name) throw ExprError(ExprError::PropertyError, "NULL property name");
        return m->m.add_property(name, value_from(value_type, words));
    });
}
hnb_expr hnb_module_prop(hnb_module* m, hnb_prop p) {
    return handle_or_zero([&] {
        if (!m->m.get_property(p)) throw ExprError(ExprError::PropertyError, "invalid property handle");
        return m->m.prop(p);
    });
}
hnb_expr hnb_module_builtin(hnb_module* m, uint32_t op, uint32_t rand_value_type) {
    return handle_or_zero([&] {
        if (op > HNB_BUILTIN_IS_ALIVE) throw ExprError(ExprError::SyntaxError, "invalid built-in operator");
        return m->m.builtin((BuiltInOperator)op, ValueType(op == HNB_BUILTIN_RAND ? rand_value_type : (uint32_t)HNB_FLOAT));
    });
}
hnb_expr hnb_module_unary(hnb_module* m, uint32_t op, hnb_expr e) {
    return handle_or_zero([&] {
        if (op > HNB_UN_Z) throw ExprError(ExprError::SyntaxError, "invalid unary operator");
        return m->m.unary((UnaryOperator)op, e);
    });
}
hnb_expr hnb_module_binary(hnb_module* m, uint32_t op, hnb_expr l, hnb_expr r) {
    return handle_or_zero([&] {
        if (op > HNB_BIN_VEC4_XYZ_W) throw ExprError(ExprError::SyntaxError, "invalid binary operator");
        return m->m.binary((BinaryOperator)op, l, r);
    });
}
hnb_expr hnb_module_ternary(hnb_module* m, uint32_t op, hnb_expr a, hnb_expr b, hnb_expr c) {
    return handle_or_zero([&] {
        if (op > HNB_TER_VEC3) throw ExprError(ExprError::SyntaxError, "invalid ternary operator");
        return m->m.ternary((TernaryOperator)op, a, b, c);
    });
}
hnb_expr hnb_module_cast(hnb_module* m, hnb_expr e, uint32_t target) {
    return handle_or_zero([&] { return m->m.cast(e, ValueType(target)); });
}
int32_t hnb_module_is_const(const hnb_module* m, hnb_expr e) {
    try { return m->m.is_const(e) ? 1 : 0; } catch (const std::exception& ex) { hnb_set_last_error_(ex.what()); return HNB_ERR_EXPR; }
}
int32_t hnb_module_has_side_effect(const hnb_module* m, hnb_expr e) {
    try { return m->m.has_side_effect(e) ? 1 : 0; } catch (const std::exception& ex) { hnb_set_last_error_(ex.what()); return HNB_ERR_EXPR; }
}
int32_t hnb_module_eval(const hnb_module* m, hnb_expr e, uint32_t context, char* out, size_t out_cap, char* stmts, size_t stmts_cap) {
    return guarded([&] {
        std::set<Attribute> all;
        for (int i = 0; i < attribute_count(); ++i) all.insert(i);
        ParticleLayout pal = ParticleLayout::build(all);
        PropertyLayout pl = PropertyLayout::make(m->m.properties());
        ShaderWriter w(context == HNB_CONTEXT_INIT ? ModifierContext::Init : ModifierContext::Update, pl, pal);
        std::string s = w.eval(m->m, e);
        copy_out(s, out, out_cap);
        copy_out(w.main_code, stmts, stmts_cap);
    });
}

uint32_t hnb_attribute_count(void) { return (uint32_t)attribute_count(); }
int32_t hnb_attribute_info(uint32_t index, const char** name, uint32_t* value_type, uint32_t default_words[4]) {
    return guarded([&] {
        const AttributeInfo& info = attribute_info((Attribute)index);
        if (name) *name = info.name;
        if (value_type) *value_type = info.type.code;
        if (default_words)
            for (int i = 0; i < 4; ++i) default_words[i] = info.default_value.bits[i];
    });
}
int32_t hnb_particle_layout_build(const char* const* names, uint32_t n_names, hnb_attr_layout* out, uint32_t cap, uint32_t* n, uint32_t* size,
                                  uint32_t* align) {
    return guarded([&] {
        std::set<Attribute> set;
        for (uint32_t i = 0; i < n_names; ++i) set.insert(attr_or_throw(names[i]));
        fill_layout(ParticleLayout::build(set), out, cap, n, size, align);
    });
}
int32_t hnb_format_f32(float value, char* out, size_t cap) {
    return guarded([&] { copy_out(f32_to_cuda_string(value), out, cap); });
}

hnb_asset* hnb_asset_create(const char* name, uint32_t capacity, const hnb_module* module) {
    auto* a = new hnb_asset();
    a->a.name = name ? name : "";
    a->a.capacity = capacity;
    if (module) a->a.module = module->m;
    return a;
}
void hnb_asset_destroy(hnb_asset* a) { delete a; }
int32_t hnb_asset_set_simulation_space(hnb_asset* a, uint32_t local) {
    a->a.simulation_space = local ? SimulationSpace::Local : SimulationSpace::Global;
    return HNB_OK;
}
int32_t hnb_asset_set_motion_integration(hnb_asset* a, uint32_t mode) {
    return guarded([&] {
        if (mode > 2) throw ExprError(ExprError::GraphEvalError, "invalid motion integration mode");
        a->a.motion_integration = (MotionIntegration)mode;
    });
}
int32_t hnb_asset_add_modifier(hnb_asset* a, uint32_t context, uint32_t kind, const hnb_expr* exprs, uint32_t n_exprs, const uint32_t* params,
                               uint32_t n_params) {
    return guarded([&] {
        if (kind < HNB_MOD_ACCEL || kind > HNB_MOD_EMIT_SPAWN_EVENT) throw ExprError(ExprError::GraphEvalError, "invalid modifier kind");
        if (context != HNB_CONTEXT_INIT && context != HNB_CONTEXT_UPDATE) throw ExprError(ExprError::GraphEvalError, "invalid modifier context");
        Modifier m;
        m.kind = (ModifierKind)kind;
        m.exprs.assign(exprs, exprs + n_exprs);
        m.params.assign(params, params + n_params);
        for (auto h : m.exprs)
            if (h) a->a.module.try_get(h);
        if ((m.kind == ModifierKind::SetAttribute || m.kind == ModifierKind::InheritAttribute)) {
            if (m.params.empty() || m.params[0] >= (uint32_t)attribute_count()) throw ExprError(ExprError::GraphEvalError, "invalid attribute index");
            if (m.kind == ModifierKind::SetAttribute && ((Attribute)m.params[0] == attr::ID || (Attribute)m.params[0] == attr::PARTICLE_COUNTER))
                throw ExprError(ExprError::GraphEvalError, "ID and PARTICLE_COUNTER are read-only pseudo-attributes, cannot be assigned.");
        }
        a->a.add_modifier(context == HNB_CONTEXT_INIT ? ModifierContext::Init : ModifierContext::Update, m);
    });
}
int32_t hnb_asset_particle_layout(const hnb_asset* a, hnb_attr_layout* out, uint32_t cap, uint32_t* n, uint32_t* size, uint32_t* align) {
    return guarded([&] { fill_layout(a->a.particle_layout(), out, cap, n, size, align); });
}
int32_t hnb_asset_property_layout(const hnb_asset* a, hnb_attr_layout* out, uint32_t cap, uint32_t* n, uint32_t* size) {
    return guarded([&] {
        PropertyLayout pl = a->a.property_layout();
        if (n) *n = (uint32_t)pl.layout.size();
        if (size) *size = pl.min_binding_size();
        const auto& props = a->a.module.properties();
        for (size_t i = 0; i < pl.layout.size() && i < cap && out; ++i) {
            // hand out the name stored in the asset's module (stable for the asset's lifetime)
            const char* nm = "?";
            for (const auto& p : props)
                if (p.name == pl.layout[i].property.name) nm = p.name.c_str();
            out[i].name = nm;
            out[i].value_type = pl.layout[i].property.default_value.type.code;
            out[i].offset = pl.layout[i].offset;
            out[i].flags = 0;
        }
    });
}
int32_t hnb_asset_serialize_properties(const hnb_asset* a, const char* const* names, const uint32_t* const* words, uint32_t n, void* blob,
                                       uint32_t blob_cap, uint32_t* blob_size) {
    return guarded([&] {
        PropertyLayout pl = a->a.property_layout();
        std::vector<std::pair<std::string, Value>> values;
        for (uint32_t i = 0; i < n; ++i) {
            PropertyHandle h = a->a.module.get_property_by_name(names[i]);
            if (!h) throw ExprError(ExprError::PropertyError, std::string("unknown property '") + names[i] + "'");
            values.push_back({names[i], value_from(a->a.module.get_property(h)->default_value.type.code, words[i])});
        }
        std::vector<uint8_t> data = pl.serialize(values);
        if (blob_size) *blob_size = (uint32_t)data.size();
        if (blob) {
            if (blob_cap < data.size()) throw ExprError(ExprError::PropertyError, "property blob buffer too small");
            memcpy(blob, data.data(), data.size());
        }
    });
}

int32_t hnb_asset_generate(const hnb_asset* a, const hnb_asset* parent, uint32_t num_event_bindings, hnb_generated** out) {
    return guarded([&] {
        if (!out) throw ExprError(ExprError::GraphEvalError, "out is NULL");
        *out = nullptr;
        ParticleLayout parent_layout;
        if (parent) parent_layout = parent->a.particle_layout();
        auto g = std::make_unique<hnb_generated>();
        g->src = a->a.generate(parent ? &parent_layout : nullptr, num_event_bindings);
        g->name = a->a.name;
        auto fill = [](const ParticleLayout& pl, std::vector<hnb_attr_layout>& v, const std::set<Attribute>* writes, bool lifetime_reap_only) {
            for (const auto& l : pl.layout) {
                if (l.is_pad) continue;
                const Attribute a = attribute_by_name(l.name);
                const bool read_only = writes && !writes->count(a);
                uint32_t flags = read_only ? uint32_t(HNB_ATTR_UPDATE_READ_ONLY) : 0u;
                if (read_only && lifetime_reap_only && a == attr::LIFETIME) flags |= HNB_ATTR_REAP_ONLY;
                v.push_back({static_name(l.name), l.type.code, l.offset, flags});
            }
        };
        fill(g->src.particle_layout, g->attrs, &g->src.update_writes, g->src.lifetime_reap_only);
        if (g->src.parent_layout) fill(*g->src.parent_layout, g->parent_attrs, nullptr, false);
        *out = g.release();
    });
}
int32_t hnb_generated_desc(const hnb_generated* g, hnb_effect_desc* d) {
    return guarded([&] {
        if (!g || !d) throw ExprError(ExprError::GraphEvalError, "NULL argument");
        memset(d, 0, sizeof(*d));
        d->name = g->name.c_str();
        d->attrs = g->attrs.data();
        d->n_attrs = (uint32_t)g->attrs.size();
        d->particle_stride = g->src.particle_layout.size();
        d->properties_struct = g->src.properties_struct.c_str();
        d->properties_size = g->src.property_layout.min_binding_size();
        d->init_code = g->src.init_code.c_str();
        d->init_extra = g->src.init_extra.c_str();
        d->sim_space_code = g->src.sim_space_code.c_str();
        d->age_code = g->src.age_code.c_str();
        d->reap_code = g->src.reap_code.c_str();
        d->update_code = g->src.update_code.c_str();
        d->update_extra = g->src.update_extra.c_str();
        d->flags = g->src.flags;
        d->parent_attrs = g->parent_attrs.empty() ? nullptr : g->parent_attrs.data();
        d->n_parent_attrs = (uint32_t)g->parent_attrs.size();
        d->parent_particle_stride = g->src.parent_layout ? g->src.parent_layout->size() : 0;
        d->num_event_bindings = g->src.num_event_bindings;
    });
}
void hnb_generated_destroy(hnb_generated* g) { delete g; }

// ---- EffectProperties: the per-instance property store (reference src/properties.rs:205-454) ----------------
// The ECS component is Bevy's; what reaches the kernels is the byte blob of `serialize`, and which values it
// holds is decided by `set` / `update`. Change detection (`Mut<>`) is reported through `*changed`.
}  // extern "C" (struct with C++ members)

struct hnb_effect_properties {
    struct Instance {  // PropertyInstance (properties.rs:183-190)
        Property def;
        Value value;
    };
    std::vector<Instance> properties;
    int find(const char* name) const {
        for (size_t i = 0; i < properties.size(); ++i)
            if (properties[i].def.name == name) return (int)i;
        return -1;
    }
};

namespace {
bool same_value(const Value& a, const Value& b) {
    return a.type == b.type && memcmp(a.bits, b.bits, sizeof(uint32_t) * (size_t)a.type.count()) == 0;
}
// EffectProperties::set / set_if_changed (properties.rs:319-376)
void props_set(hnb_effect_properties* p, const char* name, uint32_t vt, const uint32_t* words, bool only_if_changed, uint32_t* changed) {
    if (!p || !name) throw ExprError(ExprError::PropertyError, "NULL argument");
    const Value value = value_from(vt, words);
    if (changed) *changed = 1;
    const int i = p->find(name);
    if (i < 0) {
        p->properties.push_back({Property{name, value}, value});
        return;
    }
    auto& prop = p->properties[(size_t)i];
    if (prop.def.default_value.type != value.type)
        throw ExprError(ExprError::PropertyError, "Cannot assign value of type " + value.type.to_cuda_string() + " to property '" + prop.def.name +
                                                      "' of type " + prop.def.default_value.type.to_cuda_string());
    if (only_if_changed && same_value(prop.value, value)) {
        if (changed) *changed = 0;
        return;
    }
    prop.value = value;
}
}  // namespace

extern "C" {

hnb_effect_properties* hnb_effect_properties_create(void) { return new hnb_effect_properties(); }
void hnb_effect_properties_destroy(hnb_effect_properties* p) { delete p; }
uint32_t hnb_effect_properties_len(const hnb_effect_properties* p) { return p ? (uint32_t)p->properties.size() : 0; }

int32_t hnb_effect_properties_set(hnb_effect_properties* p, const char* name, uint32_t value_type, const uint32_t* words) {
    return guarded([&] { props_set(p, name, value_type, words, false, nullptr); });
}
int32_t hnb_effect_properties_set_if_changed(hnb_effect_properties* p, const char* name, uint32_t value_type, const uint32_t* words,
                                             uint32_t* changed) {
    return guarded([&] { props_set(p, name, value_type, words, true, changed); });
}
// EffectProperties::get_stored (properties.rs:305-310): 1 = found, 0 = no such property
int32_t hnb_effect_properties_get_stored(const hnb_effect_properties* p, const char* name, uint32_t* value_type, uint32_t* words16) {
    if (!p || !name) return 0;
    const int i = p->find(name);
    if (i < 0) return 0;
    const Value& v = p->properties[(size_t)i].value;
    if (value_type) *value_type = v.type.code;
    if (words16) memcpy(words16, v.bits, sizeof(v.bits));
    return 1;
}
int32_t hnb_effect_properties_get(const hnb_effect_properties* p, uint32_t index, const char** name, uint32_t* value_type,
                                  uint32_t* value_words16, uint32_t* default_words16) {
    return guarded([&] {
        if (!p || index >= p->properties.size()) throw ExprError(ExprError::PropertyError, "property index out of range");
        const auto& pi = p->properties[index];
        if (name) *name = pi.def.name.c_str();
        if (value_type) *value_type = pi.def.default_value.type.code;
        if (value_words16) memcpy(value_words16, pi.value.bits, sizeof(pi.value.bits));
        if (default_words16) memcpy(default_words16, pi.def.default_value.bits, sizeof(pi.def.default_value.bits));
    });
}
// EffectProperties::update (properties.rs:378-417): drop the instances the asset does not declare, append the
// asset's missing properties with their default value; stored values of known properties win.
int32_t hnb_effect_properties_update(hnb_effect_properties* p, const hnb_asset* asset, uint32_t* changed) {
    return guarded([&] {
        if (!p || !asset) throw ExprError(ExprError::PropertyError, "NULL argument");
        std::vector<hnb_effect_properties::Instance> fresh;
        std::set<std::string> intersect;
        for (const Property& prop : asset->a.module.properties()) {
            if (p->find(prop.name.c_str()) >= 0) {
                intersect.insert(prop.name);
                continue;
            }
            fresh.push_back({prop, prop.default_value});
        }
        bool mutated = false;
        if (intersect.size() != p->properties.size()) {
            auto& v = p->properties;
            v.erase(std::remove_if(v.begin(), v.end(), [&](const auto& pi) { return !intersect.count(pi.def.name); }), v.end());
            mutated = true;
        }
        if (!fresh.empty()) {
            p->properties.insert(p->properties.end(), fresh.begin(), fresh.end());
            mutated = true;
        }
        if (changed) *changed = mutated ? 1u : 0u;
    });
}
// EffectProperties::serialize (properties.rs:437-453): a zeroed record with every stored property the layout knows
// written at its offset. The record is padded to the layout's min_binding_size, the size hnb_upload_properties takes.
int32_t hnb_effect_properties_serialize(const hnb_effect_properties* p, const hnb_asset* asset, void* blob, uint32_t blob_cap,
                                        uint32_t* blob_size) {
    return guarded([&] {
        if (!p || !asset) throw ExprError(ExprError::PropertyError, "NULL argument");
        const PropertyLayout pl = asset->a.property_layout();
        std::vector<uint8_t> data(pl.min_binding_size(), 0);
        for (const auto& pi : p->properties) {
            const auto off = pl.offset(pi.def.name);
            if (!off) continue;
            const uint32_t size = pi.def.default_value.type.size();
            if (*off + size > data.size()) throw ExprError(ExprError::PropertyError, "property '" + pi.def.name + "' does not fit the asset's layout");
            memcpy(&data[*off], pi.value.bits, size);
        }
        if (blob_size) *blob_size = (uint32_t)data.size();
        if (blob) {
            if (blob_cap < data.size()) throw ExprError(ExprError::PropertyError, "property blob buffer too small");
            memcpy(blob, data.data(), data.size());
        }
    });
}

}  // extern "C"
