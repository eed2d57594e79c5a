// modifiers.cpp — init/update modifiers and EffectAsset code generation, lowering to CUDA C.
// Restates the `apply()` of every simulation modifier of the reference:
//   src/modifier/accel.rs    AccelModifier :79-86, RadialAccelModifier :162-189, TangentAccelModifier :281-307
//   src/modifier/force.rs    ConformToSphereModifier :175-238, LinearDragModifier :284-297
//   src/modifier/kill.rs     KillSphereModifier :76-96, KillAabbModifier :156-181
//   src/modifier/attr.rs     SetAttributeModifier :92-114, InheritAttributeModifier :173-186
//   src/modifier/position.rs SetPosition{Circle,Sphere,Cone3d}Modifier :52-109, :152-211, :267-325
//   src/modifier/velocity.rs SetVelocity{Circle,Sphere,Tangent}Modifier :45-81, :124-139, :188-224
//   src/modifier/mod.rs      EmitSpawnEventModifier :654-717
// and EffectAsset::particle_layout (src/asset.rs:605-626) / EffectShaderSources::generate
// (src/lib.rs:805-1335, init + update parts). Statement order, operand evaluation order (it fixes the
// order of PRNG draws) and parenthesisation follow the reference; only the surface syntax is C.
#include <cstring>

#include "hanabi_b200.h"
#include "hanabi_graph.h"

namespace hnb_graph {

// EvalContext::make_fn (modifier/mod.rs:332-362): the function body is generated with its own writer
// (fresh variable counter and expression cache, attribute-pointer mode).
template <typename F> void ShaderWriter::make_fn(const std::string& func_name, Module& module, F&& f) {
    ShaderWriter ctx(context_, property_layout, particle_layout, /*attribute_pointer=*/true);
    std::string body = f(module, ctx);
    extra_code += ctx.extra_code;
    extra_code += "HNB_DI void " + func_name + "(Particle* particle, Ctx& hnb_ctx) {\n    HNB_CTX_PROLOGUE\n" + ctx.main_code + body + "}\n";
}

namespace {

uint64_t fnv(const void* p, size_t n, uint64_t h = 0xcbf29ce484222325ull) {
    const unsigned char* c = (const unsigned char*)p;
    for (size_t i = 0; i < n; ++i) { h ^= c[i]; h *= 0x100000001b3ull; }
    return h;
}

// calc_func_id (modifier/mod.rs:97-101): any id unique per (modifier content, context) works; the
// reference's DefaultHasher value itself never influences results.
std::string func_name(const char* base, const Modifier& m, ModifierContext ctx) {
    uint64_t h = fnv(&m.kind, sizeof(m.kind));
    if (!m.exprs.empty()) h = fnv(m.exprs.data(), m.exprs.size() * sizeof(ExprHandle), h);
    if (!m.params.empty()) h = fnv(m.params.data(), m.params.size() * sizeof(uint32_t), h);
    char buf[32];
    snprintf(buf, sizeof(buf), "%016llX", (unsigned long long)h);
    return std::string(ctx == ModifierContext::Init ? "init_" : "update_") + base + "_" + buf;
}

ExprHandle need(const Modifier& m, size_t i, const char* what) {
    if (i >= m.exprs.size() || m.exprs[i] == 0) throw ExprError(ExprError::GraphEvalError, std::string("modifier is missing operand '") + what + "'");
    return m.exprs[i];
}
ExprHandle opt(const Modifier& m, size_t i) { return i < m.exprs.size() ? m.exprs[i] : 0; }
uint32_t param(const Modifier& m, size_t i, uint32_t def = 0) { return i < m.params.size() ? m.params[i] : def; }

const char* kPos = "position";
const char* kVel = "velocity";

}  // namespace

uint32_t Modifier::allowed_contexts() const {
    const uint32_t I = (uint32_t)ModifierContext::Init, U = (uint32_t)ModifierContext::Update;
    switch (kind) {
        case ModifierKind::Accel: case ModifierKind::RadialAccel: case ModifierKind::TangentAccel: case ModifierKind::ConformToSphere:
        case ModifierKind::LinearDrag: case ModifierKind::KillSphere: case ModifierKind::KillAabb: case ModifierKind::EmitSpawnEvent:
            return U;
        case ModifierKind::InheritAttribute: return I;
        default: return I | U;
    }
}

std::vector<Attribute> Modifier::attributes() const {
    switch (kind) {
        case ModifierKind::Accel: case ModifierKind::LinearDrag: return {attr::VELOCITY};
        case ModifierKind::RadialAccel: case ModifierKind::TangentAccel: case ModifierKind::ConformToSphere:
        case ModifierKind::SetVelocityCircle: case ModifierKind::SetVelocitySphere: case ModifierKind::SetVelocityTangent:
            return {attr::POSITION, attr::VELOCITY};
        case ModifierKind::KillSphere: case ModifierKind::KillAabb:
        case ModifierKind::SetPositionCircle: case ModifierKind::SetPositionSphere: case ModifierKind::SetPositionCone3d:
            return {attr::POSITION};
        case ModifierKind::SetAttribute: case ModifierKind::InheritAttribute: return {(Attribute)param(*this, 0)};
        case ModifierKind::EmitSpawnEvent: return {};
    }
    return {};
}

std::vector<Attribute> Modifier::update_writes() const {
    switch (kind) {
        case ModifierKind::Accel: case ModifierKind::RadialAccel: case ModifierKind::TangentAccel: case ModifierKind::ConformToSphere:
        case ModifierKind::LinearDrag: case ModifierKind::SetVelocityCircle: case ModifierKind::SetVelocitySphere:
        case ModifierKind::SetVelocityTangent:
            return {attr::VELOCITY};
        case ModifierKind::SetPositionCircle: case ModifierKind::SetPositionSphere: case ModifierKind::SetPositionCone3d:
            return {attr::POSITION};
        case ModifierKind::SetAttribute: case ModifierKind::InheritAttribute: return {(Attribute)param(*this, 0)};
        case ModifierKind::KillSphere: case ModifierKind::KillAabb: case ModifierKind::EmitSpawnEvent: return {};
    }
    return {};
}

void Modifier::apply(Module& module, ShaderWriter& context) const {
    const ModifierContext mc = context.modifier_context();
    if (!((uint32_t)mc & allowed_contexts())) throw ExprError(ExprError::InvalidModifierContext, "modifier used in an invalid context");
    const Modifier& self = *this;
    switch (kind) {
        case ModifierKind::Accel: {  // accel.rs:79-86
            ExprHandle a = module.attr(attr::VELOCITY);
            std::string attr_s = context.eval(module, a);
            std::string expr = context.eval(module, need(self, 0, "accel"));
            context.main_code += attr_s + " += (" + expr + ") * sim_params.delta_time;";
            break;
        }
        case ModifierKind::RadialAccel: {  // accel.rs:162-189
            std::string fn = func_name("radial_accel", self, mc);
            context.make_fn(fn, module, [&](Module& m, ShaderWriter& ctx) {
                std::string origin = ctx.eval(m, need(self, 0, "origin"));
                std::string accel = ctx.eval(m, need(self, 1, "accel"));
                return "const auto radial = normalize((*particle)." + std::string(kPos) + " - " + origin + ");\n" +
                       "            (*particle)." + kVel + " += radial * ((" + accel + ") * sim_params.delta_time);\n        ";
            });
            context.main_code += fn + "(&particle, hnb_ctx);\n";
            break;
        }
        case ModifierKind::TangentAccel: {  // accel.rs:281-307 — operands are evaluated in the CALLER's context
            std::string fn = func_name("tangent_accel", self, mc);
            std::string origin = context.eval(module, need(self, 0, "origin"));
            std::string axis = context.eval(module, need(self, 1, "axis"));
            std::string accel = context.eval(module, need(self, 2, "accel"));
            // operands evaluated in the caller refer to `particle.` (a value there); inside the function the
            // particle is a pointer, so give the body a reference of the same name to keep the text valid
            context.extra_code += "HNB_DI void " + fn + "(Particle* particle_ptr, Ctx& hnb_ctx) {\n    HNB_CTX_PROLOGUE\n    Particle& particle = *particle_ptr;\n" +
                                  "    const auto radial = normalize(particle." + kPos + " - " + origin + ");\n" +
                                  "    const auto tangent = normalize(cross(" + axis + ", radial));\n" +
                                  "    particle." + kVel + " += tangent * ((" + accel + ") * sim_params.delta_time);\n}\n";
            context.main_code += fn + "(&particle, hnb_ctx);\n";
            break;
        }
        case ModifierKind::ConformToSphere: {  // force.rs:175-238
            std::string fn = func_name("force_field", self, mc);
            context.make_fn(fn, module, [&](Module& m, ShaderWriter& ctx) {
                std::string origin = ctx.eval(m, need(self, 0, "origin"));
                std::string radius = ctx.eval(m, need(self, 1, "radius"));
                std::string influence_dist = ctx.eval(m, need(self, 2, "influence_dist"));
                std::string shell = opt(self, 5) ? ctx.eval(m, opt(self, 5)) : "0.1f";
                std::string max_speed = ctx.eval(m, need(self, 4, "max_attraction_speed"));
                std::string accel = ctx.eval(m, need(self, 3, "attraction_accel"));
                std::string sticky = opt(self, 6) ? ctx.eval(m, opt(self, 6)) : "2.0f";
                const std::string pos = std::string("(*particle).") + kPos, vel = std::string("(*particle).") + kVel;
                return "    const auto c = " + origin + ";\n"
                       "    const auto r = " + radius + ";\n"
                       "    const auto rel_pos = c - " + pos + ";\n"
                       "    const auto origin_dist = length(rel_pos);\n"
                       "    const auto origin_dir = normalize(rel_pos);\n"
                       "    const auto surface_dist = origin_dist - r;\n"
                       "    const auto influence_dist = " + influence_dist + ";\n"
                       "    if (surface_dist > influence_dist) {\n        return;\n    }\n"
                       "    const auto cur_radial_speed = dot(" + vel + ", origin_dir);\n"
                       "    const auto shell_half_thickness = " + shell + ";\n"
                       "    const auto shell_factor = smoothstep(0.f, shell_half_thickness, abs(surface_dist));\n"
                       "    const auto max_attraction_speed = " + max_speed + ";\n"
                       "    const auto max_radial_speed = sign(surface_dist) * shell_factor * max_attraction_speed;\n"
                       "    const auto delta_speed = max_radial_speed - cur_radial_speed;\n"
                       "    const auto attraction_accel = " + accel + ";\n"
                       "    const auto sticky_accel = attraction_accel * " + sticky + ";\n"
                       "    const auto conforming_accel = mix(sticky_accel, attraction_accel, shell_factor);\n"
                       "    const auto conforming_delta_speed = sim_params.delta_time * conforming_accel;\n"
                       "    " + vel + " += sign(delta_speed) * min(abs(delta_speed), conforming_delta_speed) * origin_dir;\n";
            });
            context.main_code += fn + "(&particle, hnb_ctx);\n";
            break;
        }
        case ModifierKind::LinearDrag: {  // force.rs:284-297 (the expression is built through the module)
            ExprHandle a = module.attr(attr::VELOCITY);
            ExprHandle dt = module.builtin(BuiltInOperator::DeltaTime);
            ExprHandle drag_dt = module.mul(need(self, 0, "drag"), dt);
            ExprHandle one = module.lit(1.f);
            ExprHandle one_minus = module.sub(one, drag_dt);
            ExprHandle zero = module.lit(0.f);
            ExprHandle expr = module.max(zero, one_minus);
            std::string attr_s = context.eval(module, a);
            std::string expr_s = context.eval(module, expr);
            context.main_code += attr_s + " *= " + expr_s + ";";
            break;
        }
        case ModifierKind::KillSphere: {  // kill.rs:76-96
            const bool kill_inside = param(self, 0) != 0;
            ExprHandle pos = module.attr(attr::POSITION);
            ExprHandle diff = module.sub(pos, need(self, 0, "center"));
            ExprHandle sqr_dist = module.dot(diff, diff);
            ExprHandle cmp = kill_inside ? module.lt(sqr_dist, need(self, 1, "sqr_radius")) : module.gt(sqr_dist, need(self, 1, "sqr_radius"));
            context.main_code += "if (" + context.eval(module, cmp) + ") {\n    is_alive = false;\n}\n";
            break;
        }
        case ModifierKind::KillAabb: {  // kill.rs:156-181
            const bool kill_inside = param(self, 0) != 0;
            ExprHandle pos = module.attr(attr::POSITION);
            ExprHandle diff = module.sub(pos, need(self, 0, "center"));
            ExprHandle dist = module.abs(diff);
            ExprHandle cmp = kill_inside ? module.lt(dist, need(self, 1, "half_size")) : module.gt(dist, need(self, 1, "half_size"));
            ExprHandle reduce = kill_inside ? module.all(cmp) : module.any(cmp);
            context.main_code += "if (" + context.eval(module, reduce) + ") {\n    is_alive = false;\n}\n";
            break;
        }
        case ModifierKind::SetAttribute: {  // attr.rs:92-114
            const Attribute at = (Attribute)param(self, 0);
            if (at == attr::ID) throw ExprError(ExprError::GraphEvalError, "The particle's ID is a read-only pseudo-attribute, cannot be assigned.");
            if (at == attr::PARTICLE_COUNTER) throw ExprError(ExprError::GraphEvalError, "The PARTICLE_COUNTER attribute is a read-only pseudo-attribute, cannot be assigned.");
            ExprHandle value = need(self, 0, "value");
            if (auto vt = module.value_type(value)) {
                ValueType want = attribute_info(at).type;
                if (*vt != want) {
                    std::string up = attribute_info(at).name;
                    for (auto& ch : up) ch = (char)toupper(ch);
                    throw ExprError(ExprError::TypeError, "Mismatching expression type in SetAttributeModifer: attribute '" + up + "' requires an expression producing a value of type " +
                                                              want.to_cuda_string() + ", but a value of type " + vt->to_cuda_string() + " was produced instead");
                }
            }
            ExprHandle a = module.attr(at);
            std::string attr_s = context.eval(module, a);
            std::string expr = context.eval(module, value);
            context.main_code += attr_s + " = " + expr + ";\n";
            break;
        }
        case ModifierKind::InheritAttribute: {  // attr.rs:173-186
            const Attribute at = (Attribute)param(self, 0);
            ExprHandle a = module.attr(at);
            context.main_code += context.eval(module, a) + " = parent_particle." + attribute_info(at).name + ";\n";
            break;
        }
        case ModifierKind::SetPositionCircle: {  // position.rs:52-109
            std::string fn = func_name("set_position_circle", self, mc);
            const bool volume = param(self, 0) == (uint32_t)ShapeDimension::Volume;
            context.make_fn(fn, module, [&](Module& m, ShaderWriter& ctx) {
                std::string center = ctx.eval(m, need(self, 0, "center"));
                std::string axis = ctx.eval(m, need(self, 1, "axis"));
                std::string radius = volume ? "const auto r = sqrt(frand()) * (" + ctx.eval(m, need(self, 2, "radius")) + ");"
                                            : "const auto r = " + ctx.eval(m, need(self, 2, "radius")) + ";";
                return "    const auto c = " + center + ";\n"
                       "    const auto n = " + axis + ";\n"
                       "    const auto sign = step(0.0f, n.z) * 2.0f - 1.0f;\n"
                       "    const auto a = -1.0f / (sign + n.z);\n"
                       "    const auto b = n.x * n.y * a;\n"
                       "    const auto tangent = vec3<f32>(1.0f + sign * n.x * n.x * a, sign * b, -sign * n.x);\n"
                       "    const auto bitangent = vec3<f32>(b, sign + n.y * n.y * a, -n.y);\n"
                       "    " + radius + "\n"
                       "    const auto theta = frand() * tau;\n"
                       "    const auto dir = tangent * cos(theta) + bitangent * sin(theta);\n"
                       "    (*particle)." + kPos + " = c + r * dir;\n";
            });
            context.main_code += fn + "(&particle, hnb_ctx);\n";
            break;
        }
        case ModifierKind::SetPositionSphere: {  // position.rs:152-211
            std::string fn = func_name("set_position_sphere", self, mc);
            const bool volume = param(self, 0) == (uint32_t)ShapeDimension::Volume;
            context.make_fn(fn, module, [&](Module& m, ShaderWriter& ctx) {
                std::string center = ctx.eval(m, need(self, 0, "center"));
                std::string radius = volume ? "const auto r = pow(frand(), 1.f/3.f) * (" + ctx.eval(m, need(self, 1, "radius")) + ");"
                                            : "const auto r = " + ctx.eval(m, need(self, 1, "radius")) + ";";
                return "    const auto c = " + center + ";\n"
                       "    " + radius + "\n"
                       "    const auto theta = frand() * tau;\n"
                       "    const auto z = frand() * 2.f - 1.f;\n"
                       "    const auto phi = acos(z);\n"
                       "    const auto sinphi = sin(phi);\n"
                       "    const auto x = sinphi * cos(theta);\n"
                       "    const auto y = sinphi * sin(theta);\n"
                       "    const auto dir = vec3<f32>(x, y, z);\n"
                       "    (*particle)." + kPos + " = c + r * dir;\n";
            });
            context.main_code += fn + "(&particle, hnb_ctx);\n";
            break;
        }
        case ModifierKind::SetPositionCone3d: {  // position.rs:267-325 (`dimension` is ignored by the reference too)
            std::string fn = func_name("set_position_cone3d", self, mc);
            context.make_fn(fn, module, [&](Module& m, ShaderWriter& ctx) {
                std::string height = ctx.eval(m, need(self, 0, "height"));
                std::string top_radius = ctx.eval(m, need(self, 2, "top_radius"));
                std::string base_radius = ctx.eval(m, need(self, 1, "base_radius"));
                return "    const auto h0 = " + height + ";\n"
                       "    const auto alpha_h = pow(frand(), 1.0f / 3.0f);\n"
                       "    const auto h = h0 * alpha_h;\n"
                       "    const auto rt = " + top_radius + ";\n"
                       "    const auto rb = " + base_radius + ";\n"
                       "    const auto r0 = rb + (rt - rb) * alpha_h;\n"
                       "    const auto alpha_r = sqrt(frand());\n"
                       "    const auto r = r0 * alpha_r;\n"
                       "    const auto theta = frand() * tau;\n"
                       "    const auto cost = cos(theta);\n"
                       "    const auto sint = sin(theta);\n"
                       "    const auto x = r * cost;\n"
                       "    const auto y = h;\n"
                       "    const auto z = r * sint;\n"
                       "    const auto p = vec3<f32>(x, y, z);\n"
                       "    const auto p2 = transform * vec4<f32>(p, 0.0f);\n"
                       "    (*particle)." + kPos + " = xyz(p2);\n";
            });
            context.main_code += fn + "(&particle, hnb_ctx);\n";
            break;
        }
        case ModifierKind::SetVelocityCircle: {  // velocity.rs:45-81
            std::string fn = func_name("set_velocity_circle", self, mc);
            context.make_fn(fn, module, [&](Module& m, ShaderWriter& ctx) {
                std::string center = ctx.eval(m, need(self, 0, "center"));
                std::string axis = ctx.eval(m, need(self, 1, "axis"));
                std::string speed = ctx.eval(m, need(self, 2, "speed"));
                return "    const auto delta = (*particle)." + std::string(kPos) + " - (" + center + ");\n"
                       "    const auto radial = normalize(delta - dot(delta, " + axis + ") * (" + axis + "));\n"
                       "    const auto radial_vec4 = transform * vec4<f32>(radial, 0.0f);\n"
                       "    (*particle)." + kVel + " = xyz(radial_vec4) * (" + speed + ");\n";
            });
            context.main_code += fn + "(&particle, hnb_ctx);\n";
            break;
        }
        case ModifierKind::SetVelocitySphere: {  // velocity.rs:124-139 (inline)
            std::string center = context.eval(module, need(self, 0, "center"));
            std::string speed = context.eval(module, need(self, 1, "speed"));
            context.main_code += std::string("particle.") + kVel + " = normalize(particle." + kPos + " - (" + center + ")) * (" + speed + ");\n";
            break;
        }
        case ModifierKind::SetVelocityTangent: {  // velocity.rs:188-224
            std::string fn = func_name("set_velocity_tangent", self, mc);
            context.make_fn(fn, module, [&](Module& m, ShaderWriter& ctx) {
                std::string origin = ctx.eval(m, need(self, 0, "origin"));
                std::string axis = ctx.eval(m, need(self, 1, "axis"));
                std::string speed = ctx.eval(m, need(self, 2, "speed"));
                return "    const auto radial = (*particle)." + std::string(kPos) + " - (" + origin + ");\n"
                       "    const auto tangent = normalize(cross(" + axis + ", radial));\n"
                       "    const auto tangent_vec4 = transform * vec4<f32>(tangent, 0.0f);\n"
                       "    (*particle)." + kVel + " = xyz(tangent_vec4) * (" + speed + ");\n";
            });
            context.main_code += fn + "(&particle, hnb_ctx);\n";
            break;
        }
        case ModifierKind::EmitSpawnEvent: {  // modifier/mod.rs:654-717
            const uint32_t condition = param(self, 0), channel = param(self, 1);
            if (channel >= 4) throw ExprError(ExprError::GraphEvalError, "at most 4 child event channels are supported");
            std::string count_val = context.eval(module, need(self, 0, "count"));
            std::string count_var = context.make_local_var();
            context.push_stmt("const auto " + count_var + " = " + count_val + ";");
            const std::string call = "hnb_append_spawn_events(hnb_ctx, " + std::to_string(channel) + "u, particle_index, u32(" + count_var + "));";
            if (condition == (uint32_t)EventEmitCondition::Always) context.main_code += "if (is_alive) { " + call + " }";
            else context.main_code += "if (was_alive && !is_alive) { " + call + " }";
            context.set_emits_gpu_spawn_events(true);
            break;
        }
    }
}

// ---- EffectAsset --------------------------------------------------------------------------------
void EffectAsset::add_modifier(ModifierContext ctx, const Modifier& m) {
    if (!((uint32_t)ctx & m.allowed_contexts())) throw ExprError(ExprError::InvalidModifierContext, "modifier cannot be used in this context");
    (ctx == ModifierContext::Init ? init_modifiers : update_modifiers).push_back(m);
}

ParticleLayout EffectAsset::particle_layout() const {
    std::set<Attribute> set;
    for (const auto& m : init_modifiers)
        for (Attribute a : m.attributes()) set.insert(a);
    for (const auto& m : update_modifiers)
        for (Attribute a : m.attributes()) set.insert(a);
    module.gather_attributes(set);
    return ParticleLayout::build(set);
}

EffectShaderSource EffectAsset::generate(const ParticleLayout* parent_layout, uint32_t num_event_bindings) const {
    EffectShaderSource out;
    out.particle_layout = particle_layout();
    if (out.particle_layout.size() == 0) throw ExprError(ExprError::Validate, "Asset " + name + " has invalid empty particle layout.");
    if (parent_layout && parent_layout->size() == 0) throw ExprError(ExprError::Validate, "Effect using asset " + name + " has invalid empty parent particle layout.");
    if (!out.particle_layout.contains(attr::POSITION))
        throw ExprError(ExprError::Validate, "The particle layout of asset '" + name + "' is missing the 'POSITION' attribute. Add a modifier using that attribute, for example the SetAttributeModifier.");
    if (out.particle_layout.contains(attr::RIBBON_ID) && !out.particle_layout.contains(attr::AGE))
        throw ExprError(ExprError::Validate, "The particle layout of asset '" + name + "' uses ribbons (has the 'RIBBON_ID' attribute), but is missing the 'AGE' attribute, which is mandatory for ribbons.");
    out.property_layout = property_layout();
    out.properties_struct = out.property_layout.generate_struct_body();
    out.num_event_bindings = num_event_bindings;
    if (parent_layout) out.parent_layout = *parent_layout;

    Module mod = module;  // modifiers append expressions while applying (lib.rs:1007)
    uint32_t flags = 0;
    if (simulation_space == SimulationSpace::Local) flags |= HNB_EFFECT_LOCAL_SPACE;
    if (parent_layout) flags |= HNB_EFFECT_READ_PARENT_PARTICLE;
    if (out.particle_layout.contains(attr::RIBBON_ID)) flags |= HNB_EFFECT_RIBBONS;  // lib.rs:1018-1019

    // init (lib.rs:1026-1069)
    bool consume = false;
    {
        ShaderWriter ctx(ModifierContext::Init, out.property_layout, out.particle_layout);
        for (const auto& m : init_modifiers) m.apply(mod, ctx);
        // SimulationSpace::eval (lib.rs:518-531); `transform[3].xyz` is the emitter translation
        if (simulation_space == SimulationSpace::Global) out.sim_space_code = "    particle.position += xyz(transform[3]);";
        consume = ctx.emits_gpu_spawn_events().value_or(false) || parent_layout != nullptr;
        out.init_code = ctx.main_code;
        out.init_extra = ctx.extra_code;
    }
    // update (lib.rs:1076-1133)
    bool emit = false;
    {
        ShaderWriter ctx(ModifierContext::Update, out.property_layout, out.particle_layout);
        for (const auto& m : update_modifiers) {
            m.apply(mod, ctx);
            for (Attribute a : m.update_writes()) out.update_writes.insert(a);
        }
        emit = ctx.emits_gpu_spawn_events().value_or(false);
        out.update_code = ctx.main_code;
        out.update_extra = ctx.extra_code;
    }
    if (consume) flags |= HNB_EFFECT_CONSUME_GPU_SPAWN_EVENTS;
    if (emit) flags |= HNB_EFFECT_EMIT_GPU_SPAWN_EVENTS;
    out.flags = flags;

    // Euler motion integration (lib.rs:1106-1133)
    const bool has_position = out.particle_layout.contains(attr::POSITION), has_velocity = out.particle_layout.contains(attr::VELOCITY);
    if (motion_integration != MotionIntegration::None && has_position && has_velocity) {
        const std::string code = "\nparticle.position += particle.velocity * sim_params.delta_time;\n";
        if (motion_integration == MotionIntegration::PreUpdate) out.update_code.insert(0, code);
        else out.update_code += code;
        out.update_writes.insert(attr::POSITION);
    }

    // aging / reaping (lib.rs:1223-1264)
    const bool has_age = out.particle_layout.contains(attr::AGE), has_lifetime = out.particle_layout.contains(attr::LIFETIME);
    // The lifetime is read only by the standard age and reap code below: no update modifier writes AGE or LIFETIME, and no
    // other update code mentions the lifetime (a textual test, so it errs on the side of leaving the flag off).
    out.lifetime_reap_only = has_age && has_lifetime && !out.update_writes.count(attr::AGE) && !out.update_writes.count(attr::LIFETIME) &&
                             out.update_code.find("lifetime") == std::string::npos && out.update_extra.find("lifetime") == std::string::npos;
    if (has_age) {
        if (has_lifetime) out.age_code += "\n    const bool was_alive = particle.age < particle.lifetime; (void)was_alive;";
        else out.age_code += "\n    const bool was_alive = true; (void)was_alive;";  // the reference leaves it undeclared (latent bug)
        out.age_code += "\n    particle.age = particle.age + sim_params.delta_time;";
        out.update_writes.insert(attr::AGE);
        if (has_lifetime) out.age_code += "\n    is_alive = particle.age < particle.lifetime;";
    } else {
        out.age_code = "\n    const bool was_alive = true; (void)was_alive;\n    is_alive = true;";
    }
    if (has_age && has_lifetime) out.reap_code = "is_alive = is_alive && (particle.age < particle.lifetime);";
    return out;
}

}  // namespace hnb_graph
