// hanabi_graph.h — Level-2 authoring layer: the C++ counterpart of the reference's
//   src/graph/{mod,expr}.rs   (Value, Module, Expr, operators, EvalContext)
//   src/attributes.rs         (Attribute set, ParticleLayout)
//   src/properties.rs         (Property, PropertyLayout, serialization)
//   src/modifier/*.rs         (init/update modifiers)
//   src/asset.rs + src/lib.rs (EffectAsset, EffectShaderSources::generate)
// with one difference: expressions and modifiers lower to CUDA C (compiled by NVRTC into the kernel
// templates of csrc/kernels) instead of WGSL. It is pure CPU code with no CUDA dependency.
#pragma once
#include <cstdint>
#include <map>
#include <memory>
#include <optional>
#include <set>
#include <stdexcept>
#include <string>
#include <vector>

namespace hnb_graph {

// ---------------------------------------------------------------------------------------------
// Errors (ExprError, reference src/graph/expr.rs:~820)
// ---------------------------------------------------------------------------------------------
struct ExprError : std::runtime_error {
    enum Kind { TypeError, SyntaxError, GraphEvalError, PropertyError, InvalidExprHandleError, InvalidModifierContext, Validate };
    Kind kind;
    ExprError(Kind k, const std::string& m) : std::runtime_error(m), kind(k) {}
};

// ---------------------------------------------------------------------------------------------
// Value types (reference src/attributes.rs:152-507). The numeric code equals hnb_value_type.
// ---------------------------------------------------------------------------------------------
enum class ScalarType : uint8_t { Bool = 0, Float = 1, Int = 2, Uint = 3 };

struct ValueType {
    uint32_t code = 1;  // hnb_value_type
    ValueType() = default;
    explicit ValueType(uint32_t c) : code(c) {}
    static ValueType scalar(ScalarType s) { return ValueType((uint32_t)s); }
    static ValueType vector(ScalarType s, int count);
    static ValueType matrix(int n) { return ValueType(16u + (uint32_t)(n - 2)); }
    static ValueType matrix(int cols, int rows);  // matCxR<f32>, MatrixType::new(cols, rows) (attributes.rs:358-362)
    bool is_scalar() const { return code < 4; }
    bool is_vector() const { return code >= 4 && code < 16; }
    bool is_matrix() const { return code >= 16; }
    bool is_valid() const { return code <= 24; }
    ScalarType elem() const;
    int cols() const;               // matrices only
    int rows() const;
    int count() const;              // number of 32-bit components (matrix: cols*rows, packed column-major)
    uint32_t size() const;          // WGSL rules; a matrix is array<vecR, C>: matCx3 and matCx4 have the same size (attributes.rs:377-386)
    uint32_t align() const;         // WGSL rules: vec2 8, vec3/vec4 16, scalar 4, matrix = AlignOf(vecR)
    std::string to_cuda_string() const;  // "f32", "vec3<f32>", ...
    bool operator==(const ValueType& o) const { return code == o.code; }
    bool operator!=(const ValueType& o) const { return code != o.code; }
};
static const ValueType FLOAT = ValueType(1), INT = ValueType(2), UINT = ValueType(3), BOOL = ValueType(0);
static const ValueType VEC2F = ValueType(7), VEC3F = ValueType(8), VEC4F = ValueType(9);

// A constant (reference src/graph/mod.rs Value): up to 16 32-bit lanes. Bools are stored as 0 / 0xFFFFFFFF
// (reference graph/mod.rs:103-109).
struct Value {
    ValueType type;
    uint32_t bits[16] = {};
    static Value from_f32(float f);
    static Value from_words(ValueType t, const uint32_t* words);
    float f(int i) const;
    int32_t i(int i) const { return (int32_t)bits[i]; }
    std::string to_cuda_string() const;  // literal text, ToWgslString analogue (reference src/lib.rs:264-430)
};
// f32 literal: Rust `{:.6}` then trailing zeros trimmed (reference src/lib.rs:264-269), plus the C `f` suffix.
std::string f32_to_cuda_string(float f);

// ---------------------------------------------------------------------------------------------
// Attributes and particle layout (reference src/attributes.rs)
// ---------------------------------------------------------------------------------------------
struct AttributeInfo {
    const char* name;
    ValueType type;
    Value default_value;
};
// Index into the table of the 39 built-in attributes (reference attributes.rs:1338-1378), same order.
using Attribute = int;
int attribute_count();
const AttributeInfo& attribute_info(Attribute a);
Attribute attribute_by_name(const std::string& name);  // -1 if unknown
namespace attr {
extern const Attribute ID, PARTICLE_COUNTER, POSITION, VELOCITY, AGE, LIFETIME, COLOR, HDR_COLOR, ALPHA, SIZE, SIZE2, SIZE3,
    PREV, NEXT, AXIS_X, AXIS_Y, AXIS_Z, SPRITE_INDEX, RIBBON_ID;
}

struct AttributeLayout {
    std::string name;  // padding entries are named pad0..pad4
    ValueType type;
    uint32_t offset;
    bool is_pad;
};
// ParticleLayoutBuilder::build (reference attributes.rs:1516-1670): WGSL-compatible AoS packing.
struct ParticleLayout {
    std::vector<AttributeLayout> layout;  // includes pads, in offset order
    uint32_t align = 4;
    static ParticleLayout build(const std::set<Attribute>& attrs);
    uint32_t size() const;              // bytes incl. trailing pad
    uint32_t min_binding_size() const { return size(); }
    bool contains(Attribute a) const;
    std::optional<uint32_t> byte_offset(Attribute a) const;
};

// ---------------------------------------------------------------------------------------------
// Properties (reference src/properties.rs)
// ---------------------------------------------------------------------------------------------
struct Property {
    std::string name;
    Value default_value;
};
struct PropertyLayoutEntry {
    Property property;
    uint32_t offset;
};
struct PropertyLayout {
    std::vector<PropertyLayoutEntry> layout;
    static PropertyLayout make(const std::vector<Property>& props);  // PropertyLayout::new (properties.rs:561-699)
    bool empty() const { return layout.empty(); }
    uint32_t cpu_size() const;
    uint32_t align() const;
    uint32_t min_binding_size() const;  // cpu_size rounded up to align
    bool contains(const std::string& name) const;
    std::optional<uint32_t> offset(const std::string& name) const;
    // Body of `struct Properties { ... }` in CUDA C with explicit padding words so that field offsets
    // equal the layout's (generate_property_struct_code analogue).
    std::string generate_struct_body() const;
    // EffectProperties::serialize (properties.rs:437-453): blob of cpu_size() bytes.
    std::vector<uint8_t> serialize(const std::vector<std::pair<std::string, Value>>& values) const;
};

// ---------------------------------------------------------------------------------------------
// Expressions (reference src/graph/expr.rs)
// ---------------------------------------------------------------------------------------------
using ExprHandle = uint32_t;      // 1-based, 0 = invalid
using PropertyHandle = uint32_t;  // 1-based

enum class BuiltInOperator : uint8_t { Time, DeltaTime, VirtualTime, VirtualDeltaTime, RealTime, RealDeltaTime, Rand, AlphaCutoff, IsAlive };
enum class UnaryOperator : uint8_t {
    Abs, Acos, Asin, Atan, All, Any, Ceil, Cos, Exp, Exp2, Floor, Fract, InvSqrt, Length, Log, Log2, Normalize,
    Pack4x8snorm, Pack4x8unorm, Round, Saturate, Sign, Sin, Sqrt, Tan, Unpack4x8snorm, Unpack4x8unorm, W, X, Y, Z
};
enum class BinaryOperator : uint8_t {
    Add, Atan2, Cross, Distance, Div, Dot, GreaterThan, GreaterThanOrEqual, LessThan, LessThanOrEqual, Max, Min, Mul,
    Remainder, Step, Sub, UniformRand, NormalRand, Vec2, Vec4XyzW
};
enum class TernaryOperator : uint8_t { Mix, Clamp, SmoothStep, Vec3 };

struct Expr {
    enum Kind : uint8_t { BuiltIn, Literal, Property, Attribute, ParentAttribute, Unary, Binary, Ternary, Cast } kind;
    BuiltInOperator builtin = BuiltInOperator::Time;
    ValueType type;          // Rand value type / Cast target
    Value literal;
    PropertyHandle property = 0;
    hnb_graph::Attribute attribute = 0;
    uint8_t op = 0;          // Unary/Binary/Ternary operator
    ExprHandle a = 0, b = 0, c = 0;
};

enum class ModifierContext : uint8_t { Init = 1, Update = 2, Render = 4 };

class Module;
// EvalContext + ShaderWriter (reference src/modifier/mod.rs:198-367)
class ShaderWriter {
  public:
    std::string main_code, extra_code;
    const PropertyLayout& property_layout;
    const ParticleLayout& particle_layout;
    ShaderWriter(ModifierContext ctx, const PropertyLayout& pl, const ParticleLayout& pal, bool attribute_pointer = false)
        : property_layout(pl), particle_layout(pal), context_(ctx), is_attribute_pointer_(attribute_pointer) {}
    ModifierContext modifier_context() const { return context_; }
    bool is_attribute_pointer() const { return is_attribute_pointer_; }
    // Evaluate through the per-writer cache: an expression with side effects is emitted once (mod.rs:309-319)
    std::string eval(const Module& module, ExprHandle h);
    std::string make_local_var();
    void push_stmt(const std::string& stmt);
    // Emit `HNB_DI void name(Particle* particle, Ctx& hnb_ctx) { <stmts><body> }` into extra_code. The body
    // is produced with a fresh writer (fresh var counter and expression cache, attribute pointer mode).
    template <typename F> void make_fn(const std::string& func_name, Module& module, F&& f);
    void set_emits_gpu_spawn_events(bool use_events);
    std::optional<bool> emits_gpu_spawn_events() const { return emits_; }

  private:
    ModifierContext context_;
    uint32_t var_counter_ = 0;
    std::map<ExprHandle, std::string> expr_cache_;
    bool is_attribute_pointer_;
    std::optional<bool> emits_;
};

class Module {
  public:
    ExprHandle add_expr(const Expr& e);
    PropertyHandle add_property(const std::string& name, const Value& default_value);
    const Property* get_property(PropertyHandle h) const;
    PropertyHandle get_property_by_name(const std::string& name) const;
    const std::vector<Property>& properties() const { return properties_; }
    void gather_attributes(std::set<Attribute>& out) const;
    ExprHandle lit(const Value& v);
    ExprHandle lit(float f) { return lit(Value::from_f32(f)); }
    ExprHandle attr(Attribute a);
    ExprHandle parent_attr(Attribute a);
    ExprHandle prop(PropertyHandle p);
    ExprHandle builtin(BuiltInOperator op, ValueType rand_type = FLOAT);
    ExprHandle unary(UnaryOperator op, ExprHandle e);
    ExprHandle binary(BinaryOperator op, ExprHandle l, ExprHandle r);
    ExprHandle ternary(TernaryOperator op, ExprHandle a, ExprHandle b, ExprHandle c);
    ExprHandle cast(ExprHandle e, ValueType target);
    // shortcuts used by modifiers
    ExprHandle add(ExprHandle l, ExprHandle r) { return binary(BinaryOperator::Add, l, r); }
    ExprHandle sub(ExprHandle l, ExprHandle r) { return binary(BinaryOperator::Sub, l, r); }
    ExprHandle mul(ExprHandle l, ExprHandle r) { return binary(BinaryOperator::Mul, l, r); }
    ExprHandle dot(ExprHandle l, ExprHandle r) { return binary(BinaryOperator::Dot, l, r); }
    ExprHandle max(ExprHandle l, ExprHandle r) { return binary(BinaryOperator::Max, l, r); }
    ExprHandle lt(ExprHandle l, ExprHandle r) { return binary(BinaryOperator::LessThan, l, r); }
    ExprHandle gt(ExprHandle l, ExprHandle r) { return binary(BinaryOperator::GreaterThan, l, r); }
    ExprHandle abs(ExprHandle e) { return unary(UnaryOperator::Abs, e); }
    ExprHandle all(ExprHandle e) { return unary(UnaryOperator::All, e); }
    ExprHandle any(ExprHandle e) { return unary(UnaryOperator::Any, e); }

    const Expr& try_get(ExprHandle h) const;  // throws InvalidExprHandleError
    size_t size() const { return expressions_.size(); }
    bool is_const(ExprHandle h) const;
    bool has_side_effect(ExprHandle h) const;
    std::optional<ValueType> value_type(ExprHandle h) const;  // Expr::value_type: None for Unary/Binary/Ternary/Property
    // Expr::eval (expr.rs:1121-1258) lowered to CUDA C
    std::string eval_expr(ExprHandle h, ShaderWriter& ctx) const;

  private:
    std::vector<Expr> expressions_;
    std::vector<Property> properties_;
};

// ---------------------------------------------------------------------------------------------
// Modifiers (reference src/modifier/*.rs)
// ---------------------------------------------------------------------------------------------
enum class ModifierKind : uint32_t {
    Accel = 1, RadialAccel, TangentAccel, ConformToSphere, LinearDrag, KillSphere, KillAabb, SetAttribute, InheritAttribute,
    SetPositionCircle, SetPositionSphere, SetPositionCone3d, SetVelocityCircle, SetVelocitySphere, SetVelocityTangent,
    EmitSpawnEvent
};
enum class ShapeDimension : uint32_t { Surface = 0, Volume = 1 };
enum class EventEmitCondition : uint32_t { Always = 0, OnDie = 1 };

struct Modifier {
    ModifierKind kind;
    std::vector<ExprHandle> exprs;  // operand expressions, in the order of the reference struct's fields (0 = None)
    std::vector<uint32_t> params;   // kind-specific flags (attribute id, kill_inside, dimension, condition, child index)
    uint32_t allowed_contexts() const;          // bitmask of ModifierContext
    std::vector<Attribute> attributes() const;  // Modifier::attributes()
    std::vector<Attribute> update_writes() const;  // attributes the code apply() emits in the update context assigns
    void apply(Module& module, ShaderWriter& ctx) const;  // Modifier::apply, emitting CUDA C
};

// ---------------------------------------------------------------------------------------------
// Asset + code generation (reference src/asset.rs, src/lib.rs:805-1335)
// ---------------------------------------------------------------------------------------------
enum class SimulationSpace : uint32_t { Global = 0, Local = 1 };
enum class MotionIntegration : uint32_t { None = 0, PreUpdate = 1, PostUpdate = 2 };

struct EffectShaderSource {  // what generate() substitutes into the kernel templates
    ParticleLayout particle_layout;
    PropertyLayout property_layout;
    std::string properties_struct;
    std::string init_code, init_extra, sim_space_code, age_code, reap_code, update_code, update_extra;
    uint32_t flags = 0;  // HNB_EFFECT_* layout flags
    std::set<Attribute> update_writes;  // attributes the update body assigns; the others are HNB_ATTR_UPDATE_READ_ONLY
    bool lifetime_reap_only = false;    // LIFETIME gets HNB_ATTR_REAP_ONLY (see EffectAsset::generate)
    std::optional<ParticleLayout> parent_layout;
    uint32_t num_event_bindings = 0;
};

struct EffectAsset {
    std::string name;
    uint32_t capacity = 0;
    SimulationSpace simulation_space = SimulationSpace::Global;
    MotionIntegration motion_integration = MotionIntegration::PostUpdate;
    uint32_t prng_seed = 0;
    Module module;
    std::vector<Modifier> init_modifiers, update_modifiers;

    void add_modifier(ModifierContext ctx, const Modifier& m);  // EffectAsset::init / ::update
    ParticleLayout particle_layout() const;                      // asset.rs:605-626
    PropertyLayout property_layout() const { return PropertyLayout::make(module.properties()); }
    // EffectShaderSources::generate (lib.rs:805-1335) for the init and update passes.
    EffectShaderSource generate(const ParticleLayout* parent_layout, uint32_t num_event_bindings) const;
};

}  // namespace hnb_graph

// The C ABI's opaque module handle (include/hanabi_b200_graph.h), shared by graph_cabi.cpp and node_graph.cpp.
struct hnb_module {
    hnb_graph::Module m;
};
