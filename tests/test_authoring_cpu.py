"""CPU tests of the authoring / code-generation layer (no GPU): the counterpart of the reference's pure-CPU
unit tests and of its naga "the generated shader parses" validation tests (SURVEY.md §4):

  literal formatting        src/lib.rs:1925-1990
  expression text           src/graph/expr.rs:4219-4300 (same structure; CUDA surface syntax)
  particle layout packing   src/attributes.rs:2379-2521
  property layout           src/properties.rs:1010-1165, :1395-1422
  modifier validity         src/modifier/mod.rs:1066-1286 — here every modifier's generated translation
                            unit is compiled for sm_90a by NVRTC
  generated update body     src/lib.rs:2155-2308 / SURVEY.md Appendix E
"""
import re
import struct
from pathlib import Path

import numpy as np
import pytest

from bevy_hanabi_b200 import _native as N
from bevy_hanabi_b200 import graph as G
from bevy_hanabi_b200 import runtime as R
from bevy_hanabi_b200._native import HanabiError

A = G.Attribute


# ---- literals -------------------------------------------------------------------------------------
def test_f32_literal_formatting():
    assert G.format_f32(1.0) == "1.f"
    assert G.format_f32(-1.0) == "-1.f"
    assert G.format_f32(1.5) == "1.5f"
    assert G.format_f32(0.5) == "0.5f"
    assert G.format_f32(0.12345678) == "0.123457f"  # 6 digits, like the reference
    assert G.format_f32(1.0 / 3.0) == "0.333333f"
    assert G.format_f32(4e-7) == "0.f"               # constants below 5e-7 vanish (SURVEY App. D.1)
    assert G.format_f32(-9.8) == "-9.8f"


def test_vector_literals():
    m = G.Module()
    assert m.eval(m.lit(G.Vec2(1., 2.)))[0] == "vec2<f32>(1.f,2.f)"
    assert m.eval(m.lit(G.Vec3(1., 2., -1.)))[0] == "vec3<f32>(1.f,2.f,-1.f)"
    assert m.eval(m.lit(G.Vec4(1., 2., -1., 2.)))[0] == "vec4<f32>(1.f,2.f,-1.f,2.f)"
    assert m.eval(m.lit(G.U32(7)))[0] == "7u"
    assert m.eval(m.lit(G.I32(-3)))[0] == "-3"
    assert m.eval(m.lit(True))[0] == "true"
    assert m.eval(m.lit(G.UVec(1, 2, 3)))[0] == "vec3<u32>(1u,2u,3u)"
    assert m.eval(m.lit(G.IVec(1, -2)))[0] == "vec2<i32>(1,-2)"
    assert m.eval(m.lit((True, False, True)))[0] == "vec3<bool>(true,false,true)"


# ---- expressions ----------------------------------------------------------------------------------
def test_writer_expression_text():
    w = G.ExprWriter()
    my_prop = w.add_property("my_prop", 3.0)
    x = w.lit(3.).abs().max(w.attr(A.POSITION) * w.lit(2.)) + w.lit(-4.).min(w.prop(my_prop))
    s, stmts = w.finish().eval(x.expr())
    assert s == "(max(abs(3.f), (particle.position) * (2.f))) + (min(-4.f, properties[properties_array_index].my_prop))"
    assert stmts == ""


def test_binary_operator_formatting():
    m = G.Module()
    x = m.attr(A.POSITION)
    y = m.lit(G.Vec3(1., 1., 1.))
    for op, sym in [("add", "+"), ("sub", "-"), ("mul", "*"), ("div", "/"), ("lt", "<"), ("le", "<="), ("gt", ">"), ("ge", ">=")]:
        assert m.eval(m.binary(op, x, y))[0] == f"(particle.position) {sym} (vec3<f32>(1.f,1.f,1.f))"
    # `%` is WGSL's truncated remainder, also on floats: a function in C
    assert m.eval(m.rem(x, y))[0] == "hnb_rem(particle.position, vec3<f32>(1.f,1.f,1.f))"
    for op in ["max", "min", "dot", "cross", "distance", "step", "atan2"]:
        assert m.eval(m.binary(op, x, y))[0] == f"{op}(particle.position, vec3<f32>(1.f,1.f,1.f))"


def test_unary_ternary_cast_text():
    m = G.Module()
    x = m.attr(A.POSITION)
    assert m.eval(m.normalize(x))[0] == "normalize(particle.position)"
    assert m.eval(m.inverse_sqrt(m.lit(4.)))[0] == "inverseSqrt(4.f)"
    assert m.eval(m.x(x))[0] == "particle.position.x"
    a, b, c = m.lit(1.), m.lit(2.), m.lit(0.5)
    assert m.eval(m.mix(a, b, c))[0] == "mix(1.f, 2.f, 0.5f)"
    assert m.eval(m.clamp(a, b, c))[0] == "clamp(1.f, 2.f, 0.5f)"
    assert m.eval(m.smoothstep(a, b, c))[0] == "smoothstep(1.f, 2.f, 0.5f)"
    assert m.eval(m.vec3(a, b, c))[0] == "make_vec3(1.f, 2.f, 0.5f)"
    assert m.eval(m.vec2(a, b))[0] == "make_vec2(1.f, 2.f)"
    assert m.eval(m.vec4_xyz_w(x, a))[0] == "make_vec4(particle.position, 1.f)"
    assert m.eval(m.cast(a, G.VEC3))[0] == "vec3<f32>(1.f)"
    assert m.eval(m.cast(a, G.UINT))[0] == "u32(1.f)"
    with pytest.raises(HanabiError):  # vector -> scalar is not a valid cast (expr.rs:1468-1490)
        m.cast(x, G.FLOAT)


def test_fluent_operand_order():
    """x.step(edge) emits step(edge, x); x.smoothstep(lo, hi) emits smoothstep(lo, hi, x) (SURVEY App. D.11)."""
    w = G.ExprWriter()
    x = w.attr(A.AGE)
    m = w.module
    assert m.eval(x.step(0.5).expr())[0] == "step(0.5f, particle.age)"
    assert m.eval(x.smoothstep(0., 1.).expr())[0] == "smoothstep(0.f, 1.f, particle.age)"
    assert m.eval(x.mix(2., 0.25).expr())[0] == "mix(particle.age, 2.f, 0.25f)"


def test_builtins_and_pseudo_attributes():
    m = G.Module()
    assert m.eval(m.builtin("time"))[0] == "sim_params.time"
    assert m.eval(m.builtin("delta_time"))[0] == "sim_params.delta_time"
    assert m.eval(m.builtin("virtual_delta_time"))[0] == "sim_params.virtual_delta_time"
    assert m.eval(m.builtin("is_alive"))[0] == "is_alive"
    assert m.eval(m.attr(A.ID))[0] == "particle_index"
    assert m.eval(m.attr(A.PARTICLE_COUNTER))[0] == "particle_counter"
    assert m.eval(m.parent_attr(A.POSITION))[0] == "parent_particle.position"
    assert m.eval(m.parent_attr(A.ID))[0] == "parent_particle_index"


def test_side_effect_hoisting():
    """Rand expressions are hoisted once into a local (expr.rs:1812-1824) and cached per writer."""
    m = G.Module()
    r = m.builtin("rand", G.FLOAT)
    assert m.has_side_effect(r) and not m.is_const(r)
    e = m.add(m.mul(r, m.lit(2.)), r)
    s, stmts = m.eval(e)
    assert stmts == "const auto var0 = frand();\n"
    assert s == "((var0) * (2.f)) + (var0)"
    r3 = m.builtin("rand", G.VEC3)
    assert m.eval(r3) == ("var0", "const auto var0 = frand3();\n")
    u = m.uniform(m.lit(1.), m.lit(3.))
    assert m.eval(u) == ("var0", "const auto var0 = rand_uniform_f(1.f, 3.f);\n")
    uv = m.uniform(m.lit(G.Vec3(0, 0, 0)), m.lit(G.Vec3(1, 1, 1)))
    assert m.eval(uv)[1] == "const auto var0 = rand_uniform_vec3(vec3<f32>(0.f,0.f,0.f), vec3<f32>(1.f,1.f,1.f));\n"
    nv = m.normal(m.lit(0.), m.lit(1.))
    assert m.eval(nv)[1] == "const auto var0 = rand_normal_f(0.f, 1.f);\n"
    # operands of unknown type (a binary expression) are rejected like in the reference (expr.rs:1162-1198)
    bad = m.uniform(m.add(m.lit(1.), m.lit(1.)), m.lit(3.))
    with pytest.raises(HanabiError):
        m.eval(bad)
    with pytest.raises(HanabiError):  # mismatched operand types
        m.eval(m.uniform(m.lit(1.), m.lit(G.Vec3(1, 1, 1))))
    with pytest.raises(HanabiError):  # irand/urand/brand do not exist in vfx_common.wgsl
        m.eval(m.builtin("rand", G.UINT))
    assert m.is_const(m.add(m.lit(1.), m.lit(2.)))


def test_invalid_handles():
    m = G.Module()
    with pytest.raises(HanabiError):
        m.unary("abs", 12345)
    with pytest.raises(HanabiError):
        m.prop(3)


# ---- layouts --------------------------------------------------------------------------------------
def _lay(names):
    fields, size, align = G.particle_layout_of(names)
    return [(f.offset, f.name) for f in fields], size, align


def test_particle_layout_goldens():
    # [3, 1, 3, 2] -> [3 1 3 - 2 - -]   (attributes.rs:2464-2490)
    fields, size, align = _lay(["f32_0", "f32x3_0", "f32x2_0", "f32x3_1"])
    assert fields == [(0, "f32x3_0"), (12, "f32_0"), (16, "f32x3_1"), (28, "pad0"), (32, "f32x2_0"), (40, "pad1"), (44, "pad2")]
    assert (size, align) == (48, 16)
    # [1, 4, 3, 2, 2, 3] -> [4 3 1 2 2 3 -]   (attributes.rs:2491-2520)
    fields, size, align = _lay(["f32_0", "f32x4_0", "f32x3_0", "f32x2_0", "f32x2_1", "f32x3_1"])
    assert fields == [(0, "f32x4_0"), (16, "f32x3_0"), (28, "f32_0"), (32, "f32x2_0"), (40, "f32x2_1"), (48, "f32x3_1"), (60, "pad0")]
    assert (size, align) == (64, 16)
    # the default layout documented at attributes.rs:41-58
    fields, size, align = _lay(["position", "velocity", "age", "lifetime"])
    assert fields == [(0, "position"), (12, "age"), (16, "velocity"), (28, "lifetime")]
    assert (size, align) == (32, 16)
    # duplicates are removed; a lone scalar stays 4-byte aligned
    assert _lay(["age", "age"]) == ([(0, "age")], 4, 4)
    assert _lay(["size2"]) == ([(0, "size2")], 8, 8)
    assert _lay(["position"]) == ([(0, "position"), (12, "pad0")], 16, 16)
    # firework "trails": + color -> 48-byte stride (SURVEY §8d C2)
    fields, size, _ = _lay(["position", "velocity", "age", "lifetime", "color"])
    # scalars pair with the vec3s in alphabetical order: age, color, then lifetime alone + 3 pads
    assert size == 48 and fields == [(0, "position"), (12, "age"), (16, "velocity"), (28, "color"), (32, "lifetime"),
                                      (36, "pad0"), (40, "pad1"), (44, "pad2")]


def test_attribute_table():
    assert len(G.ATTRIBUTES) == 39
    assert A.POSITION.vt == G.VEC3 and A.LIFETIME.default.floats() == [1.0]
    assert A.COLOR.default.words == (0xFFFFFFFF,) and A.PREV.default.words == (0xFFFFFFFF,)
    assert A.AXIS_Y.default.floats() == [0.0, 1.0, 0.0] and A.HDR_COLOR.vt == G.VEC4
    assert A.SPRITE_INDEX.vt == G.INT and A.RIBBON_ID.vt == G.UINT
    assert [a.name for a in G.ATTRIBUTES[:6]] == ["id", "particle_counter", "position", "velocity", "age", "lifetime"]


def _asset_with_props(props):
    w = G.ExprWriter()
    for name, v in props:
        w.add_property(name, v)
    zero = w.lit(G.Vec3(0, 0, 0))
    return G.EffectAsset(16, w.finish()).init(G.SetAttributeModifier(A.POSITION, zero))


def test_property_layout_goldens():
    # layout_valid (properties.rs:1010-1050)
    a = _asset_with_props([("f32", 3.4), ("vec3", G.Vec3(0, 0, 0)), ("vec2", G.Vec2(0, -1)), ("vec4", G.Vec4(0, 1, 0, 0))])
    fields, size = a.property_layout()
    assert [(f.offset, f.name) for f in fields] == [(0, "vec4"), (16, "vec3"), (28, "f32"), (32, "vec2")]
    assert size == 48  # min_binding_size; cpu_size is 40
    # layout_padding_vec3 (properties.rs:1052-1090, regression #478)
    a = _asset_with_props([("vec4a", G.Vec4(0, 1, 0, 0)), ("vec3b", G.Vec3(0, 0, 0)), ("vec3c", G.Vec3(1, 1, 1))])
    fields, size = a.property_layout()
    assert [(f.offset, f.name) for f in fields] == [(0, "vec4a"), (16, "vec3b"), (32, "vec3c")]
    assert size == 48
    # tails: 3/3/2, 3/2, 2/1 (properties.rs layout_tail_*)
    a = _asset_with_props([("a", G.Vec3(0, 0, 0)), ("b", G.Vec3(0, 0, 0)), ("c", G.Vec2(0, 0))])
    assert [(f.offset, f.name) for f in a.property_layout()[0]] == [(0, "a"), (16, "b"), (32, "c")]
    a = _asset_with_props([("a", G.Vec3(0, 0, 0)), ("c", G.Vec2(0, 0))])
    assert [(f.offset, f.name) for f in a.property_layout()[0]] == [(0, "a"), (16, "c")]
    a = _asset_with_props([("c", G.Vec2(0, 0)), ("s", 1.0)])
    assert [(f.offset, f.name) for f in a.property_layout()[0]] == [(0, "c"), (8, "s")]


def test_property_serialize():
    a = _asset_with_props([("f32", 3.4), ("vec3", G.Vec3(1, 2, 3)), ("vec4", G.Vec4(0, 1, 0, 0))])
    blob = a.serialize_properties({"f32": 7.5})
    assert len(blob) == 32  # vec4 | vec3 + f32
    words = struct.unpack("<8f", blob)
    assert words[0:4] == (0, 1, 0, 0) and words[4:7] == (1, 2, 3) and words[7] == 7.5
    with pytest.raises(HanabiError):
        a.serialize_properties({"nope": 1.0})


# ---- code generation ------------------------------------------------------------------------------
def _c5_asset():
    w = G.ExprWriter()
    accel, drag, zero = w.lit(G.Vec3(0., -9.8, 0.)), w.lit(0.5), w.lit(G.Vec3(0, 0, 0))
    return (G.EffectAsset(1024, w.finish(), name="c5")
            .init(G.SetAttributeModifier(A.POSITION, zero)).init(G.SetAttributeModifier(A.VELOCITY, zero))
            .init(G.SetAttributeModifier(A.AGE, w.lit(0.))).init(G.SetAttributeModifier(A.LIFETIME, w.lit(1.)))
            .update(G.AccelModifier(accel)).update(G.LinearDragModifier(drag)))


def test_generated_update_body_matches_appendix_e():
    fx = _c5_asset().generate()
    assert fx.update_code == ("particle.velocity += (vec3<f32>(0.f,-9.8f,0.f)) * sim_params.delta_time;"
                              "particle.velocity *= max(0.f, (1.f) - ((0.5f) * (sim_params.delta_time)));\n"
                              "particle.position += particle.velocity * sim_params.delta_time;\n")
    assert "particle.age = particle.age + sim_params.delta_time;" in fx.age_code
    assert "is_alive = particle.age < particle.lifetime;" in fx.age_code
    assert fx.reap_code == "is_alive = is_alive && (particle.age < particle.lifetime);"
    assert fx.sim_space_code.strip() == "particle.position += xyz(transform[3]);"
    assert fx.particle_stride == 32 and [(a.name, a.offset) for a in fx.attrs] == [("position", 0), ("age", 12), ("velocity", 16), ("lifetime", 28)]
    pre = _c5_asset().with_motion_integration(G.MOTION_PRE_UPDATE).generate().update_code
    assert pre.startswith("\nparticle.position += particle.velocity * sim_params.delta_time;\n")
    none = _c5_asset().with_motion_integration(G.MOTION_NONE).generate().update_code
    assert "particle.position +=" not in none
    assert _c5_asset().with_simulation_space(G.LOCAL).generate().sim_space_code == ""


def test_generate_validation_errors():
    w = G.ExprWriter()
    asset = G.EffectAsset(8, w.finish()).init(G.SetAttributeModifier(A.AGE, w.lit(0.)))
    with pytest.raises(HanabiError) as e:  # POSITION is mandatory (lib.rs:836-843)
        asset.generate()
    assert "POSITION" in str(e.value)
    w = G.ExprWriter()
    with pytest.raises(HanabiError) as e:  # SetAttribute type check (attr.rs:97-113)
        G.EffectAsset(8, w.finish()).init(G.SetAttributeModifier(A.POSITION, w.lit(1.))).generate()
    assert "Mismatching expression type" in str(e.value)
    w = G.ExprWriter()
    with pytest.raises(HanabiError):  # ID is read-only (attr.rs:80-89)
        G.EffectAsset(8, w.finish()).init(G.SetAttributeModifier(A.ID, w.lit(G.U32(1))))._native()
    w = G.ExprWriter()
    with pytest.raises(HanabiError):  # update-only modifier in the init context
        G.EffectAsset(8, w.finish()).init(G.AccelModifier(w.lit(G.Vec3(0, 0, 0))))._native()


def _all_modifier_assets():
    """One asset per simulation modifier, operands exercising literals, properties, attributes and rand."""
    def base(w):
        return [G.SetAttributeModifier(A.POSITION, w.lit(G.Vec3(0, 0, 0))), G.SetAttributeModifier(A.VELOCITY, w.lit(G.Vec3(0, 1, 0))),
                G.SetAttributeModifier(A.AGE, w.lit(0.)), G.SetAttributeModifier(A.LIFETIME, w.rand(G.FLOAT) * w.lit(2.) + w.lit(1.))]
    out = {}
    def mk(name, init_extra=(), update=()):
        w = G.ExprWriter()
        mods_i, mods_u = init_extra(w) if callable(init_extra) else [], update(w) if callable(update) else []
        a = G.EffectAsset(64, w.module, name=name)
        for m in base(w) + mods_i:
            a.init(m)
        for m in mods_u:
            a.update(m)
        out[name] = a
    c = lambda w: w.lit(G.Vec3(0.5, -1., 2.))
    mk("accel", update=lambda w: [G.AccelModifier(w.lit(G.Vec3(0, -9.8, 0)))])
    mk("accel_prop", update=lambda w: [G.AccelModifier(w.prop(w.add_property("g", G.Vec3(0, -3, 0))) * w.time())])
    mk("radial", update=lambda w: [G.RadialAccelModifier(c(w), w.lit(2.5))])
    mk("tangent", update=lambda w: [G.TangentAccelModifier(c(w), w.lit(G.Vec3(0, 1, 0)), w.lit(1.5))])
    mk("conform", update=lambda w: [G.ConformToSphereModifier(c(w), w.lit(1.5), w.lit(10.), w.lit(5.), w.lit(2.))])
    mk("conform_full", update=lambda w: [G.ConformToSphereModifier(c(w), w.lit(1.5), w.lit(10.), w.lit(5.), w.lit(2.), w.lit(0.2), w.lit(3.))])
    mk("drag", update=lambda w: [G.LinearDragModifier(w.lit(0.7))])
    mk("kill_sphere", update=lambda w: [G.KillSphereModifier(c(w), w.lit(4.), False), G.KillSphereModifier(c(w), w.lit(0.01), True)])
    mk("kill_aabb", update=lambda w: [G.KillAabbModifier(c(w), w.lit(G.Vec3(3, 2, 3)), False), G.KillAabbModifier(c(w), w.lit(G.Vec3(.1, .1, .1)), True)])
    mk("set_attr_update", update=lambda w: [G.SetAttributeModifier(A.COLOR, w.attr(A.AGE).vec3(w.lit(0.), w.lit(1.)).vec4_xyz_w(w.lit(1.)).pack4x8unorm())])
    mk("pos_circle", init_extra=lambda w: [G.SetPositionCircleModifier(c(w), w.lit(G.Vec3(0, 0, 1)), w.lit(2.), G.VOLUME),
                                           G.SetPositionCircleModifier(c(w), w.lit(G.Vec3(0, 1, 0)), w.lit(2.), G.SURFACE)])
    mk("pos_sphere", init_extra=lambda w: [G.SetPositionSphereModifier(c(w), w.lit(2.), G.VOLUME), G.SetPositionSphereModifier(c(w), w.rand() + w.lit(1.), G.SURFACE)])
    mk("pos_cone", init_extra=lambda w: [G.SetPositionCone3dModifier(w.lit(3.), w.lit(1.), w.lit(0.2), G.VOLUME)])
    mk("vel_circle", init_extra=lambda w: [G.SetVelocityCircleModifier(c(w), w.lit(G.Vec3(0, 0, 1)), w.lit(2.))])
    mk("vel_sphere", init_extra=lambda w: [G.SetVelocitySphereModifier(c(w), w.rand() * w.lit(0.2) + w.lit(0.1))])
    mk("vel_tangent", init_extra=lambda w: [G.SetVelocityTangentModifier(c(w), w.lit(G.Vec3(0, 0, 1)), w.lit(2.))])
    mk("emit_events", update=lambda w: [G.EmitSpawnEventModifier(G.ON_DIE, w.lit(G.U32(3)), 0), G.EmitSpawnEventModifier(G.ALWAYS, w.lit(G.U32(1)), 1)])
    mk("pos_sphere_update", update=lambda w: [G.SetPositionSphereModifier(c(w), w.lit(2.), G.SURFACE), G.SetPositionCone3dModifier(w.lit(3.), w.lit(1.), w.lit(0.2))])
    return out


@pytest.mark.parametrize("name", sorted(_all_modifier_assets().keys()))
def test_every_modifier_compiles_for_sm100a(name):
    """≙ validate_init / validate_update (modifier/mod.rs:1066-1286): the emitted code must be valid."""
    asset = _all_modifier_assets()[name]
    fx = asset.generate(num_event_bindings=2 if name == "emit_events" else 0)
    src = fx.generate_source()
    size, log = R.nvrtc_check(src)
    assert size > 0
    assert "error" not in log.lower()
    assert "bytes spill stores" in log and " 0 bytes spill stores" in log


def test_child_effect_compiles():
    """GPU-event child: READ_PARENT_PARTICLE + CONSUME_GPU_SPAWN_EVENTS, InheritAttribute (attr.rs:173-186)."""
    parent = _all_modifier_assets()["emit_events"]
    w = G.ExprWriter()
    child = (G.EffectAsset(256, w.module, name="child")
             .init(G.InheritAttributeModifier(A.POSITION))
             .init(G.SetAttributeModifier(A.VELOCITY, w.parent_attr(A.VELOCITY) * w.lit(0.5)))
             .init(G.SetAttributeModifier(A.AGE, w.lit(0.))).init(G.SetAttributeModifier(A.LIFETIME, w.lit(1.))))
    fx = child.generate(parent=parent)
    assert fx.flags & N.EFFECT_READ_PARENT_PARTICLE and fx.flags & N.EFFECT_CONSUME_GPU_SPAWN_EVENTS
    assert "particle.position = parent_particle.position;" in fx.init_code
    size, log = R.nvrtc_check(fx.generate_source())
    assert size > 0


def test_generated_source_rejects_bad_layouts():
    fx = R.LoweredEffect("bad", [R.AttrField("position", N.VEC3, 0), R.AttrField("age", N.FLOAT, 8)], 16)
    with pytest.raises(HanabiError):  # overlapping fields
        fx.generate_source()
    with pytest.raises(HanabiError):
        R.LoweredEffect("bad", [R.AttrField("position", N.VEC3, 0)], 14).generate_source()


# ---- numpy oracle vs C oracle on the same effect (two independent restatements must agree) ----------
def test_numpy_oracle_equals_c_oracle_on_c5(orc):
    import ctypes as C
    from oracle.hanabi_oracle import EffectOracle
    from tests.helpers import Instance, RefWorld
    rng = np.random.default_rng(11)
    def world():
        w = RefWorld(3000, 8, [Instance(0, 1500, alive=1200, seed=5), Instance(1500, 1500, alive=900, seed=6)])
        for inst in w.instances:
            n = inst.alive
            p = np.zeros((n, 8), dtype=np.float32)
            p[:, 0:3] = r.uniform(-1, 1, (n, 3)); p[:, 4:7] = r.uniform(-1, 1, (n, 3)); p[:, 7] = r.uniform(0.02, 0.3, n)
            w.particles[inst.slab_offset:inst.slab_offset + n] = p.view(np.uint32)
        return w
    r = np.random.default_rng(11); a = world()
    r = np.random.default_rng(11); b = world()
    eo = EffectOracle(_c5_asset())
    k = (C.c_float * 4)(0.0, -9.8, 0.0, 0.5)
    for step in range(15):
        a.oracle_frame(orc, orc.orc_body_update_c5(), k)
        eo.frame(b, orc)
        np.testing.assert_array_equal(a.particles, b.particles, err_msg=f"step {step}")
        np.testing.assert_array_equal(a.indirect, b.indirect)
        np.testing.assert_array_equal(a.metadata_rows(), b.metadata_rows())
        np.testing.assert_array_equal(a.draw, b.draw)
    assert a.metadata[0].alive_count < 1200


def test_swizzle_of_infix_expression_is_parenthesised():
    """`(a * b).x`: the reference's text `(a) * (b).x` (expr.rs:1146 + :1209) swizzles only the right operand; the
    CUDA lowering takes the component of the whole product, as the node's value type declares."""
    w = G.ExprWriter()
    e = (w.attr(G.Attribute.VELOCITY) * w.lit(0.5)).x()
    asset = (G.EffectAsset(8, w.module).init(G.SetAttributeModifier(G.Attribute.POSITION, w.lit(G.Vec3(0, 0, 0))))
             .update(G.SetAttributeModifier(G.Attribute.F32_0, e)))
    code = asset.generate().update_code
    assert "particle.f32_0 = ((particle.velocity) * (0.5f)).x;" in code
    # swizzles of anything that is already a primary expression stay as the reference writes them
    w2 = G.ExprWriter()
    e2 = w2.attr(G.Attribute.VELOCITY).max(w2.attr(G.Attribute.POSITION)).y()
    a2 = (G.EffectAsset(8, w2.module).init(G.SetAttributeModifier(G.Attribute.POSITION, w2.lit(G.Vec3(0, 0, 0))))
          .update(G.SetAttributeModifier(G.Attribute.F32_0, e2)))
    assert "particle.f32_0 = max(particle.velocity, particle.position).y;" in a2.generate().update_code


def test_effect_properties_serialize_reference_vector():
    """properties.rs:1395-1421 `effect_properties_serialize`: {a: 3.0, b: Vec3::ONE} -> blob of cpu_size bytes with
    each value at its layout offset."""
    a = _asset_with_props([("a", 3.0), ("b", G.Vec3(1, 1, 1))])
    fields, size = a.property_layout()
    off = {f.name: f.offset for f in fields}
    assert off == {"b": 0, "a": 12} and size == 16   # vec3 first, the f32 pairs into its padding
    blob = a.serialize_properties()
    assert len(blob) == 16                            # cpu_size = offset of the last entry + its size
    assert blob[off["a"]:off["a"] + 4] == struct.pack("<f", 3.0)
    assert blob[off["b"]:off["b"] + 12] == struct.pack("<3f", 1.0, 1.0, 1.0)


def test_background_compile_job():
    """hnb_compile_job_*: the NVRTC step on its own thread, without a context (and without a GPU) — the reference
    compiles pipelines asynchronously too (spawn.rs:968-973). Several jobs run concurrently; a broken effect reports the
    compiler log; polling never blocks."""
    import time
    from bevy_hanabi_b200 import recipes
    from bevy_hanabi_b200 import runtime as R
    t0 = time.perf_counter()
    jobs = [R.CompileJob(recipes.c5_lowered()), R.CompileJob(_c5_asset().generate()), R.CompileJob(recipes.c5_lowered(relaxed_order=True))]
    started = time.perf_counter() - t0
    assert started < 0.25, "starting a job must not wait for the compiler"
    polls = 0
    while not all(j.poll() for j in jobs):
        polls += 1
        time.sleep(0.01)
        assert time.perf_counter() - t0 < 120
    assert polls > 0, "the compile really ran in the background"
    bad = recipes.c5_lowered()
    bad.update_code = "    this is not CUDA;"
    job = R.CompileJob(bad)
    with pytest.raises(HanabiError) as e:
        job.wait()
    assert e.value.code == N.HNB_ERR_NVRTC and "error" in e.value.message
    with pytest.raises(HanabiError):
        job.poll()
    for j in jobs + [job]:
        j.close()


def test_value_bytes_and_text_reference_vectors():
    """graph/mod.rs `as_bytes` (:1709-1760) and `to_wgsl_string` (:1905-1977): the byte images of scalar / vector values
    (through the property serialiser, which is where values become bytes on this path) and the literal text of the
    same inputs the reference formats (C literals here: the reference's text plus the `f` suffix)."""
    for value, fmt, expect in [
        (3.0, "<f", bytes([0, 0, 0x40, 0x40])),
        (G.U32(0x12FF89AC), "<I", bytes([0xAC, 0x89, 0xFF, 0x12])),
        (G.I32(0x12FF89AC), "<i", bytes([0xAC, 0x89, 0xFF, 0x12])),
        (G.Vec2(-2., 3.), "<2f", bytes([0, 0, 0, 0xC0, 0, 0, 0x40, 0x40])),
        (G.Vec3(-2., 3., 4.), "<3f", bytes([0, 0, 0, 0xC0, 0, 0, 0x40, 0x40, 0, 0, 0x80, 0x40])),
        (G.Vec4(-2., 3., 4., -5.), "<4f", bytes([0, 0, 0, 0xC0, 0, 0, 0x40, 0x40, 0, 0, 0x80, 0x40, 0, 0, 0xA0, 0xC0])),
    ]:
        blob = _asset_with_props([("v", value)]).serialize_properties({})
        assert blob[:len(expect)] == expect, (value, blob.hex())
        assert not any(blob[len(expect):])                      # the tail of the binding is zero padding

    m = G.Module()
    text = lambda v: m.eval(m.lit(v))[0]
    assert [G.format_f32(f) for f in (0., -1., 1., 1e-5)] == ["0.f", "-1.f", "1.f", "0.00001f"]
    assert [text(G.U32(u)) for u in (0, 1, 42, 999999)] == ["0u", "1u", "42u", "999999u"]
    assert [text(G.I32(i)) for i in (0, -1, 1, -42, 42, -100000, 100000)] == ["0", "-1", "1", "-42", "42", "-100000", "100000"]
    assert text(True) == "true" and text(False) == "false"
    assert text(G.Vec2(0., 0.)) == "vec2<f32>(0.f,0.f)" and text(G.Vec2(-1., -1.)) == "vec2<f32>(-1.f,-1.f)"
    assert text(G.Vec3(0., 0., -1.)) == "vec3<f32>(0.f,0.f,-1.f)"
    # f32(-42.578) = -42.57799911…, f32(663.449) = 663.44897460…, f32(-42558.35) = -42558.3515625 (a tie: both Rust
    # and glibc round it to even), f32(-4.2) = -4.19999980…: six decimals, trailing zeros trimmed
    assert text(G.Vec4(-42.578, 663.449, -42558.35, -4.2)) == "vec4<f32>(-42.577999f,663.448975f,-42558.351562f,-4.2f)"
    # magnitudes the reference prints in full ("{:.6}" never switches to an exponent)
    assert G.format_f32(1e20) == "100000002004087734272.f" and G.format_f32(100.0) == "100.f"
    assert G.format_f32(-0.0) == "-0.f" and G.format_f32(5.1e-7) == "0.000001f"


# ---- matrices (reference src/attributes.rs MatrixType :322-397, src/graph/mod.rs MatrixValue :1271-1470) ---------
def test_matrix_types_literals_and_bytes():
    m = G.Module()
    text = lambda v: m.eval(m.lit(v))[0]
    # graph/mod.rs `to_wgsl_string` (:1953-1976): components column by column (`mat3x3<f32>(1.,0.,…)` there)
    assert text(G.Mat3(1, 0, 0, 0, 1, 0, 0, 0, 1)) == "mat3x3f(1.f,0.f,0.f,0.f,1.f,0.f,0.f,0.f,1.f)"
    assert text(G.Mat3(*[0.] * 9)) == "mat3x3f(0.f,0.f,0.f,0.f,0.f,0.f,0.f,0.f,0.f)"
    assert text(G.Mat3((1., 2., 3.), (4., 5., 6.), (7., 8., 9.))) == "mat3x3f(1.f,2.f,3.f,4.f,5.f,6.f,7.f,8.f,9.f)"
    assert text(G.Mat(3, 2, [0., 1., 2., 1., 2., 3.])) == "mat3x2f(0.f,1.f,2.f,1.f,2.f,3.f)"      # MatrixValue::new doc example
    assert G.vt_matrix_dims(G.vt_matrix(3, 2)) == (3, 2) and G.vt_count(G.vt_matrix(4, 3)) == 12
    with pytest.raises(ValueError):
        G.Mat(5, 2, [0.] * 10)
    with pytest.raises(ValueError):
        G.Mat(2, 2, [0.] * 3)
    # `as_bytes` (:1746-1758): 16, 48 (= 3 x sizeof(vec4)) and 64 bytes; size / align of every matCxR (attributes.rs:377-397)
    for cols in (2, 3, 4):
        for rows in (2, 3, 4):
            value = G.Mat(cols, rows, [float(i + 1) for i in range(cols * rows)])
            blob = _asset_with_props([("m", value)]).serialize_properties({})
            assert len(blob) == cols * (8 if rows == 2 else 16)
            packed = struct.unpack(f"<{len(blob) // 4}f", blob)
            n = min(cols * rows, len(packed))
            assert packed[:n] == tuple(float(i + 1) for i in range(n)) and not any(packed[n:])   # the PACKED storage, zero tail
    # casts: matrix <-> matrix only (CastExpr::is_valid, expr.rs:1480-1508; tests `invalid_cast_*`, :4690-4720)
    x = m.lit(G.Mat4(*[0.] * 16))
    for target in (G.FLOAT, G.VEC3):
        with pytest.raises(HanabiError):
            m.cast(x, target)
    with pytest.raises(HanabiError):
        m.cast(m.lit(1.0), G.MAT3)
    with pytest.raises(HanabiError):
        m.cast(m.lit(G.Vec3(0, 0, 0)), G.vt_matrix(2, 4))
    assert m.eval(m.cast(x, G.MAT4))[0].startswith("mat4x4f(mat4x4f(")
    with pytest.raises(HanabiError):     # BuiltInOperator::Rand(ValueType::Matrix) panics in the reference (expr.rs:1700)
        m.builtin("rand", G.MAT3)


def test_matrix_property_layout_limits():
    """PropertyLayout::new (properties.rs:561-699) advances 16 bytes per property of 16 bytes or more: a mat2x2 is laid
    out like a vec4; a larger matrix only fits as the last entry. The reference would overlap the next field silently."""
    a = _asset_with_props([("twist", G.Mat2(1, 0, 0, 1)), ("tint", G.Vec4(1, 1, 1, 1)), ("basis", G.Mat4(*[0.] * 16))])
    fields, size = a.property_layout()
    assert [(f.offset, f.name) for f in fields] == [(0, "twist"), (16, "tint"), (32, "basis")] and size == 96
    assert "mat2x2f twist;" in a.generate().generate_source() and "mat4x4f basis;" in a.generate().generate_source()
    for bad in ([("basis", G.Mat4(*[0.] * 16)), ("gain", 1.0)],                       # a scalar lands inside the matrix
                [("a", G.Mat3(*[0.] * 9)), ("b", G.Mat4(*[0.] * 16))]):              # two large matrices
        with pytest.raises(HanabiError, match="overlaps the matrix property"):
            _asset_with_props(bad).generate()


def test_matrix_effect_compiles_for_sm100a():
    from tests.effects import matrix_asset
    src = matrix_asset(1024).generate().generate_source()
    assert "mat2x3f(1.f,0.5f,0.25f,-0.5f,1.f,2.f)" in src
    size, log = R.nvrtc_check(src)
    assert size > 0 and "error" not in log.lower() and " 0 bytes spill stores" in log


def test_writer_method_names_of_the_reference():
    """WriterExpr::{add,sub,mul,div,rem,normalized}, ExprWriter::{push,alpha_cutoff} (graph/expr.rs): same names, same text
    as the operator forms."""
    w = G.ExprWriter()
    v = w.attr(A.VELOCITY)
    named = v.add(v).sub(v).mul(w.lit(2.)).div(w.lit(3.)).rem(w.lit(1.)).normalized()
    infix = ((((v + v) - v) * w.lit(2.)) / w.lit(3.) % w.lit(1.)).normalize()
    assert w.module.eval(named.h)[0] == w.module.eval(infix.h)[0]
    assert w.module.eval(w.push(named).h)[0] == w.module.eval(named.h)[0]
    with pytest.raises(HanabiError, match="render-only"):
        w.module.eval(w.alpha_cutoff().h)


# ---- asset.rs: add_modifiers, test_apply_modifiers (simulation half), transitive_attr ------------------------
def test_asset_add_modifiers_contexts():
    """asset.rs:1191-1216 `add_modifiers`: SetAttributeModifier is accepted in the init and in the update context
    (the render context is outside the simulation path)."""
    for add in ("init", "update"):
        w = G.ExprWriter()
        asset = G.EffectAsset(8, w.module)
        getattr(asset, add)(G.SetAttributeModifier(A.POSITION, w.lit(G.Vec3(3., 3., 3.))))
        assert len(asset.init_modifiers) + len(asset.update_modifiers) == 1
        asset._native()   # hnb_asset_add_modifier checks Modifier::context() like EffectAsset::add_modifier
        names = [f.name for f in asset.particle_layout()[0]]
        assert "position" in names


def test_asset_apply_modifiers():
    """asset.rs:1218-1300 `test_apply_modifiers`, init and update contexts: every modifier applies without error on
    the asset, capacity is kept, and the generated translation unit compiles."""
    w = G.ExprWriter()
    origin, one = w.lit(G.Vec3(0., 0., 0.)), w.lit(1.)
    asset = (G.EffectAsset(4096, w.module, name="apply_modifiers")
             .init(G.SetPositionSphereModifier(w.lit(G.Vec3(0., 0., 0.)), w.lit(1.), G.VOLUME))
             .init(G.SetVelocitySphereModifier(w.lit(G.Vec3(0., 0., 0.)), w.lit(1.)))
             .init(G.SetAttributeModifier(A.AGE, one))
             .init(G.SetAttributeModifier(A.LIFETIME, one))
             .update(G.AccelModifier(w.lit(G.Vec3(1., 1., 1.))))          # AccelModifier::constant(module, Vec3::ONE)
             .update(G.LinearDragModifier(w.lit(3.5)))                    # LinearDragModifier::constant(module, 3.5)
             .update(G.ConformToSphereModifier(origin, one, one, one, one)))
    assert asset.capacity == 4096
    fx = asset.generate()
    for needle in ("particle.position", "particle.velocity", "particle.age", "particle.lifetime"):
        assert needle in fx.init_code + fx.init_extra
    assert "particle.velocity" in fx.update_code + fx.update_extra
    size, log = R.nvrtc_check(fx.generate_source())
    assert size > 0, log


def test_asset_transitive_attr():
    """asset.rs:1403-1413 `transitive_attr` (regression test for #440): an attribute only *read* by an expression
    is part of the particle layout, like the attribute the modifier writes."""
    w = G.ExprWriter()
    asset = G.EffectAsset(32, w.module).init(G.SetAttributeModifier(A.AGE, w.attr(A.F32_0)))
    names = [f.name for f in asset.particle_layout()[0]]
    assert "age" in names        # direct
    assert "f32_0" in names      # transitive


# ---- properties.rs: the EffectProperties store ------------------------------------------------------------------
def _three_props():
    return (G.EffectProperties()
            .with_properties([("a", 3.0), ("b", G.Vec3(0, 0, 0))])
            .with_properties([("a", 7.0), ("c", G.Vec2(1, 1))]))


def test_effect_properties_with_properties():
    """properties.rs:1166-1203: the second batch overwrites the *value* of `a`, keeps its default, appends `c`."""
    ep = _three_props()
    p = ep.properties()
    assert [x.name for x in p] == ["a", "b", "c"]
    assert p[0].default_value == G.Value.of(3.0) and p[0].value == G.Value.of(7.0)
    assert p[1].default_value == p[1].value == G.Vec3(0, 0, 0)
    assert p[2].default_value == p[2].value == G.Vec2(1, 1)


def test_effect_properties_type_mismatches():
    """properties.rs:1205-1211 `effect_properties_with_properties_type_mismatch`, :1243-1247
    `effect_properties_set_type_mismatch`: the reference panics, the C ABI reports and changes nothing."""
    ep = G.EffectProperties().with_properties([("a", 3.0)])
    with pytest.raises(HanabiError, match="Cannot assign value of type"):
        ep.with_properties([("a", G.Vec2(1, 1))])
    with pytest.raises(HanabiError, match="property 'a'"):
        ep.set("a", G.Vec3(0, 0, 0))
    assert ep.get_stored("a") == G.Value.of(3.0)


def test_effect_properties_get_stored_and_set():
    """properties.rs:1213-1241 `effect_properties_get_stored`, `effect_properties_set`."""
    ep = _three_props()
    assert ep.get_stored("a") is not None and ep.get_stored("b") is not None and ep.get_stored("c") is not None
    assert ep.get_stored("x") is None
    ep.set("a", 7.0)
    ep.set("x", 3.0)                      # unknown name: appended, default = the value
    assert ep.get_stored("x") == G.Value.of(3.0) and len(ep.properties()) == 4
    assert ep.set_if_changed("x", 3.0) is False and ep.set_if_changed("x", 4.0) is True
    assert ep.get_stored("x") == G.Value.of(4.0) and ep.properties()[3].default_value == G.Value.of(3.0)


def test_effect_properties_update_against_the_asset():
    """properties.rs:1249-1392 `effect_properties_update_{empty,added,removed,override,mixed}`; the returned flag is
    the `last_changed` tick those tests watch."""
    empty = _asset_with_props([])
    one = _asset_with_props([("prop1", 32.0)])
    two = _asset_with_props([("prop1", 32.0), ("prop2", False)])
    ep = G.EffectProperties()                                   # empty
    assert ep.update(empty) is False and ep.properties() == []
    ep = G.EffectProperties()                                   # added
    assert ep.update(one) is True
    assert [(p.name, p.default_value, p.value) for p in ep.properties()] == [("prop1", G.Value.of(32.0), G.Value.of(32.0))]
    ep = G.EffectProperties()                                   # removed
    ep.set("unknown", G.I32(3))
    assert ep.update(empty) is True and ep.properties() == []
    ep = G.EffectProperties()                                   # override: the runtime value wins, nothing changes
    ep.set("prop1", 5.0)
    assert ep.update(one) is False
    assert [(p.name, p.value) for p in ep.properties()] == [("prop1", G.Value.of(5.0))]
    ep = G.EffectProperties()                                   # mixed: one override, one default
    ep.set("prop1", 5.0)
    assert ep.update(two) is True
    p = ep.properties()
    assert [(x.name, x.value) for x in p] == [("prop1", G.Value.of(5.0)), ("prop2", G.Value.of(False))]
    assert p[1].default_value == G.Value.of(False)


def test_effect_properties_serialize_store():
    """properties.rs:1394-1421 `effect_properties_serialize` through the store, and the store against the asset-side
    serialiser: after update() both produce the same record."""
    a = _asset_with_props([("a", 3.0), ("b", G.Vec3(1, 1, 1))])
    ep = G.EffectProperties().with_properties([("a", 3.0), ("b", G.Vec3(1, 1, 1))])
    blob = ep.serialize(a)
    off = {f.name: f.offset for f in a.property_layout()[0]}
    assert blob[off["a"]:off["a"] + 4] == struct.pack("<f", 3.0)
    assert blob[off["b"]:off["b"] + 12] == struct.pack("<3f", 1.0, 1.0, 1.0)
    assert blob == a.serialize_properties()
    # a stored property the layout does not know is skipped; a missing one stays zero until update() adds its default
    ep2 = G.EffectProperties().with_properties([("zzz", 9.0)])
    assert ep2.serialize(a) == bytes(len(blob))
    ep2.update(a)
    ep2.set("a", 7.5)
    assert ep2.serialize(a) == a.serialize_properties({"a": 7.5})


def test_cast_validity_reference_cases():
    """graph/expr.rs:4681-4687 `invalid_cast_vector_to_scalar`, :4721-4740 `cast_expr_new`: vector -> scalar is
    rejected when the operand type is known; a cast of a property (type unknown to `is_valid`) is let through."""
    m = G.Module()
    with pytest.raises(HanabiError, match="invalid cast"):
        m.cast(m.lit(G.Vec2(1, 1)), G.FLOAT)
    x = m.attr(A.POSITION)
    assert m.cast(x, G.VEC3) != 0                               # Some(true)
    with pytest.raises(HanabiError, match="invalid cast"):
        m.cast(x, G.BOOL)                                       # Some(false)
    y = m.prop(m.add_property("my_prop", 3.0))
    assert m.cast(y, G.vt_matrix(2, 3)) != 0                    # None: not decidable at authoring time


def test_effect_asset_builder_names_of_the_reference():
    """asset.rs:430-600: with_name / with_simulation_condition / add_modifier / modifiers / properties."""
    w = G.ExprWriter()
    w.add_property("speed", 2.0)
    zero = w.lit(G.Vec3(0, 0, 0))
    a = (G.EffectAsset(32, w.module).with_name("named").with_simulation_condition(G.ALWAYS)
         .add_modifier("init", G.SetAttributeModifier(A.POSITION, zero))
         .add_modifier("update", G.AccelModifier(w.lit(G.Vec3(0, -1, 0)))))
    assert a.name == "named" and a.simulation_condition == G.ALWAYS
    assert [m.kind for m in a.modifiers()] == ["set_attribute", "accel"]
    assert a.properties() == [("speed", G.Value.of(2.0))]
    assert a.generate().name == "named"
    with pytest.raises(ValueError):
        a.add_modifier("render", G.AccelModifier(zero))


def test_value_splat():
    """graph/mod.rs:2350-2408 `splat`: VectorValue::splat for every scalar type and vector width."""
    for c in (2, 3, 4):
        b = G.Value.splat(True, c)
        assert G.vt_elem(b.vt) == "b" and G.vt_count(b.vt) == c and b == G.Value.of([True] * c)
        f = G.Value.splat(3.4, c)
        assert G.vt_elem(f.vt) == "f" and G.vt_count(f.vt) == c and f == G.Value.of([3.4] * c)
        i = G.Value.splat(G.I32(-46458), c)
        assert G.vt_elem(i.vt) == "i" and G.vt_count(i.vt) == c and i == G.IVec(*[-46458] * c)
        u = G.Value.splat(G.U32(46458), c)
        assert G.vt_elem(u.vt) == "u" and G.vt_count(u.vt) == c and u == G.UVec(*[46458] * c)
    with pytest.raises(ValueError):
        G.Value.splat(G.Vec2(1, 2), 2)
    with pytest.raises(ValueError):
        G.Value.splat(1.0, 5)
