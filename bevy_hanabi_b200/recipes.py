"""Effect recipes of the BASELINE.json configs (SURVEY.md §8d), expressed through the authoring API.

``c5_lowered()`` is additionally available as a hand-lowered description (the exact code
EffectShaderSources::generate emits for config C5, SURVEY.md Appendix E, transliterated to CUDA C) so
that the runtime can be exercised independently of the expression compiler.
"""
from __future__ import annotations

from . import _native as N
from .runtime import AttrField, LoweredEffect

C5_STRIDE = 32
C5_ATTRS = [
    AttrField("position", N.VEC3, 0),
    AttrField("age", N.FLOAT, 12),
    AttrField("velocity", N.VEC3, 16),
    AttrField("lifetime", N.FLOAT, 28),
]


def c5_lowered(relaxed_order: bool = False, slot_order: bool = False) -> LoweredEffect:
    """Config C5: attrs {POSITION, VELOCITY, AGE, LIFETIME}; update [Accel((0,-9.8,0)), LinearDrag(0.5)];
    MotionIntegration::PostUpdate. Statement order as in SURVEY.md Appendix E."""
    return LoweredEffect(
        name="c5_accel_drag",
        attrs=C5_ATTRS,
        particle_stride=C5_STRIDE,
        init_code=(
            "    particle.position = vec3<f32>(0.f,0.f,0.f);\n"
            "    particle.velocity = vec3<f32>(0.f,0.f,0.f);\n"
            "    particle.age = 0.f;\n"
            "    particle.lifetime = 1.f;\n"),
        age_code=(
            "    const bool was_alive = particle.age < particle.lifetime; (void)was_alive;\n"
            "    particle.age = particle.age + sim_params.delta_time;\n"
            "    is_alive = particle.age < particle.lifetime;"),
        reap_code="    is_alive = is_alive && (particle.age < particle.lifetime);",
        update_code=(
            "    particle.velocity += (vec3<f32>(0.f,-9.8f,0.f)) * sim_params.delta_time;"
            "particle.velocity *= max(0.f, (1.f) - ((0.5f) * (sim_params.delta_time)));\n"
            "particle.position += particle.velocity * sim_params.delta_time;\n"),
        flags=(N.EFFECT_RELAXED_ORDER if relaxed_order else 0) | (N.EFFECT_SLOT_ORDER if slot_order else 0),
    )


def c5_generated_source() -> str:
    return c5_lowered().generate_source()


def c5_asset(capacity: int):
    """Config C5 authored through the public API (the path a Hanabi user takes): the same update and init code as
    `c5_lowered()` (tests/test_authoring_cpu.py), plus the lowering's write set: LIFETIME is declared
    HNB_ATTR_UPDATE_READ_ONLY, so its column plan is [0,16) [16,24) [24,28) [28,32) where `c5_lowered()`, which declares
    no write set, keeps the default cut."""
    from . import graph as G
    w = G.ExprWriter()
    A = G.Attribute
    zero = w.lit(G.Vec3(0., 0., 0.))
    return (G.EffectAsset(capacity, w.finish(), name="c5_accel_drag")
            .init(G.SetAttributeModifier(A.POSITION, zero)).init(G.SetAttributeModifier(A.VELOCITY, zero))
            .init(G.SetAttributeModifier(A.AGE, w.lit(0.))).init(G.SetAttributeModifier(A.LIFETIME, w.lit(1.)))
            .update(G.AccelModifier(w.lit(G.Vec3(0., -9.8, 0.)))).update(G.LinearDragModifier(w.lit(0.5))))
