"""GPU parity of authored effects (init + update, every simulation modifier, properties, transforms,
multi-instance batches, dead-slot recycling) against the numpy oracle, frame by frame.

Comparison rules (BASELINE.json north_star): metadata counters, draw-indirect counts, prefix sums, alive
lists (ping/pong) and the dead stack are compared bit-exactly; fp32 attributes bit-exactly when the effect
only uses IEEE-exact operations (+ - * / sqrt min max compare, the integer PRNG), and within 1e-5 relative
to the attribute's magnitude (tests/helpers.py::assert_float_attributes_close) when it goes through
sin/cos/acos/pow/log, whose last bits differ between CUDA's and numpy's libm.
"""
import numpy as np
import pytest

from bevy_hanabi_b200 import graph as G
from oracle.hanabi_oracle import pcg_hash
from tests.effects import firework_trails, force_field
from tests.helpers import Instance, Lockstep, RefWorld

pytestmark = pytest.mark.gpu
A = G.Attribute


# ---------------------------------------------------------------------------------------------------
def test_c1_single_particle_plumbing(ctx, orc):
    """BASELINE config C1 (gpu_tests/single_particle.rs:37-45): position = lit, size3 = lit, capacity 16, no age:
    particles never die; spawn requests beyond the free slots are dropped (vfx_init.wgsl:115-137)."""
    w = G.ExprWriter()
    asset = (G.EffectAsset(16, w.module, name="single_particle")
             .init(G.SetAttributeModifier(A.POSITION, w.lit(G.Vec3(0.1, 0.2, 0.3))))
             .init(G.SetAttributeModifier(A.SIZE3, w.lit(G.Vec3(10., 10., 10.)))))
    fields, size, _ = asset.particle_layout()
    ref = RefWorld(16, size // 4, [Instance(0, 16, alive=0, seed=0)])
    Lockstep(ctx, orc, ref, asset).run([[17 if f % 2 else 3] for f in range(40)])
    assert ref.metadata[0].alive_count == 16 and ref.metadata[0].max_spawn == 0
    assert ref.metadata[0].particle_counter == 16


def test_c2_firework_bursts_with_recycling(ctx, orc):
    """Bursts of 1000 every 20 frames at dt=1/20: particles live 16-24 frames, so dead slots are recycled by later
    bursts and the dead stack / alive lists are permuted. Every operation is IEEE-exact: zero tolerance."""
    asset = firework_trails(4096)
    _, size, _ = asset.particle_layout()
    assert size == 48
    ref = RefWorld(4096, size // 4, [Instance(0, 4096, alive=0)], dt=1.0 / 20.0)
    seeds = lambda n, f: [int(pcg_hash(np.array([0x1234 + f], dtype=np.uint32))[0])]
    Lockstep(ctx, orc, ref, asset, seeds=seeds).run([[1000 if f % 20 == 0 else 0] for f in range(70)])
    assert ref.metadata[0].particle_counter == 4000


def test_c2_relaxed_order_same_sets(ctx, orc):
    """HNB_EFFECT_RELAXED_ORDER (reference-style atomics): counts and per-segment index SETS must be identical."""
    asset = firework_trails(2048)
    ref = RefWorld(2048, 12, [Instance(0, 2048, alive=0)], dt=1.0 / 20.0)
    Lockstep(ctx, orc, ref, asset, relaxed=True).run([[700 if f % 12 == 0 else 0] for f in range(24)], check_every=3)


def test_c3_force_field(ctx, orc):
    asset = force_field(8192)
    _, size, _ = asset.particle_layout()
    ref = RefWorld(8192, size // 4, [Instance(0, 8192, alive=0, seed=77)])
    props = [{"attraction_accel": 18.0, "repulsor_position": G.Vec3(0.25, 0.5, 0.1)}]
    Lockstep(ctx, orc, ref, asset, rtol=1e-5, props=props).run([[5000 if f == 0 else (30 if f % 5 == 0 else 0)] for f in range(25)])


def test_fast_math_effects_stay_within_tolerance(ctx, orc):
    """HNB_EFFECT_FAST_MATH (FMA contraction, approximate division / square root): fp32 attributes within the 1e-5
    per-step bound of BASELINE.json, every integer structure still exact."""
    from bevy_hanabi_b200 import _native as N
    asset = force_field(8192)
    assert asset.generate(fast_math=True).flags & N.EFFECT_FAST_MATH
    _, size, _ = asset.particle_layout()
    ref = RefWorld(8192, size // 4, [Instance(0, 8192, alive=0, seed=77)])
    props = [{"attraction_accel": 18.0, "repulsor_position": G.Vec3(0.25, 0.5, 0.1)}]
    Lockstep(ctx, orc, ref, asset, rtol=1e-5, props=props, fast_math=True).run([[5000 if f == 0 else (30 if f % 5 == 0 else 0)] for f in range(25)])
    asset = firework_trails(4096)
    ref = RefWorld(4096, 12, [Instance(0, 4096, alive=0)], dt=1.0 / 20.0)
    Lockstep(ctx, orc, ref, asset, rtol=1e-5, fast_math=True).run([[1000 if f % 20 == 0 else 0] for f in range(30)])


def test_many_instances_properties_transforms(ctx, orc):
    """One batch of instances sharing an effect: per-instance seed, spawn count, property record and emitter
    translation (Global simulation space adds transform[3].xyz at init, lib.rs:525-528)."""
    w = G.ExprWriter()
    speed = w.add_property("speed", 1.0)
    tint = w.add_property("tint", G.U32(0))
    asset = (G.EffectAsset(300, w.module, name="instanced")
             .init(G.SetAttributeModifier(A.POSITION, w.rand(G.VEC3) * w.lit(2.) - w.lit(1.)))
             .init(G.SetAttributeModifier(A.VELOCITY, (w.rand(G.VEC3) - w.lit(0.5)) * w.prop(speed)))
             .init(G.SetAttributeModifier(A.AGE, w.lit(0.)))
             .init(G.SetAttributeModifier(A.LIFETIME, w.lit(0.3).uniform(w.lit(0.9))))
             .init(G.SetAttributeModifier(A.COLOR, w.prop(tint)))
             .init(G.SetAttributeModifier(A.U32_0, w.attr(A.PARTICLE_COUNTER)))
             .init(G.SetAttributeModifier(A.U32_1, w.attr(A.ID)))
             .update(G.AccelModifier(w.lit(G.Vec3(0., -2., 0.)) * w.prop(speed))))
    _, size, _ = asset.particle_layout()
    n_inst = 37
    insts = [Instance(i * 300, 300, alive=0, seed=1000 + i) for i in range(n_inst)]
    ref = RefWorld(n_inst * 300, size // 4, insts, dt=1.0 / 30.0)
    for i in range(n_inst):
        tr = list(ref.spawners[i].transform)
        tr[3], tr[7], tr[11] = float(i), -0.5 * i, 2.0  # translation = last element of each row
        for k in range(12):
            ref.spawners[i].transform[k] = tr[k]
    props = [{"speed": 0.5 + 0.25 * i, "tint": G.U32(0x01010101 * (i % 200))} for i in range(n_inst)]
    rng = np.random.default_rng(4)
    sched = [[int(x) for x in rng.integers(0, 40, n_inst)] for _ in range(45)]
    Lockstep(ctx, orc, ref, asset, props=props).run(sched, check_every=3)
    assert all(ref.metadata[i].particle_counter > 0 for i in range(n_inst))


def test_shapes_and_transformed_velocities(ctx, orc):
    """SetPosition{Circle,Cone3d} + SetVelocity{Circle,Tangent} under a rotated/scaled emitter transform,
    Radial/Tangent accel in update."""
    w = G.ExprWriter()
    axis = w.lit(G.Vec3(0., 0., 1.))
    center = w.lit(G.Vec3(0.5, -0.25, 0.))
    asset = (G.EffectAsset(3000, w.module, name="shapes", simulation_space=G.LOCAL)
             .init(G.SetPositionCircleModifier(center, axis, w.lit(2.), G.VOLUME))
             .init(G.SetVelocityTangentModifier(center, axis, w.lit(1.5)))
             .init(G.SetAttributeModifier(A.AGE, w.lit(0.)))
             .init(G.SetAttributeModifier(A.LIFETIME, w.lit(5.)))
             .update(G.RadialAccelModifier(center, w.lit(-0.5)))
             .update(G.TangentAccelModifier(center, axis, w.lit(0.25))))
    w2 = G.ExprWriter()
    asset2 = (G.EffectAsset(3000, w2.module, name="cone")
              .init(G.SetPositionCone3dModifier(w2.lit(3.), w2.lit(1.), w2.lit(0.25)))
              .init(G.SetVelocityCircleModifier(w2.lit(G.Vec3(0, 0, 0)), w2.lit(G.Vec3(0., 1., 0.)), w2.lit(0.1).uniform(w2.lit(2.))))
              .init(G.SetAttributeModifier(A.AGE, w2.lit(0.)))
              .init(G.SetAttributeModifier(A.LIFETIME, w2.lit(5.))))
    for a in (asset, asset2):
        _, size, _ = a.particle_layout()
        ref = RefWorld(3000, size // 4, [Instance(0, 3000, alive=0, seed=31337)])
        c, s = np.float32(np.cos(0.7)), np.float32(np.sin(0.7))
        rows = [1.5 * c, -1.5 * s, 0., 4.,   1.5 * s, 1.5 * c, 0., -1.,   0., 0., 0.5, 2.]
        for k in range(12):
            ref.spawners[0].transform[k] = rows[k]
        Lockstep(ctx, orc, ref, a, rtol=1e-5).run([[2000 if f == 0 else 100] for f in range(6)])


def test_expression_operators_end_to_end(ctx, orc):
    """A grab bag of expression operators evaluated on the GPU vs the oracle's interpreter."""
    w = G.ExprWriter()
    t = w.time()
    pos = w.attr(A.POSITION)
    e1 = (pos.x().abs().sqrt() + pos.y().fract() * w.lit(3.)).max(pos.z().floor()).min(w.lit(5.))
    e2 = pos.cross(w.lit(G.Vec3(0., 1., 0.))).length().mix(w.lit(2.), w.lit(0.25)).clamp(w.lit(0.), w.lit(1.5))
    e3 = pos.dot(pos).step(w.lit(0.5)) + (pos.x() % w.lit(0.3)) + pos.distance(w.lit(G.Vec3(1., 1., 1.))).smoothstep(w.lit(0.), w.lit(4.))
    packed = pos.vec4_xyz_w(w.lit(1.)).saturate().pack4x8unorm()
    asset = (G.EffectAsset(2000, w.module, name="ops")
             .init(G.SetAttributeModifier(A.POSITION, w.rand(G.VEC3) * w.lit(4.) - w.lit(2.)))
             .init(G.SetAttributeModifier(A.AGE, w.lit(0.)))
             .init(G.SetAttributeModifier(A.LIFETIME, w.lit(100.)))
             .update(G.SetAttributeModifier(A.F32_0, e1 + t))
             .update(G.SetAttributeModifier(A.F32_1, e2))
             .update(G.SetAttributeModifier(A.F32_2, e3))
             .update(G.SetAttributeModifier(A.U32_0, packed))
             .update(G.SetAttributeModifier(A.F32X4_0, w.attr(A.U32_0).unpack4x8unorm()))
             .update(G.SetAttributeModifier(A.F32X2_0, pos.x().vec2(pos.z()).sign() * w.lit(G.Vec2(2., 3.)))))
    _, size, _ = asset.particle_layout()
    ref = RefWorld(2000, size // 4, [Instance(0, 2000, alive=0, seed=5)])
    Lockstep(ctx, orc, ref, asset).run([[1500 if f == 0 else 0] for f in range(4)])


def test_transcendental_operators(ctx, orc):
    w = G.ExprWriter()
    x = w.attr(A.F32_0)
    asset = (G.EffectAsset(1500, w.module, name="transc")
             .init(G.SetAttributeModifier(A.POSITION, w.lit(G.Vec3(0, 0, 0))))
             .init(G.SetAttributeModifier(A.F32_0, w.rand() * w.lit(3.) + w.lit(0.01)))
             .update(G.SetAttributeModifier(A.F32_1, x.sin() + x.cos() * x.tan().atan()))
             .update(G.SetAttributeModifier(A.F32_2, x.exp().log() + x.exp2().log2() + (x * w.lit(0.3)).acos().asin()))
             .update(G.SetAttributeModifier(A.F32_3, x.atan2(w.lit(2.)) + w.lit(0.).normal(w.lit(1.)) + x.inverse_sqrt() + x.round() + x.ceil())))
    _, size, _ = asset.particle_layout()
    ref = RefWorld(1500, size // 4, [Instance(0, 1500, alive=0, seed=99)])
    Lockstep(ctx, orc, ref, asset, rtol=1e-5).run([[1500 if f == 0 else 0] for f in range(3)])
