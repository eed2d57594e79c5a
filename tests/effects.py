"""Effect recipes and constants shared by test modules and tools. The asset names and literals reach the generated
source, so they must not change unless the generated code is meant to."""
import ctypes as C

import numpy as np

from bevy_hanabi_b200 import graph as G
from oracle import c_oracle as O

A = G.Attribute

ACCEL_DRAG = (C.c_float * 4)(0.0, -9.8, 0.0, 0.5)  # the C oracle's constants of C5's update: Accel((0,-9.8,0)), LinearDrag(0.5)
EVENT_CAP = 256  # the reference hard-codes 256 events per child (event.rs:266-267)


def firework_trails(capacity):
    """BASELINE config C2 (examples/firework.rs:184-251 made parent-less, SURVEY §8d)."""
    w = G.ExprWriter()
    vel = (w.rand(G.VEC3) * w.lit(2.) - w.lit(1.)).normalize() * w.lit(40.).uniform(w.lit(60.))
    return (G.EffectAsset(capacity, w.module, name="firework_trails")
            .init(G.SetAttributeModifier(A.POSITION, w.lit(G.Vec3(0, 0, 0))))
            .init(G.SetAttributeModifier(A.VELOCITY, vel))
            .init(G.SetAttributeModifier(A.AGE, w.lit(0.)))
            .init(G.SetAttributeModifier(A.LIFETIME, w.lit(0.8).uniform(w.lit(1.2))))
            .init(G.SetAttributeModifier(A.COLOR, w.lit(G.U32(0xFFFFFFFF))))
            .update(G.LinearDragModifier(w.lit(4.)))
            .update(G.AccelModifier(w.lit(G.Vec3(0., -16., 0.)))))


def force_field(capacity, aabb_half=(3., 2., 3.), kill_center=(-2., 1., 0.), kill_r2=0.36):
    """BASELINE config C3 (examples/force_field.rs:126-203 scaled): sphere spawn, two ConformToSphere, two kills.
    (The kill volumes are parameters so that a test can make them bite within a few frames.)"""
    w = G.ExprWriter()
    attractor = w.add_property("attraction_accel", 20.0)
    repulsor = w.add_property("repulsor_position", G.Vec3(0.2, 0.6, 0.))
    m = (G.EffectAsset(capacity, w.module, name="force_field")
         .init(G.SetPositionSphereModifier(w.lit(G.Vec3(0, 0, 0)), w.lit(0.05), G.SURFACE))
         .init(G.SetVelocitySphereModifier(w.lit(G.Vec3(0, 0, 0)), w.rand() * w.lit(0.2) + w.lit(0.1)))
         .init(G.SetAttributeModifier(A.AGE, w.lit(0.)))
         .init(G.SetAttributeModifier(A.LIFETIME, w.lit(10.)))
         .update(G.ConformToSphereModifier(w.prop(repulsor), w.lit(0.2), w.lit(0.4), w.lit(-10.), w.lit(-2.), w.lit(0.1), w.lit(2.)))
         .update(G.ConformToSphereModifier(w.lit(G.Vec3(0.6, -0.2, 0.)), w.lit(0.3), w.lit(30.), w.prop(attractor), w.lit(5.)))
         .update(G.KillAabbModifier(w.lit(G.Vec3(0, 0, 0)), w.lit(G.Vec3(*aabb_half))))
         .update(G.KillSphereModifier(w.lit(G.Vec3(*kill_center)), w.lit(kill_r2), True)))
    return m


def drifting_sparks(capacity, name="sparks", lifetime=(0.2, 0.9)):
    """32-byte sparks under gravity and drag, dying after `lifetime` seconds (uniform)."""
    w = G.ExprWriter()
    return (G.EffectAsset(capacity, w.module, name=name)
            .init(G.SetAttributeModifier(A.POSITION, w.rand(G.VEC3) * w.lit(2.) - w.lit(1.)))
            .init(G.SetAttributeModifier(A.VELOCITY, w.rand(G.VEC3) * w.lit(2.) - w.lit(1.)))
            .init(G.SetAttributeModifier(A.AGE, w.lit(0.)))
            .init(G.SetAttributeModifier(A.LIFETIME, w.lit(lifetime[0]).uniform(w.lit(lifetime[1]))))
            .update(G.AccelModifier(w.lit(G.Vec3(0., -9.8, 0.))))
            .update(G.LinearDragModifier(w.lit(0.5))))


def growing_dust(capacity):
    """No age / lifetime: particles never die (like C1), a size attribute grows, a kill box culls."""
    w = G.ExprWriter()
    return (G.EffectAsset(capacity, w.module, name="dust")
            .init(G.SetAttributeModifier(A.POSITION, w.rand(G.VEC3) - w.lit(0.5)))
            .init(G.SetAttributeModifier(A.VELOCITY, (w.rand(G.VEC3) - w.lit(0.5)) * w.lit(3.)))
            .init(G.SetAttributeModifier(A.SIZE, w.lit(0.01)))
            .update(G.SetAttributeModifier(A.SIZE, w.attr(A.SIZE) * w.lit(1.0625) + w.time() * w.lit(0.001)))
            .update(G.KillAabbModifier(w.lit(G.Vec3(0., 0., 0.)), w.lit(G.Vec3(1.5, 1.0, 1.25)))))


def ribbon_asset(capacity, ribbons=5.0, lifetime=(0.15, 0.6)):
    w = G.ExprWriter()
    return (G.EffectAsset(capacity, w.module, name="ribbons")
            .init(G.SetAttributeModifier(A.POSITION, w.rand(G.VEC3) * w.lit(2.) - w.lit(1.)))
            .init(G.SetAttributeModifier(A.VELOCITY, w.rand(G.VEC3) - w.lit(0.5)))
            .init(G.SetAttributeModifier(A.AGE, w.rand(G.FLOAT) * w.lit(0.1)))
            .init(G.SetAttributeModifier(A.LIFETIME, w.lit(lifetime[0]).uniform(w.lit(lifetime[1]))))
            .init(G.SetAttributeModifier(A.RIBBON_ID, (w.rand(G.FLOAT) * w.lit(ribbons)).cast(G.UINT))))


def instancing(capacity):
    """BASELINE config C4's recipe (examples/instancing.rs:224-249, main effect): SetPositionSphere(Volume, r=1),
    SetVelocitySphere(speed 2), age 0, lifetime 12; no update modifier (Euler integration + age / reap only)."""
    w = G.ExprWriter()
    return (G.EffectAsset(capacity, w.module, name="instancing")
            .init(G.SetPositionSphereModifier(w.lit(G.Vec3(0, 0, 0)), w.lit(1.), G.VOLUME))
            .init(G.SetVelocitySphereModifier(w.lit(G.Vec3(0, 0, 0)), w.lit(2.)))
            .init(G.SetAttributeModifier(A.AGE, w.lit(0.)))
            .init(G.SetAttributeModifier(A.LIFETIME, w.lit(12.))))


def matrix_asset(capacity):
    """Matrix values (reference src/graph/mod.rs MatrixValue, src/attributes.rs MatrixType) in literals and
    properties, through every WGSL matrix product and sum."""
    w = G.ExprWriter()
    rot = w.lit(G.Mat3((0., 1., 0.), (-1., 0., 0.), (0., 0., 1.)))            # quarter turn about z
    lift = w.lit(G.Mat(2, 3, [1., 0.5, 0.25, -0.5, 1., 2.]))                   # mat2x3: vec2 -> vec3
    squash = w.lit(G.Mat(3, 2, [0.5, 0.125, -0.25, 1., 0.75, -1.5]))           # mat3x2: vec3 -> vec2
    twist = w.prop(w.add_property("twist", G.Mat2(0.8, 0.6, -0.6, 0.8)))       # 16 bytes: laid out like a vec4
    gain = w.prop(w.add_property("gain", G.Vec4(1.5, 0., 0., 0.))).x()
    # 64 bytes: must be the last entry of the layout (PropertyLayout::new advances 16 bytes per property of 16 bytes or
    # more and places smaller properties after them, properties.rs:572-580), so no scalar / vec2 / vec3 property here
    basis = w.prop(w.add_property("basis", G.Mat4(*[float(i) for i in range(16)])))
    wide = w.lit(G.Mat(2, 4, [0.5, -1., 2., 0.25, 1.5, 0.75, -0.5, 1.]))     # mat2x4: vec2 -> vec4
    tall = w.lit(G.Mat(4, 2, [1., -2., 0.5, 0.25, -0.75, 1.25, 2., -0.125]))  # mat4x2: vec4 -> vec2
    m34 = w.lit(G.Mat(3, 4, [0.1 * (i - 5) for i in range(12)]))              # mat3x4: vec3 -> vec4 (literals rounded to 1e-6)
    m43 = w.lit(G.Mat(4, 3, [0.3 * (7 - i) for i in range(12)]))              # mat4x3: vec4 -> vec3
    v, p = w.attr(A.VELOCITY), w.attr(A.POSITION)
    q = w.attr(A.F32X4_1)
    return (G.EffectAsset(capacity, w.module, name="matrices")
            .init(G.SetAttributeModifier(A.POSITION, w.rand(G.VEC3) * w.lit(4.) - w.lit(2.)))
            .init(G.SetAttributeModifier(A.VELOCITY, w.rand(G.VEC3) - w.lit(0.5)))
            .init(G.SetAttributeModifier(A.AGE, w.lit(0.)))
            .init(G.SetAttributeModifier(A.LIFETIME, w.lit(0.3).uniform(w.lit(0.9))))
            .init(G.SetAttributeModifier(A.F32X2_0, squash * (rot * (w.rand(G.VEC3) * gain))))                  # m*v twice, at init
            .update(G.SetAttributeModifier(A.F32X3_0, (rot * v) * w.lit(0.875) + lift * (twist * v.x().vec2(v.y()))))    # m*v, prop m*v
            .update(G.SetAttributeModifier(A.F32X3_1, v * (rot * rot + rot * w.lit(0.5)) - p * (w.lit(2.) * rot - rot)))  # v*m, m*m, m+m, m-m, m*s, s*m
            .update(G.SetAttributeModifier(A.F32X4_1, wide * v.x().vec2(v.y()) + m34 * p + v * m43))           # the other four shapes, m*v and v*m
            .update(G.SetAttributeModifier(A.F32X3_2, (lift * squash) * p + m43 * q + q * m34))                 # mat2x3 * mat3x2 -> mat3x3
            .update(G.SetAttributeModifier(A.F32X2_1, (squash * lift) * w.attr(A.F32X2_0) + p * lift))          # -> mat2x2; vec3 * mat2x3 -> vec2
            .update(G.SetAttributeModifier(A.F32X4_0, basis * p.vec4_xyz_w(gain) + v.vec4_xyz_w(w.lit(1.)) * basis))
            .update(G.SetAttributeModifier(A.F32X2_2, tall * q + q * wide)))


MATRIX_PROPS = {"twist": G.Mat2(0.28, 0.96, -0.96, 0.28), "gain": G.Vec4(0.75, 9., 9., 9.),
                "basis": G.Mat4((1., 0., 0., 0.), (0., 2., 0., 0.), (0., 0., -1., 0.), (0.5, -0.25, 3., 1.))}


# ---- GPU spawn events -------------------------------------------------------------------------------------------------
def event_assets():
    """A rocket that emits 3 events on death (channel 0) and the sparks that consume them."""
    wp = G.ExprWriter()
    parent = (G.EffectAsset(512, wp.module, name="rocket")
              .init(G.SetAttributeModifier(A.POSITION, wp.rand(G.VEC3) * wp.lit(8.) - wp.lit(4.)))
              .init(G.SetAttributeModifier(A.VELOCITY, wp.lit(G.Vec3(0., 3., 0.))))
              .init(G.SetAttributeModifier(A.AGE, wp.lit(0.)))
              .init(G.SetAttributeModifier(A.LIFETIME, wp.lit(0.05).uniform(wp.lit(0.4))))
              .update(G.EmitSpawnEventModifier(G.ON_DIE, wp.lit(G.U32(3)), 0)))
    wc = G.ExprWriter()
    child = (G.EffectAsset(2048, wc.module, name="sparks")
             .init(G.InheritAttributeModifier(A.POSITION))
             .init(G.SetAttributeModifier(A.VELOCITY, wc.parent_attr(A.VELOCITY) * wc.lit(-0.5) + (wc.rand(G.VEC3) - wc.lit(0.5))))
             .init(G.SetAttributeModifier(A.AGE, wc.lit(0.)))
             .init(G.SetAttributeModifier(A.LIFETIME, wc.lit(0.3)))
             .init(G.SetAttributeModifier(A.U32_0, wc.parent_attr(A.ID))))
    return parent, child


def emitter_assets(pcap):
    """One parent of `pcap` slots, two event channels: channel 0 fed every frame by particles that are alive
    (EventEmitCondition::Always, count 0 or 1 drawn per particle), channel 1 by dying particles (OnDie, 4 events each); and
    the two children of 4096 slots that consume them."""
    wp = G.ExprWriter()
    parent = (G.EffectAsset(pcap, wp.module, name="emitter")
              .init(G.SetAttributeModifier(A.POSITION, wp.rand(G.VEC3) * wp.lit(2.) - wp.lit(1.)))
              .init(G.SetAttributeModifier(A.VELOCITY, wp.rand(G.VEC3) - wp.lit(0.5)))
              .init(G.SetAttributeModifier(A.AGE, wp.lit(0.)))
              .init(G.SetAttributeModifier(A.LIFETIME, wp.lit(0.1).uniform(wp.lit(0.5))))
              .update(G.EmitSpawnEventModifier(G.ALWAYS, (wp.rand(G.FLOAT) * wp.lit(1.25)).cast(G.UINT), 0))
              .update(G.EmitSpawnEventModifier(G.ON_DIE, wp.lit(G.U32(4)), 1)))
    children = []
    for tag in (0, 1):
        wc = G.ExprWriter()
        children.append(G.EffectAsset(4096, wc.module, name=f"child{tag}")
                        .init(G.InheritAttributeModifier(A.POSITION))
                        .init(G.SetAttributeModifier(A.VELOCITY, wc.parent_attr(A.VELOCITY) * wc.lit(0.25 + tag) + (wc.rand(G.VEC3) - wc.lit(0.5))))
                        .init(G.SetAttributeModifier(A.AGE, wc.lit(0.)))
                        .init(G.SetAttributeModifier(A.LIFETIME, wc.lit(0.2 + 0.1 * tag)))
                        .init(G.SetAttributeModifier(A.U32_0, wc.parent_attr(A.ID))))
    return parent, children


# ---- tile shapes: one effect per record width -------------------------------------------------------------------------
ROWS_PER_LANE = 16  # HNB_ROWS_PER_LANE's default


def tile_k(stride):
    """choose_tile_k restated: rows a lane keeps in flight for records of `stride` bytes (index + record ~ 40 words)."""
    k = 40 // (stride // 4 + 1)
    return 4 if k >= 4 else 2 if k >= 2 else 1


def edge_counts(k, chunks):
    """Alive counts at the edges of a sub-tile (32 K rows) and of a tile of `chunks` sub-tiles."""
    sub, S = 32 * k, 32 * k * chunks
    return sorted({sub - 1, sub + 1, S - 1, S, S + 1, 2 * S + 1})


def _vec4s(capacity, n):
    """A 32-byte spark plus `n` vec4 attributes, each updated from itself, its neighbour and a per-instance property:
    64 bytes with 2 of them, 96 bytes with 4 (adds and multiplies only: IEEE-exact)."""
    w = G.ExprWriter()
    gain = w.prop(w.add_property("gain", 1.0))
    slots = [A.F32X4_0, A.F32X4_1, A.F32X4_2, A.F32X4_3][:n]
    asset = (G.EffectAsset(capacity, w.module, name=f"vec4x{n}")
             .init(G.SetAttributeModifier(A.POSITION, w.rand(G.VEC3) * w.lit(2.) - w.lit(1.)))
             .init(G.SetAttributeModifier(A.VELOCITY, w.rand(G.VEC3) - w.lit(0.5)))
             .init(G.SetAttributeModifier(A.AGE, w.lit(0.)))
             .init(G.SetAttributeModifier(A.LIFETIME, w.lit(0.25).uniform(w.lit(0.6)))))
    for s in slots:
        asset = asset.init(G.SetAttributeModifier(s, w.rand(G.VEC4)))
    for i, s in enumerate(slots):
        asset = asset.update(G.SetAttributeModifier(s, w.attr(s) * w.lit(0.75) + w.attr(slots[i - 1]) * gain))
    return asset.update(G.AccelModifier(w.lit(G.Vec3(0., -3., 0.)) * gain))


# name -> (builder, record bytes, dt: lifetimes of 2-6 frames, properties of instance i or None)
EFFECTS = {
    "trails48": (firework_trails, 48, 0.25, None),
    "vec4x2_64": (lambda cap: _vec4s(cap, 2), 64, 0.1, lambda i: {"gain": 0.5 + 0.125 * i}),
    "vec4x4_96": (lambda cap: _vec4s(cap, 4), 96, 0.1, lambda i: {"gain": 1.5 - 0.125 * i}),
    "matrix144": (matrix_asset, 144, 0.15, lambda i: MATRIX_PROPS if i % 2 == 0 else {}),
}


def table_asset(name, capacity):
    build, size, _, _ = EFFECTS[name]
    asset = build(capacity)
    assert asset.particle_layout()[1] == size, f"{name}: record size"
    return asset


def table_props(name, n):
    """The property records of instances 0 .. n-1 of EFFECTS[name], or None when the effect has no properties."""
    props = EFFECTS[name][3]
    return None if props is None else [props(i) for i in range(n)]


# ---- C5 under the C oracle --------------------------------------------------------------------------------------------
def c5_init():
    """The C5 effect's init: position = velocity = 0, age 0, lifetime 1."""
    ci = O.ConstInit()
    ci.stride_words = 8
    ci.words[7] = int(np.float32(1.0).view(np.uint32))
    return ci


def fill_c5(ref, rng, life_lo, life_hi):
    """C5 records of the initially alive rows of every instance: random positions and velocities, age 0, lifetimes in
    [life_lo, life_hi)."""
    for inst in ref.instances:
        n = inst.alive
        rows = slice(inst.slab_offset, inst.slab_offset + n)
        p = np.zeros((n, 8), dtype=np.float32)
        p[:, 0:3] = rng.uniform(-1, 1, (n, 3))
        p[:, 3] = 0.0
        p[:, 4:7] = rng.uniform(-1, 1, (n, 3))
        p[:, 7] = rng.uniform(life_lo, life_hi, n)
        ref.particles[rows] = p.view(np.uint32)


# ---- random expressions -----------------------------------------------------------------------------------------------
def exact_expr(draw, w, depth, kind):
    """Draw an expression of `kind` ('f' scalar / 'v' vec3) using only IEEE-exact operators (`draw`: hypothesis's)."""
    from hypothesis import strategies as st
    lit_f = lambda: w.lit(float(np.float32(draw(st.floats(-4, 4, allow_nan=False, width=32)))))
    if depth == 0:
        if kind == "f":
            c = draw(st.integers(0, 4))
            return [lit_f, lambda: w.attr(A.AGE), lambda: w.attr(A.F32_1), lambda: w.attr(A.POSITION).y(), lambda: w.time()][c]()
        c = draw(st.integers(0, 2))
        if c == 0:
            return w.lit(G.Vec3(*[float(np.float32(draw(st.floats(-3, 3, allow_nan=False, width=32)))) for _ in range(3)]))
        return [None, lambda: w.attr(A.POSITION), lambda: w.attr(A.VELOCITY)][c]()
    sub = lambda k: exact_expr(draw, w, depth - 1, k)
    if kind == "f":
        c = draw(st.integers(0, 13))
        if c == 0: return sub("f") + sub("f")
        if c == 1: return sub("f") - sub("f")
        if c == 2: return sub("f") * sub("f")
        if c == 3: return sub("f") / (sub("f").abs() + w.lit(1.))
        if c == 4: return sub("f").min(sub("f"))
        if c == 5: return sub("f").max(sub("f"))
        if c == 6: return sub("f").abs().sqrt()
        if c == 7: return sub("f").floor() + sub("f").fract()
        if c == 8: return sub("f").sign() * sub("f").ceil()
        if c == 9: return sub("v").dot(sub("v"))
        if c == 10: return sub("f").clamp(w.lit(-1.), w.lit(2.))
        if c == 11: return sub("f").mix(sub("f"), w.lit(0.25))
        if c == 12: return sub("f").step(sub("f")) + sub("v").x()
        return sub("v").length()
    c = draw(st.integers(0, 7))
    if c == 0: return sub("v") + sub("v")
    if c == 1: return sub("v") * sub("f")
    if c == 2: return sub("v").cross(sub("v"))
    if c == 3: return sub("f").vec3(sub("f"), sub("f"))
    if c == 4: return sub("v").abs().min(sub("v"))
    if c == 5: return sub("f").cast(G.VEC3) - sub("v")
    if c == 6: return sub("v") / (sub("v").abs() + w.lit(G.Vec3(1., 1., 1.)))
    return sub("v").max(sub("v")) * w.lit(0.5)
