"""CPU-side fuzz of the expression lowering over the WHOLE operator table (reference src/graph/expr.rs:1833-2360):
random typed expression trees over scalars, vec2/3/4, uint and bool values are lowered to CUDA C and

  * compiled for sm_90a with NVRTC (no GPU needed) — catches text that is not valid C++ against hnb_wgsl.cuh
    (missing overloads, ambiguous calls, precedence of pasted text), and
  * interpreted by the numpy oracle on a few particles — catches operators the oracle cannot evaluate or evaluates
    with the wrong shape / type.

The GPU suite compares values (tests/test_gpu_misc.py::test_random_expression_graphs_bit_exact for the IEEE-exact
operators, test_gpu_effects.py for the transcendental ones); this test widens the structural coverage.
"""
import numpy as np
import pytest

from bevy_hanabi_b200 import graph as G
from bevy_hanabi_b200 import runtime as R
from oracle.hanabi_oracle import EffectOracle
from tests.helpers import Instance, RefWorld

hypothesis = pytest.importorskip("hypothesis")
from hypothesis import HealthCheck, Phase, given, settings, strategies as st  # noqa: E402

A = G.Attribute


def build(draw, w, depth, kind):
    """kind: f (f32) | v2 | v3 | v4 | u (u32) | b (bool)"""
    i = lambda n: draw(st.integers(0, n))
    lit = lambda lo=-3.0, hi=3.0: float(np.float32(draw(st.floats(lo, hi, allow_nan=False, width=32))))
    sub = lambda k: build(draw, w, depth - 1, k)
    if depth == 0:
        if kind == "f":
            return [lambda: w.lit(lit()), lambda: w.attr(A.AGE), lambda: w.attr(A.LIFETIME), lambda: w.attr(A.F32_1), lambda: w.time(),
                    lambda: w.delta_time(), lambda: w.attr(A.POSITION).z()][i(6)]()
        if kind == "v2":
            return [lambda: w.lit(G.Vec2(lit(), lit())), lambda: w.attr(A.SIZE2)][i(1)]()
        if kind == "v3":
            return [lambda: w.lit(G.Vec3(lit(), lit(), lit())), lambda: w.attr(A.POSITION), lambda: w.attr(A.VELOCITY)][i(2)]()
        if kind == "v4":
            return [lambda: w.lit(G.Vec4(lit(), lit(), lit(), lit())), lambda: w.attr(A.HDR_COLOR)][i(1)]()
        if kind == "u":
            return [lambda: w.lit(G.U32(draw(st.integers(0, 2**32 - 1)))), lambda: w.attr(A.ID), lambda: w.attr(A.PARTICLE_COUNTER), lambda: w.attr(A.COLOR)][i(3)]()
        return [lambda: w.lit(True), lambda: w.lit(False), lambda: w.is_alive()][i(2)]()
    if kind == "f":
        c = i(29)
        un = ["abs", "acos", "asin", "atan", "ceil", "cos", "exp", "exp2", "floor", "fract", "log", "log2", "round", "saturate", "sign", "sin", "sqrt", "tan"]
        if c < len(un): return getattr(sub("f"), un[c])()
        c -= len(un)
        if c == 0: return sub("f").inverse_sqrt()
        if c == 1: return sub("v3").length() + sub("v2").length() - sub("v4").length()
        if c == 2: return sub("v3").dot(sub("v3")) * sub("v4").dot(sub("v4"))
        if c == 3: return sub("v3").distance(sub("v3"))
        if c == 4: return sub("f").atan2(sub("f"))
        if c == 5: return (sub("f") % (sub("f").abs() + w.lit(0.5))).min(sub("f")).max(sub("f"))
        if c == 6: return sub("f").mix(sub("f"), sub("f")).clamp(sub("f"), sub("f"))
        if c == 7: return sub("f").smoothstep(sub("f"), sub("f")) + sub("f").step(sub("f"))
        if c == 8: return sub("v4").w() * sub("v2").y() + sub("v3").x()
        if c == 9: return sub("u").cast(G.FLOAT) + sub("b").cast(G.FLOAT)
        # rand_uniform / rand_normal need operands whose type is known without evaluation (expr.rs:1162-1176):
        # literals, attributes, casts
        if c == 10: return w.lit(lit()).uniform(w.attr(A.LIFETIME)) + sub("f").cast(G.FLOAT).normal(w.lit(lit())) + w.rand()
        return sub("f") / sub("f") - sub("f") * sub("f")
    if kind == "v2":
        c = i(4)
        if c == 0: return sub("f").vec2(sub("f"))
        if c == 1: return (sub("v2") + sub("v2")) * sub("f")
        if c == 2: return sub("v2").abs().max(sub("v2")).normalize()
        if c == 3: return sub("v2").mix(sub("v2"), sub("f")) + w.rand(G.VEC2)
        return sub("f").cast(G.VEC2) - sub("v2").fract()
    if kind == "v3":
        c = i(8)
        if c == 0: return sub("v3").cross(sub("v3"))
        if c == 1: return sub("f").vec3(sub("f"), sub("f"))
        if c == 2: return sub("v3").normalize() * sub("f") + sub("v3") / (sub("v3").abs() + w.lit(1.))
        if c == 3: return sub("v3").clamp(sub("v3"), sub("v3")).mix(sub("v3"), sub("v3"))
        if c == 4: return sub("v3").sin() + sub("v3").exp2().sqrt() - sub("v3").floor()
        if c == 5: return sub("f").cast(G.VEC3) * sub("v3").sign()
        if c == 6: return w.lit(G.Vec3(lit(), lit(), lit())).uniform(w.attr(A.VELOCITY)) + sub("v3").cast(G.VEC3).normal(w.attr(A.POSITION)) + w.rand(G.VEC3)
        if c == 7: return sub("v3").step(sub("v3")) + sub("v3").smoothstep(sub("v3"), sub("v3"))
        return sub("v3").min(sub("v3")) % (sub("v3").abs() + w.lit(0.25))
    if kind == "v4":
        c = i(4)
        if c == 0: return sub("v3").vec4_xyz_w(sub("f"))
        if c == 1: return sub("u").unpack4x8unorm() + sub("u").unpack4x8snorm()
        if c == 2: return sub("v4") * sub("v4") - sub("v4").saturate()
        if c == 3: return sub("f").cast(G.VEC4).max(sub("v4")) + w.rand(G.VEC4)
        return sub("v4").normalize().mix(sub("v4"), sub("f"))
    if kind == "u":
        c = i(3)
        if c == 0: return sub("v4").pack4x8unorm()
        if c == 1: return sub("v4").pack4x8snorm()
        if c == 2: return sub("f").abs().cast(G.UINT) + sub("u")
        return sub("u") * sub("u") - sub("u")
    c = i(5)
    if c == 0: return sub("f").lt(sub("f"))
    if c == 1: return sub("f").ge(sub("f"))
    if c == 2: return sub("v3").gt(sub("v3")).all()
    if c == 3: return sub("v3").le(sub("v3")).any()
    if c == 4: return sub("u").lt(sub("u"))
    return sub("v2").lt(sub("v2")).any()


@settings(max_examples=25, deadline=None, suppress_health_check=list(HealthCheck), phases=[Phase.generate], derandomize=True)
@given(st.data())
def test_random_typed_graphs_compile_and_interpret(orc, data):
    w = G.ExprWriter()
    d = data.draw(st.integers(1, 3))
    exprs = {k: build(data.draw, w, d, k) for k in ("f", "v2", "v3", "v4", "u", "b")}
    asset = (G.EffectAsset(64, w.module, name="typed_fuzz")
             .init(G.SetAttributeModifier(A.POSITION, w.rand(G.VEC3) * w.lit(4.) - w.lit(2.)))
             .init(G.SetAttributeModifier(A.VELOCITY, w.rand(G.VEC3) - w.lit(0.5)))
             .init(G.SetAttributeModifier(A.AGE, w.lit(0.)))
             .init(G.SetAttributeModifier(A.LIFETIME, w.lit(5.)))
             .init(G.SetAttributeModifier(A.F32_1, w.rand() * w.lit(3.)))
             .init(G.SetAttributeModifier(A.SIZE2, w.rand(G.VEC2)))
             .init(G.SetAttributeModifier(A.HDR_COLOR, w.rand(G.VEC4)))
             .init(G.SetAttributeModifier(A.COLOR, w.rand(G.VEC4).pack4x8unorm()))
             .update(G.SetAttributeModifier(A.F32_0, exprs["f"]))
             .update(G.SetAttributeModifier(A.F32X2_0, exprs["v2"]))
             .update(G.SetAttributeModifier(A.F32X3_0, exprs["v3"]))
             .update(G.SetAttributeModifier(A.F32X4_0, exprs["v4"]))
             .update(G.SetAttributeModifier(A.U32_0, exprs["u"]))
             .update(G.SetAttributeModifier(A.F32_2, exprs["b"].cast(G.FLOAT))))
    fx = asset.generate()
    try:
        R.nvrtc_check(fx.generate_source())
    except Exception as e:  # show the offending text
        raise AssertionError(f"generated update code does not compile:\n{fx.update_code}\n{str(e)[:2000]}") from None
    _, size, _ = asset.particle_layout()
    ref = RefWorld(64, size // 4, [Instance(0, 64, alive=0, seed=data.draw(st.integers(0, 2**32 - 1)))])
    eo = EffectOracle(asset)
    with np.errstate(all="ignore"):
        for f in range(2):
            ref.sim.time = np.float32(f) * ref.sim.delta_time
            ref.set_spawns([40 if f == 0 else 5])
            eo.frame(ref, orc)
    assert ref.metadata[0].particle_counter == 45


@settings(max_examples=30, deadline=None, suppress_health_check=list(HealthCheck), phases=[Phase.generate], derandomize=True)
@given(st.data())
def test_random_exact_graphs_generated_code_equals_interpreter(orc, data):
    """Values, not just syntax: random graphs over the IEEE-exact operators (the generator of the GPU fuzz test), with
    the generated code executed on the CPU (tests/host_exec.py) and compared bit for bit with the interpreter."""
    from tests.host_exec import HostEffect, replay_frame
    from tests.effects import exact_expr
    w = G.ExprWriter()
    f_expr = exact_expr(data.draw, w, data.draw(st.integers(1, 3)), "f")
    v_expr = exact_expr(data.draw, w, data.draw(st.integers(1, 3)), "v")
    asset = (G.EffectAsset(256, w.module, name="exact_fuzz")
             .init(G.SetAttributeModifier(A.POSITION, w.rand(G.VEC3) * w.lit(4.) - w.lit(2.)))
             .init(G.SetAttributeModifier(A.VELOCITY, w.rand(G.VEC3) - w.lit(0.5)))
             .init(G.SetAttributeModifier(A.AGE, w.lit(0.)))
             .init(G.SetAttributeModifier(A.LIFETIME, w.lit(0.05).uniform(w.lit(0.2))))
             .init(G.SetAttributeModifier(A.F32_1, w.rand() * w.lit(3.)))
             .update(G.SetAttributeModifier(A.F32_0, f_expr))
             .update(G.SetAttributeModifier(A.F32X3_0, v_expr)))
    fx = asset.generate()
    host = HostEffect(fx)
    _, size, _ = asset.particle_layout()
    ref = RefWorld(256, size // 4, [Instance(0, 256, alive=0, seed=data.draw(st.integers(0, 2**32 - 1)))])
    eo = EffectOracle(asset)

    def canon(a, b):
        a, b = a.copy(), b.copy()
        fa, fb = a.view(np.float32), b.view(np.float32)
        same = (np.isnan(fa) & np.isnan(fb)) | ((fa == 0) & (fb == 0))  # any NaN == any NaN; min/max may return either zero
        a[same] = 0
        b[same] = 0
        return a, b

    with np.errstate(all="ignore"):
        for f in range(3):
            ref.sim.time = np.float32(f) * ref.sim.delta_time
            ref.set_spawns([120 if f == 0 else 30])
            ih, io, uh, uo, ah, ao = replay_frame(host, eo, ref, orc)
            np.testing.assert_array_equal(*canon(ih, io), err_msg="init records\n" + fx.init_code)
            np.testing.assert_array_equal(*canon(uh, uo), err_msg="update records\n" + fx.update_code)
            np.testing.assert_array_equal(ah, ao)


def build_linear(draw, w, depth, kind):
    """Random graphs over matCxR / vecN / f32 values joined by the WGSL linear-algebra operators only (+, -, *, dot):
    every operation is one IEEE rounding, so generated code and interpreter must agree bit for bit.
    kind: "f" | ("v", n) | ("m", cols, rows)"""
    i = lambda n: draw(st.integers(0, n))
    dim = lambda: draw(st.integers(2, 4))
    lit = lambda: float(np.float32(draw(st.floats(-2.0, 2.0, allow_nan=False, width=32))))
    sub = lambda k: build_linear(draw, w, depth - 1, k)
    if kind == "f":
        if depth == 0:
            return [lambda: w.lit(lit()), lambda: w.attr(A.AGE), lambda: w.attr(A.F32_1)][i(2)]()
        c, n = i(2), dim()
        if c == 0: return sub("f") * sub("f") - sub("f")
        if c == 1: return sub(("v", n)).dot(sub(("v", n)))
        return (sub(("v", n)) * sub(("m", 3, n))).y()                      # component of an infix product
    if kind[0] == "v":
        n = kind[1]
        if depth == 0:
            attr = {2: A.SIZE2, 3: [A.POSITION, A.VELOCITY][i(1)], 4: A.HDR_COLOR}[n]
            return [lambda: w.lit(Value_vec(n, [lit() for _ in range(n)])), lambda: w.attr(attr)][i(1)]()
        c, k = i(3), dim()
        if c == 0: return sub(("m", k, n)) * sub(("v", k))                 # matKxN * vecK -> vecN
        if c == 1: return sub(("v", k)) * sub(("m", n, k))                 # vecK * matNxK -> vecN
        if c == 2: return sub(kind) * sub("f") + sub(kind)
        return sub(kind) - sub(kind) * sub(kind)
    _, cols, rows = kind
    if depth == 0:
        return w.lit(G.Mat(cols, rows, [lit() for _ in range(cols * rows)]))
    c, k = i(4), dim()
    if c == 0: return sub(("m", k, rows)) * sub(("m", cols, k))            # matKxR * matCxK -> matCxR
    if c == 1: return sub(kind) + sub(kind)
    if c == 2: return sub(kind) - sub(kind)
    if c == 3: return sub(kind) * sub("f")
    return sub("f") * sub(kind)


def Value_vec(n, xs):
    return {2: G.Vec2, 3: G.Vec3, 4: G.Vec4}[n](*xs)


@settings(max_examples=30, deadline=None, suppress_health_check=list(HealthCheck), phases=[Phase.generate], derandomize=True)
@given(st.data())
def test_random_matrix_graphs_generated_code_equals_interpreter(orc, data):
    """Matrix values (all nine matCxR shapes, chosen at random) in random product / sum graphs: the generated code must
    compile for sm_90a and, run on the CPU, equal the interpreter bit for bit."""
    from tests.host_exec import HostEffect, replay_frame
    w = G.ExprWriter()
    depth = lambda: data.draw(st.integers(1, 3))
    exprs = {"f": build_linear(data.draw, w, depth(), "f"), 2: build_linear(data.draw, w, depth(), ("v", 2)),
             3: build_linear(data.draw, w, depth(), ("v", 3)), 4: build_linear(data.draw, w, depth(), ("v", 4))}
    asset = (G.EffectAsset(128, w.module, name="matrix_fuzz")
             .init(G.SetAttributeModifier(A.POSITION, w.rand(G.VEC3) * w.lit(4.) - w.lit(2.)))
             .init(G.SetAttributeModifier(A.VELOCITY, w.rand(G.VEC3) - w.lit(0.5)))
             .init(G.SetAttributeModifier(A.AGE, w.lit(0.)))
             .init(G.SetAttributeModifier(A.LIFETIME, w.lit(0.05).uniform(w.lit(0.2))))
             .init(G.SetAttributeModifier(A.F32_1, w.rand() * w.lit(3.)))
             .init(G.SetAttributeModifier(A.SIZE2, w.rand(G.VEC2)))
             .init(G.SetAttributeModifier(A.HDR_COLOR, w.rand(G.VEC4)))
             .update(G.SetAttributeModifier(A.F32_0, exprs["f"]))
             .update(G.SetAttributeModifier(A.F32X2_0, exprs[2]))
             .update(G.SetAttributeModifier(A.F32X3_0, exprs[3]))
             .update(G.SetAttributeModifier(A.F32X4_0, exprs[4])))
    fx = asset.generate()
    try:
        R.nvrtc_check(fx.generate_source())
    except Exception as e:
        raise AssertionError(f"generated update code does not compile:\n{fx.update_code}\n{str(e)[:2000]}") from None
    host = HostEffect(fx)
    _, size, _ = asset.particle_layout()
    ref = RefWorld(128, size // 4, [Instance(0, 128, alive=0, seed=data.draw(st.integers(0, 2**32 - 1)))])
    eo = EffectOracle(asset)

    def canon(a, b):
        a, b = a.copy(), b.copy()
        fa, fb = a.view(np.float32), b.view(np.float32)
        same = np.isnan(fa) & np.isnan(fb)
        a[same] = 0
        b[same] = 0
        return a, b

    with np.errstate(all="ignore"):
        for f in range(2):
            ref.sim.time = np.float32(f) * ref.sim.delta_time
            ref.set_spawns([80 if f == 0 else 20])
            ih, io, uh, uo, ah, ao = replay_frame(host, eo, ref, orc)
            np.testing.assert_array_equal(*canon(ih, io), err_msg="init records\n" + fx.init_code)
            np.testing.assert_array_equal(*canon(uh, uo), err_msg="update records\n" + fx.update_code)
            np.testing.assert_array_equal(ah, ao)
