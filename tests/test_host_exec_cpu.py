"""The GENERATED effect code, executed on the CPU (tests/host_exec.py), against the numpy interpreter of the
expression graph: checks the values the lowered text computes — both passes, every record, the is_alive flag —
without a GPU. IEEE-exact effects must agree bit for bit; effects going through libm within 1e-5 of the attribute's
magnitude (glibc and numpy round sin/cos/acos/pow differently in the last place, like CUDA's libm does)."""
import numpy as np
import pytest

from bevy_hanabi_b200 import graph as G
from oracle.hanabi_oracle import EffectOracle, pcg_hash
from tests.effects import MATRIX_PROPS, drifting_sparks, firework_trails, force_field, growing_dust, matrix_asset, ribbon_asset
from tests.helpers import Instance, RefWorld, assert_float_attributes_close, float_word_mask
from tests.host_exec import HostEffect, replay_frame

A = G.Attribute


def _world(asset, capacity, seed=5, dt=1.0 / 30.0):
    _, size, _ = asset.particle_layout()
    return RefWorld(capacity, size // 4, [Instance(0, capacity, alive=0, seed=seed)], dt=dt)


def _run(orc, asset, frames, spawns, exact=True, props=None, capacity=2048):
    fx = asset.generate()
    host = HostEffect(fx)
    ref = _world(asset, capacity)
    blob = None
    if props is not None:
        blob = asset.serialize_properties(props)
        ref.metadata[0].properties_array_index = 0
    eo = EffectOracle(asset, {0: props} if props else None)
    mask, fattrs = float_word_mask(asset)
    checked_init = checked_update = deaths = 0
    for f in range(frames):
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        ref.set_spawns([spawns(f)], [int(pcg_hash(np.array([77 + f], dtype=np.uint32))[0])])
        ih, io, uh, uo, ah, ao = replay_frame(host, eo, ref, orc, blob)
        if exact:
            np.testing.assert_array_equal(ih, io, err_msg=f"frame {f}: init records")
            np.testing.assert_array_equal(uh, uo, err_msg=f"frame {f}: update records")
        else:
            np.testing.assert_array_equal(ih[:, ~mask], io[:, ~mask])
            np.testing.assert_array_equal(uh[:, ~mask], uo[:, ~mask])
            if len(ih):
                assert_float_attributes_close(ih, io, fattrs, 1e-5, f"frame {f}: init")
            if len(uh):
                assert_float_attributes_close(uh, uo, fattrs, 1e-5, f"frame {f}: update")
        np.testing.assert_array_equal(ah, ao, err_msg=f"frame {f}: is_alive")
        checked_init += len(ih)
        checked_update += len(uh)
        deaths += int((~ao).sum())
    return checked_init, checked_update, deaths


def test_trails_generated_code_equals_interpreter(orc):
    ci, cu, deaths = _run(orc, firework_trails(2048), 30, lambda f: 700 if f % 10 == 0 else 0)
    assert ci > 1500
    assert cu > 10_000 and deaths > 100


@pytest.mark.parametrize("name", ["sparks", "dust", "ribbons"])
def test_scene_assets_generated_code_equals_interpreter(orc, name):
    asset = {"sparks": drifting_sparks, "dust": growing_dust, "ribbons": ribbon_asset}[name](2048)
    ci, cu, deaths = _run(orc, asset, 20, lambda f: 300 if f % 4 == 0 else 11)
    assert ci > 800 and cu > 5000
    if name != "ribbons":
        assert deaths > 0


def test_force_field_generated_code_within_tolerance(orc):
    props = {"attraction_accel": 18.0, "repulsor_position": G.Vec3(0.25, 0.5, 0.1)}
    ci, cu, _ = _run(orc, force_field(4096), 6, lambda f: 3000 if f == 0 else 20, exact=False, props=props, capacity=4096)
    assert ci > 3000 and cu > 15_000


def test_operator_table_generated_code(orc):
    """Every IEEE-exact operator family in one effect (same graph as the GPU operator test uses for its exact part)."""
    w = G.ExprWriter()
    x, v = w.attr(A.F32_0), w.attr(A.VELOCITY)
    asset = (G.EffectAsset(512, w.module, name="ops")
             .init(G.SetAttributeModifier(A.POSITION, w.rand(G.VEC3) * w.lit(4.) - w.lit(2.)))
             .init(G.SetAttributeModifier(A.VELOCITY, w.rand(G.VEC3) - w.lit(0.5)))
             .init(G.SetAttributeModifier(A.F32_0, w.rand() * w.lit(3.) - w.lit(1.)))
             .init(G.SetAttributeModifier(A.AGE, w.lit(0.)))
             .init(G.SetAttributeModifier(A.LIFETIME, w.lit(0.2).uniform(w.lit(0.6))))
             .update(G.SetAttributeModifier(A.F32_1, x.abs().sqrt() + x.floor() - x.fract() * x.ceil() + x.sign() + x.saturate() + x.round()))
             .update(G.SetAttributeModifier(A.F32_2, x.min(w.lit(0.5)).max(w.lit(-0.25)).clamp(w.lit(-0.1), w.lit(0.4)).mix(x, w.lit(0.25))
                                            + x.step(w.lit(0.3)) + x.smoothstep(w.lit(-1.), w.lit(2.)) + (x % w.lit(0.7))))
             .update(G.SetAttributeModifier(A.F32X3_0, v.cross(w.attr(A.POSITION)) + v.normalize() * v.length() - v.abs().min(w.attr(A.POSITION))
                                            + v.x().vec3(v.dot(v), v.distance(w.attr(A.POSITION)))))
             .update(G.SetAttributeModifier(A.U32_0, (x.abs() * w.lit(1000.)).cast(G.UINT) + w.attr(A.ID) * w.attr(A.PARTICLE_COUNTER)))
             .update(G.SetAttributeModifier(A.F32_3, v.gt(w.attr(A.POSITION)).any().cast(G.FLOAT) + v.le(w.attr(A.POSITION)).all().cast(G.FLOAT)
                                            + w.is_alive().cast(G.FLOAT) + w.time() * w.delta_time())))
    ci, cu, deaths = _run(orc, asset, 12, lambda f: 400 if f == 0 else 15, capacity=512)
    assert ci > 400 and cu > 2000 and deaths > 50


def test_matrix_values_generated_code_equals_interpreter(orc):
    """Every product only multiplies and adds in a fixed order, so the lowered text and the interpreter agree bit for bit."""
    ci, cu, deaths = _run(orc, matrix_asset(1024), 10, lambda f: 500 if f == 0 else 25, props=MATRIX_PROPS, capacity=1024)
    assert ci > 500 and cu > 3000 and deaths > 20
    # and with the default property values
    ci, cu, _ = _run(orc, matrix_asset(1024), 3, lambda f: 200, props={}, capacity=1024)
    assert ci == 600


def test_three_row_matrix_property_keeps_the_reference_byte_image(orc):
    """MatrixValue::as_bytes (graph/mod.rs:1387-1391) uploads the PACKED column-major storage, which the shader reads with
    WGSL's 16-byte column stride: a mat3x3 / mat2x3 / mat4x3 property is seen with shifted columns. Same bytes, same
    read here (tests/test_authoring_cpu.py pins the bytes); this checks the lowered code against the interpreter."""
    w = G.ExprWriter()
    m = w.prop(w.add_property("m", G.Mat3(*[float(i + 1) for i in range(9)])))
    asset = (G.EffectAsset(256, w.module, name="mat3prop")
             .init(G.SetAttributeModifier(A.POSITION, w.rand(G.VEC3)))
             .init(G.SetAttributeModifier(A.AGE, w.lit(0.))).init(G.SetAttributeModifier(A.LIFETIME, w.lit(10.)))
             .update(G.SetAttributeModifier(A.F32X3_0, m * w.attr(A.POSITION))))
    _run(orc, asset, 2, lambda f: 100, props={}, capacity=256)
    # the columns the shader sees: (1 2 3) (5 6 7) (9 0 0), not (1 2 3) (4 5 6) (7 8 9)
    from oracle.hanabi_oracle import literal_array
    seen = literal_array(G.Mat3(*[float(i + 1) for i in range(9)]), 1, as_shader_text=False)[0]
    np.testing.assert_array_equal(seen, np.array([[1, 2, 3], [5, 6, 7], [9, 0, 0]], dtype=np.float32))
