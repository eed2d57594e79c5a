"""CPU-only sanity of the numpy oracle on the authored effects used by the GPU parity tests: structural
invariants of the reference's bookkeeping (SURVEY.md §3.5) must hold after every frame."""
import numpy as np
import pytest

from bevy_hanabi_b200 import graph as G
from oracle.hanabi_oracle import EffectOracle, pcg_hash
from tests.effects import firework_trails, force_field, ribbon_asset
from tests.helpers import Instance, RefWorld


def _check_invariants(ref):
    for i, inst in enumerate(ref.instances):
        md = ref.metadata[i]
        base, cap = inst.slab_offset, inst.capacity
        assert md.alive_count == ref.draw[5 * md.indirect_render_index + 1]           # alive_count == instance_count
        assert md.max_spawn == cap - md.alive_count
        alive = ref.indirect[base:base + md.alive_count, md.indirect_write_index].astype(np.int64)
        dead = ref.indirect[base + md.alive_count:base + cap, 2].astype(np.int64) - base
        both = np.concatenate([alive, dead])
        assert sorted(both.tolist()) == list(range(cap)), "alive list + dead stack must partition the instance's slots"


@pytest.mark.parametrize("name", ["firework", "force_field"])
def test_oracle_invariants(orc, name):
    if name == "firework":
        asset = firework_trails(2048)
        ref = RefWorld(2048, 12, [Instance(0, 2048, alive=0)], dt=1.0 / 20.0)
        spawns = lambda f: [700 if f % 12 == 0 else 0]
        props = None
    else:
        asset = force_field(4096)
        _, size, _ = asset.particle_layout()
        ref = RefWorld(4096, size // 4, [Instance(0, 4096, alive=0, seed=77)])
        spawns = lambda f: [3000 if f == 0 else 10]
        props = {0: {"attraction_accel": 18.0, "repulsor_position": G.Vec3(0.25, 0.5, 0.1)}}
    eo = EffectOracle(asset, props)
    died = False
    for f in range(40):
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        ref.set_spawns(spawns(f), [int(pcg_hash(np.array([f], dtype=np.uint32))[0])])
        before = ref.metadata[0].alive_count
        eo.frame(ref, orc)
        _check_invariants(ref)
        died |= ref.metadata[0].alive_count < before + spawns(f)[0]
    assert ref.metadata[0].particle_counter > 0
    if name == "firework":
        assert died, "the scenario must exercise kills and slot recycling"


def test_oracle_runs_all_gpu_scenarios_shapes(orc):
    """Every effect of the GPU parity suite is interpretable by the oracle (catches oracle bugs without a GPU)."""
    w = G.ExprWriter()
    axis, center = w.lit(G.Vec3(0., 0., 1.)), w.lit(G.Vec3(0.5, -0.25, 0.))
    A = G.Attribute
    asset = (G.EffectAsset(500, w.module, simulation_space=G.LOCAL)
             .init(G.SetPositionCircleModifier(center, axis, w.lit(2.), G.VOLUME))
             .init(G.SetVelocityTangentModifier(center, axis, w.lit(1.5)))
             .init(G.SetAttributeModifier(A.AGE, w.lit(0.))).init(G.SetAttributeModifier(A.LIFETIME, w.lit(5.)))
             .update(G.RadialAccelModifier(center, w.lit(-0.5))).update(G.TangentAccelModifier(center, axis, w.lit(0.25))))
    _, size, _ = asset.particle_layout()
    ref = RefWorld(500, size // 4, [Instance(0, 500, alive=0, seed=3)])
    eo = EffectOracle(asset)
    for f in range(3):
        ref.set_spawns([200])
        eo.frame(ref, orc)
        _check_invariants(ref)
    pos = ref.particles[:400, 0:3].view(np.float32)
    assert np.all(np.isfinite(pos))
    # circle of radius 2 around `center` in the z = 0 plane
    d = pos[:, :2] - np.array([0.5, -0.25], dtype=np.float32)
    assert np.all(np.abs(pos[:, 2]) < 0.2)


def test_float_literals_are_seen_through_six_decimals():
    """The reference embeds f32 literals as `{:.6}` text (src/lib.rs:264-269): both the generated CUDA code and the
    oracle must evaluate with the rounded value; properties travel as bytes and keep every bit."""
    from oracle.hanabi_oracle import literal_array
    x = float(np.float32(1.018241286277771))
    w = G.ExprWriter()
    e = w.lit(x).fract()
    asset = (G.EffectAsset(8, w.module).init(G.SetAttributeModifier(G.Attribute.POSITION, w.lit(G.Vec3(0, 0, 0))))
             .update(G.SetAttributeModifier(G.Attribute.F32_0, e)))
    assert "fract(1.018241f)" in asset.generate().update_code
    lit = [nd for nd in w.module.nodes if nd.kind == "lit"][0]
    assert literal_array(lit.value, 1)[0] == np.float32(1.018241)
    assert literal_array(lit.value, 1)[0] != np.float32(x)
    assert literal_array(lit.value, 1, as_shader_text=False)[0] == np.float32(x)
    w.lit(-1e-8)
    v = literal_array(w.module.nodes[-1].value, 1)[0]
    assert v == 0 and np.signbit(v)  # "-0.f"


def test_ribbon_sort_restatement_equals_stable_sort(orc):
    """The literal restatement of vfx_sort_fill / vfx_sort (insertion sort) / vfx_sort_copy and the vectorised
    stable sort used for large instances are the same function (ties keep the alive list's order)."""
    rng = np.random.default_rng(5)
    for n, cap, base in ((0, 8, 0), (1, 8, 3), (2, 8, 0), (257, 400, 16), (1500, 1600, 5)):
        worlds = []
        for literal in (True, False):
            ref = RefWorld(base + cap, 6, [Instance(base, cap, alive=n)])
            r2 = np.random.default_rng(n)
            ref.particles[:] = r2.integers(0, 2**32, ref.particles.shape, dtype=np.uint32)
            ref.particles[:, 4] = r2.integers(0, 4, base + cap, dtype=np.uint32)                      # key: few ribbons
            ref.particles[:, 1] = r2.choice(np.array([0.0, 0.5, 1.0], dtype=np.float32), base + cap).view(np.uint32)  # key2: ties
            ref.indirect[:] = r2.integers(0, 2**32, ref.indirect.shape, dtype=np.uint32)
            ref.indirect[base:base + n, 1] = r2.permutation(cap)[:n]
            ref.metadata[0].indirect_write_index = 1
            ref.metadata[0].sort_key_offset, ref.metadata[0].sort_key2_offset = 4, 1
            before = ref.indirect.copy()
            ref.oracle_sort_ribbons(orc, literal=literal)
            untouched = np.ones_like(before, dtype=bool)
            untouched[base:base + n, 1] = False
            np.testing.assert_array_equal(ref.indirect[untouched], before[untouched])
            assert sorted(ref.indirect[base:base + n, 1].tolist()) == sorted(before[base:base + n, 1].tolist())
            worlds.append(ref.indirect.copy())
        np.testing.assert_array_equal(worlds[0], worlds[1], err_msg=f"n={n}")


def test_ribbon_layout_sets_the_ribbons_flag():
    from bevy_hanabi_b200 import _native as N
    assert ribbon_asset(16).generate().flags & N.EFFECT_RIBBONS
    assert not firework_trails(16).generate().flags & N.EFFECT_RIBBONS
