"""BASELINE.json's C2 and C3 at their quoted sizes.

tests/test_gpu_effects.py runs the same effects at 4096 / 8192 particles; tests/test_gpu_fullsize.py covers C4 and C5 at
full size through checksums. These two compare EVERY record with the numpy interpreter at the sizes BASELINE.json names
(the interpreter needs a few seconds per frame at 1 Mi particles)."""
import numpy as np
import pytest

from bevy_hanabi_b200 import graph as G
from oracle.hanabi_oracle import pcg_hash
from tests.helpers import Instance, RefWorld
from tests.test_gpu_effects import _firework_trails, _force_field, _run

pytestmark = pytest.mark.gpu


def test_c2_firework_at_32768(ctx, orc):
    """configs[1]: "firework.rs effect, 32768 capacity": bursts into recycled slots, IEEE-exact, zero tolerance."""
    asset = _firework_trails(32768)
    _, size, _ = asset.particle_layout()
    ref = RefWorld(32768, size // 4, [Instance(0, 32768, alive=0)], dt=1.0 / 20.0)
    seeds = lambda f: [int(pcg_hash(np.array([0x4321 + f], dtype=np.uint32))[0])]
    _run(ctx, orc, asset, ref, 50, lambda f: [9000 if f % 20 == 0 else 150], seeds=seeds, check_every=5)
    assert ref.metadata[0].particle_counter > 30000 and 0 < ref.metadata[0].alive_count < 32768


def test_c3_force_field_at_1m(ctx, orc):
    """configs[2]: "force_field.rs: 1M particles": 1e-5 of the attribute's magnitude per step (sphere sampling and the
    ConformToSphere modifiers go through libm), every integer structure exact."""
    n = 1 << 20
    asset = _force_field(n)
    _, size, _ = asset.particle_layout()
    ref = RefWorld(n, size // 4, [Instance(0, n, alive=0, seed=77)])
    props = [{"attraction_accel": 18.0, "repulsor_position": G.Vec3(0.25, 0.5, 0.1)}]
    _run(ctx, orc, asset, ref, 6, lambda f: [n - 4096 if f == 0 else 500], rtol=1e-5, props=props)
    assert ref.metadata[0].alive_count > (n >> 1)


def _instancing(capacity):
    """BASELINE config C4's recipe (examples/instancing.rs:224-249, main effect): SetPositionSphere(Volume, r=1),
    SetVelocitySphere(speed 2), age 0, lifetime 12; no update modifier (Euler integration + age / reap only)."""
    w = G.ExprWriter()
    A = G.Attribute
    return (G.EffectAsset(capacity, w.module, name="instancing")
            .init(G.SetPositionSphereModifier(w.lit(G.Vec3(0, 0, 0)), w.lit(1.), G.VOLUME))
            .init(G.SetVelocitySphereModifier(w.lit(G.Vec3(0, 0, 0)), w.lit(2.)))
            .init(G.SetAttributeModifier(A.AGE, w.lit(0.)))
            .init(G.SetAttributeModifier(A.LIFETIME, w.lit(12.))))


def test_c4_instancing_recipe_1024_instances_one_batch(ctx, orc):
    """configs[3]: "instancing.rs: 1024 effect instances x 65536 particles, batched dispatch" with ITS recipe and ITS
    topology (one batch of 1024 instances of 65536 slots: init and update locate their instance with a depth-10 search of
    the 1024-entry prefix sums; 1024 independent look-back chains), SURVEY.md §8d row C4: a burst per instance through the
    real init kernel, then "spawn 1 / instance / step" frames (init of 1024 threads spread over 1024 instances + update), then
    one long step that expires every particle (1024 dead-stack pushes of whole populations). EVERY record and list entry of
    the 64 Mi-slot slab is compared with the numpy interpreter: integers exact, fp32 within 1e-5 of the attribute (sphere
    sampling goes through pow / sin / cos). Per-instance seeds = pcg_hash(i)."""
    from tests.test_gpu_effects import _float_word_mask
    from oracle.hanabi_oracle import EffectOracle
    from tests.helpers import GpuWorld, assert_world_equal
    n_inst, cap, burst = 1024, 65536, 8192
    asset = _instancing(cap)
    _, size, _ = asset.particle_layout()
    assert size == 32
    seeds = pcg_hash(np.arange(n_inst, dtype=np.uint32))
    ref = RefWorld(n_inst * cap, size // 4, [Instance(i * cap, cap, alive=0, seed=int(seeds[i])) for i in range(n_inst)])
    eo = EffectOracle(asset, None)
    gpu = GpuWorld(ctx, ref, asset.generate())
    mask, fattrs = _float_word_mask(asset)
    dt = ref.sim.delta_time
    for f in range(6):
        ref.sim.time = np.float32(f) * dt
        ref.sim.virtual_time = ref.sim.real_time = ref.sim.time
        if f == 5:  # everything expires: age + 12 >= lifetime for every particle, the ones spawned this frame included
            ref.sim.delta_time = ref.sim.virtual_delta_time = ref.sim.real_delta_time = np.float32(12.0)
        ref.set_spawns([burst if f == 0 else 1 + (i & 1) * (f & 1) for i in range(n_inst)])  # 1 (or 2) per instance per step
        eo.frame(ref, orc)
        gpu.frame()
        if f in (0, 4, 5):
            got = gpu.pull()
            assert_world_equal(ref, got, float_words=mask, rtol=1e-5, what=f"frame {f}", float_attrs=fattrs)
            if f != 5:
                ctx.slab_upload_aos(gpu.slab, 0, ref.particles)  # 1e-5 is a per-step bound (see test_gpu_effects._run)
    md = ref.metadata_rows()
    assert int(ref.metadata[0].particle_counter) == burst + 5 and int(ref.metadata[1].particle_counter) == burst + 8
    assert all(ref.metadata[i].alive_count == 0 and ref.metadata[i].max_spawn == cap for i in range(n_inst)), md[:4]
    ctx.slab_destroy(gpu.slab)


def test_c3_force_field_free_running_60_frames(ctx, orc):
    """The rtol tests above restart every compared frame from the oracle's state (the 1e-5 bound is per step). This one does
    NOT: a 64 Ki-particle force field runs 60 frames on the device and in the interpreter independently, and the
    divergence is REPORTED (printed) and bounded:
      * kill decisions that flip (a particle crossing a kill surface one frame earlier or later on one side) show up as
        the symmetric difference of the two alive SETS;
      * fp32 drift of the particles alive on both sides, relative to the attribute's magnitude.
    No spawning after the burst, so a slot always holds the same particle on both sides and the sets are comparable."""
    from tests.test_gpu_effects import _float_word_mask
    from oracle.hanabi_oracle import EffectOracle
    from tests.helpers import GpuWorld
    n = 1 << 16
    # kill volumes pulled in so that they bite: the box is left by ~80 % of the particles between frames 10 and 30, the
    # small sphere sits on the attractor
    asset = _force_field(n, aabb_half=(0.8, 0.6, 0.8), kill_center=(0.6, -0.2, 0.), kill_r2=0.0025)
    _, size, _ = asset.particle_layout()
    ref = RefWorld(n, size // 4, [Instance(0, n, alive=0, seed=77)])
    props = [{"attraction_accel": 18.0, "repulsor_position": G.Vec3(0.25, 0.5, 0.1)}]
    ref.metadata[0].properties_array_index = 0
    eo = EffectOracle(asset, {0: props[0]})
    gpu = GpuWorld(ctx, ref, asset.generate(), property_blobs=[asset.serialize_properties(props[0])])
    _, fattrs = _float_word_mask(asset)
    rows = []
    for f in range(60):
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        ref.sim.virtual_time = ref.sim.real_time = ref.sim.time
        ref.set_spawns([n if f == 0 else 0])
        eo.frame(ref, orc)
        gpu.frame()
        if f % 10 == 9 or f == 0:
            got = gpu.pull()
            w_ref, w_gpu = ref.metadata[0].indirect_write_index, int(got["metadata"][0][4])
            a_ref, a_gpu = int(ref.metadata[0].alive_count), int(got["metadata"][0][1])
            s_ref = ref.indirect[:a_ref, w_ref]
            s_gpu = got["indirect"][:a_gpu, w_gpu]
            flipped = np.setxor1d(s_ref, s_gpu)
            common = np.intersect1d(s_ref, s_gpu)
            drift = drift99 = 0.0
            for first, cnt in fattrs:
                a = np.ascontiguousarray(got["particles"][common, first:first + cnt]).view(np.float32).astype(np.float64)
                b = np.ascontiguousarray(ref.particles[common, first:first + cnt]).view(np.float32).astype(np.float64)
                scale = np.maximum(np.max(np.abs(b), axis=1, keepdims=True), 1e-3)
                rel = np.max(np.abs(a - b) / scale, axis=1)
                drift = max(drift, float(np.max(rel)))
                drift99 = max(drift99, float(np.percentile(rel, 99)))
            # the order of the survivors both sides agree on is still the canonical one on both sides
            assert np.array_equal(s_ref[np.isin(s_ref, common)], s_gpu[np.isin(s_gpu, common)])
            rows.append({"frame": f, "alive_oracle": a_ref, "alive_device": a_gpu, "kill_decisions_flipped": int(flipped.size), "max_rel_drift": drift, "p99_rel_drift": drift99})
    print(rows)
    assert rows[0]["kill_decisions_flipped"] == 0
    assert rows[-1]["alive_oracle"] < n // 2, "the scenario must kill a good part of the particles"
    assert max(r["kill_decisions_flipped"] for r in rows) <= n // 100, rows   # <= 1 % of the particles at any compared frame
    assert rows[-1]["p99_rel_drift"] < 1e-2, rows                              # 60 free-running steps of a stiff force field
