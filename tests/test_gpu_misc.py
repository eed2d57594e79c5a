"""GPU tests of the edges: error behaviour of the C ABI (≙ simulate()'s "skip the frame rather than desynchronise
buffers", reference mod.rs:6994-7022), odd particle layouts through the AoS<->SoA interop, the >2047-instance
batch path (tile-prefix search in global memory), slab slice reset, and randomised expression graphs
(hypothesis) compared bit-for-bit with the oracle's interpreter."""
import ctypes as C

import numpy as np
import pytest

from bevy_hanabi_b200 import _native as N
from bevy_hanabi_b200 import graph as G
from bevy_hanabi_b200 import recipes
from bevy_hanabi_b200 import runtime as R
from bevy_hanabi_b200._native import HanabiError
from oracle.hanabi_oracle import EffectOracle
from tests.effects import exact_expr
from tests.helpers import GpuWorld, Instance, RefWorld, assert_world_equal

pytestmark = pytest.mark.gpu
A = G.Attribute


def test_error_paths_leave_state_untouched(ctx):
    fx32 = ctx.effect_compile(recipes.c5_lowered())
    slab32 = ctx.slab_create(1024, 32)
    slab48 = ctx.slab_create(1024, 48)
    ctx.metadata_insert(0, R.initial_metadata(1024, 0, 8))
    ctx.draw_args_insert(0)
    ctx.upload_spawners([R.make_spawner(seed=1)])
    ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, 1)], [0])
    ctx.set_sim_params(1 / 60, 0.0, 1)
    before = bytes(ctx.read_metadata(0))
    with pytest.raises(HanabiError) as e:  # effect compiled for a 32-byte record, slab holds 48-byte records
        ctx.simulate([N.BatchLaunch.make(fx32, slab48, 0, 0)])
    assert e.value.code == N.HNB_ERR_LAYOUT
    with pytest.raises(HanabiError) as e:  # unknown handles
        ctx.simulate([N.BatchLaunch.make(fx32, 99, 0, 0)])
    assert e.value.code == N.HNB_ERR_INVALID_ARG
    with pytest.raises(HanabiError) as e:
        ctx.simulate([N.BatchLaunch.make(77, slab32, 0, 0)])
    assert e.value.code == N.HNB_ERR_INVALID_ARG
    with pytest.raises(HanabiError) as e:  # batch index beyond the uploaded table
        ctx.simulate([N.BatchLaunch.make(fx32, slab32, 3, 0)])
    assert e.value.code == N.HNB_ERR_OUT_OF_RANGE
    with pytest.raises(HanabiError) as e:  # an uploaded batch is not launched
        ctx.simulate([])
    assert e.value.code == N.HNB_ERR_NOT_READY
    ctx.set_sim_params(1 / 60, 0.0, 2)     # more effects than spawner rows
    with pytest.raises(HanabiError) as e:
        ctx.simulate([N.BatchLaunch.make(fx32, slab32, 0, 0)])
    assert e.value.code == N.HNB_ERR_NOT_READY
    ctx.set_sim_params(1 / 60, 0.0, 1)
    ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, 1), N.BatchInfo(0, 0, 0, 0, 0, 1)], [0])  # overlapping batches
    with pytest.raises(HanabiError) as e:
        ctx.simulate([N.BatchLaunch.make(fx32, slab32, 0, 0), N.BatchLaunch.make(fx32, slab32, 1, 0)])
    assert e.value.code == N.HNB_ERR_BATCH_COVERAGE
    ctx.sync()
    assert bytes(ctx.read_metadata(0)) == before, "a rejected frame must not touch device state"
    # out-of-range row accesses
    with pytest.raises(HanabiError):
        ctx.slab_download_aos(slab32, 1000, 100, 32)
    with pytest.raises(HanabiError):
        ctx.read_metadata(12345)
    # a generated kernel that does not compile reports the NVRTC log
    bad = recipes.c5_lowered()
    bad.update_code = "    this is not CUDA;"
    with pytest.raises(HanabiError) as e:
        ctx.effect_compile(bad)
    assert e.value.code == N.HNB_ERR_NVRTC and "error" in e.value.message
    # and the context is still usable
    ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, 1)], [0])
    ctx.simulate([N.BatchLaunch.make(fx32, slab32, 0, 0)])
    ctx.sync()


def test_properties_required(ctx):
    w = G.ExprWriter()
    p = w.add_property("g", G.Vec3(0, -1, 0))
    asset = (G.EffectAsset(64, w.module).init(G.SetAttributeModifier(A.POSITION, w.lit(G.Vec3(0, 0, 0))))
             .init(G.SetAttributeModifier(A.VELOCITY, w.prop(p))))
    fx = ctx.effect_compile(asset.generate())
    slab = ctx.slab_create(64, asset.particle_layout()[1])
    ctx.metadata_insert(0, R.initial_metadata(64, 0, 8, properties_array_index=0))
    ctx.draw_args_insert(0)
    ctx.upload_spawners([R.make_spawner(spawn=4)])
    ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, 1)], [0])
    ctx.set_sim_params(1 / 60, 0.0, 1)
    with pytest.raises(HanabiError) as e:
        ctx.simulate([N.BatchLaunch.make(fx, slab, 0, 4)])
    assert e.value.code == N.HNB_ERR_NOT_READY
    with pytest.raises(HanabiError):  # wrong blob size
        ctx.upload_properties(fx, 0, b"\0" * 4)
    ctx.upload_properties(fx, 0, asset.serialize_properties())
    ctx.simulate([N.BatchLaunch.make(fx, slab, 0, 4)])
    ctx.sync()
    assert ctx.read_metadata(0).alive_count == 4


@pytest.mark.parametrize("stride", [4, 8, 12, 16, 20, 28, 48, 52, 100])
def test_aos_soa_roundtrip_odd_strides(ctx, stride):
    """Planes of 16/8/4 bytes: every record size that is a multiple of 4 must round-trip through the SoA store."""
    rng = np.random.default_rng(stride)
    rows = 1000
    slab = ctx.slab_create(rows, stride)
    data = rng.integers(0, 2**32, (rows, stride // 4), dtype=np.uint32)
    ctx.slab_upload_aos(slab, 0, data)
    np.testing.assert_array_equal(ctx.slab_download_aos(slab, 0, rows, stride), data)
    part = rng.integers(0, 2**32, (100, stride // 4), dtype=np.uint32)
    ctx.slab_upload_aos(slab, 450, part)
    data[450:550] = part
    np.testing.assert_array_equal(ctx.slab_download_aos(slab, 0, rows, stride), data)
    np.testing.assert_array_equal(ctx.slab_download_aos(slab, 440, 30, stride), data[440:470])
    ind = rng.integers(0, 2**32, (rows, 3), dtype=np.uint32)
    ctx.slab_upload_indirect(slab, 0, ind)
    np.testing.assert_array_equal(ctx.slab_download_indirect(slab, 0, rows), ind)
    ctx.slab_reset_rows(slab, 100, 50)  # dead[i] = i, ping = pong = 0 (effect_cache.rs:309-322)
    got = ctx.slab_download_indirect(slab, 0, rows)
    ind[100:150, 0:2] = 0
    ind[100:150, 2] = np.arange(100, 150)
    np.testing.assert_array_equal(got, ind)


def test_slab_create_initial_contents(ctx):
    slab = ctx.slab_create(300, 32)
    ind = ctx.slab_download_indirect(slab, 0, 300)
    assert np.all(ind[:, 0] == 0) and np.all(ind[:, 1] == 0)
    np.testing.assert_array_equal(ind[:, 2], np.arange(300))
    assert not ctx.slab_download_aos(slab, 0, 300, 32).any()


def test_batch_with_more_instances_than_the_shared_memory_table(ctx, orc):
    """3000 instances in ONE batch: the tile-prefix table does not fit the 2047-entry shared-memory stage, so tiles
    are located by binary search in global memory. Also: many empty and single-tile instances."""
    rng = np.random.default_rng(8)
    n_inst = 3000
    caps = rng.integers(1, 90, n_inst)
    alive = [int(rng.integers(0, c + 1)) if rng.random() > 0.1 else 0 for c in caps]
    insts, off = [], 0
    for c, a in zip(caps, alive):
        insts.append(Instance(off, int(c), alive=a, seed=off * 7 + 1))
        off += int(c)
    ref = RefWorld(off, 8, insts)
    for inst in ref.instances:
        n = inst.alive
        p = np.zeros((n, 8), dtype=np.float32)
        p[:, 0:3] = rng.uniform(-1, 1, (n, 3)); p[:, 4:7] = rng.uniform(-1, 1, (n, 3)); p[:, 7] = rng.uniform(0.02, 0.2, n)
        ref.particles[inst.slab_offset:inst.slab_offset + n] = p.view(np.uint32)
    gpu = GpuWorld(ctx, ref, recipes.c5_lowered())
    k = (C.c_float * 4)(0.0, -9.8, 0.0, 0.5)
    for step in range(8):
        ref.oracle_frame(orc, orc.orc_body_update_c5(), k)
        gpu.frame()
        if step in (0, 3, 7):
            assert_world_equal(ref, gpu.pull(), what=f"step {step}")


def test_empty_frames(ctx):
    """No effects at all, then an instance that is empty and asks for nothing: frames must be no-ops."""
    ctx.set_sim_params(1 / 60, 0.0, 0)
    ctx.simulate([])
    ctx.sync()
    fx = ctx.effect_compile(recipes.c5_lowered())
    slab = ctx.slab_create(256, 32)
    ctx.metadata_insert(0, R.initial_metadata(256, 0, 8))
    ctx.draw_args_insert(0)
    ctx.upload_spawners([R.make_spawner(seed=1)])
    ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, 1)], [0])
    ctx.set_sim_params(1 / 60, 0.0, 1)
    for _ in range(3):
        ctx.simulate([N.BatchLaunch.make(fx, slab, 0, 0)])
    md = ctx.read_metadata(0)
    assert (md.alive_count, md.max_update, md.max_spawn, md.particle_counter) == (0, 0, 256, 0)
    assert ctx.read_draw_args(0).instance_count == 0
    assert ctx.read_batch_info(0).total_update_count == 0
    ind = ctx.slab_download_indirect(slab, 0, 256)
    np.testing.assert_array_equal(ind[:, 2], np.arange(256))


def test_effect_from_background_compile_job(ctx, orc):
    """hnb_compile_job_* + hnb_effect_create_from_job: compiled off-thread, loaded into the context, same results as
    the synchronous path; one job serves several contexts."""
    job = R.CompileJob(recipes.c5_lowered())
    job.wait()
    effect = ctx.effect_create_from_job(job)
    rng = np.random.default_rng(11)
    n = 5000
    ref = RefWorld(n, 8, [Instance(0, n, alive=n, seed=9)])
    p = np.zeros((n, 8), dtype=np.float32)
    p[:, 0:3] = rng.uniform(-1, 1, (n, 3)); p[:, 4:7] = rng.uniform(-1, 1, (n, 3)); p[:, 7] = rng.uniform(0.01, 0.2, n)
    ref.particles[:] = p.view(np.uint32)
    gpu = GpuWorld(ctx, ref, None, effect=effect)
    k = (C.c_float * 4)(0.0, -9.8, 0.0, 0.5)
    for step in range(4):
        ref.oracle_frame(orc, orc.orc_body_update_c5(), k)
        gpu.frame()
    assert_world_equal(ref, gpu.pull(), what="effect from a compile job")
    assert ctx.effect_create_from_job(job) != effect   # registering again gives a new handle on the cached module
    job.close()


def test_epoch_wrap(native, orc, monkeypatch):
    """The look-back's tile states carry a 30-bit frame epoch; frames across the wrap must stay exact."""
    monkeypatch.setenv("HNB_EPOCH_START", str(0x3fffffff - 3))
    c = native.Context(0)
    try:
        rng = np.random.default_rng(3)
        n = 200_000
        ref = RefWorld(n, 8, [Instance(0, n, alive=n, seed=9)])
        p = np.zeros((n, 8), dtype=np.float32)
        p[:, 0:3] = rng.uniform(-1, 1, (n, 3)); p[:, 4:7] = rng.uniform(-1, 1, (n, 3)); p[:, 7] = rng.uniform(0.01, 0.2, n)
        ref.particles[:] = p.view(np.uint32)
        gpu = GpuWorld(c, ref, recipes.c5_lowered())
        k = (C.c_float * 4)(0.0, -9.8, 0.0, 0.5)
        for step in range(8):
            ref.oracle_frame(orc, orc.orc_body_update_c5(), k)
            gpu.frame()
            assert_world_equal(ref, gpu.pull(), what=f"step {step}")
    finally:
        c.close()


# ---- randomised expression graphs ---------------------------------------------------------------------
hypothesis = pytest.importorskip("hypothesis")
from hypothesis import HealthCheck, Phase, given, settings, strategies as st  # noqa: E402


# no shrinking: every example costs an NVRTC compile and a few GPU frames
@settings(max_examples=20, deadline=None, suppress_health_check=list(HealthCheck), phases=[Phase.generate], derandomize=True)
@given(st.data())
def test_random_expression_graphs_bit_exact(ctx, orc, data):
    w = G.ExprWriter()
    f_expr = exact_expr(data.draw, w, data.draw(st.integers(1, 3)), "f")
    v_expr = exact_expr(data.draw, w, data.draw(st.integers(1, 3)), "v")
    asset = (G.EffectAsset(600, w.module, name="fuzz")
             .init(G.SetAttributeModifier(A.POSITION, w.rand(G.VEC3) * w.lit(4.) - w.lit(2.)))
             .init(G.SetAttributeModifier(A.VELOCITY, w.rand(G.VEC3) - w.lit(0.5)))
             .init(G.SetAttributeModifier(A.AGE, w.lit(0.)))
             .init(G.SetAttributeModifier(A.LIFETIME, w.lit(0.05).uniform(w.lit(0.2))))
             .init(G.SetAttributeModifier(A.F32_1, w.rand() * w.lit(3.)))
             .update(G.SetAttributeModifier(A.F32_0, f_expr))
             .update(G.SetAttributeModifier(A.F32X3_0, v_expr)))
    _, size, _ = asset.particle_layout()
    ref = RefWorld(600, size // 4, [Instance(0, 600, alive=0, seed=data.draw(st.integers(0, 2**32 - 1)))])
    eo = EffectOracle(asset)
    gpu = GpuWorld(ctx, ref, asset.generate())
    for f in range(4):
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        ref.set_spawns([300 if f == 0 else 40])
        eo.frame(ref, orc)
        gpu.frame()
    got = gpu.pull()
    # NaNs may legitimately appear (0 * inf ...); compare bit patterns except that any NaN equals any NaN
    a, b = got["particles"].copy(), ref.particles.copy()
    fa, fb = a.view(np.float32), b.view(np.float32)
    both_nan = np.isnan(fa) & np.isnan(fb)
    both_zero = (fa == 0) & (fb == 0)  # min/max of (+0, -0) may legitimately return either zero (IEEE minNum/maxNum)
    a[both_nan | both_zero] = 0
    b[both_nan | both_zero] = 0
    fx = asset.generate()
    np.testing.assert_array_equal(a, b, err_msg="generated update code:\n" + fx.update_code)
    np.testing.assert_array_equal(got["indirect"], ref.indirect)
    np.testing.assert_array_equal(got["metadata"], ref.metadata_rows())


def test_second_standalone_init_before_indirect_is_refused(ctx):
    """ADVICE r1: init accounting is deferred to the indirect pass; a second stand-alone init of the same batch before it
    would pop the same dead slots. The library refuses it instead of corrupting the counters."""
    from bevy_hanabi_b200 import _native as N, recipes, runtime as R
    slab = ctx.slab_create(256, 32)
    effect = ctx.effect_compile(recipes.c5_lowered())
    ctx.metadata_insert(0, R.initial_metadata(256, 0, 8))
    ctx.draw_args_insert(0)
    ctx.upload_spawners([R.make_spawner(spawn=10, seed=1)])
    ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, 1)], [0])
    ctx.set_sim_params(1 / 60, 0.0, 1)
    la = N.BatchLaunch.make(effect, slab, 0, 10)
    ctx.pass_init(la)
    with pytest.raises(Exception, match="init pass pending"):
        ctx.pass_init(la)
    ctx.pass_indirect()
    assert ctx.read_metadata(0).alive_count == 10
    ctx.pass_init(la)   # fine again once the accounting has been applied
    ctx.pass_indirect()
    assert ctx.read_metadata(0).alive_count == 20 and ctx.read_metadata(0).particle_counter == 20
