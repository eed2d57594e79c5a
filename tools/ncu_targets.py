"""Exactly the launches an `ncu --profile-from-start off` capture should see, one scenario per process.

usage (on a GPU box):
  ncu --set full --clock-control none --import-source on --profile-from-start off -o gpurun_out/r2_ncu_<scenario> \
      python tools/ncu_targets.py <scenario>
Every scenario sets its state up and warms the kernels OUTSIDE the profiled range, then brackets ONE frame (or one call)
with cudaProfilerStart / cudaProfilerStop, so a report holds one launch of each kernel of that frame: hnb_init (when the
frame spawns), k_bookkeeping, hnb_update. `tools/ncu_summary.py` turns the report into a text summary.
"""
import os, sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import bevy_hanabi_b200 as hb
from bevy_hanabi_b200 import _native as N, graph as G, recipes, runtime as R

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import perf_matrix as PM   # scenario helpers (single_instance, recipes of the other configs)

A = G.Attribute
stream = PM.stream


def profiled(fn):
    torch.cuda.synchronize()
    torch.cuda.profiler.start()
    fn()
    torch.cuda.synchronize()
    torch.cuda.profiler.stop()


def c5(mi, slot_order=False):
    P = mi << 20
    ctx = hb.Context(0, stream.cuda_stream)
    slab = ctx.slab_create(P, 32)
    ctx.slab_fill_c5(slab, 0, P, 42, 1e9, 1e9)
    PM.single_instance(ctx, P, 32, alive=P)
    la = [N.BatchLaunch.make(ctx.effect_compile(recipes.c5_lowered(slot_order=slot_order)), slab, 0, 0)]
    for _ in range(5):
        ctx.simulate(la)
    profiled(lambda: ctx.simulate(la))
    ctx.close()


def burst(asset, P, spawn, props=None, update_frames=1):
    """frame 1 (profiled): init of `spawn` particles + bookkeeping + update of them; then `update_frames` plain frames."""
    ctx = hb.Context(0, stream.cuda_stream)
    fx = asset.generate()
    stride = fx.particle_stride
    slab = ctx.slab_create(P, stride)
    effect = ctx.effect_compile(fx)
    if props is not None:
        ctx.upload_properties(effect, 0, props)
    md = R.initial_metadata(P, 0, stride // 4, properties_array_index=0 if props is not None else N.INVALID)
    ctx.metadata_insert(0, md)
    ctx.draw_args_insert(0)
    ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, 1)], [0])
    ctx.set_sim_params(1 / 60, 0.0, 1)
    ctx.upload_spawners([R.make_spawner(spawn=1024, seed=1)])
    ctx.simulate([N.BatchLaunch.make(effect, slab, 0, 1024)])   # warm-up pair of kernels
    ctx.sync()
    ctx.slab_reset_rows(slab, 0, P)
    ctx.metadata_insert(0, md)
    ctx.upload_spawners([R.make_spawner(spawn=spawn, seed=7)])
    profiled(lambda: ctx.simulate([N.BatchLaunch.make(effect, slab, 0, spawn)]))
    ctx.upload_spawners([R.make_spawner(spawn=0, seed=8)])
    la = [N.BatchLaunch.make(effect, slab, 0, 0)]
    ctx.simulate(la)
    profiled(lambda: [ctx.simulate(la) for _ in range(update_frames)])
    ctx.close()


def c5_init():
    w = G.ExprWriter()
    asset = (G.EffectAsset(64 << 20, w.module, name="c5_spawned")
             .init(G.SetAttributeModifier(A.POSITION, w.rand(G.VEC3) * w.lit(2.) - w.lit(1.)))
             .init(G.SetAttributeModifier(A.VELOCITY, w.rand(G.VEC3) * w.lit(2.) - w.lit(1.)))
             .init(G.SetAttributeModifier(A.AGE, w.lit(0.)))
             .init(G.SetAttributeModifier(A.LIFETIME, w.lit(1e9)))
             .update(G.AccelModifier(w.lit(G.Vec3(0., -9.8, 0.))))
             .update(G.LinearDragModifier(w.lit(0.5))))
    burst(asset, 64 << 20, 32 << 20)


def c3(mi):
    from tests.effects import force_field
    P = mi << 20
    asset = force_field(P)
    burst(asset, P, P, props=asset.serialize_properties())


def c2():
    """firework trails at its BASELINE capacity: 32768 slots, a burst of 30000, then plain frames."""
    from tests.effects import firework_trails
    burst(firework_trails(32768), 32768, 30000, update_frames=2)


def c4():
    """C4: 1024 instances x 65536 slots in one batch with the instancing.rs recipe: a frame that spawns one particle per
    instance into a nearly full slab (init with a depth-10 prefix search + bookkeeping of 1024 instances + update of 64 Mi)."""
    from tests.effects import instancing
    n_inst, cap = 1024, 65536
    ctx = hb.Context(0, stream.cuda_stream)
    fx = instancing(cap).generate()
    slab = ctx.slab_create(n_inst * cap, fx.particle_stride)
    effect = ctx.effect_compile(fx)
    for i in range(n_inst):
        ctx.metadata_insert(i, R.initial_metadata(cap, i, fx.particle_stride // 4))
        ctx.draw_args_insert(i)
    ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, n_inst)], [i * (cap - 64) for i in range(n_inst)])
    ctx.set_sim_params(1 / 60, 0.0, n_inst)
    mk = lambda spawn: [R.make_spawner(spawn=spawn, seed=1000 + i, effect_metadata_index=i, draw_indirect_index=i, slab_offset=i * cap) for i in range(n_inst)]
    ctx.upload_spawners(mk(cap - 64))
    ctx.simulate([N.BatchLaunch.make(effect, slab, 0, n_inst * (cap - 64))])     # fill through the real init kernel
    ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, n_inst)], list(range(n_inst)))
    ctx.upload_spawners(mk(1))
    la = [N.BatchLaunch.make(effect, slab, 0, n_inst)]
    ctx.simulate(la)
    profiled(lambda: ctx.simulate(la))
    assert ctx.read_metadata(5).alive_count == cap - 64 + 2
    ctx.close()


def churn(slot_order=False):
    """The steady-state churn world of perf_matrix.churn (16 Mi slots, ~13 Mi alive in recycled slots): one profiled frame."""
    from tests.effects import drifting_sparks
    P = 16 << 20
    ctx = hb.Context(0, stream.cuda_stream)
    fx = drifting_sparks(P).generate(slot_order=slot_order)
    slab = ctx.slab_create(P, fx.particle_stride)
    effect = ctx.effect_compile(fx)
    ctx.metadata_insert(0, R.initial_metadata(P, 0, fx.particle_stride // 4))
    ctx.draw_args_insert(0)
    ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, 1)], [0])
    dt, rate = 1 / 60, P // 40
    la = [N.BatchLaunch.make(effect, slab, 0, rate)]

    def frame(f):
        ctx.set_sim_params(dt, f * dt, 1)
        ctx.upload_spawners([R.make_spawner(spawn=rate, seed=1000 + f)])
        ctx.simulate(la)
    for f in range(240):
        frame(f)
    profiled(lambda: frame(240))
    print("alive", ctx.read_metadata(0).alive_count, flush=True)
    ctx.close()


def interop():
    P = 64 << 20
    ctx = hb.Context(0, stream.cuda_stream)
    slab = ctx.slab_create(P, 32)
    buf, ibuf = ctx.device_alloc(P * 32), ctx.device_alloc(P * 12)
    ctx.slab_export_aos_device(slab, 0, P, buf)
    ctx.slab_export_indirect_device(slab, 0, P, ibuf)

    def calls():
        ctx.slab_export_aos_device(slab, 0, P, buf)
        ctx.slab_import_aos_device(slab, 0, P, buf)
        ctx.slab_export_indirect_device(slab, 0, P, ibuf)
        ctx.slab_import_indirect_device(slab, 0, P, ibuf)
    profiled(calls)
    ctx.close()


SCENARIOS = {"c5_64m": lambda: c5(64), "c5_32m": lambda: c5(32), "c5_16m": lambda: c5(16), "c5_8m": lambda: c5(8), "c5_1m": lambda: c5(1), "c5_64m_slot": lambda: c5(64, True), "c5_init": c5_init, "c3_16m": lambda: c3(16),
             "c3_1m": lambda: c3(1), "c2": c2, "c4": c4, "churn": churn, "churn_slot": lambda: churn(True), "interop": interop}
if __name__ == "__main__":
    SCENARIOS[sys.argv[1]]()
