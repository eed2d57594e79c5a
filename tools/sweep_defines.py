"""Kernel-variant sweep: time hnb_update for several HNB_DEFINES settings on the C5 workload."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bevy_hanabi_b200 as hb
from bevy_hanabi_b200 import _native as N, recipes, runtime as R
stream = torch.cuda.Stream(); torch.cuda.set_stream(stream)
ctx = hb.Context(0, stream.cuda_stream)
P = int(os.environ.get("SWEEP_P", 64 << 20))
slab = ctx.slab_create(P, 32); ctx.slab_fill_c5(slab, 0, P, 42, 1e9, 1e9)
md = R.initial_metadata(P, 0, 8); md.alive_count = P; md.max_spawn = 0
ctx.metadata_insert(0, md); ctx.draw_args_insert(0)
sp = (N.Spawner*1)(R.make_spawner(seed=42)); bi = (N.BatchInfo*1)(N.BatchInfo(0,0,0,0,0,1)); pre=(N.u32*1)(0)
ctx.upload_spawners_raw(sp,1); ctx.upload_batches_raw(bi,1,pre,1); ctx.set_sim_params(1/60,0,1)
for defs in sys.argv[1:]:
    os.environ["HNB_DEFINES"] = defs
    try:
        fx = ctx.effect_compile(recipes.c5_lowered())
    except Exception as e:
        print(f"{defs[:90]:90s} COMPILE ERROR {str(e)[:300]}"); continue
    la = (N.BatchLaunch*1)(N.BatchLaunch.make(fx, slab, 0, 0))
    for _ in range(5): ctx.simulate_raw(la,1)
    ctx.sync(); ctx.enable_kernel_timing(True); ctx.kernel_time_ms()
    for _ in range(40): ctx.simulate_raw(la,1)
    ms,k = ctx.kernel_time_ms()
    print(f"{defs[:90]:90s} update {ms/k:.4f} ms  {72*P/(ms/k*1e-3)/1e9:.0f} GB/s")
