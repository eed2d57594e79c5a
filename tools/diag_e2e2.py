import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bevy_hanabi_b200 as hb
from bevy_hanabi_b200 import _native as N, recipes, runtime as R
stream = torch.cuda.Stream(); torch.cuda.set_stream(stream)
ctx = hb.Context(0, stream.cuda_stream)
P = 64<<20
slab = ctx.slab_create(P, 32); ctx.slab_fill_c5(slab, 0, P, 42, 1e9, 1e9)
md = R.initial_metadata(P, 0, 8); md.alive_count = P; md.max_spawn = 0
ctx.metadata_insert(0, md); ctx.draw_args_insert(0)
sp = (N.Spawner*1)(R.make_spawner(seed=42)); bi = (N.BatchInfo*1)(N.BatchInfo(0,0,0,0,0,1)); pre=(N.u32*1)(0)
ctx.upload_spawners_raw(sp,1); ctx.upload_batches_raw(bi,1,pre,1); ctx.set_sim_params(1/60,0,1)
x = torch.empty(1<<26, device="cuda", dtype=torch.float32); y = torch.empty_like(x)
for relaxed in (False, True):
    fx = ctx.effect_compile(recipes.c5_lowered(relaxed_order=relaxed))
    la = (N.BatchLaunch*1)(N.BatchLaunch.make(fx, slab, 0, 0))
    for _ in range(5): ctx.simulate_raw(la,1)
    ctx.sync(); ctx.enable_kernel_timing(True); ctx.kernel_time_ms()
    def seq(n, pre=None):
        out=[]
        for i in range(n):
            if pre and i == 0: pre()
            ctx.simulate_raw(la,1)
            # time each kernel separately by draining per launch AFTER all are queued is impossible; so queue n, then read total
        ms,k = ctx.kernel_time_ms()
        return ms/k
    print("relaxed" if relaxed else "ordered")
    for n in (1,2,3,4,6,8,16):
        tot=[]
        for rep in range(6):
            ctx.sync(); time.sleep(0.001)
            for i in range(n): ctx.simulate_raw(la,1)
            ms,k = ctx.kernel_time_ms(); tot.append(ms)
        tot.sort()
        print(f"   {n:2d} kernels queued after a sync: total {tot[len(tot)//2]:.3f} ms  (avg {tot[len(tot)//2]/n:.3f})")
    ctx.sync(); time.sleep(0.001)
    torch.add(x, 1.0, out=y); ctx.simulate_raw(la,1); ms,k = ctx.kernel_time_ms(); print(f"   after sync: torch add 256MB first, then 1 kernel: {ms:.3f} ms")
    ctx.sync(); time.sleep(0.001)
    for _ in range(20): torch.add(x, 1.0, out=y)
    ctx.simulate_raw(la,1); ms,k = ctx.kernel_time_ms(); print(f"   after sync: 20x torch add (2 ms busy), then 1 kernel: {ms:.3f} ms")
