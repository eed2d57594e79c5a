import sys, time, os
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
os.environ["HNB_DEFINES"] = "HNB_PROFILE=1"
fx = ctx.effect_compile(recipes.c5_lowered())
la = (N.BatchLaunch*1)(N.BatchLaunch.make(fx, slab, 0, 0))
for _ in range(5): ctx.simulate_raw(la,1)
ctx.sync(); ctx.enable_kernel_timing(True); ctx.kernel_time_ms(); ctx.read_debug()
def show(tag):
    ms,k = ctx.kernel_time_ms(); d = ctx.read_debug()
    w = max(d[5],1)
    print(f"{tag:28s} kernel {ms/k:.3f} ms | per-warp Mcycles: pass1 {d[0]/w/1e6:.3f} lookback {d[1]/w/1e6:.3f} pass2 {d[2]/w/1e6:.3f} | polls/tile {d[3]/max(d[4],1):.2f} tiles {d[4]} warps {d[5]} longest warp {d[6]/1e6:.3f} Mcyc")
for rep in range(3):
    ctx.sync(); time.sleep(0.001)
    ctx.simulate_raw(la,1); show("1st after sync")
    ctx.sync(); time.sleep(0.001)
    ctx.simulate_raw(la,1); ctx.simulate_raw(la,1); ctx.simulate_raw(la,1); ctx.simulate_raw(la,1)
    # can't split counters per kernel when queued; so measure aggregated over 4 (2 slow + 2 fast)
    show("4 queued after sync (sum/4)")
for _ in range(10): ctx.simulate_raw(la,1)
ctx.read_debug(); ctx.kernel_time_ms()
for _ in range(1): ctx.simulate_raw(la,1)
show("11th in a queued run")
