"""Diagnostics: why does hnb_update run slower when the host synchronises every step?"""
import os, sys, time, ctypes as C
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bevy_hanabi_b200 as hb
from bevy_hanabi_b200 import _native as N, recipes, runtime as R
stream = torch.cuda.Stream(); torch.cuda.set_stream(stream)
ctx = hb.Context(0, stream.cuda_stream)
P = 64*1024*1024
slab = ctx.slab_create(P, 32); fx = ctx.effect_compile(recipes.c5_lowered())
ctx.slab_fill_c5(slab, 0, P, 42, 1e9, 1e9)
md = R.initial_metadata(P, 0, 8); md.alive_count = P; md.max_spawn = 0
ctx.metadata_insert(0, md); ctx.draw_args_insert(0)
sp = (N.Spawner*1)(R.make_spawner(seed=42)); bi = (N.BatchInfo*1)(N.BatchInfo(0,0,0,0,0,1)); pre=(N.u32*1)(0)
la = (N.BatchLaunch*1)(N.BatchLaunch.make(fx, slab, 0, 0))
def up():
    ctx.upload_spawners_raw(sp,1); ctx.upload_batches_raw(bi,1,pre,1); ctx.set_sim_params(1/60,0,1)
up()
for _ in range(5): ctx.simulate_raw(la,1)
ctx.sync()
ctx.enable_kernel_timing(True); ctx.kernel_time_ms()
n=30
def run(name, body):
    ctx.sync(); t0=time.perf_counter()
    for i in range(n): body(i)
    ctx.sync(); el=(time.perf_counter()-t0)/n*1e3
    ms,k = ctx.kernel_time_ms()
    print(f"{name:45s} wall/step {el:.3f} ms   update kernel {ms/max(k,1):.3f} ms")
run("resident, no sync", lambda i: ctx.simulate_raw(la,1))
run("resident, sync each step", lambda i: (ctx.simulate_raw(la,1), ctx.sync()))
run("resident, sync + sleep 2ms", lambda i: (ctx.simulate_raw(la,1), ctx.sync(), time.sleep(0.002)))
run("upload + simulate, no sync", lambda i: (up(), ctx.simulate_raw(la,1)))
run("upload + simulate, sync each step", lambda i: (up(), ctx.simulate_raw(la,1), ctx.sync()))
x = torch.empty(256*1024*1024, device="cuda", dtype=torch.uint8)
run("resident, sync, then 256MB memset (L2 flush)", lambda i: (ctx.simulate_raw(la,1), ctx.sync(), x.zero_()))
run("resident no sync, 256MB memset between", lambda i: (ctx.simulate_raw(la,1), x.zero_()))
