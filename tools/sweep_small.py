"""Shard-size sweep: hnb_update time vs particles per GPU for each tile-chunk setting (HNB_TILE_CHUNKS) and
optional HNB_DEFINES variants. Usage: sweep_small.py [defines ...]  (env SWEEP_PS="4,8,16,32" in Mi rows)"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bevy_hanabi_b200 as hb
from bevy_hanabi_b200 import _native as N, recipes, runtime as R
stream = torch.cuda.Stream(); torch.cuda.set_stream(stream)
PS = [int(float(x) * (1 << 20)) for x in os.environ.get("SWEEP_PS", "4,8,16,32").split(",")]
CH = os.environ.get("SWEEP_CHUNKS", "0,1,2,4").split(",")
variants = sys.argv[1:] or [""]
for P in PS:
    for defs in variants:
        for ch in CH:
            os.environ["HNB_DEFINES"] = defs
            if ch == "0": os.environ.pop("HNB_TILE_CHUNKS", None)
            else: os.environ["HNB_TILE_CHUNKS"] = ch
            ctx = hb.Context(0, stream.cuda_stream)
            slab = ctx.slab_create(P, 32); ctx.slab_fill_c5(slab, 0, P, 42, 1e9, 1e9)
            md = R.initial_metadata(P, 0, 8); md.alive_count = P; md.max_spawn = 0
            ctx.metadata_insert(0, md); ctx.draw_args_insert(0)
            sp = (N.Spawner*1)(R.make_spawner(seed=42)); bi = (N.BatchInfo*1)(N.BatchInfo(0,0,0,0,0,1)); pre=(N.u32*1)(0)
            ctx.upload_spawners_raw(sp,1); ctx.upload_batches_raw(bi,1,pre,1); ctx.set_sim_params(1/60,0,1)
            fx = ctx.effect_compile(recipes.c5_lowered())
            la = (N.BatchLaunch*1)(N.BatchLaunch.make(fx, slab, 0, 0))
            for _ in range(10): ctx.simulate_raw(la,1)
            ctx.sync()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(100): ctx.simulate_raw(la,1)
            e1.record(stream); e1.synchronize()
            step = e0.elapsed_time(e1) / 100
            ctx.enable_kernel_timing(True); ctx.kernel_time_ms()
            for _ in range(40): ctx.simulate_raw(la,1)
            ms,k = ctx.kernel_time_ms()
            print(f"P={P/(1<<20):8.4f}Mi chunks={ch} {defs[:50]:50s} update {ms/k:.4f} ms {72*P/(ms/k*1e-3)/1e9:5.0f} GB/s  step {step:.4f} ms", flush=True)
            ctx.close()
