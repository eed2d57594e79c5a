"""Where does the fixed cost of one hnb_update launch go? Timeline probes of the HNB_PROFILE build (%globaltimer)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ["HNB_DEFINES"] = os.environ.get("HNB_DEFINES", "") + ";HNB_PROFILE=1"
import torch
import bevy_hanabi_b200 as hb
from bevy_hanabi_b200 import _native as N, recipes, runtime as R
stream = torch.cuda.Stream(); torch.cuda.set_stream(stream)
M = (1 << 64) - 1
for P in [int(float(x) * (1 << 20)) for x in os.environ.get("SWEEP_PS", "0.0625,1,8,64").split(",")]:
    ctx = hb.Context(0, stream.cuda_stream)
    slab = ctx.slab_create(P, 32); ctx.slab_fill_c5(slab, 0, P, 42, 1e9, 1e9)
    md = R.initial_metadata(P, 0, 8); md.alive_count = P; md.max_spawn = 0
    ctx.metadata_insert(0, md); ctx.draw_args_insert(0)
    ctx.upload_spawners([R.make_spawner(seed=42)]); ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, 1)], [0]); ctx.set_sim_params(1 / 60, 0, 1)
    la = [N.BatchLaunch.make(ctx.effect_compile(recipes.c5_lowered()), slab, 0, 0)]
    for _ in range(10): ctx.simulate(la)
    ctx.sync(); ctx.read_debug(True)
    rows = []
    for _ in range(8):
        ctx.enable_kernel_timing(True); ctx.kernel_time_ms()
        ctx.simulate(la)
        ms, k = ctx.kernel_time_ms()
        d = ctx.read_debug(True)
        t0 = M - d[8]
        rows.append((ms * 1e3, d[9] - t0, (M - d[12]) - t0, d[10] - t0, (M - d[13]) - t0, d[11] - t0, d[4], d[5], d[3]))
    rows.sort()
    r = rows[len(rows) // 2]
    print(f"P={P/(1<<20):8.4f}Mi event {r[0]:7.1f} us | first warp start=0, last warp started {r[1]/1e3:6.1f} us, first pass-1 done {r[2]/1e3:6.1f}..{r[3]/1e3:6.1f} us, "
          f"warps end {r[4]/1e3:6.1f}..{r[5]/1e3:6.1f} us | tiles {r[6]} warps {r[7]} polls {r[8]}", flush=True)
    ctx.close()
