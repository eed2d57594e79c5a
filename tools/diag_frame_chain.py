"""Where does a frame's time go when frames are chained with programmatic dependent launch? Per-frame %globaltimer probes
of the HNB_PROFILE build (ring of 64 frames): for consecutive frames N, N+1 of a C5 instance it prints, relative to the end
of frame N's last warp: when the first CTA of N+1 became resident, when the first warp of N+1 passed the dependency wait,
when the first sub-tile (128 rows) of N+1 was done, and when N+1's last warp ended. Usage: python tools/diag_frame_chain.py [Mi ...]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ["HNB_DEFINES"] = os.environ.get("HNB_DEFINES", "") + ";HNB_PROFILE=1"
import numpy as np
import torch
import bevy_hanabi_b200 as hb
from bevy_hanabi_b200 import _native as N, recipes, runtime as R
stream = torch.cuda.Stream(); torch.cuda.set_stream(stream)
M = (1 << 64) - 1
for mi in [float(x) for x in (sys.argv[1:] or ["1", "8", "64"])]:
    P = int(mi * (1 << 20))
    ctx = hb.Context(0, stream.cuda_stream)
    slab = ctx.slab_create(P, 32); ctx.slab_fill_c5(slab, 0, P, 42, 1e9, 1e9)
    md = R.initial_metadata(P, 0, 8); md.alive_count = P; md.max_spawn = 0
    ctx.metadata_insert(0, md); ctx.draw_args_insert(0)
    ctx.upload_spawners([R.make_spawner(seed=42)]); ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, 1)], [0]); ctx.set_sim_params(1 / 60, 0, 1)
    la = [N.BatchLaunch.make(ctx.effect_compile(recipes.c5_lowered()), slab, 0, 0)]
    for _ in range(10): ctx.simulate(la)
    ctx.sync(); ctx.read_debug_ring(True)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(48): ctx.simulate(la)
    e1.record(stream); e1.synchronize()
    ring = np.array(ctx.read_debug_ring(True), dtype=np.uint64).reshape(64, 4)
    fr = [(int(M - int(r[0])), int(M - int(r[1])), int(M - int(r[2])), int(r[3])) for r in ring if r[3] != 0]
    fr.sort(key=lambda r: r[3])
    gaps = []
    for a, b in zip(fr[4:-1], fr[5:]):   # skip the first frames of the burst
        end_n = a[3]
        gaps.append(((b[0] - end_n) / 1e3, (b[1] - end_n) / 1e3, (b[2] - end_n) / 1e3, (b[3] - end_n) / 1e3))
    g = np.median(np.array(gaps), axis=0)
    print(f"C5 {mi:5.2f} Mi: frame {e0.elapsed_time(e1) / 48 * 1e3:7.1f} us | after frame N's last warp: N+1 resident {g[0]:+6.1f} us, "
          f"past the wait {g[1]:+6.1f} us, first sub-tile done {g[2]:+6.1f} us, last warp ends {g[3]:+7.1f} us ({len(gaps)} frame pairs)", flush=True)
    ctx.close()
