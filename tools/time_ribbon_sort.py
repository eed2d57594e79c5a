"""Time hnb_pass_sort (ribbon sort) for several sizes; wide = all eight radix passes, narrow = typical ribbon keys."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import bevy_hanabi_b200 as hb
from bevy_hanabi_b200 import _native as N, runtime as R
from tests.test_gpu_ribbons import _ribbon_asset
stream = torch.cuda.Stream(); torch.cuda.set_stream(stream)
ctx = hb.Context(0, stream.cuda_stream)
asset = _ribbon_asset(16); fx = asset.generate(); fields, size, _ = asset.particle_layout()
off = {f.name: f.offset // 4 for f in fields}; words = size // 4
effect = ctx.effect_compile(fx)
for n in (512, 2048, 16384, 1 << 18, 1 << 20, 1 << 22):
    for wide in (False, True):
        rng = np.random.default_rng(n)
        slab = ctx.slab_create(n, size)
        particles = np.zeros((n, words), dtype=np.uint32)
        if wide:
            particles[:, off["ribbon_id"]] = rng.integers(0, 2**32, n, dtype=np.uint32)
            particles[:, off["age"]] = rng.integers(0, 2**32, n, dtype=np.uint32)
        else:
            particles[:, off["ribbon_id"]] = rng.integers(0, 64, n, dtype=np.uint32)
            particles[:, off["age"]] = rng.uniform(0, 2, n).astype(np.float32).view(np.uint32)
        ctx.slab_upload_aos(slab, 0, particles)
        ind = np.zeros((n, 3), dtype=np.uint32); ind[:, 0] = rng.permutation(n)
        md = R.initial_metadata(n, 0, words); md.alive_count = n; md.indirect_write_index = 0
        md.sort_key_offset, md.sort_key2_offset = off["ribbon_id"], off["age"]
        ctx.metadata_insert(0, md); ctx.draw_args_insert(0)
        ctx.upload_spawners([R.make_spawner()]); ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, 1)], [0]); ctx.set_sim_params(1 / 60, 0.0, 1)
        la = N.BatchLaunch.make(effect, slab, 0, 0)
        ts = []
        for it in range(6):
            ctx.slab_upload_indirect(slab, 0, ind)   # unsorted again
            ctx.sync()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream); ctx.pass_sort(la); e1.record(stream); e1.synchronize()
            ts.append(e0.elapsed_time(e1))
        t = min(ts[1:])
        print(f"n={n:8d} {'wide  ' if wide else 'narrow'} sort {t*1e3:9.1f} us  {n/t/1e3:8.1f} Mkeys/s", flush=True)
