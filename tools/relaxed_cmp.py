import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__)))); sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import perf_matrix as PM
from perf_matrix import *
for mi in (64, 8):
    for relaxed in (False, True):
        P = mi << 20
        ctx = hb.Context(0, stream.cuda_stream)
        slab = ctx.slab_create(P, 32)
        ctx.slab_fill_c5(slab, 0, P, 42, 1e9, 1e9)
        single_instance(ctx, P, 32, alive=P)
        la = [N.BatchLaunch.make(ctx.effect_compile(recipes.c5_lowered(relaxed_order=relaxed)), slab, 0, 0)]
        for _ in range(10): ctx.simulate(la)
        fr = min(frame_ms(ctx, la, 100) for _ in range(3))
        k = timed_update(ctx, la, 30)
        report(f"C5 {mi} Mi {'RELAXED (atomic per tile, no look-back)' if relaxed else 'ordered (look-back)'}", fr, 72 * P, f"isolated {k:.4f} ms")
        ctx.close()
