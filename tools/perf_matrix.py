"""Performance matrix beyond the headline bench line: the same kernels on the other BASELINE configurations.

Every row reports the hnb_update launch time (CUDA events inside the context, as in bench.py), the algorithmic
traffic (8 + 2*stride bytes per UPDATED particle, SURVEY.md §8d) and the fraction of the measured HBM peak; init
rows report whole frames (init + bookkeeping + update of the newly spawned particles) because the init kernel is
not timed separately.  Usage: python tools/perf_matrix.py [scenario ...]
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import bevy_hanabi_b200 as hb
from bevy_hanabi_b200 import _native as N, graph as G, recipes, runtime as R

A = G.Attribute
PEAK = 3350.0  # GB/s, H100 SXM data sheet
stream = torch.cuda.Stream()
torch.cuda.set_stream(stream)


def report(name, ms, bytes_, extra=""):
    gbs = bytes_ / (ms * 1e-3) / 1e9
    print(f"{name:44s} {ms:8.4f} ms  {gbs:7.0f} GB/s  {100 * gbs / PEAK:5.1f} % of {PEAK:.0f}  {extra}", flush=True)


def timed_update(ctx, launches, steps):
    ctx.sync()
    ctx.enable_kernel_timing(True)
    ctx.kernel_time_ms()
    for _ in range(steps):
        ctx.simulate(launches)
    ms, k = ctx.kernel_time_ms()
    ctx.enable_kernel_timing(False)
    return ms / k


def frame_ms(ctx, launches, steps=1):
    ctx.sync()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(steps):
        ctx.simulate(launches)
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) / steps


def single_instance(ctx, capacity, stride, alive=0, spawn=0, seed=42):
    md = R.initial_metadata(capacity, 0, stride // 4)
    md.alive_count, md.max_spawn = alive, capacity - alive
    ctx.metadata_insert(0, md)
    ctx.draw_args_insert(0)
    ctx.upload_spawners([R.make_spawner(spawn=spawn, seed=seed)])
    ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, 1)], [0])
    ctx.set_sim_params(1 / 60, 0.0, 1)


def c5_update():
    P = 64 << 20
    ctx = hb.Context(0, stream.cuda_stream)
    slab = ctx.slab_create(P, 32)
    ctx.slab_fill_c5(slab, 0, P, 42, 1e9, 1e9)
    single_instance(ctx, P, 32, alive=P)
    la = [N.BatchLaunch.make(ctx.effect_compile(recipes.c5_lowered()), slab, 0, 0)]
    for _ in range(5):
        ctx.simulate(la)
    ms = timed_update(ctx, la, 30)
    report("C5 64Mi update, nobody dies", ms, 72 * P)
    ctx.close()


def c5_dying():
    """Lifetimes U(0, 0.5 s): ~3 % of the survivors die every step; dead-stack pushes + compaction at work."""
    P = 64 << 20
    ctx = hb.Context(0, stream.cuda_stream)
    slab = ctx.slab_create(P, 32)
    ctx.slab_fill_c5(slab, 0, P, 42, 0.0, 0.5)
    single_instance(ctx, P, 32, alive=P)
    la = [N.BatchLaunch.make(ctx.effect_compile(recipes.c5_lowered()), slab, 0, 0)]
    alive = P
    for step in range(12):
        ms = timed_update(ctx, la, 1)
        after = ctx.read_metadata(0).alive_count
        if step in (0, 1, 5, 11):
            report(f"C5 64Mi dying, step {step}: {alive >> 10} Ki -> {after >> 10} Ki", ms, 72 * alive, f"{100 * (alive - after) / max(alive, 1):.1f} % died")
        alive = after
    ctx.close()


def c4_topology():
    n_inst, cap = 1024, 65536
    P = n_inst * cap
    ctx = hb.Context(0, stream.cuda_stream)
    slab = ctx.slab_create(P, 32)
    sp = []
    for i in range(n_inst):
        ctx.slab_fill_c5(slab, i * cap, cap, 7000 + i, 1e9, 1e9)
        m = R.initial_metadata(cap, i, 8)
        m.alive_count, m.max_spawn = cap, 0
        ctx.metadata_insert(i, m)
        ctx.draw_args_insert(i)
        sp.append(R.make_spawner(seed=i, effect_metadata_index=i, draw_indirect_index=i, slab_offset=i * cap))
    ctx.upload_spawners(sp)
    ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, n_inst)], [0] * n_inst)
    ctx.set_sim_params(1 / 60, 0.0, n_inst)
    la = [N.BatchLaunch.make(ctx.effect_compile(recipes.c5_lowered()), slab, 0, 0)]
    for _ in range(5):
        ctx.simulate(la)
    ms = timed_update(ctx, la, 30)
    report("C4 shape: 1024 instances x 65536, one batch", ms, 72 * P, f"frame {frame_ms(ctx, la, 20):.4f} ms")
    # the same with one spawn per instance per frame (init + update): needs free slots -> kill a few first
    ctx.close()


def _burst(name, asset, P, spawn, props=None, steps=10, fast_math=False, sector_planes=False):
    ctx = hb.Context(0, stream.cuda_stream)
    fx = asset.generate(fast_math=fast_math, sector_planes=sector_planes)
    stride = fx.particle_stride
    slab = ctx.slab_create(P, stride, sector_planes=sector_planes)
    effect = ctx.effect_compile(fx)
    if props is not None:
        ctx.upload_properties(effect, 0, props)
    md = R.initial_metadata(P, 0, stride // 4, properties_array_index=0 if props is not None else N.INVALID)
    ctx.metadata_insert(0, md)
    ctx.draw_args_insert(0)
    ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, 1)], [0])
    ctx.set_sim_params(1 / 60, 0.0, 1)
    # warm the kernels on a throw-away frame pair, then reset the instance
    ctx.upload_spawners([R.make_spawner(spawn=1024, seed=1)])
    ctx.simulate([N.BatchLaunch.make(effect, slab, 0, 1024)])
    ctx.sync()
    ctx.slab_reset_rows(slab, 0, P)
    ctx.metadata_insert(0, md)
    ctx.upload_spawners([R.make_spawner(spawn=spawn, seed=7)])
    t_burst = frame_ms(ctx, [N.BatchLaunch.make(effect, slab, 0, spawn)])
    alive = ctx.read_metadata(0).alive_count
    ctx.upload_spawners([R.make_spawner(spawn=0, seed=8)])
    la = [N.BatchLaunch.make(effect, slab, 0, 0)]
    for _ in range(3):
        ctx.simulate(la)
    ms = timed_update(ctx, la, steps)
    alive2 = ctx.read_metadata(0).alive_count
    upd_bytes = (8 + 2 * stride) * alive
    report(f"{name}: update, {alive2 >> 10} Ki alive, stride {stride}", ms, (8 + 2 * stride) * alive2)
    t_plain = frame_ms(ctx, la, 5)
    init_bytes = (stride + 8) * alive
    report(f"{name}: burst frame (init {alive >> 10} Ki + update)", t_burst, init_bytes + upd_bytes, f"init alone ~{t_burst - t_plain:.4f} ms = {init_bytes / max(t_burst - t_plain, 1e-6) / 1e6:.0f} GB/s")
    ctx.close()


def c5_init_burst():
    w = G.ExprWriter()
    asset = (G.EffectAsset(64 << 20, w.module, name="c5_spawned")
             .init(G.SetAttributeModifier(A.POSITION, w.rand(G.VEC3) * w.lit(2.) - w.lit(1.)))
             .init(G.SetAttributeModifier(A.VELOCITY, w.rand(G.VEC3) * w.lit(2.) - w.lit(1.)))
             .init(G.SetAttributeModifier(A.AGE, w.lit(0.)))
             .init(G.SetAttributeModifier(A.LIFETIME, w.lit(1e9)))
             .update(G.AccelModifier(w.lit(G.Vec3(0., -9.8, 0.))))
             .update(G.LinearDragModifier(w.lit(0.5))))
    _burst("C5 recipe, 32Mi burst", asset, 64 << 20, 32 << 20)


def c2_trails():
    from tests.effects import firework_trails
    _burst("C2 trails, 32Mi burst", firework_trails(40 << 20), 40 << 20, 32 << 20)


def c3_force_field():
    from tests.effects import force_field
    for P in (1 << 20, 16 << 20):
        asset = force_field(P)
        _burst(f"C3 force field, {P >> 20}Mi burst", asset, P, P, props=asset.serialize_properties())


def c3_fast_math():
    from tests.effects import force_field
    asset = force_field(16 << 20)
    _burst("C3 force field FAST_MATH, 16Mi burst", asset, 16 << 20, 16 << 20, props=asset.serialize_properties(), fast_math=True)


def many_batches():
    """Typical game frame: many effect assets -> many batches -> one init/update launch each."""
    for nb, cap in ((64, 16 << 10), (64, 256 << 10), (256, 4 << 10)):
        ctx = hb.Context(0, stream.cuda_stream)
        effect = ctx.effect_compile(recipes.c5_lowered())
        sp, bis, la = [], [], []
        for b in range(nb):
            slab = ctx.slab_create(cap, 32)
            ctx.slab_fill_c5(slab, 0, cap, 100 + b, 1e9, 1e9)
            m = R.initial_metadata(cap, b, 8)
            m.alive_count, m.max_spawn = cap, 0
            ctx.metadata_insert(b, m)
            ctx.draw_args_insert(b)
            sp.append(R.make_spawner(seed=b, effect_metadata_index=b, draw_indirect_index=b, slab_offset=0))
            bis.append(N.BatchInfo(0, 0, b, 0, b, 1))
            la.append(N.BatchLaunch.make(effect, slab, b, 0))
        ctx.upload_spawners(sp)
        ctx.upload_batches(bis, [0] * nb)
        ctx.set_sim_params(1 / 60, 0.0, nb)
        for _ in range(5):
            ctx.simulate(la)
        ms = frame_ms(ctx, la, 30)
        report(f"{nb} batches x {cap >> 10} Ki particles: frame", ms, 72 * nb * cap, f"{ms * 1e3 / nb:.1f} us per batch")
        ctx.close()


def _churned(sector_planes: bool = False, slot_order: bool = False):
    """16 Mi slots of drifting sparks after 240 frames of constant spawning into recycled slots."""
    from tests.effects import drifting_sparks
    P = 16 << 20
    ctx = hb.Context(0, stream.cuda_stream)
    asset = drifting_sparks(P)          # lifetimes U(0.2, 0.9) s
    fx = asset.generate(sector_planes=sector_planes, slot_order=slot_order)
    stride = fx.particle_stride
    slab = ctx.slab_create(P, stride, sector_planes=sector_planes)
    effect = ctx.effect_compile(fx)
    ctx.metadata_insert(0, R.initial_metadata(P, 0, stride // 4))
    ctx.draw_args_insert(0)
    ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, 1)], [0])
    dt, rate = 1 / 60, P // 40           # ~33 frames mean life -> the population settles around 0.8 P
    for f in range(240):                 # 4 s of simulated time: every slot has been recycled several times
        ctx.set_sim_params(dt, f * dt, 1)
        ctx.upload_spawners([R.make_spawner(spawn=rate, seed=1000 + f)])
        ctx.simulate([N.BatchLaunch.make(effect, slab, 0, rate)])
    return P, ctx, slab, effect, stride, dt, rate


def churn(sector_planes: bool = False, slot_order: bool = False):
    """Steady-state churn: constant spawn rate into recycled slots until the alive list is a random-looking permutation
    of the slab (survivors keep their relative order, new particles land in whatever slots died). The gathers then touch
    scattered 16-byte plane elements (half-used 32-byte sectors): the honest number for long-running effects, unlike the
    freshly filled slabs of the other rows."""
    P, ctx, slab, effect, stride, dt, rate = _churned(sector_planes, slot_order)
    alive = ctx.read_metadata(0).alive_count
    ind = ctx.slab_download_indirect(slab, 0, 1 << 16)
    col = ctx.read_metadata(0).indirect_write_index
    jumps = np.abs(np.diff(ind[:, col].astype(np.int64)))
    la = [N.BatchLaunch.make(effect, slab, 0, rate)]
    ctx.sync(); ctx.enable_kernel_timing(True); ctx.kernel_time_ms()
    for f in range(240, 250):
        ctx.set_sim_params(dt, f * dt, 1)
        ctx.upload_spawners([R.make_spawner(spawn=rate, seed=1000 + f)])
        ctx.simulate(la)
    ms, k = ctx.kernel_time_ms()
    ctx.enable_kernel_timing(False)
    alive2 = ctx.read_metadata(0).alive_count
    report(f"churn steady state{' (sector planes)' if sector_planes else ''}{' (SLOT ORDER)' if slot_order else ''}: {alive2 >> 10} Ki of {P >> 10} Ki alive, stride {stride}", ms / k, (8 + 2 * stride) * alive2,
           f"median |slot jump| between consecutive alive-list entries {np.median(jumps):.0f} (1 = identity order)")
    ctx.close()


def churn_slot():
    """The same with HNB_EFFECT_SLOT_ORDER: the update walks the slots, not the (permuted) alive list."""
    churn(slot_order=True)


def c5_slot():
    """C5 in slot order, nobody dies: the headline workload without the alive-list read (68 B instead of 72 B per particle;
    reported against the same 72 B so that the rows compare)."""
    for mi in (8, 64):
        P = mi << 20
        ctx = hb.Context(0, stream.cuda_stream)
        slab = ctx.slab_create(P, 32)
        ctx.slab_fill_c5(slab, 0, P, 42, 1e9, 1e9)
        single_instance(ctx, P, 32, alive=P)
        la = [N.BatchLaunch.make(ctx.effect_compile(recipes.c5_lowered(slot_order=True)), slab, 0, 0)]
        for _ in range(10):
            ctx.simulate(la)
        fr = min(frame_ms(ctx, la, 100) for _ in range(3))
        k = timed_update(ctx, la, 30)
        assert ctx.read_metadata(0).alive_count == P
        report(f"C5 {mi:2d}Mi SLOT ORDER frame chain", fr, 72 * P, f"isolated update kernel {k:.4f} ms = {68 * P / k / 1e6:.0f} GB/s of its own 68 B per particle")
        ctx.close()
    # dying: the population thins out but every access stays inside contiguous spans
    P = 64 << 20
    ctx = hb.Context(0, stream.cuda_stream)
    slab = ctx.slab_create(P, 32)
    ctx.slab_fill_c5(slab, 0, P, 42, 0.0, 0.5)
    single_instance(ctx, P, 32, alive=P)
    la = [N.BatchLaunch.make(ctx.effect_compile(recipes.c5_lowered(slot_order=True)), slab, 0, 0)]
    alive = P
    for step in range(12):
        ms = timed_update(ctx, la, 1)
        after = ctx.read_metadata(0).alive_count
        if step in (0, 1, 5, 11):
            report(f"C5 64Mi SLOT ORDER dying, step {step}: {alive >> 10} Ki -> {after >> 10} Ki", ms, 72 * alive, f"{100 * (alive - after) / max(alive, 1):.1f} % died")
        alive = after
    ctx.close()


def churn_sector():
    """The same with HNB_SLAB_SECTOR_PLANES (32-byte-wide columns): one full sector per gathered record."""
    churn(sector_planes=True)


def _card():
    """Name and power limit of cuda:0 (read-only query), printed with the numbers they qualify."""
    import subprocess
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        q = f"nvidia-smi unavailable ({type(e).__name__})"
    print(f"card: {torch.cuda.get_device_name(0)} | {q}", flush=True)


def _repack_bytes(ctx, slab, rows, alive):
    """Bytes hnb_slab_repack moves: per column a gather (src word + scattered element read + scratch write) and the copy
    back (read + write); then ping / pong below n, dead from n, and the alive bitmap."""
    v = ctx.slab_device_view(slab)
    widths = [v.plane_width[p] for p in range(v.num_planes)]
    return sum(rows * (4 + 4 * w) for w in widths) + 8 * alive + 4 * (rows - alive) + rows // 8


def _timed_repack(ctx, slab, effect, rows):
    ctx.sync()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    ctx.slab_repack(slab, effect, 0, 0, rows)
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1)


def churn_repack():
    """hnb_slab_repack on the churn steady state: the update time of the churned slab, the repack's own time (CUDA events
    around the call: gathers, copies back, lists; the scratch comes from cudaMallocAsync inside the window), then the update
    time at frames +1..+10, +60 and +240 under the same constant spawning, and a second repack at +240. Then an init-filled
    C5 instance (64 Mi rows, one burst through hnb_init: identity list, no claim) before and after a repack."""
    _card()
    P, ctx, slab, effect, stride, dt, rate = _churned()
    frame = [240]

    def step_ms():
        f = frame[0]
        ctx.set_sim_params(dt, f * dt, 1)
        ctx.upload_spawners([R.make_spawner(spawn=rate, seed=1000 + f)])
        frame[0] += 1
        return timed_update(ctx, [N.BatchLaunch.make(effect, slab, 0, rate)], 1)

    ms = sum(step_ms() for _ in range(10)) / 10
    alive = ctx.read_metadata(0).alive_count
    report(f"churn_repack: churned update, {alive >> 10} Ki of {P >> 10} Ki alive", ms, (8 + 2 * stride) * alive, "mean of 10 frames")
    def repack(label):
        alive = ctx.read_metadata(0).alive_count
        rp = _timed_repack(ctx, slab, effect, P)
        report(f"churn_repack: {label} repack of {P >> 20} Mi rows, {alive >> 10} Ki alive", rp, _repack_bytes(ctx, slab, P, alive),
               "bytes: gathers + copies back + lists")

    repack("first")
    since, out = 0, []
    for target in list(range(1, 11)) + [60, 240]:
        while since < target:
            t = step_ms()
            since += 1
        out.append((target, t, ctx.read_metadata(0).alive_count))
    for target, t, a in out:
        report(f"churn_repack: update at frame +{target} after the repack", t, (8 + 2 * stride) * a, f"{a >> 10} Ki alive")
    repack("second (+240)")
    ctx.close()

    # init-filled C5-like instance: the identity list of a burst into a fresh slab carries no claim until a repack
    P = 64 << 20
    w = G.ExprWriter()
    asset = (G.EffectAsset(P, w.module, name="c5_spawned")
             .init(G.SetAttributeModifier(A.POSITION, w.rand(G.VEC3) * w.lit(2.) - w.lit(1.)))
             .init(G.SetAttributeModifier(A.VELOCITY, w.rand(G.VEC3) * w.lit(2.) - w.lit(1.)))
             .init(G.SetAttributeModifier(A.AGE, w.lit(0.)))
             .init(G.SetAttributeModifier(A.LIFETIME, w.lit(1e9)))
             .update(G.AccelModifier(w.lit(G.Vec3(0., -9.8, 0.))))
             .update(G.LinearDragModifier(w.lit(0.5))))
    ctx = hb.Context(0, stream.cuda_stream)
    fx = asset.generate()
    slab = ctx.slab_create(P, fx.particle_stride)
    effect = ctx.effect_compile(fx)
    ctx.metadata_insert(0, R.initial_metadata(P, 0, fx.particle_stride // 4))
    ctx.draw_args_insert(0)
    ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, 1)], [0])
    ctx.set_sim_params(1 / 60, 0.0, 1)
    ctx.upload_spawners([R.make_spawner(spawn=P, seed=7)])
    ctx.simulate([N.BatchLaunch.make(effect, slab, 0, P)])
    ctx.upload_spawners([R.make_spawner(spawn=0, seed=8)])
    la = [N.BatchLaunch.make(effect, slab, 0, 0)]
    for _ in range(3):
        ctx.simulate(la)
    alive = ctx.read_metadata(0).alive_count
    before = timed_update(ctx, la, 30)
    rp = _timed_repack(ctx, slab, effect, P)
    for _ in range(3):
        ctx.simulate(la)
    after = timed_update(ctx, la, 30)
    report(f"churn_repack: init-filled C5 {alive >> 20} Mi, update before repack", before, 72 * alive, "72 B per particle-step")
    report(f"churn_repack: init-filled C5 {alive >> 20} Mi, repack", rp, _repack_bytes(ctx, slab, P, alive))
    report(f"churn_repack: init-filled C5 {alive >> 20} Mi, update after repack", after, 64 * alive,
           f"64 B per particle-step; {100 * (after - before) / before:+.1f} % per launch")
    ctx.close()


def _events_ms(fn, reps=5):
    """Best of `reps` CUDA-event windows around fn() on the scenario's stream, in ms."""
    best = float("inf")
    for _ in range(reps):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        fn()
        e1.record(stream)
        e1.synchronize()
        best = min(best, e0.elapsed_time(e1))
    return best


def _snapshot_pair(label, ctx, slab, effect, rows, stride, alive):
    """Time hnb_instance_snapshot of metadata row 0 and hnb_instance_restore of it into a second slab (metadata row 1).
    Bytes: a snapshot reads 4 B of list and S B of record and writes S B per live particle; a restore reads and writes
    S B, then writes 8 B of lists per particle, 4 B of dead stack per free slot and the alive bitmap."""
    nbytes = ctx.instance_snapshot_bytes(stride, rows)
    buf = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    dst = ctx.slab_create(rows, stride, sector_planes=False)
    ctx.metadata_insert(1, R.initial_metadata(rows, 1, stride // 4))
    snap = _events_ms(lambda: ctx.instance_snapshot(slab, effect, 0, 0, rows, buf.data_ptr(), nbytes))
    rest = _events_ms(lambda: ctx.instance_restore(dst, effect, 1, 0, rows, buf.data_ptr(), nbytes))
    assert ctx.read_metadata(1).alive_count == alive
    report(f"snapshot_restore: {label} snapshot", snap, (4 + 2 * stride) * alive, f"{alive >> 10} Ki alive, best of 5")
    report(f"snapshot_restore: {label} restore", rest, (8 + 2 * stride) * alive + 4 * (rows - alive) + rows // 8, "into another slab, best of 5")
    del buf
    ctx.slab_destroy(dst)


def snapshot_restore():
    """hnb_instance_snapshot / hnb_instance_restore: a filled 64 Mi C5 instance (identity list), the 16 Mi-slot churn steady
    state (gathers through a permuted list), and a 2 GiB device-to-device torch copy for scale."""
    _card()
    a = torch.empty(2 << 30, dtype=torch.uint8, device="cuda")
    b = torch.empty_like(a)
    ms = _events_ms(lambda: b.copy_(a))
    report("snapshot_restore: 2 GiB device-to-device copy", ms, 2 * a.numel(), "torch copy_, best of 5")
    del a, b
    torch.cuda.empty_cache()

    P = 64 << 20
    ctx = hb.Context(0, stream.cuda_stream)
    slab = ctx.slab_create(P, 32)
    ctx.slab_fill_c5(slab, 0, P, 42, 1e9, 1e9)
    single_instance(ctx, P, 32, alive=P)
    effect = ctx.effect_compile(recipes.c5_lowered())
    _snapshot_pair(f"filled C5 {P >> 20} Mi", ctx, slab, effect, P, 32, P)
    ctx.close()
    torch.cuda.empty_cache()

    P, ctx, slab, effect, stride, dt, rate = _churned()
    _snapshot_pair(f"churned {P >> 20} Mi slots", ctx, slab, effect, P, stride, ctx.read_metadata(0).alive_count)
    ctx.close()


def _timed_append(label, ctx, slab, effect, rows, stride, src, src_bytes, md):
    """Best of 5 CUDA-event windows around hnb_instance_append of `src` into metadata row 0, after a warm-up call. Before
    every call the metadata row is put back to `md` (outside the window), so each call makes the same m appends into the
    same slots. Bytes: 4 B of dead-stack entry, S B of record read, S B of record written and 4 B of list per record."""
    best = float("inf")
    for rep in range(6):
        ctx.metadata_insert(0, md)
        ctx.sync()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        ctx.instance_append(slab, effect, 0, 0, rows, src, src_bytes)
        e1.record(stream)
        e1.synchronize()
        if rep:
            best = min(best, e0.elapsed_time(e1))
    m = ctx.read_metadata(0).alive_count - md.alive_count
    report(f"append: {label}", best, (8 + 2 * stride) * m, f"{m} records, best of 5")
    return m


def append():
    """hnb_instance_append: 1, 64 and 4096 records into a small C5 instance (latency); 1 Mi records into the 16 Mi-slot
    churn steady state (permuted dead stack, scattered slots); 1 Mi records into a 64 Mi-row C5 instance whose last 1 Mi
    slots are free, in stack order and permuted; a 2 GiB device-to-device torch copy for scale."""
    _card()
    a = torch.empty(2 << 30, dtype=torch.uint8, device="cuda")
    b = torch.empty_like(a)
    ms = _events_ms(lambda: b.copy_(a))
    report("append: 2 GiB device-to-device copy", ms, 2 * a.numel(), "torch copy_, best of 5")
    del a, b
    torch.cuda.empty_cache()

    def c5_source(k):
        """A version-1 snapshot of k random C5 records, in device memory (torch)."""
        g = torch.Generator(device="cuda").manual_seed(k)
        words = torch.empty(16 + 8 * k, dtype=torch.int32, device="cuda")
        words[16:] = (torch.rand(8 * k, device="cuda", generator=g) * 2 - 1).view(torch.int32)
        words[:16] = torch.tensor([0x53424E48, 1, 32, k] + [0] * 12, dtype=torch.int64).to(torch.int32).cuda()
        return words

    # latency: a 64 Ki-row C5 instance, 16 Ki alive
    P, alive = 64 << 10, 16 << 10
    ctx = hb.Context(0, stream.cuda_stream)
    slab = ctx.slab_create(P, 32)
    ctx.slab_fill_c5(slab, 0, alive, 42, 1e9, 1e9)
    effect = ctx.effect_compile(recipes.c5_lowered())
    md = R.initial_metadata(P, 0, 8)
    md.alive_count, md.max_spawn = alive, P - alive
    for k in (1, 64, 4096):
        src = c5_source(k)
        _timed_append(f"{k} records into a {P >> 10} Ki-row C5 instance", ctx, slab, effect, P, 32, src.data_ptr(), 4 * src.numel(), md)
    ctx.close()

    # the churn steady state: records from a snapshot of the instance itself, src_bytes cut to 1 Mi records
    P, ctx, slab, effect, stride, dt, rate = _churned()
    md = ctx.read_metadata(0)
    F = 1 << 20
    assert md.max_spawn >= F
    nbytes = ctx.instance_snapshot_bytes(stride, P)
    buf = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    ctx.instance_snapshot(slab, effect, 0, 0, P, buf.data_ptr(), nbytes)
    ind = ctx.slab_download_indirect(slab, md.alive_count, F)
    jumps = np.abs(np.diff(ind[:, 2].astype(np.int64)))
    _timed_append(f"1 Mi records into the 16 Mi churn steady state, {md.alive_count >> 10} Ki alive", ctx, slab, effect, P, stride,
                  buf.data_ptr(), 64 + F * stride, md)
    print(f"    median |slot jump| between consecutive dead-stack entries {np.median(jumps):.0f}", flush=True)
    del buf
    ctx.close()
    torch.cuda.empty_cache()

    # a 64 Mi-row C5 instance with its last 1 Mi slots free
    P = 64 << 20
    ctx = hb.Context(0, stream.cuda_stream)
    slab = ctx.slab_create(P, 32)
    ctx.slab_fill_c5(slab, 0, P, 42, 1e9, 1e9)
    effect = ctx.effect_compile(recipes.c5_lowered())
    md = R.initial_metadata(P, 0, 8)
    md.alive_count, md.max_spawn = P - F, F
    src = c5_source(F)
    _timed_append("1 Mi records into a 64 Mi C5 instance, stack order", ctx, slab, effect, P, 32, src.data_ptr(), 4 * src.numel(), md)
    rows3 = ctx.slab_download_indirect(slab, P - F, F)
    rows3[:, 2] = np.random.default_rng(1).permutation(rows3[:, 2])
    ctx.slab_upload_indirect(slab, P - F, rows3)
    _timed_append("1 Mi records into a 64 Mi C5 instance, permuted", ctx, slab, effect, P, 32, src.data_ptr(), 4 * src.numel(), md)
    ctx.close()


def _timed_bounds(label, ctx, launch, instances, bytes_, extra=""):
    """hnb_batch_bounds of `launch`'s batch into a device buffer: one warm-up call, then the best of 5 CUDA-event windows.
    `bytes_`: what the pass must read (16 B of position per live particle, 4 B of list where no claim covers the row)."""
    out = torch.empty(32 * instances, dtype=torch.uint8, device="cuda")
    ctx.batch_bounds(launch, out.data_ptr(), instances)
    ms = _events_ms(lambda: ctx.batch_bounds(launch, out.data_ptr(), instances))
    rec = np.frombuffer(out.cpu().numpy().tobytes(), dtype=R.BOUNDS_DTYPE)
    report(f"bounds: {label}", ms, bytes_, f"{ms * 1e3:.1f} us per call, {int(rec['count'].sum()) >> 10} Ki particles in {instances} records, best of 5{extra}")
    return rec


def bounds():
    """hnb_batch_bounds: the filled 64 Mi C5 instance under its claim (16 B per particle), the same size spawned by one
    init burst (identity list without a claim: 20 B), C4's topology in one call, the 16 Mi-slot churn steady state
    (gathers through a permuted list) and one small instance (latency), beside a 2 GiB device-to-device copy."""
    _card()
    a = torch.empty(2 << 30, dtype=torch.uint8, device="cuda")
    b = torch.empty_like(a)
    ms = _events_ms(lambda: b.copy_(a))
    report("bounds: 2 GiB device-to-device copy", ms, 2 * a.numel(), "torch copy_ (reads 2 GiB and writes 2 GiB), best of 5")
    del a, b
    torch.cuda.empty_cache()

    P = 64 << 20
    ctx = hb.Context(0, stream.cuda_stream)
    effect = ctx.effect_compile(recipes.c5_lowered())
    slab = ctx.slab_create(P, 32)
    ctx.slab_fill_c5(slab, 0, P, 42, 1e9, 1e9)
    single_instance(ctx, P, 32, alive=P)
    la = N.BatchLaunch.make(effect, slab, 0, 0)
    ctx.simulate([la])
    rec = _timed_bounds("C5 64Mi filled, claim over every row", ctx, la, 1, 16 * P)
    assert rec["count"][0] == P and (rec["min"][0] < -0.99).all() and (rec["max"][0] > 0.99).all()
    ctx.slab_destroy(slab)
    slab = ctx.slab_create(P, 32)
    single_instance(ctx, P, 32, alive=0, spawn=P)
    ctx.simulate([N.BatchLaunch.make(effect, slab, 0, P)])
    ctx.upload_spawners([R.make_spawner(spawn=0, seed=43)])
    la = N.BatchLaunch.make(effect, slab, 0, 0)
    ctx.simulate([la])
    rec = _timed_bounds("C5 64Mi from one init burst, no claim", ctx, la, 1, 20 * P)
    assert rec["count"][0] == P
    ctx.close()
    torch.cuda.empty_cache()

    n_inst, cap = 1024, 65536
    ctx = hb.Context(0, stream.cuda_stream)
    effect = ctx.effect_compile(recipes.c5_lowered())
    slab = ctx.slab_create(n_inst * cap, 32)
    sp = []
    for i in range(n_inst):
        ctx.slab_fill_c5(slab, i * cap, cap, 7000 + i, 1e9, 1e9)  # the last fill holds the slab's claim
        m = R.initial_metadata(cap, i, 8)
        m.alive_count, m.max_spawn = cap, 0
        ctx.metadata_insert(i, m)
        ctx.draw_args_insert(i)
        sp.append(R.make_spawner(seed=i, effect_metadata_index=i, draw_indirect_index=i, slab_offset=i * cap))
    ctx.upload_spawners(sp)
    ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, n_inst)], [0] * n_inst)
    ctx.set_sim_params(1 / 60, 0.0, n_inst)
    la = N.BatchLaunch.make(effect, slab, 0, 0)
    ctx.simulate([la])
    rec = _timed_bounds("C4 shape: 1024 x 65536 in one batch", ctx, la, n_inst, 20 * n_inst * cap - 4 * cap)
    assert (rec["count"] == cap).all()
    ctx.close()
    torch.cuda.empty_cache()

    for cap in (4096, 16 << 10):
        ctx = hb.Context(0, stream.cuda_stream)
        slab = ctx.slab_create(cap, 32)
        ctx.slab_fill_c5(slab, 0, cap, 100, 1e9, 1e9)
        single_instance(ctx, cap, 32, alive=cap)
        la = N.BatchLaunch.make(ctx.effect_compile(recipes.c5_lowered()), slab, 0, 0)
        ctx.simulate([la])
        _timed_bounds(f"one instance of {cap >> 10} Ki particles (latency)", ctx, la, 1, 16 * cap)
        ctx.close()

    P, ctx, slab, effect, stride, dt, rate = _churned()
    alive = ctx.read_metadata(0).alive_count
    _timed_bounds(f"churned {P >> 20} Mi slots, {alive >> 10} Ki alive, permuted list", ctx, N.BatchLaunch.make(effect, slab, 0, rate), 1, 20 * alive,
                  "; GB/s counts 4 B of list + 16 B of position, the gather moves whole 32 B sectors")
    ctx.close()


def _timed_depth_order(label, ctx, launch, instances, rows, alive, claimed, extra=""):
    """hnb_batch_depth_order of `launch`'s batch into a device order buffer of `rows`: one warm-up call, then the best of 5
    CUDA-event windows. GB/s counts what any depth sort must move: 16 B of position (and 4 B of list where no claim covers
    the row) read and a 4 B entry written per live particle."""
    order = torch.empty(rows, dtype=torch.int32, device="cuda")
    planes = torch.tensor([[0.48, -0.6, 0.64, 0.25]] * instances, dtype=torch.float32, device="cuda")
    ctx.batch_depth_order(launch, planes.data_ptr(), instances, order.data_ptr(), rows)
    ms = _events_ms(lambda: ctx.batch_depth_order(launch, planes.data_ptr(), instances, order.data_ptr(), rows))
    report(f"depth_order: {label}", ms, (20 if claimed else 24) * alive, f"{ms * 1e3:.1f} us per call, {alive >> 10} Ki particles, best of 5{extra}")
    return order


def depth_order():
    """hnb_batch_depth_order: the filled 64 Mi C5 instance under its claim, the same size spawned by one init burst, C4's
    topology in one call, the 16 Mi-slot churn steady state and single instances of 4 Ki and 16 Ki (latency), beside a
    2 GiB device-to-device copy and torch's stable argsort (CUB radix sort) of the same 64 Mi depths, already computed."""
    _card()
    a = torch.empty(2 << 30, dtype=torch.uint8, device="cuda")
    b = torch.empty_like(a)
    ms = _events_ms(lambda: b.copy_(a))
    report("depth_order: 2 GiB device-to-device copy", ms, 2 * a.numel(), "torch copy_ (reads 2 GiB and writes 2 GiB), best of 5")
    del a, b
    torch.cuda.empty_cache()

    P = 64 << 20
    ctx = hb.Context(0, stream.cuda_stream)
    effect = ctx.effect_compile(recipes.c5_lowered())
    slab = ctx.slab_create(P, 32)
    ctx.slab_fill_c5(slab, 0, P, 42, 1e9, 1e9)
    single_instance(ctx, P, 32, alive=P)
    la = N.BatchLaunch.make(effect, slab, 0, 0)
    ctx.simulate([la])
    order = _timed_depth_order("C5 64Mi filled, claim over every row", ctx, la, 1, P, P, True)
    view = ctx.slab_device_view(slab)
    col = torch.as_tensor(_DeviceColumn(view.planes[0], (P, 4)), device="cuda")
    depth = ((col[:, 0] * 0.48 + col[:, 1] * -0.6) + col[:, 2] * 0.64) + 0.25
    ms = _events_ms(lambda: torch.argsort(depth, descending=True, stable=True))
    report("depth_order: torch.argsort(stable=True) of the 64Mi depths", ms, 8 * P, "CUB radix sort of float32 keys with int64 indices, best of 5")
    del order, depth, col
    ctx.slab_destroy(slab)
    slab = ctx.slab_create(P, 32)
    single_instance(ctx, P, 32, alive=0, spawn=P)
    ctx.simulate([N.BatchLaunch.make(effect, slab, 0, P)])
    ctx.upload_spawners([R.make_spawner(spawn=0, seed=43)])
    la = N.BatchLaunch.make(effect, slab, 0, 0)
    ctx.simulate([la])
    _timed_depth_order("C5 64Mi from one init burst, no claim", ctx, la, 1, P, P, False)
    ctx.close()
    torch.cuda.empty_cache()

    n_inst, cap = 1024, 65536
    ctx = hb.Context(0, stream.cuda_stream)
    effect = ctx.effect_compile(recipes.c5_lowered())
    slab = ctx.slab_create(n_inst * cap, 32)
    sp = []
    for i in range(n_inst):
        ctx.slab_fill_c5(slab, i * cap, cap, 7000 + i, 1e9, 1e9)  # the last fill holds the slab's claim
        m = R.initial_metadata(cap, i, 8)
        m.alive_count, m.max_spawn = cap, 0
        ctx.metadata_insert(i, m)
        ctx.draw_args_insert(i)
        sp.append(R.make_spawner(seed=i, effect_metadata_index=i, draw_indirect_index=i, slab_offset=i * cap))
    ctx.upload_spawners(sp)
    ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, n_inst)], [0] * n_inst)
    ctx.set_sim_params(1 / 60, 0.0, n_inst)
    la = N.BatchLaunch.make(effect, slab, 0, 0)
    ctx.simulate([la])
    _timed_depth_order("C4 shape: 1024 x 65536 in one batch", ctx, la, n_inst, n_inst * cap, n_inst * cap, False)
    ctx.close()
    torch.cuda.empty_cache()

    for cap in (4096, 16 << 10):
        ctx = hb.Context(0, stream.cuda_stream)
        slab = ctx.slab_create(cap, 32)
        ctx.slab_fill_c5(slab, 0, cap, 100, 1e9, 1e9)
        single_instance(ctx, cap, 32, alive=cap)
        la = N.BatchLaunch.make(ctx.effect_compile(recipes.c5_lowered()), slab, 0, 0)
        ctx.simulate([la])
        _timed_depth_order(f"one instance of {cap >> 10} Ki particles (latency)", ctx, la, 1, cap, cap, True)
        ctx.close()

    P, ctx, slab, effect, stride, dt, rate = _churned()
    alive = ctx.read_metadata(0).alive_count
    _timed_depth_order(f"churned {P >> 20} Mi slots, {alive >> 10} Ki alive, permuted list", ctx, N.BatchLaunch.make(effect, slab, 0, rate), 1, P,
                           alive, False)
    ctx.close()


# Frusta for the cull cases, as (a, b, c, d) planes: x in [0, 2] and the other two axes in [-2, 2] keeps about half of a
# cloud over [-1, 1]^3; x in [0.998, 2] keeps about 0.1 % of it.
CULL_HALF = [[1, 0, 0, 0], [-1, 0, 0, 2], [0, 1, 0, 2], [0, -1, 0, 2], [0, 0, 1, 2], [0, 0, -1, 2]]
CULL_FEW = [[1, 0, 0, -0.998]] + CULL_HALF[1:]


def _timed_cull(label, ctx, launch, instances, rows, alive, claimed, frustum, bounds_bytes):
    """hnb_batch_cull of `launch`'s batch (alive-list source) into device buffers of `rows`, then hnb_batch_bounds of the
    same batch: one warm-up call each, then the best of 5 CUDA-event windows. GB/s counts what the cull must move: 16 B of
    position (and 4 B of list where no claim covers the row) read per live particle and 4 B written per visible one."""
    visible = torch.empty(rows, dtype=torch.int32, device="cuda")
    args = torch.empty(5 * instances, dtype=torch.int32, device="cuda")
    frusta = torch.tensor([frustum] * instances, dtype=torch.float32, device="cuda")
    call = lambda: ctx.batch_cull(launch, frusta.data_ptr(), instances, 0, 0, visible.data_ptr(), rows, args.data_ptr(), instances)  # noqa: E731
    call()
    ms = _events_ms(call)
    m = int(args.view(-1, 5)[:, 1].sum())
    report(f"cull: {label}", ms, (16 if claimed else 20) * alive + 4 * m,
           f"{ms * 1e3:.1f} us per call, {m >> 10} Ki of {alive >> 10} Ki particles visible, best of 5")
    _timed_bounds(f"{label} (beside cull)", ctx, launch, instances, bounds_bytes)


def _cull_worlds(small_caps):
    """The cull cases, one at a time: (label, ctx, launch, instances, rows, alive, claimed, bounds_bytes, filled) for the
    filled 64 Mi C5 instance under its claim, the same size spawned by one init burst, C4's topology in one call, single
    instances of each of `small_caps` (latency) and the 16 Mi-slot churn steady state. Each context is closed after its
    case."""
    P = 64 << 20
    ctx = hb.Context(0, stream.cuda_stream)
    effect = ctx.effect_compile(recipes.c5_lowered())
    slab = ctx.slab_create(P, 32)
    ctx.slab_fill_c5(slab, 0, P, 42, 1e9, 1e9)
    single_instance(ctx, P, 32, alive=P)
    la = N.BatchLaunch.make(effect, slab, 0, 0)
    ctx.simulate([la])
    yield "C5 64Mi filled, claim", ctx, la, 1, P, P, True, 16 * P, True
    ctx.slab_destroy(slab)
    slab = ctx.slab_create(P, 32)
    single_instance(ctx, P, 32, alive=0, spawn=P)
    ctx.simulate([N.BatchLaunch.make(effect, slab, 0, P)])
    ctx.upload_spawners([R.make_spawner(spawn=0, seed=43)])
    la = N.BatchLaunch.make(effect, slab, 0, 0)
    ctx.simulate([la])
    yield "C5 64Mi from one init burst, no claim", ctx, la, 1, P, P, False, 20 * P, False
    ctx.close()
    torch.cuda.empty_cache()

    n_inst, cap = 1024, 65536
    ctx = hb.Context(0, stream.cuda_stream)
    effect = ctx.effect_compile(recipes.c5_lowered())
    slab = ctx.slab_create(n_inst * cap, 32)
    sp = []
    for i in range(n_inst):
        ctx.slab_fill_c5(slab, i * cap, cap, 7000 + i, 1e9, 1e9)  # the last fill holds the slab's claim
        m = R.initial_metadata(cap, i, 8)
        m.alive_count, m.max_spawn = cap, 0
        ctx.metadata_insert(i, m)
        ctx.draw_args_insert(i)
        sp.append(R.make_spawner(seed=i, effect_metadata_index=i, draw_indirect_index=i, slab_offset=i * cap))
    ctx.upload_spawners(sp)
    ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, n_inst)], [0] * n_inst)
    ctx.set_sim_params(1 / 60, 0.0, n_inst)
    la = N.BatchLaunch.make(effect, slab, 0, 0)
    ctx.simulate([la])
    yield "C4 shape: 1024 x 65536 in one batch", ctx, la, n_inst, n_inst * cap, n_inst * cap, False, 20 * n_inst * cap - 4 * cap, False
    ctx.close()
    torch.cuda.empty_cache()

    for cap in small_caps:
        ctx = hb.Context(0, stream.cuda_stream)
        slab = ctx.slab_create(cap, 32)
        ctx.slab_fill_c5(slab, 0, cap, 100, 1e9, 1e9)
        single_instance(ctx, cap, 32, alive=cap)
        la = N.BatchLaunch.make(ctx.effect_compile(recipes.c5_lowered()), slab, 0, 0)
        ctx.simulate([la])
        yield f"one instance of {cap >> 10} Ki particles (latency)", ctx, la, 1, cap, cap, True, 16 * cap, False
        ctx.close()

    P, ctx, slab, effect, stride, dt, rate = _churned()
    alive = ctx.read_metadata(0).alive_count
    yield (f"churned {P >> 20} Mi slots, {alive >> 10} Ki alive, permuted list", ctx, N.BatchLaunch.make(effect, slab, 0, rate), 1, P,
           alive, False, 20 * alive, False)
    ctx.close()


def _copy_for_scale(name):
    a = torch.empty(2 << 30, dtype=torch.uint8, device="cuda")
    b = torch.empty_like(a)
    ms = _events_ms(lambda: b.copy_(a))
    report(f"{name}: 2 GiB device-to-device copy", ms, 2 * a.numel(), "torch copy_ (reads 2 GiB and writes 2 GiB), best of 5")
    del a, b
    torch.cuda.empty_cache()


def cull():
    """hnb_batch_cull: the filled 64 Mi C5 instance under its claim with about half and with about 0.1 % of it visible,
    the same size spawned by one init burst, C4's topology in one call, the 16 Mi-slot churn steady state and single
    instances of 4 Ki and 16 Ki (latency); each beside hnb_batch_bounds of the same batch, and a 2 GiB device-to-device
    copy for scale."""
    _card()
    _copy_for_scale("cull")
    for label, ctx, la, instances, rows, alive, claimed, bounds_bytes, filled in _cull_worlds((4096, 16 << 10)):
        if filled:
            _timed_cull(f"{label}, ~half visible", ctx, la, instances, rows, alive, claimed, CULL_HALF, bounds_bytes)
            _timed_cull(f"{label}, ~0.1 % visible", ctx, la, instances, rows, alive, claimed, CULL_FEW, bounds_bytes)
        else:
            _timed_cull(label, ctx, la, instances, rows, alive, claimed, CULL_HALF, bounds_bytes)


def view_frusta(views):
    """One frustum per view, each keeping about half of a cloud around the origin from a different direction: the half
    space n_v . p >= 0, with n_v turning around the y axis and tilting up and down, inside a box of half-width 2. (views,
    6, 4) float32."""
    out = []
    for v in range(views):
        t = 2 * np.pi * v / max(views, 1)
        n = np.array([np.cos(t), 0.3 * (-1) ** v, np.sin(t)])
        n /= np.linalg.norm(n)
        out.append([[*n, 0.0]] + CULL_HALF[1:])
    return np.array(out, dtype=np.float32)


def _timed_cull_views(label, ctx, launch, instances, rows, alive, claimed):
    """hnb_batch_cull_views of `launch`'s batch (alive-list source) at 1, 2, 4 and 8 views, beside as many hnb_batch_cull
    calls over the same stacked buffers: one warm-up each, then the best of 5 CUDA-event windows for each. GB/s counts
    what one multi-view call must move: 16 B of position (and 4 B of list where no claim covers the row) read per live
    particle once, and 4 B written per visible entry of each view."""
    vr = (rows + 63) // 64 * 64  # each view's slice 256-byte aligned
    visible = torch.empty(8 * vr, dtype=torch.int32, device="cuda")
    args = torch.empty(8 * 5 * instances, dtype=torch.int32, device="cuda")
    for views in (1, 2, 4, 8):
        frusta = torch.tensor(np.repeat(view_frusta(views)[:, None], instances, axis=1), device="cuda")
        fp, vp, ap = frusta.data_ptr(), visible.data_ptr(), args.data_ptr()
        one = lambda: ctx.batch_cull_views(launch, views, fp, instances, 0, 0, vp, vr, ap, instances)  # noqa: E731

        def separate():
            for v in range(views):
                ctx.batch_cull(launch, fp + 96 * v * instances, instances, 0, 0, vp + 4 * v * vr, vr, ap + 20 * v * instances, instances)
        one()
        ms_one = _events_ms(one)
        m = [int(x) for x in args.view(8, -1, 5)[:views, :, 1].sum(dim=1).tolist()]
        separate()
        ms_sep = _events_ms(separate)
        read = (16 if claimed else 20) * alive
        report(f"cull_views: {label}, V={views}", ms_one, read + 4 * sum(m),
               f"{ms_one * 1e3:.1f} us per call; {views} x cull: {ms_sep:.4f} ms ({ms_sep / ms_one:.2f}x); "
               f"visible per view {', '.join(f'{100 * x / max(alive, 1):.0f} %' for x in m)}; best of 5")


def cull_views():
    """hnb_batch_cull_views at 1, 2, 4 and 8 views, each view seeing about half of the cloud from another direction,
    beside as many hnb_batch_cull calls, on the cull cases: the filled 64 Mi C5 instance under its claim, the same size
    from one init burst, C4's topology in one call, the 16 Mi-slot churn steady state and one 4 Ki instance."""
    _card()
    _copy_for_scale("cull_views")
    for label, ctx, la, instances, rows, alive, claimed, _, _ in _cull_worlds((4096,)):
        _timed_cull_views(label, ctx, la, instances, rows, alive, claimed)


class _DeviceColumn:
    """A device column as torch sees it through __cuda_array_interface__."""

    def __init__(self, ptr, shape):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": "<f4", "data": (ptr, False), "version": 2}


def fresh_sector():
    """Cost of sector planes when access IS coalesced: C5 recipe burst + update, like `c5_init`, on a sector slab."""
    w = G.ExprWriter()
    asset = (G.EffectAsset(64 << 20, w.module, name="c5_spawned_sector")
             .init(G.SetAttributeModifier(A.POSITION, w.rand(G.VEC3) * w.lit(2.) - w.lit(1.)))
             .init(G.SetAttributeModifier(A.VELOCITY, w.rand(G.VEC3) * w.lit(2.) - w.lit(1.)))
             .init(G.SetAttributeModifier(A.AGE, w.lit(0.)))
             .init(G.SetAttributeModifier(A.LIFETIME, w.lit(1e9)))
             .update(G.AccelModifier(w.lit(G.Vec3(0., -9.8, 0.))))
             .update(G.LinearDragModifier(w.lit(0.5))))
    _burst("C5 recipe on SECTOR planes, 32Mi burst", asset, 64 << 20, 32 << 20, sector_planes=True)


def frame_chain():
    """Whole frames (bookkeeping + update, state resident, no table changes) back to back: what one step costs beyond its
    update kernel, at the shard sizes of the strong-scaling runs."""
    for mi in (1, 2, 4, 8, 16, 64):
        P = mi << 20
        ctx = hb.Context(0, stream.cuda_stream)
        slab = ctx.slab_create(P, 32)
        ctx.slab_fill_c5(slab, 0, P, 42, 1e9, 1e9)
        single_instance(ctx, P, 32, alive=P)
        la = [N.BatchLaunch.make(ctx.effect_compile(recipes.c5_lowered()), slab, 0, 0)]
        for _ in range(10):
            ctx.simulate(la)
        fr = min(frame_ms(ctx, la, 200) for _ in range(3))
        k = timed_update(ctx, la, 50)
        report(f"C5 {mi:2d}Mi frame chain", fr, 72 * P, f"isolated update kernel {k:.4f} ms; frame - kernel = {1e3 * (fr - k):+.1f} us")
        ctx.close()


def chunks_sweep():
    """Tile size (HNB_TILE_CHUNKS sub-tiles of 128 rows) and CTAs per SM under the pipelined frame chain."""
    import os
    for mi in (2, 4, 8, 16, 32):
        P = mi << 20
        for defines in ("", "HNB_MIN_BLOCKS=4"):
            for chunks in ("1", "2", "4"):
                os.environ["HNB_TILE_CHUNKS"] = chunks
                if defines:
                    os.environ["HNB_DEFINES"] = defines
                else:
                    os.environ.pop("HNB_DEFINES", None)
                ctx = hb.Context(0, stream.cuda_stream)
                slab = ctx.slab_create(P, 32)
                ctx.slab_fill_c5(slab, 0, P, 42, 1e9, 1e9)
                single_instance(ctx, P, 32, alive=P)
                la = [N.BatchLaunch.make(ctx.effect_compile(recipes.c5_lowered()), slab, 0, 0)]
                for _ in range(10):
                    ctx.simulate(la)
                fr = min(frame_ms(ctx, la, 200) for _ in range(3))
                report(f"C5 {mi:2d}Mi frame chain, chunks={chunks} {defines}", fr, 72 * P)
                ctx.close()
    os.environ.pop("HNB_TILE_CHUNKS", None)
    os.environ.pop("HNB_DEFINES", None)


def interop():
    """Device-resident export of the reference layouts (what a renderer binds, SURVEY §8 f-2): SoA planes -> AoS records and
    {ping,pong,dead} columns -> interleaved rows, device to device; bytes = read + written."""
    for stride, P in ((32, 64 << 20), (48, 32 << 20), (20, 32 << 20)):
        ctx = hb.Context(0, stream.cuda_stream)
        slab = ctx.slab_create(P, stride)
        buf = ctx.device_alloc(P * stride)
        ibuf = ctx.device_alloc(P * 12)
        for name, fn, nbytes in (("export AoS", lambda: ctx.slab_export_aos_device(slab, 0, P, buf), 2 * P * stride),
                                 ("import AoS", lambda: ctx.slab_import_aos_device(slab, 0, P, buf), 2 * P * stride),
                                 ("export indirect rows", lambda: ctx.slab_export_indirect_device(slab, 0, P, ibuf), 2 * P * 12),
                                 ("import indirect rows", lambda: ctx.slab_import_indirect_device(slab, 0, P, ibuf), 2 * P * 12)):
            for _ in range(3):
                fn()
            ctx.sync()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(10):
                fn()
            e1.record(stream)
            e1.synchronize()
            report(f"interop {name}, stride {stride}, {P >> 20} Mi rows", e0.elapsed_time(e1) / 10, nbytes)
        ctx.device_free(buf)
        ctx.device_free(ibuf)
        ctx.close()


def c2_small():
    """BASELINE configs[1] at ITS size: firework trails, 32768 slots (48-byte records). The whole population is 1.5 MB: a
    frame is pure fixed cost (launch chain + dependent-load latency), reported in microseconds per frame."""
    from tests.effects import firework_trails
    P = 32768
    ctx = hb.Context(0, stream.cuda_stream)
    fx = firework_trails(P).generate()
    slab = ctx.slab_create(P, fx.particle_stride)
    effect = ctx.effect_compile(fx)
    ctx.metadata_insert(0, R.initial_metadata(P, 0, fx.particle_stride // 4))
    ctx.draw_args_insert(0)
    ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, 1)], [0])
    ctx.set_sim_params(1 / 600, 0.0, 1)     # short steps: nobody expires during the measurement
    ctx.upload_spawners([R.make_spawner(spawn=30000, seed=7)])
    t_burst = frame_ms(ctx, [N.BatchLaunch.make(effect, slab, 0, 30000)])
    ctx.upload_spawners([R.make_spawner(spawn=0, seed=8)])
    la = [N.BatchLaunch.make(effect, slab, 0, 0)]
    for _ in range(10):
        ctx.simulate(la)
    fr = min(frame_ms(ctx, la, 200) for _ in range(3))
    k = timed_update(ctx, la, 50)
    alive = ctx.read_metadata(0).alive_count
    report(f"C2 firework @ 32768 slots: steady frame, {alive} alive", fr, (8 + 2 * 48) * alive, f"{fr * 1e3:.1f} us per frame (update kernel alone {k * 1e3:.1f} us); first burst frame of 30000 spawns (cold) {t_burst * 1e3:.1f} us")
    # a frame that also spawns: 100 particles per frame into free slots
    ctx.upload_spawners([R.make_spawner(spawn=8, seed=9)])
    la8 = [N.BatchLaunch.make(effect, slab, 0, 8)]
    for _ in range(5):
        ctx.simulate(la8)
    fr8 = min(frame_ms(ctx, la8, 100) for _ in range(3))
    report("C2 firework @ 32768 slots: frame with 8 spawns (init + bookkeeping + update)", fr8, (8 + 2 * 48) * alive, f"{fr8 * 1e3:.1f} us per frame")
    ctx.close()


def c4_recipe():
    """BASELINE configs[3] as stated (SURVEY 8d row C4): instancing.rs recipe, 1024 instances x 65536 slots in ONE batch, filled
    through the real init kernel; update-only frames, then frames that spawn one particle per instance (init with a
    depth-10 prefix search over 1024 instances + bookkeeping of 1024 instances + update)."""
    from tests.effects import instancing
    n_inst, cap = 1024, 65536
    ctx = hb.Context(0, stream.cuda_stream)
    fx = instancing(cap).generate()
    stride = fx.particle_stride
    slab = ctx.slab_create(n_inst * cap, stride)
    effect = ctx.effect_compile(fx)
    for i in range(n_inst):
        ctx.metadata_insert(i, R.initial_metadata(cap, i, stride // 4))
        ctx.draw_args_insert(i)
    fill = cap - 1024
    mk = lambda spawn: [R.make_spawner(spawn=spawn, seed=1000 + i, effect_metadata_index=i, draw_indirect_index=i, slab_offset=i * cap) for i in range(n_inst)]
    ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, n_inst)], [i * fill for i in range(n_inst)])
    ctx.set_sim_params(1 / 60, 0.0, n_inst)
    ctx.upload_spawners(mk(fill))
    t_fill = frame_ms(ctx, [N.BatchLaunch.make(effect, slab, 0, n_inst * fill)])
    alive = n_inst * fill
    report(f"C4 recipe: fill frame (init {alive >> 10} Ki over 1024 instances + update)", t_fill, (stride + 8) * alive + (8 + 2 * stride) * alive)
    ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, n_inst)], [0] * n_inst)
    ctx.upload_spawners(mk(0))
    la = [N.BatchLaunch.make(effect, slab, 0, 0)]
    for _ in range(5):
        ctx.simulate(la)
    fr = min(frame_ms(ctx, la, 30) for _ in range(2))
    k = timed_update(ctx, la, 20)
    report(f"C4 recipe: update-only frame, {alive >> 10} Ki alive in 1024 instances", fr, (8 + 2 * stride) * alive, f"update kernel alone {k:.4f} ms")
    ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, n_inst)], list(range(n_inst)))
    ctx.upload_spawners(mk(1))
    la1 = [N.BatchLaunch.make(effect, slab, 0, n_inst)]
    for _ in range(5):
        ctx.simulate(la1)
    fr1 = min(frame_ms(ctx, la1, 30) for _ in range(2))
    alive1 = sum(ctx.read_metadata(i).alive_count for i in (0, 511, 1023)) // 3 * n_inst
    report(f"C4 recipe: spawn 1 / instance / step frame (init 1024 + update {alive1 >> 10} Ki)", fr1, (8 + 2 * stride) * alive1, f"+{(fr1 - fr) * 1e3:.1f} us over the update-only frame")
    ctx.close()


def c3_chain():
    """C3 at its BASELINE size (1 Mi) as a frame chain (what a running effect costs per frame), strict and fast-math."""
    from tests.effects import force_field
    P = 1 << 20
    for fast in (False, True):
        asset = force_field(P)
        ctx = hb.Context(0, stream.cuda_stream)
        fx = asset.generate(fast_math=fast)
        slab = ctx.slab_create(P, fx.particle_stride)
        effect = ctx.effect_compile(fx)
        ctx.upload_properties(effect, 0, asset.serialize_properties())
        ctx.metadata_insert(0, R.initial_metadata(P, 0, fx.particle_stride // 4, properties_array_index=0))
        ctx.draw_args_insert(0)
        ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, 1)], [0])
        ctx.set_sim_params(1 / 6000, 0.0, 1)
        ctx.upload_spawners([R.make_spawner(spawn=P, seed=7)])
        ctx.simulate([N.BatchLaunch.make(effect, slab, 0, P)])
        ctx.upload_spawners([R.make_spawner(spawn=0, seed=8)])
        la = [N.BatchLaunch.make(effect, slab, 0, 0)]
        for _ in range(10):
            ctx.simulate(la)
        fr = min(frame_ms(ctx, la, 200) for _ in range(3))
        k = timed_update(ctx, la, 50)
        alive = ctx.read_metadata(0).alive_count
        report(f"C3 force field 1Mi frame chain{' FAST_MATH' if fast else ''}, {alive >> 10} Ki alive", fr, (8 + 2 * fx.particle_stride) * alive, f"isolated update kernel {k:.4f} ms")
        ctx.close()


def emitter_relocation():
    """hnb_slab_repack_events, hnb_instance_snapshot_events and hnb_instance_restore_events on an emitting parent of 16 Mi
    slots in a churned state, with two channels of 512 Ki entries, both full and overflowing (channel 0: Always, count 1;
    channel 1: OnDie, count 4). The first repack runs on the churned lists (one window); snapshot and restore (into a
    second slab) are best of 5."""
    _card()
    P, CAP = 16 << 20, 1 << 19
    w = G.ExprWriter()
    asset = (G.EffectAsset(P, w.module, name="relocated_emitter")
             .init(G.SetAttributeModifier(A.POSITION, w.rand(G.VEC3) * w.lit(2.) - w.lit(1.)))
             .init(G.SetAttributeModifier(A.VELOCITY, w.rand(G.VEC3) - w.lit(0.5)))
             .init(G.SetAttributeModifier(A.AGE, w.lit(0.)))
             .init(G.SetAttributeModifier(A.LIFETIME, w.lit(0.1).uniform(w.lit(0.5))))
             .update(G.EmitSpawnEventModifier(G.ALWAYS, w.lit(G.U32(1)), 0))
             .update(G.EmitSpawnEventModifier(G.ON_DIE, w.lit(G.U32(4)), 1)))
    fx = asset.generate(num_event_bindings=2)
    stride = fx.particle_stride
    ctx = hb.Context(0, stream.cuda_stream)
    slab, effect = ctx.slab_create(P, stride), ctx.effect_compile(fx)
    ev = [ctx.event_buffer_create(CAP) for _ in range(4)]
    for row in range(4):
        ctx.child_info_insert(row, 0, 0)
    for row in (0, 1):
        md = R.initial_metadata(P, row, stride // 4)
        md.base_child_index = 2 * row
        ctx.metadata_insert(row, md)
        ctx.draw_args_insert(row)
    ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, 1)], [0])
    dt, rate = 1 / 60, P // 24
    for f in range(40):  # lifetimes of 6 to 30 frames: the list is a permutation of the slice by now
        ctx.set_sim_params(dt, f * dt, 1)
        ctx.upload_spawners([R.make_spawner(spawn=rate, seed=100 + f)])
        ctx.simulate([N.BatchLaunch.make(effect, slab, 0, rate, emit_events=ev[:2])])
    ctx.sync()
    alive = ctx.read_metadata(0).alive_count
    counts = [ctx.read_child_info(k).event_count for k in (0, 1)]
    assert min(counts) > CAP, counts
    events = 12 * 2 * CAP  # per entry: the entry read and written, one inverse word read
    rp = _events_ms(lambda: ctx.slab_repack_events(slab, effect, 0, 0, P, ev[:2]), reps=1)
    report(f"emitter_relocation: repack of {P >> 20} Mi rows, {alive >> 10} Ki alive, 2 x {CAP >> 10} Ki events", rp,
           _repack_bytes(ctx, slab, P, alive) + 8 * P + events, "one window; bytes: repack + inverse + events")
    nbytes = ctx.instance_snapshot_events_bytes(stride, P, [CAP, CAP])
    buf = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    dst = ctx.slab_create(P, stride)
    snap = _events_ms(lambda: ctx.instance_snapshot_events(slab, effect, 0, 0, P, ev[:2], buf.data_ptr(), nbytes))
    rest = _events_ms(lambda: ctx.instance_restore_events(dst, effect, 1, 0, P, ev[2:], buf.data_ptr(), nbytes))
    md = ctx.read_metadata(1)
    records = md.max_update
    restored = [ctx.read_child_info(k).event_count for k in (2, 3)]
    report("emitter_relocation: snapshot", snap, (4 + 2 * stride) * records + 8 * P + events, f"{records >> 10} Ki records, best of 5")
    report("emitter_relocation: restore", rest, (8 + 2 * stride) * records + 4 * (P - alive) + P // 8 + 8 * 2 * CAP,
           f"into another slab, best of 5; event counts {counts} -> {restored}, alive {alive} -> {md.alive_count}")
    del buf
    ctx.close()


SCENARIOS = {"append": append, "cull": cull, "cull_views": cull_views, "c2_small": c2_small, "c4_recipe": c4_recipe, "c3_chain": c3_chain, "churn_slot": churn_slot, "c5_slot": c5_slot, "chunks": chunks_sweep, "interop": interop, "frame_chain": frame_chain, "churn": churn, "churn_sector": churn_sector, "churn_repack": churn_repack, "snapshot_restore": snapshot_restore, "bounds": bounds, "depth_order": depth_order, "emitter_relocation": emitter_relocation, "fresh_sector": fresh_sector, "many": many_batches, "c5": c5_update, "c5_dying": c5_dying, "c4": c4_topology, "c5_init": c5_init_burst, "c2": c2_trails, "c3": c3_force_field, "c3_fast": c3_fast_math}
if __name__ == "__main__":
    for name in (sys.argv[1:] or list(SCENARIOS)):
        try:
            SCENARIOS[name]()
        except Exception as e:  # keep going: one scenario must not hide the others
            print(f"{name}: FAILED {type(e).__name__}: {str(e)[:400]}", flush=True)
