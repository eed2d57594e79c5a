"""Parity at BASELINE.json's FULL size (config C5: 67,108,864 particles on one GPU), where downloading and diffing
buffers is impractical: the whole-slab state is compared through order-independent 64-bit checksums computed by the
device (hnb_slab_checksum*) and by the oracle (orc_checksum) over identical counter-based initial states, plus
size-independent invariants of the bookkeeping (SURVEY.md §3.5).

Each C5 case runs both device modules: the hand-lowered recipes.c5_lowered (default cut, no lifetime floors) and the
authored recipes.c5_asset that bench.py times (its own column plan, HNB_LIFE_FLOOR 1: the fill's identity claim lets the
update prove rows alive from a floor per 32 rows and skip their lifetime loads)."""
import ctypes as C
import time

import numpy as np
import pytest

from oracle import c_oracle as O

pytestmark = pytest.mark.gpu


def _module(recipe, n):
    from bevy_hanabi_b200 import recipes
    if recipe == "lowered":
        return recipes.c5_lowered()
    fx = recipes.c5_asset(n).generate()
    assert "\n#define HNB_LIFE_FLOOR 1\n" in fx.generate_source()
    return fx


def _oracle_run(orc, n, seed, lo, hi, steps, dt, checks=None):
    """The oracle's state after `steps` frames, or after each frame count of `checks` (a list of states)."""
    particles = np.empty((n, 8), dtype=np.float32)
    indirect = np.zeros((n, 3), dtype=np.uint32)
    indirect[:, 2] = np.arange(n, dtype=np.uint32)
    orc.orc_fill_c5(O.ptr(particles), O.ptr(indirect), 0, n, seed, lo, hi)
    sim = O.SimParams(dt, 0, dt, 0, dt, 0, 1)
    md = (O.EffectMetadata * 1)()
    md[0].capacity, md[0].alive_count, md[0].max_spawn = n, n, 0
    sp = (O.Spawner * 1)()
    sp[0].seed = 42
    draw = np.zeros(5, dtype=np.uint32)
    prefix = np.zeros(1, dtype=np.uint32)
    bi = (O.BatchInfo * 1)(O.BatchInfo(0, 0, 0, 0, 0, 1))
    dispatch = np.zeros(3, dtype=np.uint32)
    k = (C.c_float * 4)(0.0, -9.8, 0.0, 0.5)
    flags = np.zeros(n, dtype=np.uint8)
    u32p = C.POINTER(C.c_uint32)
    from oracle.host_threads import oracle_threads
    threads = oracle_threads()
    out = []
    for step in range(1, max(checks or [steps]) + 1):
        orc.orc_indirect(C.byref(sim), md, draw.ctypes.data_as(u32p), sp, prefix.ctypes.data_as(u32p), None, 0)
        orc.orc_prefix_sum(bi, 1, prefix.ctypes.data_as(u32p), dispatch.ctypes.data_as(u32p))
        orc.orc_update_c5_parallel(C.byref(sim), draw.ctypes.data_as(u32p), O.ptr(particles), O.ptr(indirect), sp, md, k, O.ptr(flags), threads)
        if step in (checks or [steps]):
            out.append({"alive": md[0].alive_count, "max_spawn": md[0].max_spawn, "instance_count": int(draw[1]),
                        "write_index": md[0].indirect_write_index, "particles": orc.orc_checksum(O.ptr(particles.view(np.uint32)), 0, n, 8),
                        "indirect": orc.orc_checksum(O.ptr(indirect), 0, n, 3)})
    return out if checks else out[0]


def _gpu_run(ctx, n, seed, lo, hi, steps, dt, recipe="lowered", checks=None):
    from bevy_hanabi_b200 import _native as N, runtime as R
    slab = ctx.slab_create(n, 32)
    effect = ctx.effect_compile(_module(recipe, n))
    ctx.slab_fill_c5(slab, 0, n, seed, lo, hi)
    md = R.initial_metadata(n, 0, 8)
    md.alive_count, md.max_spawn = n, 0
    ctx.metadata_insert(0, md)
    ctx.draw_args_insert(0, N.DrawIndexedIndirectArgs(0, 0, 0, 0, 0))
    ctx.upload_spawners([R.make_spawner(seed=42)])
    ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, 1)], [0])
    ctx.set_sim_params(dt, 0.0, 1)
    launches = [N.BatchLaunch.make(effect, slab, 0, 0)]
    out = []
    for step in range(1, max(checks or [steps]) + 1):
        ctx.simulate(launches)
        if step in (checks or [steps]):
            m = ctx.read_metadata(0)
            out.append({"alive": m.alive_count, "max_spawn": m.max_spawn, "instance_count": ctx.read_draw_args(0).instance_count,
                        "write_index": m.indirect_write_index, "particles": ctx.slab_checksum(slab, 0, n),
                        "indirect": ctx.slab_checksum_indirect(slab, 0, n)})
    ctx.slab_destroy(slab)
    ctx.effect_destroy(effect)
    return out if checks else out[0]


@pytest.mark.parametrize("n,lo,hi,steps", [
    (1 << 20, 0.02, 0.3, 12),          # 1M with deaths: the checksum machinery itself, cross-checked cheaply
    (64 << 20, 1e9, 1e9, 3),           # BASELINE C5: 64M, nothing dies (the benchmarked steady state)
    (64 << 20, 0.02, 0.12, 5),         # BASELINE C5 variant B: lifetimes expire -> kills, dead stack, compaction at 64M
])
def test_c5_checksum_parity(ctx, orc, n, lo, hi, steps):
    dt = 1.0 / 60.0
    want = _oracle_run(orc, n, 1234, lo, hi, steps, dt)
    for recipe in ("lowered", "authored"):
        got = _gpu_run(ctx, n, 1234, lo, hi, steps, dt, recipe)
        assert got == want, recipe
    assert got["alive"] == got["instance_count"] and got["max_spawn"] == n - got["alive"]
    if hi > 1e8:
        assert got["alive"] == n
    else:
        assert 0 < got["alive"] < n  # the scenario must actually kill some and keep some


def test_authored_c5_floors_at_64_mi_rows(ctx, orc):
    """The authored C5 at BASELINE's 64 Mi rows for 150 frames, lifetimes U(2.0, 2.5) at dt = 1/60: floors prove every row
    alive until about frame 120, then deaths begin in every group and end the claim. Checked after frames 119 (nobody has
    died yet), 130 and 150."""
    n, dt, lo, hi, checks = 64 << 20, 1.0 / 60.0, 2.0, 2.5, [119, 130, 150]
    t0 = time.perf_counter()
    want = _oracle_run(orc, n, 4321, lo, hi, 150, dt, checks)
    t1 = time.perf_counter()
    got = _gpu_run(ctx, n, 4321, lo, hi, 150, dt, "authored", checks)
    t2 = time.perf_counter()
    print(f"64 Mi rows x 150 frames: oracle {t1 - t0:.1f} s, device (with its checksums) {t2 - t1:.1f} s")
    for step, g, w in zip(checks, got, want):
        assert g == w, f"after frame {step}"
    assert got[0]["alive"] == n and 0 < got[1]["alive"] < n and got[2]["alive"] < got[1]["alive"]


def test_c4_instancing_topology_checksum(ctx, orc):
    """BASELINE config C4's shape at full size: 1024 instances x 65536 particles in ONE batch (one launch, prefix
    search depth 10, 1024 independent look-back chains), with kills. Whole-slab checksums vs the oracle."""
    _c4_topology(ctx, orc, "lowered", 3, 0.02, 0.12)


def test_c4_topology_authored_claim_in_the_middle(ctx, orc):
    """The C4 topology with the authored C5: instance 517 is filled last and holds the claim, so the floors of one
    instance in the middle of the batch are stored on frame 0 and prove its rows alive until deaths begin at frame 6
    (lifetimes U(0.1, 0.3)); the other 1023 instances keep none."""
    _c4_topology(ctx, orc, "authored", 10, 0.1, 0.3, claimed=517)


def _c4_topology(ctx, orc, recipe, steps, lo, hi, claimed=None):
    """`claimed`: the instance filled last (the fill holds the identity claim), the others in order."""
    from bevy_hanabi_b200 import _native as N, runtime as R
    n_inst, cap = 1024, 65536
    n = n_inst * cap
    dt = 1.0 / 60.0
    order = [i for i in range(n_inst) if i != claimed] + ([claimed] if claimed is not None else [])
    # ---- oracle
    particles = np.empty((n, 8), dtype=np.float32)
    indirect = np.zeros((n, 3), dtype=np.uint32)
    indirect[:, 2] = np.arange(n, dtype=np.uint32)
    for i in order:
        orc.orc_fill_c5(O.ptr(particles), O.ptr(indirect), i * cap, cap, 7000 + i, lo, hi)
    sim = O.SimParams(dt, 0, dt, 0, dt, 0, n_inst)
    md = (O.EffectMetadata * n_inst)()
    sp = (O.Spawner * n_inst)()
    for i in range(n_inst):
        md[i].capacity, md[i].alive_count, md[i].max_spawn, md[i].indirect_render_index = cap, cap, 0, i
        sp[i].seed, sp[i].effect_metadata_index, sp[i].draw_indirect_index, sp[i].slab_offset = i, i, i, i * cap
    draw = np.zeros(5 * n_inst, dtype=np.uint32)
    prefix = np.zeros(n_inst, dtype=np.uint32)
    bi = (O.BatchInfo * 1)(O.BatchInfo(0, 0, 0, 0, 0, n_inst))
    dispatch = np.zeros(3, dtype=np.uint32)
    k = (C.c_float * 4)(0.0, -9.8, 0.0, 0.5)
    flags = np.zeros(cap, dtype=np.uint8)
    u32p = C.POINTER(C.c_uint32)
    from oracle.host_threads import oracle_threads
    threads = oracle_threads()
    for _ in range(steps):
        orc.orc_indirect(C.byref(sim), md, draw.ctypes.data_as(u32p), sp, prefix.ctypes.data_as(u32p), None, 0)
        orc.orc_prefix_sum(bi, 1, prefix.ctypes.data_as(u32p), dispatch.ctypes.data_as(u32p))
        for i in range(n_inst):
            orc.orc_update_c5_parallel(C.byref(sim), draw.ctypes.data_as(u32p), O.ptr(particles), O.ptr(indirect), C.byref(sp[i]), C.byref(md[i]), k,
                                       O.ptr(flags), threads)
    want = {"particles": orc.orc_checksum(O.ptr(particles.view(np.uint32)), 0, n, 8), "indirect": orc.orc_checksum(O.ptr(indirect), 0, n, 3),
            "alive": [md[i].alive_count for i in range(n_inst)], "total_update": bi[0].total_update_count}
    # ---- GPU
    slab = ctx.slab_create(n, 32)
    effect = ctx.effect_compile(_module(recipe, cap))
    for i in order:
        ctx.slab_fill_c5(slab, i * cap, cap, 7000 + i, lo, hi)
    spawners = []
    for i in range(n_inst):
        m = R.initial_metadata(cap, i, 8)
        m.alive_count, m.max_spawn = cap, 0
        ctx.metadata_insert(i, m)
        ctx.draw_args_insert(i, N.DrawIndexedIndirectArgs(0, 0, 0, 0, 0))
        spawners.append(R.make_spawner(seed=i, effect_metadata_index=i, draw_indirect_index=i, slab_offset=i * cap))
    ctx.upload_spawners(spawners)
    ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, n_inst)], [0] * n_inst)
    ctx.set_sim_params(dt, 0.0, n_inst)
    launches = [N.BatchLaunch.make(effect, slab, 0, 0)]
    for _ in range(steps):
        ctx.simulate(launches)
    got = {"particles": ctx.slab_checksum(slab, 0, n), "indirect": ctx.slab_checksum_indirect(slab, 0, n),
           "alive": [ctx.read_metadata(i).alive_count for i in range(n_inst)], "total_update": ctx.read_batch_info(0).total_update_count}
    assert got["alive"] == want["alive"]
    assert got["total_update"] == want["total_update"]
    assert got["indirect"] == want["indirect"]
    assert got["particles"] == want["particles"]
    assert 0 < sum(got["alive"]) < n
    assert all(ctx.read_draw_args(i).instance_count == got["alive"][i] for i in range(0, n_inst, 97))
    if claimed is not None:
        assert 0 < got["alive"][claimed] < cap
