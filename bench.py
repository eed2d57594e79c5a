#!/usr/bin/env python
"""bench.py — particle-update throughput of the hot path on config C5 (BASELINE.json configs[4]).

    python bench.py --gpus N --steps K --warmup W            # this framework (CUDA, sm_90a)
    python bench.py --impl reference --gpus N --steps K ...  # the reference's path on the host CPU

Workload (SURVEY.md §8d, C5): one effect instance of 64 Mi particles, attributes {position, velocity,
age, lifetime} (32 B AoS record -> two float4 SoA planes), update = [Accel((0,-9.8,0)), LinearDrag(0.5)]
+ Euler integration + age/lifetime kill, dt = 1/60, lifetime 1e9 (nothing dies: steady state), alive
list = identity. A "step" is one full simulate(): (init skipped: 0 spawns) -> fused indirect+prefix-sum
bookkeeping kernel -> update kernel. For N GPUs the 64 Mi particles are sharded by index range
(64Mi/N per rank, strong scaling), no collective on the data path.

One JSON line is printed by rank 0 (see the task contract): value = particle-steps/s over the whole
job with all state resident in HBM; e2e = same metric through the C ABI with the per-frame HOST tables
(spawners, batch infos, prefix sums, sim params) uploaded and the draw-indirect instance count read
back every step; roofline = update kernel algorithmic bytes (72 B/particle-step) / its CUDA-event
duration vs the HBM peak (MEASURED_PEAKS.json when present, else the H100 SXM data sheet's 3.35 TB/s); cpu_baseline = the CPU oracle (C port, OpenMP) on a bounded
sample of the same workload.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import threading
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))

TOTAL_PARTICLES = 64 * 1024 * 1024
BYTES_PER_PARTICLE_STEP = 72  # 4 (alive idx read) + 32 (record read) + 32 (record write) + 4 (alive idx write); SURVEY §8d
DT = 1.0 / 60.0
METRIC = "particle-steps/sec at 64M particles"
UNIT = "particle-steps/s"


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--particles", type=int, default=TOTAL_PARTICLES, help="total particles over all GPUs")
    ap.add_argument("--scaling", default="strong", choices=["strong", "weak"])
    ap.add_argument("--cpu-seconds", type=float, default=12.0, help="budget of the cpu_baseline leg")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", help="write what the last timed step computed as DIR/<name>.npy")
    return ap.parse_args()


# ---------------------------------------------------------------------------------------------------
# clocks sampling during the timed region
# ---------------------------------------------------------------------------------------------------
class ClockSampler:
    """SM clock and throttle reasons sampled DURING the timed region. NVML in a thread (a query takes microseconds,
    so even a 40 ms timed region gets dozens of samples); `nvidia-smi -lms` as a fallback when pynvml is missing."""
    QUERY = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
             "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index: int):
        self.gpu = gpu_index
        self.samples = []          # nvidia-smi csv lines (fallback)
        self.sm, self.reason_bits = [], 0
        self.sm_max = None
        self.proc = None
        self.thread = None
        self.stop_flag = threading.Event()
        self.source = None

    def _nvml_handle(self):
        import pynvml
        pynvml.nvmlInit()
        try:
            import torch
            uuid = str(torch.cuda.get_device_properties(self.gpu).uuid)
            return pynvml, pynvml.nvmlDeviceGetHandleByUUID(("GPU-" + uuid).encode())
        except Exception:
            return pynvml, pynvml.nvmlDeviceGetHandleByIndex(self.gpu)

    def start(self):
        try:
            nv, h = self._nvml_handle()
            self.sm_max = float(nv.nvmlDeviceGetMaxClockInfo(h, nv.NVML_CLOCK_SM))
            def poll():
                while not self.stop_flag.is_set():
                    try:
                        self.sm.append(float(nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM)))
                        self.reason_bits |= int(nv.nvmlDeviceGetCurrentClocksEventReasons(h))
                    except Exception:
                        pass
                    time.sleep(0.001)
            self.nv = nv
            self.source = "nvml"
            self.thread = threading.Thread(target=poll, daemon=True)
            self.thread.start()
            return
        except Exception:
            self.source = None
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--id={self.gpu}", f"--query-gpu={self.QUERY}", "--format=csv,noheader,nounits",
                                          "-lms", "20"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        except Exception:
            self.proc = None
            return
        self.source = "nvidia-smi"
        def pump():
            for line in self.proc.stdout:
                self.samples.append(line.strip())
        self.thread = threading.Thread(target=pump, daemon=True)
        self.thread.start()

    def stop(self):
        if self.source == "nvml":
            self.stop_flag.set()
            self.thread.join(timeout=2)
            nv, bits = self.nv, self.reason_bits
            names = (("hw_slowdown", nv.nvmlClocksEventReasonHwSlowdown), ("hw_thermal_slowdown", nv.nvmlClocksEventReasonHwThermalSlowdown),
                     ("sw_thermal_slowdown", nv.nvmlClocksEventReasonSwThermalSlowdown), ("sw_power_cap", nv.nvmlClocksEventReasonSwPowerCap),
                     ("hw_power_brake_slowdown", nv.nvmlClocksEventReasonHwPowerBrakeSlowdown))
            return {"sm_mhz": statistics.median(self.sm) if self.sm else None, "sm_max_mhz": self.sm_max,
                    "reasons": sorted(n for n, b in names if bits & b), "samples": len(self.sm), "source": "nvml"}
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["no NVML, no nvidia-smi"], "samples": 0}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except Exception:
            self.proc.kill()
        sm, smax, reasons = [], [], set()
        for s in self.samples:
            f = [x.strip() for x in s.split(",")]
            if len(f) < 9:
                continue
            try:
                sm.append(float(f[1])); smax.append(float(f[2]))
            except ValueError:
                continue
            for name, val in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[5:9]):
                if val.lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": max(smax) if smax else None,
                "reasons": sorted(reasons), "samples": len(sm), "source": "nvidia-smi"}


def device_info(gpu_index: int):
    """The card's name and power limit: a measured time is only meaningful next to them."""
    import torch
    info = {"name": torch.cuda.get_device_name(gpu_index), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", f"--id={gpu_index}", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_w"] = float(out)
    except Exception:
        pass
    return info


# ---------------------------------------------------------------------------------------------------
# CPU arm: the oracle's multi-threaded C5 update (oracle/vfx_oracle.c::orc_update_c5_parallel)
# ---------------------------------------------------------------------------------------------------
def usable_cpus():
    """(logical CPUs, usable physical cores, how it was decided) — oracle/host_threads.py (shared with the tests' oracle runs)."""
    from oracle.host_threads import usable_cpus as f
    return f()


def cpu_workload_particles():
    """The 64 Mi-particle C5 instance itself when the host has the memory for it (2.9 GiB of buffers), else 8 Mi."""
    need = TOTAL_PARTICLES * (32 + 12 + 1)
    try:
        import psutil
        avail = psutil.virtual_memory().available
    except Exception:
        avail = None
    if avail is None or avail > 3 * need:
        return TOTAL_PARTICLES, "the full 64 Mi-particle instance"
    return 8 * 1024 * 1024, f"an 8 Mi-particle instance (host has {avail >> 20} MiB available, the 64 Mi one needs {need >> 20} MiB)"


class CpuC5:
    """One C5 instance on the host, stepped with the oracle's OpenMP port of the reference's passes."""

    def __init__(self, particles: int, threads: int):
        import numpy as np
        # one thread per physical core, pinned, neighbours first (must be in the environment before libgomp starts)
        os.environ.setdefault("OMP_PROC_BIND", "close")
        os.environ.setdefault("OMP_PLACES", "cores")
        from oracle import c_oracle as O
        self.np, self.O = np, O
        self.orc = O.load()
        self.n = particles
        self.threads = threads
        self.orc.orc_set_threads(threads)  # for the fill / reset loops; the update takes its own count
        self.particles = np.empty((particles, 8), dtype=np.float32)
        self.indirect = np.empty((particles, 3), dtype=np.uint32)
        # first touch by the threads that will own the rows (static schedule, same partition as the update)
        self.orc.orc_indirect_reset(O.ptr(self.indirect), 0, particles)
        self.orc.orc_fill_c5(O.ptr(self.particles), O.ptr(self.indirect), 0, particles, 42, 1e9, 1e9)
        self.flags = np.zeros(particles, dtype=np.uint8)
        self.sim = O.SimParams(DT, 0, DT, 0, DT, 0, 1)
        self.md = (O.EffectMetadata * 1)()
        self.md[0].capacity = particles
        self.md[0].alive_count = particles
        self.md[0].max_spawn = 0
        self.md[0].indirect_render_index = 0
        self.sp = (O.Spawner * 1)()
        self.sp[0].seed = 42
        self.draw = np.zeros(5, dtype=np.uint32)
        self.prefix = np.zeros(1, dtype=np.uint32)
        self.bi = (O.BatchInfo * 1)()
        self.bi[0].prefix_sum_count = 1
        self.dispatch = np.zeros(3, dtype=np.uint32)
        self.k = (C.c_float * 4)(0.0, -9.8, 0.0, 0.5)
        self.frames = 0

    def step(self, threads=None):
        """One full frame: indirect -> prefix sum -> update (all of vfx_*.wgsl's work for this config)."""
        o, P, u32 = self.orc, C.POINTER, C.c_uint32
        o.orc_indirect(C.byref(self.sim), self.md, self.draw.ctypes.data_as(P(u32)), self.sp, self.prefix.ctypes.data_as(P(u32)), None, 0)
        o.orc_prefix_sum(self.bi, 1, self.prefix.ctypes.data_as(P(u32)), self.dispatch.ctypes.data_as(P(u32)))
        alive = o.orc_update_c5_parallel(C.byref(self.sim), self.draw.ctypes.data_as(P(u32)), self.O.ptr(self.particles),
                                         self.O.ptr(self.indirect), self.sp, self.md, self.k, self.O.ptr(self.flags),
                                         self.threads if threads is None else threads)
        if alive != self.n:
            raise RuntimeError(f"CPU arm: {alive} of {self.n} particles alive")
        self.frames += 1
        return alive

    def checksum(self):
        return int(self.orc.orc_checksum(self.O.ptr(self.particles), 0, self.n, 8))

    def timed_steps(self, steps, threads=None):
        out = []
        for _ in range(steps):
            t0 = time.perf_counter()
            self.step(threads)
            out.append(time.perf_counter() - t0)
        return out


def measure_cpu_arm(steps: int, warmup: int, budget_s: float):
    """The CPU arm of both the `cpu_baseline` block and `--impl reference`: same workload, same threads, same timing, so
    that the two agree on the same box. Returns (value over the timed steps, per-step seconds, description dict)."""
    n, what = cpu_workload_particles()
    logical, cores, how = usable_cpus()
    arm = CpuC5(n, cores)
    w = arm.timed_steps(max(1, warmup))
    est = min(w)
    steps = max(1, min(steps, int(budget_s / max(est, 1e-6))))  # exactly the K asked for unless that would take minutes
    ts = arm.timed_steps(steps)
    total = sum(ts)
    med5 = statistics.median((ts + arm.timed_steps(max(0, 5 - steps)))[:5])  # BASELINE.md §3: median of five timed steps
    # BASELINE.md §3 also asks for the single-thread figure: one warm step, two timed
    one = arm.timed_steps(3, threads=1)[1:]
    desc = {
        "cores": cores, "kind": "port", "particles_per_step": n, "steps": steps,
        "sample": f"{steps} full frames (indirect + prefix-sum + update) of {what}, {total:.1f} s wall, oracle/vfx_oracle.c, "
                  f"OpenMP x{cores} (one thread per physical core, OMP_PROC_BIND={os.environ.get('OMP_PROC_BIND')}; {how}; "
                  f"OMP_NUM_THREADS={os.environ.get('OMP_NUM_THREADS', 'unset')} from the launcher ignored); the Rust/wgpu "
                  "reference cannot be built in this image (no Rust toolchain, no Vulkan ICD)",
        "median_of_5_value": n / med5, "single_thread_value": n / statistics.median(one),
        "gbps": BYTES_PER_PARTICLE_STEP * n * steps / total / 1e9,
    }
    return n * steps / total, ts, desc, arm


def cpu_baseline(seconds: float):
    value, _, desc, arm = measure_cpu_arm(20, 2, seconds)
    return {"value": value, "unit": UNIT, **desc}, arm


def run_reference(args):
    """--impl reference: the reference's path cannot be built here (no Rust toolchain, no Vulkan ICD —
    SURVEY.md §0.3), so this times the oracle's C port of it on all host cores. Rank 0 only."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    value, ts, desc, _ = measure_cpu_arm(args.steps, min(args.warmup, 2), 60.0)
    steps = desc["steps"]
    n = desc["particles_per_step"]
    line = {
        "impl": "reference", "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": args.gpus, "steps": steps,
        "warmup": args.warmup, "ms_per_step": sum(ts) / steps * 1e3, "higher_is_better": True, "scaling": args.scaling,
        "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": "C5 synthetic 64M-particle SoA buffer, Accel+LinearDrag update, sharded by index range",
                   "particles_total": n, "particles_per_step": n, "dt": DT,
                   "note": "CPU arm: one host runs the whole instance whatever --gpus says"},
        "cpu_baseline": {"value": value, "unit": UNIT, **desc},
        "e2e": {"value": value, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    print(json.dumps(line), flush=True)


# ---------------------------------------------------------------------------------------------------
# GPU arm
# ---------------------------------------------------------------------------------------------------
DUMP_SAMPLE_ROWS = 1 << 20   # over all ranks: 56 B per sampled row (record + three indices) = 56 MiB, under 64 MB
DUMP_LIMIT_BYTES = 64 * 10**6
DUMP_BLOCK_ROWS = 4096       # rows are sampled as whole blocks, so only the sampled rows leave the device


def dump_outputs(ctx, slab, rows, logical_first, out_dir, rank, world):
    """What a caller of simulate() receives after the last timed step: the particle records, the alive list and the
    counts, as .npy files (suffixed _rank<r> when several ranks write). Records and list entries are a fixed, seeded
    sample of blocks of rows; the ranks share the DUMP_SAMPLE_ROWS budget."""
    import numpy as np

    from bevy_hanabi_b200 import recipes
    out_dir.mkdir(parents=True, exist_ok=True)
    suffix = f"_rank{rank}" if world > 1 else ""
    md = ctx.read_metadata(0)
    n_blocks = -(-rows // DUMP_BLOCK_ROWS)
    k = min(n_blocks, max(1, DUMP_SAMPLE_ROWS // world // DUMP_BLOCK_ROWS))
    blocks = np.sort(np.random.default_rng([20240607, logical_first]).choice(n_blocks, k, replace=False))
    recs, idx, pick = [], [], []
    for b in blocks:
        first = int(b) * DUMP_BLOCK_ROWS
        count = min(DUMP_BLOCK_ROWS, rows - first)
        recs.append(ctx.slab_download_aos(slab, first, count, recipes.C5_STRIDE))
        idx.append(ctx.slab_download_indirect(slab, first, count)[:, md.indirect_write_index])
        pick.append(np.arange(first, first + count))
    pick, idx = np.concatenate(pick), np.concatenate(idx)
    alive = pick < md.alive_count
    arrays = {
        "particles": np.concatenate(recs).view(np.float32),  # (rows, 8): position.xyz, age, velocity.xyz, lifetime
        "particle_rows": (pick + logical_first).astype(np.float64),
        "alive_list": idx[alive].astype(np.float64),
        "alive_list_positions": pick[alive].astype(np.float64),
        "counts": np.array([md.alive_count, md.max_update, md.max_spawn, ctx.read_draw_args(0).instance_count], dtype=np.float64),
    }
    total = sum(a.nbytes for a in arrays.values())
    if total * world > DUMP_LIMIT_BYTES:
        raise RuntimeError(f"bench.py: dump of {total} bytes per rank x {world} ranks exceeds {DUMP_LIMIT_BYTES}")
    for name, a in arrays.items():
        np.save(out_dir / f"{name}{suffix}.npy", a)


def run_b200(args):
    import torch
    import torch.distributed as dist

    import bevy_hanabi_b200 as hb
    from bevy_hanabi_b200 import _native as N
    from bevy_hanabi_b200 import recipes, runtime as R

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device — hanabi_b200 has no CPU path (use --impl reference for the CPU arm)")
    torch.cuda.set_device(local_rank)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    n_gpus = max(world, 1)
    from bevy_hanabi_b200.sharding import shard_range
    if args.scaling == "strong":
        first_row, end_row = shard_range(args.particles, rank, n_gpus)   # index-range shard of the logical instance
        per_rank = end_row - first_row
        total = args.particles
    else:
        per_rank = args.particles
        total = per_rank * n_gpus

    # all work goes on ONE explicit non-default stream shared by torch (events, barriers) and the backend
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    assert stream.cuda_stream != 0
    ctx = hb.Context(local_rank, stream.cuda_stream)
    slab = ctx.slab_create(per_rank, recipes.C5_STRIDE)
    # the C5 effect authored through the Module/Modifier/EffectAsset API and lowered to CUDA C by the library
    effect = ctx.effect_compile(recipes.c5_asset(per_rank).generate())
    # shard `rank` owns logical rows [first_row, end_row) of the 64M instance under shard-local indices: the same
    # counter-based values a 1-GPU run holds for those rows (one seed for the whole instance, hashed with the LOGICAL row)
    logical_first = first_row if args.scaling == "strong" else rank * per_rank
    ctx.slab_fill_c5(slab, 0, per_rank, 42, 1e9, 1e9, logical_first=logical_first)
    md = R.initial_metadata(per_rank, 0, 8)
    md.alive_count = per_rank
    md.max_spawn = 0
    ctx.metadata_insert(0, md)
    ctx.draw_args_insert(0)
    spawners = (N.Spawner * 1)(R.make_spawner(spawn=0, seed=42))
    batches = (N.BatchInfo * 1)(N.BatchInfo(0, 0, 0, 0, 0, 1))
    prefix = (N.u32 * 1)(0)
    launches = (N.BatchLaunch * 1)(N.BatchLaunch.make(effect, slab, 0, 0))
    sim_t = [0.0]

    def upload_tables():
        ctx.upload_spawners_raw(spawners, 1)
        ctx.upload_batches_raw(batches, 1, prefix, 1)
        ctx.set_sim_params(DT, sim_t[0], 1)
        sim_t[0] += DT

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    per_rank_ms = []

    def timed(fn, steps):
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(steps):
            fn()
        e1.record(stream)
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        per_rank_ms.clear()
        per_rank_ms.append(ms)
        if world > 1:
            t = torch.tensor([ms], device="cuda", dtype=torch.float64)
            allt = [torch.zeros_like(t) for _ in range(world)]
            dist.all_gather(allt, t)
            per_rank_ms[:] = [float(x.item()) for x in allt]
            ms = max(per_rank_ms)  # device time, MAX over ranks
        barrier()
        return ms

    # -- device-resident loop (value): tables uploaded once, only the 64-byte frame header moves per step
    upload_tables()
    def step_resident():
        ctx.simulate_raw(launches, 1)
    for _ in range(max(args.warmup, 3)):
        step_resident()
    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
    l0 = ctx.launch_count
    ms = timed(step_resident, args.steps)
    value_per_rank_ms = [m / args.steps for m in per_rank_ms]
    gpu_launches = ctx.launch_count - l0
    clocks = sampler.stop() if rank == 0 else None
    value = total * args.steps / (ms * 1e-3)
    if args.dump_outputs:
        dump_outputs(ctx, slab, per_rank, logical_first, Path(args.dump_outputs), rank, world)

    # -- roofline leg: the update kernel alone, timed by CUDA events recorded around each launch on the launching stream
    ctx.enable_kernel_timing(True)
    ctx.kernel_time_ms()
    for _ in range(args.steps):
        step_resident()
    k_ms, k_n = ctx.kernel_time_ms()
    ctx.enable_kernel_timing(False)
    k_avg_ms = k_ms / max(k_n, 1)
    if world > 1:
        t = torch.tensor([k_avg_ms], device="cuda", dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        k_avg_ms = float(t.item())
    achieved = BYTES_PER_PARTICLE_STEP * per_rank / (k_avg_ms * 1e-3) / 1e9

    # -- end-to-end loop: host tables up, simulate, instance count back, every step. Like a renderer, the host keeps
    # two frames in flight: the count of step i is checked while step i+1 is already queued, so the host's wake-up
    # latency is not on the critical path (every step's count is still checked, on the host, against the expected value).
    # Both transfers are the library's own low-latency paths (DESIGN.md §4.1): the step's tables (header, batch info, tile word,
    # spawner row, range / spawn-prefix words: 232 bytes of the pinned host arena) reach the device in the parameter space of the
    # frame's first kernel launch, and the result comes back as one 64-bit (epoch, instance_count) word that the update pass
    # stores into pinned host memory — no copy-engine operation and no event sits between two kernels of the chain.
    FRAMES_IN_FLIGHT = 2
    ctx.set_count_mailbox(rows=1, ring=4)
    e2e_state = {"step": 0, "checked": 0, "epochs": []}
    def check_epoch(epoch):
        got = ctx.mailbox_count(epoch, 0)   # spins until the word of that frame has landed in host memory
        if got != per_rank:
            raise RuntimeError(f"instance_count {got} != {per_rank}")
        e2e_state["checked"] += 1
    def step_e2e():
        i = e2e_state["step"]
        if i >= FRAMES_IN_FLIGHT:
            check_epoch(e2e_state["epochs"][i - FRAMES_IN_FLIGHT])
        spawners[0].seed = 0x9E3779B9 * (i + 1) & 0xFFFFFFFF  # the tables differ from the previous step's (identical uploads are
        upload_tables()                                       # elided by the library); C5's update draws no random numbers
        ctx.simulate_raw(launches, 1)
        e2e_state["epochs"].append(ctx.last_epoch())
        e2e_state["step"] = i + 1
    def drain_e2e():
        ctx.sync()
        n = e2e_state["step"]
        for e in e2e_state["epochs"][max(0, n - FRAMES_IN_FLIGHT):n]:
            check_epoch(e)
        e2e_state["step"] = 0
        e2e_state["epochs"] = []
    copies0 = ctx.frame_block_copies
    for _ in range(3):
        step_e2e()
    drain_e2e()
    # K steps, three times; the MEDIAN run is reported (all three are listed): the timed region is short at 8 GPUs, where a
    # single scheduling hiccup of one rank's host process (the max over ranks sees it) shifts the result by tens of percent
    e2e_runs = []
    for _ in range(3):
        e2e_state["checked"] = 0
        e2e_runs.append(timed(step_e2e, args.steps))  # ends with a device synchronisation
        drain_e2e()
        assert e2e_state["checked"] == args.steps, "every step's instance count must have been checked on the host"
    ms_e2e = sorted(e2e_runs)[1]
    e2e_copy_engine_ops = ctx.frame_block_copies - copies0
    e2e_value = total * args.steps / (ms_e2e * 1e-3)
    h2d = 64 + 24 + 4 + 4 + 128 + 8  # frame header + batch info + tile size (+pad) + spawner row + range / spawn-prefix words
    ctx.set_count_mailbox(rows=0)

    # -- correctness guard inside the bench: nothing died, and the checksum of the whole logical instance (each shard
    # hashes its rows under their LOGICAL index; the sum over the shards is independent of how many GPUs hold it)
    mdr = ctx.read_metadata(0)
    assert mdr.alive_count == per_rank and mdr.max_update == per_rank, "bench state corrupted"
    frames_run = ctx.frames_simulated
    shard_sum = ctx.slab_checksum(slab, 0, per_rank, index_base=logical_first)
    state_sum = shard_sum
    if world > 1:
        t = torch.tensor([shard_sum - (1 << 64) if shard_sum >= (1 << 63) else shard_sum], device="cuda", dtype=torch.int64)
        dist.all_reduce(t, op=dist.ReduceOp.SUM)  # wraps mod 2^64
        state_sum = int(t.item()) % (1 << 64)

    peaks_path = ROOT / "MEASURED_PEAKS.json"
    if peaks_path.exists():
        peak = json.loads(peaks_path.read_text()).get("hbm_gbs", 3350.0)
        peak_src = "measured (MEASURED_PEAKS.json hbm_gbs)"
    else:
        peak, peak_src = 3350.0, "fallback (H100 SXM data sheet, 3.35 TB/s HBM3)"

    if rank == 0:
        line = {
            "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": n_gpus, "steps": args.steps, "warmup": max(args.warmup, 3),
            "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": args.scaling, "vs_baseline": None,
            "dtype": "f32", "data": "synthetic",
            "config": {"workload": "C5 synthetic 64M-particle SoA buffer, Accel+LinearDrag update, sharded by index range",
                       "particles_total": total, "particles_per_gpu": per_rank, "dt": DT, "steps_per_sec": args.steps / (ms * 1e-3),
                       "ms_per_step_by_rank": value_per_rank_ms,
                       "l2": "inputs larger than L2 (per-GPU working set %.0f MB per step)" % (per_rank * 72 / 1e6),
                       "parallelism": f"index-range shards x{n_gpus}, no collective",
                       "state_checksum": {"frames": int(frames_run), "sum_over_shards": f"0x{state_sum:016x}",
                                          "note": "order-independent 64-bit checksum of all particle records after `frames` frames, rows hashed "
                                                  "under their logical index: equal for every --gpus N at equal `frames`"}},
            "e2e": {"value": e2e_value, "unit": UNIT, "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": 8,
                    "ms_per_step": ms_e2e / args.steps, "frames_in_flight": FRAMES_IN_FLIGHT,
                    "h2d_path": "kernel parameter space of the frame's bookkeeping launch (from the pinned host arena)",
                    "d2h_path": "64-bit (epoch, instance_count) word stored by the update kernel into pinned host memory",
                    "copy_engine_ops_in_timed_region": int(e2e_copy_engine_ops),
                    "ms_per_step_runs": [r / args.steps for r in e2e_runs], "reported": "median of 3 runs of `steps` steps",
                    "note": "every step the host rewrites its per-frame tables (spawner row, batch info, prefix sums, sim params) and "
                            "they travel to the device with that step's first kernel launch; the draw-indirect instance_count of every "
                            "step comes back through the count mailbox and is checked on the host (two frames in flight: step i is "
                            "checked while step i+1 is queued); particle state stays in HBM as in the reference (it is never on the "
                            "host there either)"},
            "gpu_launches": int(gpu_launches),
            "roofline": {"bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
                         "traffic": None, "kernel": "hnb_update", "kernel_ms": k_avg_ms, "peak_source": peak_src,
                         "bytes_per_particle_step": BYTES_PER_PARTICLE_STEP},
            "clocks": clocks,
            "device": device_info(local_rank),
        }
        if not args.no_cpu_baseline and n_gpus == 1:
            cb, arm = cpu_baseline(args.cpu_seconds)
            line["cpu_baseline"] = cb
            # parity inside the bench: replay as many frames as the CPU arm ran on a fresh slab of the same instance and
            # compare the whole-state checksums (C5 is IEEE-exact: bit-for-bit)
            n_cpu, frames_cpu = cb["particles_per_step"], arm.frames
            c2 = hb.Context(local_rank, stream.cuda_stream)
            s2 = c2.slab_create(n_cpu, recipes.C5_STRIDE)
            e2 = c2.effect_compile(recipes.c5_asset(n_cpu).generate())
            c2.slab_fill_c5(s2, 0, n_cpu, 42, 1e9, 1e9)
            md2 = R.initial_metadata(n_cpu, 0, 8)
            md2.alive_count, md2.max_spawn = n_cpu, 0
            c2.metadata_insert(0, md2)
            c2.draw_args_insert(0)
            c2.upload_spawners_raw(spawners, 1)
            c2.upload_batches_raw(batches, 1, prefix, 1)
            c2.set_sim_params(DT, 0.0, 1)
            l2 = (N.BatchLaunch * 1)(N.BatchLaunch.make(e2, s2, 0, 0))
            for _ in range(frames_cpu):
                c2.simulate_raw(l2, 1)
            gpu_sum = c2.slab_checksum(s2, 0, n_cpu)
            cpu_sum = arm.checksum()
            c2.close()
            line["parity_check"] = {"particles": n_cpu, "frames": frames_cpu, "gpu_checksum": f"0x{gpu_sum:016x}",
                                    "cpu_oracle_checksum": f"0x{cpu_sum:016x}", "match": gpu_sum == cpu_sum}
            if gpu_sum != cpu_sum:
                raise SystemExit("bench.py: GPU state differs from the CPU oracle's after the same number of frames")
        print(json.dumps(line), flush=True)
    ctx.close()
    if world > 1:
        dist.destroy_process_group()


def main():
    args = parse_args()
    if args.impl == "reference":
        run_reference(args)
    else:
        run_b200(args)


if __name__ == "__main__":
    main()
