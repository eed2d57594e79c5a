"""Long-running fuzz of the kernels under the CPU emulation (tests/kernel_emu.py): random worlds, effects, tile sizes and
grids for a time budget; stops at the first mismatch with the oracle and prints the seed.

    python tools/emu_fuzz.py [seconds] [first_seed] [sector]     # "sector": half of the worlds on HNB_SLAB_SECTOR_PLANES slabs
"""
import os
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from oracle import c_oracle  # noqa: E402
from oracle.hanabi_oracle import EffectOracle, pcg_hash  # noqa: E402
from tests import static_emu  # noqa: E402
from tests.effects import drifting_sparks, firework_trails, growing_dust, ribbon_asset  # noqa: E402
from tests.helpers import Instance, RefWorld  # noqa: E402
from tests.kernel_emu import EmuWorld, assert_same  # noqa: E402


def one(seed, orc, slib, sector_mix=False):
    rng = np.random.default_rng(seed)
    kind = int(rng.integers(0, 4))
    asset = [drifting_sparks, firework_trails, growing_dust, ribbon_asset][kind](1)
    fields, size, _ = asset.particle_layout()
    n_inst = int(rng.integers(1, 10))
    caps = [int(rng.choice([1, 2, 31, 32, 33, 64, 127, 128, 129, 255, 256, 257, 511, 512, 513, 1023, 1024, 1025, 1500, 2049, 2600])) for _ in range(n_inst)]
    insts, off = [], 0
    for i, c in enumerate(caps):
        insts.append(Instance(off, c, alive=0, seed=seed * 100 + i))
        off += c
    dt = float(rng.choice([1 / 30, 1 / 10, 1 / 4, 1.0]))
    ref = RefWorld(off, size // 4, insts, dt=dt)
    if kind == 3:
        ref.set_sort_keys(fields)
    eo = EffectOracle(asset)
    chunks, ctas = int(rng.choice([1, 2, 4])), int(rng.integers(1, 4))
    sector = sector_mix and bool(int(pcg_hash(np.array([seed], dtype=np.uint32))[0]) & 1)   # independent of `rng`: same worlds as without the option
    fx = asset.generate(sector_planes=sector)
    k = {32: 4, 48: 2}.get(size, 1)
    if chunks * k > 16:
        chunks = 1
    emu = EmuWorld(ref, fx, chunks=chunks, update_ctas=ctas, static_lib=slib)
    frames = int(rng.integers(3, 9))
    for f in range(frames):
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        mode = rng.random()
        spawns = [0 if mode < 0.15 else (int(rng.integers(0, c + 60)) if rng.random() < 0.7 else 0) for c in caps]
        seeds = [int(pcg_hash(np.array([seed * 64 + f * 16 + i], dtype=np.uint32))[0]) for i in range(n_inst)]
        ref.set_spawns(spawns, seeds)
        eo.frame(ref, orc)
        emu.frame_step(orc, ref.sim, spawns, seeds)
        assert_same(ref, emu.pull(), f"seed {seed} kind {kind} caps {caps} chunks {chunks} ctas {ctas} sector {sector} frame {f}")
    return kind


def main():
    budget = float(sys.argv[1]) if len(sys.argv) > 1 else 120.0
    seed = int(sys.argv[2]) if len(sys.argv) > 2 else 0
    sector_mix = len(sys.argv) > 3 and sys.argv[3] == "sector"
    orc, slib = c_oracle.load(), static_emu.build()
    t0, n, kinds = time.time(), 0, [0, 0, 0, 0]
    while time.time() - t0 < budget:
        kinds[one(seed, orc, slib, sector_mix)] += 1
        seed += 1
        n += 1
        if n % 25 == 0:
            print(f"{n} worlds ok ({time.time() - t0:.0f} s), next seed {seed}, per effect {kinds}", flush=True)
    print(f"done: {n} random worlds bit-exact against the oracle, seeds up to {seed - 1}, per effect {kinds}" + (", half of them on sector-plane slabs" if sector_mix else ""))


if __name__ == "__main__":
    main()
