"""CPU estimate of the gather locality of a long-running effect (no GPU): run the churn scenario of tools/perf_matrix.py with the
numpy oracle at a small scale and count, per group of 32 consecutive alive-list entries (one warp's gathers), how many
32-byte DRAM sectors a 16-byte-per-row plane touches, versus the 16 sectors of the perfectly coalesced case."""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from oracle import c_oracle  # noqa: E402
from oracle.hanabi_oracle import EffectOracle  # noqa: E402
from tests.helpers import Instance, RefWorld  # noqa: E402
from tests.effects import drifting_sparks  # noqa: E402

orc = c_oracle.load()
P = 1 << 16
asset = drifting_sparks(P)
_, size, _ = asset.particle_layout()
ref = RefWorld(P, size // 4, [Instance(0, P, alive=0, seed=1)], dt=1 / 60)
eo = EffectOracle(asset)
rate = P // 40
for f in range(300):
    ref.sim.time = np.float32(f) * ref.sim.delta_time
    ref.set_spawns([rate], [1000 + f])
    eo.frame(ref, orc)
    if f in (0, 30, 60, 120, 299):
        md = ref.metadata[0]
        lst = ref.indirect[:md.alive_count, md.indirect_write_index].astype(np.int64)
        groups = lst[:len(lst) // 32 * 32].reshape(-1, 32)
        sectors = np.array([len(np.unique(g // 2)) for g in groups])      # 2 rows of 16 B per 32-byte sector
        lines = np.array([len(np.unique(g // 8)) for g in groups])        # 8 rows per 128-byte line
        print(f"frame {f:3d}: alive {md.alive_count:6d} ({100 * md.alive_count / P:.0f} % of capacity)  sectors per warp gather "
              f"{sectors.mean():5.1f} (ideal 16 -> x{sectors.mean() / 16:.2f} traffic)  128-B lines {lines.mean():5.1f} (ideal 4)")
