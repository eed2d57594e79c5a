"""Long-running fuzz of GPU spawn events under the CPU emulation: tests/kernel_emu.py::random_event_scene (the scenes of
tests/test_kernel_emu_cpu.py::test_random_event_scenes) over many seeds, default (atomic) and ordered append.   python tools/emu_fuzz_events.py [seconds] [first_seed]"""
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from oracle import c_oracle  # noqa: E402
from tests.kernel_emu import random_event_scene  # noqa: E402

budget = float(sys.argv[1]) if len(sys.argv) > 1 else 120.0
seed = int(sys.argv[2]) if len(sys.argv) > 2 else 3
orc = c_oracle.load()
t0, n = time.time(), 0
while time.time() - t0 < budget:
    for ordered in (False, True):
        random_event_scene(orc, ordered, seed)
        n += 1
    seed += 1
    if n % 10 == 0:
        print(f"{n} scenes ok ({time.time() - t0:.0f} s), next seed {seed}", flush=True)
print(f"done: {n} random event scenes exact against the oracle (seeds up to {seed - 1}, default and ordered append)")
