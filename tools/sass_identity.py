#!/usr/bin/env python
"""Guard for changes that must not touch the default device code: dump the SASS of four representative generated
effects (C5 recipe, an event-emitting parent, its child, a force-field effect with properties) and compare it with a
saved baseline.

    python tools/sass_identity.py save  [dir]     # before the change (default dir: /tmp/sass_baseline)
    python tools/sass_identity.py check [dir]     # after the change: prints IDENTICAL / DIFFERENT per effect

Compiles with nvcc offline (no GPU needed), with the flags the NVRTC path uses for default effects.
"""
import os
import subprocess
import sys
from pathlib import Path

CUDA = Path(os.environ.get("CUDA_HOME", "/usr/local/cuda"))  # the same nvcc as bevy_hanabi_b200/build.py

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))


def sources():
    from bevy_hanabi_b200 import recipes
    from tests.effects import event_assets, force_field
    p, c = event_assets()
    return {"c5": recipes.c5_lowered().generate_source(), "parent": p.generate(num_event_bindings=1).generate_source(),
            "child": c.generate(parent=p).generate_source(), "ff": force_field(10).generate().generate_source()}


def sass(name, src, d: Path):
    cu, cubin = d / f"{name}.cu", d / f"{name}.cubin"
    cu.write_text(src)
    subprocess.run([str(CUDA / "bin" / "nvcc"), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--fmad=false",
                    "-diag-suppress", "550,177", "-cubin", str(cu), "-o", str(cubin)], check=True)
    return subprocess.run(["cuobjdump", "-sass", str(cubin)], capture_output=True, text=True, check=True).stdout


def main():
    mode = sys.argv[1] if len(sys.argv) > 1 else "check"
    d = Path(sys.argv[2] if len(sys.argv) > 2 else "/tmp/sass_baseline")
    d.mkdir(parents=True, exist_ok=True)
    bad = 0
    for name, src in sources().items():
        out = sass(name, src, d)
        ref = d / f"{name}.sass"
        if mode == "save":
            ref.write_text(out)
            print(name, "saved", len(out))
        else:
            same = ref.exists() and ref.read_text() == out
            bad += not same
            print(name, "IDENTICAL" if same else "DIFFERENT")
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
