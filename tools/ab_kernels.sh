#!/bin/bash
# Same-machine A/B of the kernel sources: current tree vs the files under tools/ab_old/ (rebuilt in place), C5 at 64 / 8 / 1 Mi.
# tools/ab_old/ is not kept in the repository: fill it before the run, e.g.
#   mkdir -p tools/ab_old && for f in hnb_particle_kernels.cuh hnb_static_kernels.cu hnb_wgsl.cuh; do git show <rev>:bevy_hanabi_b200/csrc/kernels/$f > tools/ab_old/$f; done
set -e
K=bevy_hanabi_b200/csrc/kernels
run() { SWEEP_PS="64,8,1" SWEEP_CHUNKS=0 timeout 300 python tools/sweep_small.py 2>&1 | grep "^P=" | sed "s/^/$1 /"; }
run new
mkdir -p /tmp/ab_new && cp $K/hnb_particle_kernels.cuh $K/hnb_static_kernels.cu $K/hnb_wgsl.cuh /tmp/ab_new/
cp tools/ab_old/* $K/
python -c "import __graft_entry__ as g; g.build()" > /dev/null 2>&1
run old
cp /tmp/ab_new/* $K/
python -c "import __graft_entry__ as g; g.build()" > /dev/null 2>&1
run new
