#!/bin/bash
# compute-sanitizer over the GPU tests that exercise the round-2 kernel changes (slot order, ordered events, bookkeeping paths,
# init with the staged spawn prefix, sector planes, interop transposes). Output: $OUT/r2_sanitizer.txt (OUT defaults to tool_out)
OUT=${OUT:-tool_out}
mkdir -p $OUT
O=$OUT/r2_sanitizer.txt
echo "# compute-sanitizer (round 2 kernels): memcheck on update_c5 + slot_order + golden + events + ordered_events + sector_planes + interop + scene; racecheck on update_c5 + slot_order + golden + interop; synccheck on update_c5 + slot_order" > $O
T="tests/test_gpu_update_c5.py tests/test_gpu_slot_order.py tests/test_gpu_golden.py tests/test_gpu_events.py tests/test_gpu_ordered_events.py tests/test_gpu_sector_planes.py tests/test_gpu_interop.py tests/test_gpu_scene.py"
(timeout 1200 compute-sanitizer --tool memcheck python -m pytest $T -m gpu -q -x -k "not 2200000 and not 400000" 2>&1 | grep -E "COMPUTE-SANITIZER|passed|failed|ERROR SUMMARY|Invalid|at 0x" | head -40) >> $O
echo "--- racecheck" >> $O
(timeout 900 compute-sanitizer --tool racecheck python -m pytest tests/test_gpu_update_c5.py tests/test_gpu_slot_order.py tests/test_gpu_golden.py tests/test_gpu_interop.py -m gpu -q -x -k "not 2200000 and not 400000" 2>&1 | grep -E "COMPUTE-SANITIZER|passed|failed|RACECHECK SUMMARY|hazard" | head -40) >> $O
echo "--- synccheck" >> $O
(timeout 600 compute-sanitizer --tool synccheck python -m pytest tests/test_gpu_update_c5.py tests/test_gpu_slot_order.py -m gpu -q -x -k "not 2200000 and not 400000" 2>&1 | grep -E "COMPUTE-SANITIZER|passed|failed|ERROR SUMMARY" | head -20) >> $O
cat $O
