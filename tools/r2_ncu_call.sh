#!/bin/bash
# An ncu --set full capture of every kernel of the path in every BASELINE shape (tools/ncu_targets.py), each summarised
# right away (the reports together are large; only those named in NCU_KEEP are kept), then the launch list of a short
# bench run. Outputs under $OUT (default tool_out/).
OUT=${OUT:-tool_out}
mkdir -p $OUT
for s in ${NCU_SCENARIOS:-c5_64m c5_8m c5_1m c5_64m_slot c5_init c3_16m c3_1m c2 c4 churn churn_slot interop}; do
  timeout 600 ncu --set full --clock-control none --import-source on --profile-from-start off -f -o $OUT/r2_ncu_$s \
      python tools/ncu_targets.py $s > $OUT/r2_ncu_$s.log 2>&1
  echo "$s rc=$?" >> $OUT/r2_ncu_rc.txt
  python tools/ncu_summary.py $OUT/r2_ncu_$s.ncu-rep $OUT/r2_ncu_${s}_summary.txt > /dev/null 2>&1
  case " ${NCU_KEEP:-c3_16m c5_8m} " in *" $s "*) ;; *) rm -f $OUT/r2_ncu_$s.ncu-rep ;; esac
done
timeout 600 ncu --metrics gpu__time_duration.sum --clock-control none -c 400 --csv --log-file $OUT/r2_launches.csv \
    python bench.py --steps 5 --warmup 3 > $OUT/r2_launches_bench.log 2>&1
cat $OUT/r2_ncu_rc.txt; du -sh $OUT
