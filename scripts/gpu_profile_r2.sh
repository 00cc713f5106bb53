#!/bin/bash
# Round-2 profiling call: ncu launch list + --set full captures of the fused tile kernel (cfg3 and cfg4), the
# recompute kernel and the wire kernels; compute-sanitizer on the new kernels.  usage: scripts/gpu_profile_r2.sh <tag>
TAG=${1:-r02}; OUT=runs/$TAG; mkdir -p $OUT
PROF="python bench.py --profile --steps 8 --warmup 3"
timeout 600 ncu --metrics gpu__time_duration.sum --clock-control none --csv --log-file $OUT/launches.csv $PROF > $OUT/ncu_launches.log 2>&1
timeout 900 ncu --set full --clock-control none --import-source on -k regex:step_tile_kernel -s 6 -c 1 -f -o $OUT/prof_fused $PROF > $OUT/ncu_fused.log 2>&1
timeout 900 ncu --set full --clock-control none --import-source on -k regex:step_tile_kernel -s 6 -c 1 -f -o $OUT/prof_fused_cfg4 $PROF --workload cfg4 > $OUT/ncu_fused_cfg4.log 2>&1
timeout 900 ncu --set full --clock-control none --import-source on -k regex:recompute_kernel -s 4 -c 1 -f -o $OUT/prof_recompute python scripts/micro_recompute.py > $OUT/ncu_recompute.log 2>&1
timeout 900 ncu --set full --clock-control none --import-source on -k regex:wire_ -c 2 -f -o $OUT/prof_wire python scripts/micro_wire.py > $OUT/ncu_wire.log 2>&1
ls -la $OUT | tail -n 12
