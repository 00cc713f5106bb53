#!/bin/bash
# One GPU round: parity tests, smoke, bench (fused default + scatter), ncu launch lists + full captures.
# usage: scripts/gpu_round.sh <tag> [skip_tests]
TAG=${1:-r}; OUT=runs/$TAG; mkdir -p $OUT
if [ -z "$2" ]; then
  timeout 300 python __graft_entry__.py smoke > $OUT/smoke.txt 2>&1; echo "smoke rc=$?" >> $OUT/smoke.txt
  timeout 1800 python -m pytest tests -m gpu -x -q > $OUT/pytest_gpu.txt 2>&1; echo "pytest rc=$?" >> $OUT/pytest_gpu.txt
fi
timeout 900 python bench.py --steps 100 --warmup 10 > $OUT/bench.json 2> $OUT/bench.err; echo "bench rc=$?" >> $OUT/bench.err
timeout 900 python bench.py --steps 100 --warmup 10 --scatter --no-cpu-baseline --e2e-steps 8 > $OUT/bench_scatter.json 2> $OUT/bench_scatter.err
timeout 900 python bench.py --steps 100 --warmup 10 --compact-device --no-cpu-baseline --e2e-steps 8 > $OUT/bench_compact.json 2> $OUT/bench_compact.err
PROF="python bench.py --profile --steps 8 --warmup 3"
timeout 900 ncu --metrics gpu__time_duration.sum --clock-control none --csv --log-file $OUT/launches.csv $PROF > $OUT/ncu_launches.log 2>&1
timeout 900 ncu --metrics gpu__time_duration.sum --clock-control none --csv --log-file $OUT/launches_scatter.csv $PROF --scatter > $OUT/ncu_launches_scatter.log 2>&1
timeout 900 ncu --set full --clock-control none --import-source on -k regex:step_tile_kernel -s 6 -c 1 -f -o $OUT/prof_fused $PROF > $OUT/ncu_fused.log 2>&1
timeout 900 ncu --set full --clock-control none --import-source on -k regex:step_tile_compact_kernel -s 6 -c 1 -f -o $OUT/prof_ctile $PROF --compact-device > $OUT/ncu_ctile.log 2>&1
timeout 900 ncu --set full --clock-control none --import-source on -k regex:recompute_kernel -s 6 -c 1 -f -o $OUT/prof_recompute $PROF --scatter > $OUT/ncu_recompute.log 2>&1
timeout 900 ncu --set full --clock-control none --import-source on -k regex:apply_kernel -s 6 -c 1 -f -o $OUT/prof_apply $PROF --scatter > $OUT/ncu_apply.log 2>&1
for f in smoke.txt pytest_gpu.txt bench.err; do [ -f $OUT/$f ] && { echo "== $f"; tail -n 3 $OUT/$f; }; done
python - <<PY
import json
for n in ("bench","bench_scatter","bench_compact"):
    try:
        d=json.loads(open("$OUT/%s.json"%n).read().strip().splitlines()[-1])
        print(n, "value=%.3e ms/step=%.4f"%(d["value"],d["ms_per_step"]), [(k["kernel"],round(k["avg_us"],1),round(k["frac"],3)) for k in d["kernels"]], "staged=%.3e (%.3f ms)"%(d["e2e_staged"]["value"],d["e2e_staged"]["ms_per_step"]), "e2e(zero-copy)=%.3e"%d["e2e"]["value"], "cpu=", d.get("cpu_baseline",{}).get("value"))
    except Exception as e:
        print(n, "failed", e)
PY
