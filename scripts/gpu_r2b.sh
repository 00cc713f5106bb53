#!/bin/bash
# e2e staging diagnosis: step_begin_records traced at several staging-thread counts
OUT=runs/${1:-r2b}; mkdir -p $OUT
for T in ${2:-32 48 56 64}; do
  RAFTGPU_TRACE=1 timeout 600 python bench.py --steps 5 --warmup 3 --e2e-steps 24 --e2e-threads $T --no-sublegs --no-cpu-baseline > $OUT/bench_T$T.json 2> $OUT/bench_T$T.err
  echo "== T=$T"; grep "step_begin_records n=" $OUT/bench_T$T.err | tail -n 2; grep "step_wait" $OUT/bench_T$T.err | tail -n 2
  python - <<PY
import json
d=json.loads(open("$OUT/bench_T$T.json").read().strip().splitlines()[-1])
print({a:(round(b,4) if isinstance(b,float) else b) for a,b in d["e2e"].items() if a!="api"})
PY
done
