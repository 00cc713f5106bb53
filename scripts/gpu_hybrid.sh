#!/bin/bash
# hybrid staging: smoke, then the e2e leg in its modes at several staging-thread counts (strict timeouts)
OUT=runs/${1:-hyb}; mkdir -p $OUT
timeout 200 python __graft_entry__.py smoke 2>&1 | tail -2
for T in ${2:-48 12}; do
  for M in ${3:-hybrid packed raw}; do
    BENCH_E2E_MODE=$M timeout 150 python bench.py --steps 5 --warmup 3 --e2e-steps 40 --e2e-threads $T --no-sublegs --no-cpu-baseline > $OUT/bench_${M}_T$T.json 2> $OUT/bench_${M}_T$T.err
    python - <<PY
import json
try:
    d=json.loads(open("$OUT/bench_${M}_T$T.json").read().strip().splitlines()[-1])
    e=d["e2e"]; print("T=$T $M: e2e %.3e  %.3f ms/step  h2d %.1f MB  begin %.2f wait %.2f ms | value %.3e" % (e["value"], e["ms_per_step"], e["h2d_bytes_per_step"]/1e6, e["host_ms_per_step"]["begin"], e["host_ms_per_step"]["wait"], d["value"]))
except Exception as ex:
    print("T=$T $M failed", ex); print(open("$OUT/bench_${M}_T$T.err").read()[-800:])
PY
  done
done
