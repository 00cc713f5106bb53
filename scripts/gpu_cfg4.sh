#!/bin/bash
# cfg4 (1M x 7 joint) measurements: fused, scatter, with CPU arm
OUT=runs/cfg4; mkdir -p $OUT
timeout 600 python bench.py --workload cfg4 --steps 60 --warmup 6 --e2e-steps 8 > $OUT/fused.json 2> $OUT/fused.err
timeout 600 python bench.py --workload cfg4 --steps 60 --warmup 6 --e2e-steps 8 --no-cpu-baseline --scatter > $OUT/scatter.json 2> $OUT/scatter.err
python - <<PY
import json
for f in ("fused","scatter"):
    try:
        d=json.loads(open("$OUT/%s.json"%f).read().strip().splitlines()[-1])
        print(f,"value=%.3e ms/step=%.4f"%(d["value"],d["ms_per_step"]), [(k["kernel"],round(k["avg_us"],1),round(k["frac"],3)) for k in d["kernels"]], "e2e=%.3e staged=%.3e"%(d["e2e"]["value"],d["e2e_staged"]["value"]), d.get("cpu_baseline",{}).get("value"))
    except Exception as e:
        print(f,"failed", e); print(open("$OUT/%s.err"%f).read()[-1500:])
PY
