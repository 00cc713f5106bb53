#!/bin/bash
# quick GPU iteration: selected parity tests, then the device-resident bench with phase timing
# usage: gpu_quick.sh [pytest -k expression]
OUT=runs/quick; mkdir -p $OUT
timeout 1500 python -m pytest tests -m gpu -x -q -k "${1:-fused or every_ingest or golden}" > $OUT/pytest.txt 2>&1; tail -n 4 $OUT/pytest.txt
RAFTGPU_TILE_DEBUG=1 timeout 600 python bench.py --steps 60 --warmup 6 --no-cpu-baseline --e2e-steps 4 > $OUT/bench.json 2> $OUT/bench.err
grep "tile debug" $OUT/bench.err
python - <<PY
import json
try:
    d=json.loads(open("$OUT/bench.json").read().strip().splitlines()[-1])
    print("value=%.3e ms/step=%.4f"%(d["value"],d["ms_per_step"]), [(k["kernel"],round(k["avg_us"],1),round(k["frac"],3)) for k in d["kernels"]], "e2e=%.3e"%d["e2e"]["value"])
except Exception as e:
    print("failed", e); print(open("$OUT/bench.err").read()[-2000:])
PY
