#!/bin/bash
# Round-2 GPU call: parity tests, the host packer's thread scaling on the box's CPUs, the bench line.
# usage: scripts/gpu_r2.sh <tag> [steps]
TAG=${1:-r2}; STEPS=${2:-20}; OUT=runs/$TAG; mkdir -p $OUT
lscpu | grep -E "Model name|^CPU\(s\)|Thread|Socket|NUMA" > $OUT/env.txt
timeout 900 python -m pytest tests -m gpu -x -q > $OUT/pytest_gpu.txt 2>&1; echo "pytest rc=$?" >> $OUT/pytest_gpu.txt
tail -n 3 $OUT/pytest_gpu.txt
[ -x scripts/micro/pack_bench ] && { timeout 300 scripts/micro/pack_bench 1000000 4 8 16 32 64 > $OUT/pack_bench.txt 2>&1; RAFTGPU_PACK_SCALAR=1 timeout 300 scripts/micro/pack_bench 1000000 32 >> $OUT/pack_bench.txt 2>&1; cat $OUT/pack_bench.txt; }
timeout 900 python bench.py --steps $STEPS --warmup 5 > $OUT/bench.json 2> $OUT/bench.err; echo "bench rc=$?" >> $OUT/bench.err
tail -n 5 $OUT/bench.err
python - <<PY
import json
try:
    d=json.loads(open("$OUT/bench.json").read().strip().splitlines()[-1])
    print("value=%.3e ms/step=%.4f frac=%.3f"%(d["value"],d["ms_per_step"],d["roofline"]["frac"]))
    for k in ("e2e","e2e_prepacked","e2e_wire","scatter","recompute_only","cpu_baseline"):
        if d.get(k): print(k, {a:(round(b,4) if isinstance(b,float) else b) for a,b in d[k].items() if a not in ("api","sample")})
except Exception as e:
    print("failed", e)
PY
