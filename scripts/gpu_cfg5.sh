#!/bin/bash
# cfg5-sized run: 10M groups x 5 peers over 8 GPUs (1.25M per GPU), as the driver launches bench.py
N=${1:-8}; OUT=runs/multi; mkdir -p $OUT
python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port 29541 \
  bench.py --gpus $N --steps 40 --warmup 4 --e2e-steps 8 --groups 1250000 > $OUT/bench_cfg5_n$N.json 2> $OUT/bench_cfg5_n$N.err
echo "rc=$?"
python - <<PY
import json
d=json.loads(open("$OUT/bench_cfg5_n$N.json").read().strip().splitlines()[-1])
print("N=%d groups/gpu=%d value=%.3e ms/step=%.4f frac=%.3f e2e=%.3e staged=%.3e records_api=%.3e"%(d["n_gpus"],d["config"]["groups_per_gpu"],d["value"],d["ms_per_step"],d["roofline"]["frac"],d["e2e"]["value"],d["e2e_staged"]["value"],d["e2e_records_api"]["value"]), d["clocks"])
PY
