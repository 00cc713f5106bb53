#!/bin/bash
# multi-GPU bench under torchrun, as the driver launches it (strict timeouts)
N=${1:-2}; OUT=runs/multi; mkdir -p $OUT
nvidia-smi --query-gpu=index,name --format=csv,noheader | head -8
timeout ${2:-240} python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port 29533 \
  bench.py --gpus $N --steps 20 --warmup 5 --no-sublegs --no-cpu-baseline > $OUT/bench_n$N.json 2> $OUT/bench_n$N.err
echo "rc=$?"; grep -v Warning $OUT/bench_n$N.err | tail -5 | cut -c1-300
python - <<PY
import json
d=json.loads(open("$OUT/bench_n$N.json").read().strip().splitlines()[-1])
e=d["e2e"]
print("N=%d value=%.3e ms/step=%.4f frac=%.3f | e2e=%.3e (%.3f ms/step, %s threads, mode %s, h2d %.1f MB) begin %.2f wait %.2f" % (d["n_gpus"], d["value"], d["ms_per_step"], d["roofline"]["frac"], e["value"], e["ms_per_step"], e.get("host_threads"), e.get("mode"), e["h2d_bytes_per_step"]/1e6, e["host_ms_per_step"]["begin"], e["host_ms_per_step"]["wait"]))
PY
