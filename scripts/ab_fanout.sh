#!/bin/bash
# A/B of the fan-out kernel variants on one GPU (every command under its own short timeout)
OUT=${OUT:-bench_outputs}
mkdir -p $OUT
timeout 200 python -m pytest tests/test_gpu_xshard.py tests/test_gpu_parity.py -m gpu -x -q 2>&1 | tail -4
run() {  # variant
  SDB_FANOUT_VARIANT=$1 timeout 60 python scripts/proxy_import8.py 2>&1 | tail -1 | sed "s/^/v$1 proxy: /"
}
bench() {
  timeout 100 python bench.py --steps 32 --warmup 4 --variant $1 --cpu-budget 0 > $OUT/ab.json 2> $OUT/ab.err
  python - <<PY
import json
d=json.loads(open("$OUT/ab.json").read().strip().splitlines()[-1])
print("v$1 bench:", round(d["value"]/1e9,3), round(d["ms_per_step"],4), {k:round(x["ms_per_launch"],4) for k,x in d["kernels"].items()}, round(d["roofline"]["frac"],4))
PY
}
for v in 0 1 2 3; do run $v; done
for v in 0 1 2 3; do bench $v; done
