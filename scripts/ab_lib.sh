#!/bin/bash
# usage: scripts/ab_lib.sh LIB_A LIB_B [rounds] [steps]
# A/B of two builds of the library on one GPU: the c2 step (bench.py --no-extras) and the per-kernel times from the
# profiler, alternated in both orders (rounds of A,B then rounds of B,A) so drift on a shared host shows as spread.
OUT=${OUT:-bench_outputs}
A=$1; B=$2; R=${3:-3}; K=${4:-32}
mkdir -p $OUT
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv,noheader
one() {  # label lib
  SWARMDB_B200_LIB=$2 timeout 200 python bench.py --steps $K --warmup 4 --no-extras --cpu-budget 0 > $OUT/ab_$1.json 2> $OUT/ab_$1.err
  python - "$1" "$OUT/ab_$1.json" <<'PY'
import json, sys
d = json.loads(open(sys.argv[2]).read().strip().splitlines()[-1])
k = {n: round(x, 4) for n, x in d["kernels"].items() if x is not None}
print(sys.argv[1], "step_ms", round(d["ms_per_step"], 4), k, flush=True)
PY
}
for r in $(seq $R); do one A $A; one B $B; done
for r in $(seq $R); do one B $B; one A $A; done
