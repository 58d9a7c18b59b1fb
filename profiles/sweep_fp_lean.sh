#!/bin/bash
# k_filter_project_tma with the lean consumer loop: offset-resolve delay, lag, stages and tile size around the
# defaults (delay 2, lag = max(delay, L2 budget), K = 8 for C2 / 4 for C3).  The lag must be >= the delay; the
# flag shift register allows up to 128 / K - 1 tiles (15 at K = 8, 24 at K <= 4).
run() { echo "== $*"; env "$@" FP_SHORT=1 timeout 100 python profiles/microbench_fp.py 2>&1 | grep -E "^(c2|sel1|c3|sel99)"; }
run X=1
for d in 1 2 3; do
  for l in 1 2 3 4 6; do
    [ $l -ge $d ] || continue
    run DFGPU_FP_DELAY=$d DFGPU_FP_LAG=$l
    run DFGPU_FP_DELAY=$d DFGPU_FP_LAG=$l DFGPU_FP_K=4
  done
done
run DFGPU_FP_STAGES=4,2
run DFGPU_FP_STAGES=2,4
run DFGPU_FP_LEAN=0
