#!/bin/bash
# k_filter_project_tma with the lean consumer loop: lag, stages and tile size around the defaults
run() { echo "== $*"; env "$@" FP_SHORT=1 timeout 100 python profiles/microbench_fp.py 2>&1 | grep -E "^(c2|sel1|c3|sel99)"; }
run X=1
for l in 6 10 12; do run DFGPU_FP_LAG=$l; done
run DFGPU_FP_STAGES=4,2
run DFGPU_FP_STAGES=2,4
run DFGPU_FP_K=4
run DFGPU_FP_K=4 DFGPU_FP_LAG=12
run DFGPU_FP_K=4 DFGPU_FP_LAG=24
run DFGPU_FP_LEAN=0
