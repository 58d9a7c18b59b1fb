#!/bin/bash
# k_filter_project_tma: dual-ring vs stash mode, and the lag of each
run() { echo "== $*"; env "$@" timeout 100 python profiles/microbench_fp.py 2>&1 | grep -E "^(c2|sel1|c3|copy|sel99|and2)"; }
run X=1
for l in 8 12 16 20; do run DFGPU_FP_MODE=stash DFGPU_FP_LAG=$l; done
