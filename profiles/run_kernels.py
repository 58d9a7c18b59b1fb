#!/usr/bin/env python
"""Short driver for ncu captures: runs each hot-path operator a few times on BASELINE-sized inputs.
  ncu --set full --clock-control none --import-source on -k regex:k_filter_project -s 2 -c 1 -o fp python profiles/run_kernels.py c2
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from datafusion_archive_b200 import engine, workloads  # noqa: E402

which = sys.argv[1] if len(sys.argv) > 1 else "c2"
n = int(float(sys.argv[2])) if len(sys.argv) > 2 else 100_000_000
reps = int(sys.argv[3]) if len(sys.argv) > 3 else 3
ctx = engine.GpuContext(0)
if which in ("c2", "c3", "sel1"):
    arrays, pred, proj = (workloads.c3 if which == "c3" else workloads.c2)(n)
    if which == "sel1":  # 1 % selectivity: the predicate pass alone
        from datafusion_archive_b200.expr import col, lit
        pred = col(0) > lit(0.99)
    b = ctx.upload(arrays)
    for _ in range(reps):
        r = ctx.filter_project(b, pred, proj)
        print(which, "rows out", r.nrows)
        r.free()
elif which == "deep":
    from datafusion_archive_b200.expr import col, lit
    import numpy as np
    b = ctx.upload([np.random.default_rng(1).random(n)])
    pred = (col(0) * col(0)) < lit(0.3)
    proj = [(col(0) + col(0)) * (col(0) - lit(1.0)) / (col(0) + lit(2.0))]
    ctx.profile_enable(True)
    for _ in range(reps):
        r = ctx.filter_project(b, pred, proj)
        r.free()
    ms, k = ctx.profile_get()
    print(which, "kernel ms", ms / k)
elif which == "reduce":
    from datafusion_archive_b200.expr import AggregateFunction, col
    import numpy as np
    b = ctx.upload([np.random.default_rng(47).random(n)])
    aggs = [AggregateFunction(f, col(0)) for f in ("min", "max", "sum", "count")]
    for _ in range(reps):
        r = ctx.aggregate(b, [], aggs)
        print(which, "rows", r.nrows)
        r.free()
else:
    arrays, keys, aggs, _ = (workloads.c4 if which == "c4" else workloads.c5)(n)
    b = ctx.upload(arrays)
    for _ in range(reps):
        r = ctx.aggregate(b, keys, aggs)
        print(which, "groups", r.nrows)
        r.free()
b.free()
ctx.close()
