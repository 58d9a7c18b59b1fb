#!/usr/bin/env python
"""COUNT(DISTINCT) next to SUM(v), COUNT(v) on the same data: whole aggregate call (CUDA events, median of 5).
Cases: the C4 shape (1e8 rows, 1e5 mixed Int64 keys) with v ~ UniformInt[0,100); the same keys with every v distinct;
no GROUP BY over 1e8 Int64 values with 1e6 distinct.  Prints the card name and power limit read in the same run.
usage: microbench_distinct.py [rows]"""
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from datafusion_archive_b200 import engine, workloads  # noqa: E402
from datafusion_archive_b200.expr import AggregateFunction, col  # noqa: E402

n = int(float(sys.argv[1])) if len(sys.argv) > 1 else 100_000_000
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print("card: %s" % card.splitlines()[0] if card else "card: unknown")
ctx = engine.GpuContext(0)
rng = np.random.default_rng(46)
k = workloads.mix_keys(rng.integers(0, 100_000, n, dtype=np.int64))
cases = [("C4 keys, v in [0,100)", [k, rng.integers(0, 100, n, dtype=np.int64)], [col(0)]),
         ("C4 keys, every v distinct", [k, rng.permutation(n).astype(np.int64)], [col(0)]),
         ("no GROUP BY, 1e6 distinct", [rng.integers(0, 1_000_000, n, dtype=np.int64)], [])]
for name, arrays, keys in cases:
    b = ctx.upload(arrays)
    arg = col(len(arrays) - 1)
    for label, aggs in [("SUM(v), COUNT(v)", [AggregateFunction("sum", arg), AggregateFunction("count", arg)]),
                        ("COUNT(DISTINCT v)", [AggregateFunction("count", arg, distinct=True)])]:
        ctx.aggregate(b, keys, aggs).free()  # warm-up
        walls = []
        for _ in range(5):
            ctx.timer_start()
            ctx.aggregate(b, keys, aggs).free()
            walls.append(ctx.timer_stop())
        wall = float(np.median(walls))
        print("%-28s %-18s %9.3f ms  %7.2f Grows/s  (median of 5, max %.3f ms)" % (name, label, wall, n / wall / 1e6, max(walls)))
    b.free()
ctx.close()
