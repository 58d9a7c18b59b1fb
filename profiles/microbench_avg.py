#!/usr/bin/env python
"""AVG(v) next to SUM(v), COUNT(v) on the C4 data (1e8 rows, 1e5 scrambled Int64 keys, v ~ U[0,1) f64), the same keys with
an Int32 v, and no GROUP BY over the f64 column.  Variants of a case alternate, 7 rounds each; reported per variant:
the summed time of the scan / reduce kernels (dfgpu_profile_*) and of the whole aggregate call (CUDA events), each the
median over the rounds.  Prints the card name and power limit read in the same run.
usage: microbench_avg.py [rows]"""
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from datafusion_archive_b200 import engine, workloads  # noqa: E402
from datafusion_archive_b200.expr import AggregateFunction, col  # noqa: E402

n = int(float(sys.argv[1])) if len(sys.argv) > 1 else 100_000_000
ROUNDS = 7
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print("card: %s" % (card.splitlines()[0] if card else "unknown"))
ctx = engine.GpuContext(0)
arrays, keys, _, _ = workloads.c4(n)
v32 = np.random.default_rng(47).integers(-1000, 1000, n).astype(np.int32)


def sum_count(c):
    return [AggregateFunction("sum", c), AggregateFunction("count", c)]


def avg(c):
    return [AggregateFunction("avg", c)]


cases = [("C4, f64 v", arrays, keys, [("SUM(v), COUNT(v)", sum_count(col(1))), ("AVG(v)", avg(col(1)))]),
         ("C4 keys, Int32 v", [arrays[0], v32], keys, [("SUM(v), COUNT(v)", sum_count(col(1))), ("AVG(v)", avg(col(1)))]),
         ("no GROUP BY, f64 v", [arrays[1]], [], [("SUM(v)", [AggregateFunction("sum", col(0))]), ("AVG(v)", avg(col(0)))])]


def once(b, keys, aggs):
    ctx.profile_enable(True)
    ctx.timer_start()
    ctx.aggregate(b, keys, aggs).free()
    wall = ctx.timer_stop()
    kern, _ = ctx.profile_get()
    ctx.profile_enable(False)
    return kern, wall


for name, cols, ks, variants in cases:
    b = ctx.upload(cols)
    for _, aggs in variants:
        once(b, ks, aggs)  # warm-up
    t = {label: ([], []) for label, _ in variants}
    for _ in range(ROUNDS):
        for label, aggs in variants:
            kern, wall = once(b, ks, aggs)
            t[label][0].append(kern)
            t[label][1].append(wall)
    for label, _ in variants:
        kern, wall = t[label]
        print("%-20s %-18s kernel %8.3f ms (min %.3f, max %.3f)  call %8.3f ms (min %.3f, max %.3f)  median of %d" %
              (name, label, np.median(kern), min(kern), max(kern), np.median(wall), min(wall), max(wall), ROUNDS))
    b.free()
ctx.close()
