#!/usr/bin/env python
"""What a scalar function costs on the interpreter path, 1e8 rows resident in HBM:
  filter  SELECT a FROM t WHERE a > 0.5   against sqrt(a) > 0.5 and sin(a) > 0.5   (a ~ U[0,1) f64)
  group   SELECT k, SUM(v) ... GROUP BY k against SUM(sqrt(v))                      (the C4 data: 1e5 Int64 keys)
Variants of a case alternate, 7 rounds each; reported per variant: the summed time of the scan kernels
(dfgpu_profile_*, the kernel events bench.py uses) and of the whole call (CUDA events), each the median over the rounds.
Prints the card name and power limit read in the same run.
usage: microbench_fn.py [rows]"""
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from datafusion_archive_b200 import engine, workloads  # noqa: E402
from datafusion_archive_b200.expr import AggregateFunction, col, fn  # noqa: E402

n = int(float(sys.argv[1])) if len(sys.argv) > 1 else 100_000_000
ROUNDS = 7
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print("card: %s" % (card.splitlines()[0] if card else "unknown"))
ctx = engine.GpuContext(0)
a = np.random.default_rng(48).random(n)
arrays, keys, _, _ = workloads.c4(n)


def filt(pred):
    return lambda b: ctx.filter_project(b, pred, [col(0)]).free()


def group(arg):
    return lambda b: ctx.aggregate(b, keys, [AggregateFunction("sum", arg)]).free()


cases = [("filter", [a], [("a > 0.5", filt(col(0) > 0.5)), ("sqrt(a) > 0.5", filt(fn("sqrt", col(0)) > 0.5)),
                          ("sin(a) > 0.5", filt(fn("sin", col(0)) > 0.5))]),
         ("GROUP BY k", arrays, [("SUM(v)", group(col(1))), ("SUM(sqrt(v))", group(fn("sqrt", col(1))))])]


def once(run, b):
    ctx.profile_enable(True)
    ctx.timer_start()
    run(b)
    wall = ctx.timer_stop()
    kern, _ = ctx.profile_get()
    ctx.profile_enable(False)
    return kern, wall


for name, cols, variants in cases:
    b = ctx.upload(cols)
    for _, run in variants:
        once(run, b)  # warm-up
    t = {label: ([], []) for label, _ in variants}
    for _ in range(ROUNDS):
        for label, run in variants:
            kern, wall = once(run, b)
            t[label][0].append(kern)
            t[label][1].append(wall)
    for label, _ in variants:
        kern, wall = t[label]
        print("%-11s %-15s kernel %8.3f ms (min %.3f, max %.3f)  call %8.3f ms (min %.3f, max %.3f)  median of %d" %
              (name, label, np.median(kern), min(kern), max(kern), np.median(wall), min(wall), max(wall), ROUNDS))
    b.free()
ctx.close()
