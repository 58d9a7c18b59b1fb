#!/usr/bin/env python
"""What CASE costs, 1e8 rows resident in HBM:
  project  SELECT CASE WHEN x > 0.5 THEN x ELSE 0.0 END FROM t   against SELECT x FROM t          (x ~ U[0,1) f64)
  group    SELECT k, SUM(CASE WHEN v > 0.5 THEN v ELSE 0.0 END) ... GROUP BY k
           against SELECT k, SUM(v) ... WHERE v > 0.5 GROUP BY k                                  (the C4 data)
  wide     SELECT k, j, SUM(sqrt(v)) ... GROUP BY k, j: a function under a two-Int64-key GROUP BY, the wide-key
           interpreter kernel (k_hash_agg_wide<kFnDepth>); runs on libraries without CASE too, for an A/B via DFGPU_LIB
Variants of a case alternate, 7 rounds each; reported per variant: the summed time of the scan kernels
(dfgpu_profile_*, the kernel events bench.py uses) and of the whole call (CUDA events), each the median over the rounds,
and the share of the data sheet's HBM bandwidth (3.35 TB/s) that the algorithmic bytes (every input column read once,
every output column written once) over the kernel time come to.  Prints the card name and power limit read in the
same run.  With a library that has no CASE (DFGPU_LIB), the CASE variants are skipped.
usage: microbench_case.py [rows]"""
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from datafusion_archive_b200 import engine, workloads  # noqa: E402
from datafusion_archive_b200.expr import AggregateFunction, case, col, fn  # noqa: E402

n = int(float(sys.argv[1])) if len(sys.argv) > 1 else 100_000_000
ROUNDS = 7
HBM = 3.35e12
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print("card: %s" % (card.splitlines()[0] if card else "unknown"))
print("library: %s" % (os.environ.get("DFGPU_LIB") or "the tree's build"))
ctx = engine.GpuContext(0)
x = np.random.default_rng(48).random(n)
arrays, keys, _, _ = workloads.c4(n)
j = np.random.default_rng(49).integers(0, 4, n, dtype=np.int64)


def project(e, pred=None):
    return lambda b: ctx.filter_project(b, pred, [e]).free()


def group(ks, arg, pred=None):
    return lambda b: ctx.aggregate(b, ks, [AggregateFunction("sum", arg)], pred=pred).free()


def has_case():
    b = ctx.upload([x[:64]])
    try:
        ctx.filter_project(b, None, [case([(col(0) > 0.5, col(0))], 0.0)]).free()
        return True
    except engine.DfGpuError:
        return False
    finally:
        b.free()


CASE = has_case()
proj_bytes = 16.0 * n  # x read, one Float64 output written (all n rows)
group_bytes = 16.0 * n  # k and v read; the table is L2-resident
cases = [("project", [x], proj_bytes, [("SELECT x", project(col(0)), True),
                                       ("CASE WHEN x > 0.5 THEN x ELSE 0.0 END", project(case([(col(0) > 0.5, col(0))], 0.0)), False)]),
         ("GROUP BY k", arrays, group_bytes, [("SUM(v) WHERE v > 0.5", group(keys, col(1), col(1) > 0.5), True),
                                               ("SUM(CASE WHEN v > 0.5 THEN v ELSE 0.0 END)",
                                                group(keys, case([(col(1) > 0.5, col(1))], 0.0)), False)]),
         ("GROUP BY k, j", arrays + [j], 24.0 * n, [("SUM(sqrt(v))", group([col(0), col(2)], fn("sqrt", col(1))), True)])]


def once(run, b):
    ctx.profile_enable(True)
    ctx.timer_start()
    run(b)
    wall = ctx.timer_stop()
    kern, _ = ctx.profile_get()
    ctx.profile_enable(False)
    return kern, wall


for name, cols, nbytes, variants in cases:
    variants = [(label, run) for label, run, any_lib in variants if any_lib or CASE]
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
        k = float(np.median(kern))
        print("%-13s %-42s kernel %8.3f ms (min %.3f, max %.3f)  call %8.3f ms  HBM %5.1f %%  median of %d" %
              (name, label, k, min(kern), max(kern), np.median(wall), 100.0 * nbytes / (k * 1e-3) / HBM, ROUNDS))
    b.free()
if not CASE:
    print("this library has no CASE: CASE variants skipped")
ctx.close()
