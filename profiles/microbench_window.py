#!/usr/bin/env python
"""What window functions cost, on a resident batch of an Int64 key k with P distinct values and a Float64 v.
  (a) dfgpu_sort by (k, v): the baseline
  (b) ROW_NUMBER + SUM(v) + MIN(v) + AVG(v) OVER (PARTITION BY k ORDER BY v): one dfgpu_window call
  (c) SUM(v) OVER (PARTITION BY k): one dfgpu_window call
  (d) SELECT k, SUM(v) OVER (PARTITION BY k) FROM t end to end through ExecutionContext.sql() from host buffers: the
      host concatenation, the upload, (c), the download and the projection's extra round trip of its input columns
For (a)-(c): the CUDA time of each kernel from torch.profiler (median over the rounds of the per-round sum per kernel
name), and for the post-sort kernels the bytes a simple model says they move (each array read or written once,
random accesses counted at their element size) over their time.  Prints the card name and power limit read in the same
run.
usage: microbench_window.py [max_rows]"""
import os
import re
import subprocess
import sys
import time
from collections import defaultdict

import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from datafusion_archive_b200 import _abi as A  # noqa: E402
from datafusion_archive_b200 import engine, host  # noqa: E402
from datafusion_archive_b200.expr import col  # noqa: E402

max_rows = int(float(sys.argv[1])) if len(sys.argv) > 1 else 100_000_000
ROUNDS = 3
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print("card: %s" % (card.splitlines()[0] if card else "unknown"))
ctx = engine.GpuContext(0)
torch.cuda.init()


def short(name):
    m = re.search(r"(k_[a-z0-9_]+)", name)
    return m.group(1) if m else name[:30]


def kernel_times(fn):
    """{kernel: median ms per round} and the median wall ms of fn()"""
    per = defaultdict(list)
    walls = []
    for _ in range(ROUNDS):
        ctx.sync()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            t0 = time.perf_counter()
            fn()
            ctx.sync()
            walls.append((time.perf_counter() - t0) * 1e3)
        acc = defaultdict(float)
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in e.name and "Memset" not in e.name:
                acc[short(e.name)] += e.device_time_total / 1e3
        for k, v in acc.items():
            per[k].append(v)
    return {k: float(np.median(v)) for k, v in per.items()}, float(np.median(walls))


def model_bytes(n, G, nfn_scan, nfn_out):
    """bytes per post-sort kernel (summed over calls): 4-byte row ids, flags and numbers, 8-byte keys and values"""
    return {
        "k_win_flags": n * (4 + 2 * 2 * 8 + 8),       # perm, two rows of two 8-byte keys, two flag words
        "k_win_bounds": n * (4 + 8 + 16 + 4) + 8 * G,  # perm, flags, numbers read + written, inverse, first positions
        "k_win_tile_reduce": nfn_scan * n * (4 + 8 + 4),
        "k_win_tile_scan": nfn_scan * (n * (4 + 8 + 4 + 4 + 4) + 12 * G),
        "k_win_out": nfn_out * n * (4 + 4 + 4 + 12 + 8 + 1 / 8),
    }


def report(label, times, wall, mb=None):
    total = sum(times.values())
    print("  %s: wall %.2f ms, kernels %.2f ms" % (label, wall, total))
    for k in sorted(times, key=lambda k: -times[k]):
        extra = ""
        if mb and k in mb:
            extra = "  model %.2f GB, %.0f GB/s" % (mb[k] / 1e9, mb[k] / 1e9 / (times[k] / 1e3))
        print("    %-20s %8.3f ms%s" % (k, times[k], extra))
    return total


for n in [10_000_000, 100_000_000]:
    if n > max_rows:
        continue
    for P in [100, 100_000, 10_000_000]:
        rng = np.random.default_rng(1)
        k = rng.integers(0, P, n)
        v = rng.standard_normal(n)
        b = ctx.upload([k, v])
        print("n=%d P=%d" % (n, P))
        ta, wa = kernel_times(lambda: ctx.sort(b, keys=[col(0), col(1)]).free())
        a = report("(a) sort by (k, v)", ta, wa)
        fb = [(A.WIN_ROW_NUMBER, None, 0), (A.AGG_SUM, col(1), 0), (A.AGG_MIN, col(1), 0), (A.AGG_AVG, col(1), 0)]
        tb, wb = kernel_times(lambda: ctx.window(b, fb, partition=[col(0)], order=[col(1)]).free())
        G = n  # a continuous v: every row its own peer group
        bb = report("(b) ROW_NUMBER+SUM+MIN+AVG OVER (PARTITION BY k ORDER BY v)", tb, wb, model_bytes(n, G, 3, 4))
        print("    (b) - (a): %.2f ms (%.0f%% of (a))" % (bb - a, 100 * (bb - a) / a))
        tc, wc = kernel_times(lambda: ctx.window(b, [(A.AGG_SUM, col(1), 0)], partition=[col(0)]).free())
        report("(c) SUM(v) OVER (PARTITION BY k)", tc, wc, model_bytes(n, min(P, n), 1, 1))
        b.free()
        sql = host.ExecutionContext(0)
        walls = []
        for _ in range(2 if n > 10_000_000 else ROUNDS):
            sql.register_memory("t", [("k", k), ("v", v)])
            t0 = time.perf_counter()
            out = sql.sql("SELECT k, SUM(v) OVER (PARTITION BY k) FROM t").collect()
            walls.append((time.perf_counter() - t0) * 1e3)
            del out
        sql.close()
        print("  (d) SELECT k, SUM(v) OVER (PARTITION BY k) FROM t via sql(): %.1f ms (median of %d)" % (float(np.median(walls)), len(walls)))
ctx.close()
