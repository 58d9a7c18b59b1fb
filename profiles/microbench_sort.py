#!/usr/bin/env python
"""What ORDER BY / LIMIT costs.
  (a) dfgpu_sort alone over a resident batch, at 1e6 / 1e7 / 1e8 rows, for three key sets:
        i64       one Int64 key, uniform over the whole range (8 live digits)
        f64+i64   Float64 DESC (standard normal), then an Int64 tie-break uniform in [0, 1e6)
        utf8      one Utf8 key of 8 to 24 random lower-case bytes (1e6 and 1e7 rows only: the strings are built on the host)
      Reported: the summed time of the sort's kernels (dfgpu_profile_*: every sort kernel and its scans and gathers), the
      median over 5 rounds; the live passes (digits not constant over all rows, computed here from the same encoding);
      the bytes those passes move (count: key read; scatter: key + row id read and written) plus the encode sweeps and
      the final gather of the key and a row-number payload; and that traffic over the data sheet's HBM bandwidth
      (3.35 TB/s) per kernel time, named as such.
  (b) the C5 shape (1e6 groups over min(1.25e8, max_rows) rows, SELECT k, MIN(v), MAX(v), SUM(v) .. GROUP BY k), end to end from host
      buffers, with and without ORDER BY SUM(v) DESC LIMIT 10 (dfgpu_sort of the aggregate's device result, the GROUP BY
      key as the tie-break), alternated over 5 rounds; the median of each and the difference.
Prints the card name and power limit read in the same run.
usage: microbench_sort.py [max_rows]"""
import os
import subprocess
import sys
import time

import numpy as np
import pyarrow as pa

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from datafusion_archive_b200 import engine, workloads  # noqa: E402
from datafusion_archive_b200 import _abi as A  # noqa: E402
from datafusion_archive_b200.expr import col  # noqa: E402

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import sort_ref as R  # noqa: E402

max_rows = int(float(sys.argv[1])) if len(sys.argv) > 1 else 100_000_000
ROUNDS = 5
HBM = 3.35e12
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print("card: %s" % (card.splitlines()[0] if card else "unknown"))
ctx = engine.GpuContext(0)


def live_digits(enc, width):
    if len(enc) == 0:
        return 0
    v = np.bitwise_or.reduce(enc) ^ np.bitwise_and.reduce(enc)
    return sum(1 for d in range(width) if (int(v) >> (8 * d)) & 255)


def utf8_column(rng, n):
    lens = rng.integers(8, 25, n).astype(np.int32)
    offs = np.zeros(n + 1, np.int32)
    np.cumsum(lens, out=offs[1:])
    data = rng.integers(97, 123, int(offs[-1]), dtype=np.uint8)
    return pa.StringArray.from_buffers(n, pa.py_buffer(offs), pa.py_buffer(data)), offs, data


def sort_case(name, n, rng):
    """(arrays, keys, desc, traffic bytes)"""
    m = n
    if name == "i64":
        k = rng.integers(-(1 << 63), (1 << 63) - 1, n, dtype=np.int64, endpoint=True)
        p = live_digits(R.encode(A.INT64, k), 8)
        traffic = (m * 4 + m * 8 + m * 8) + p * (m * 8 + 2 * m * 12)
        return [k, np.arange(n, dtype=np.int64)], [col(0)], [False], traffic, p
    if name == "f64+i64":
        f = rng.standard_normal(n)
        t = rng.integers(0, 1_000_000, n, dtype=np.int64)
        p1, p2 = live_digits(R.encode(A.FLOAT64, f), 8), live_digits(R.encode(A.INT64, t), 8)
        traffic = 2 * (m * 4 + m * 8 + m * 8) + (p1 + p2) * (m * 8 + 2 * m * 12)
        return [f, t, np.arange(n, dtype=np.int64)], [col(0), col(1)], [True, False], traffic, p1 + p2
    arr, offs, data = utf8_column(rng, n)
    # not computed: the rank's MSD rounds and their passes depend on the ties in the data
    traffic = None
    return [arr, np.arange(n, dtype=np.int64)], [col(0)], [False], traffic, None


print("(a) dfgpu_sort, kernel time (median of %d)" % ROUNDS)
print("%-8s %12s %10s %8s %14s %10s" % ("keys", "rows", "ms", "passes", "pass bytes", "HBM share"))
for name in ("i64", "f64+i64", "utf8"):
    for n in (1_000_000, 10_000_000, 100_000_000):
        if n > max_rows or (name == "utf8" and n > 10_000_000):
            continue
        rng = np.random.default_rng(n)
        arrays, keys, desc, traffic, passes = sort_case(name, n, rng)
        b = ctx.upload(arrays)
        ctx.sort(b, keys=keys, desc=desc).free()  # warm-up
        times = []
        for _ in range(ROUNDS):
            ctx.profile_enable(True)
            ctx.sort(b, keys=keys, desc=desc).free()
            ms, _ = ctx.profile_get()
            times.append(ms)
        ctx.profile_enable(False)
        b.free()
        ms = float(np.median(times))
        share = "%.1f%%" % (100 * traffic / HBM / (ms * 1e-3)) if traffic else "n/a"
        print("%-8s %12d %10.3f %8s %14s %10s" % (name, n, ms, passes if passes is not None else "-", traffic if traffic else "-", share), flush=True)

print("(b) C5 shape end to end, with and without ORDER BY SUM(v) DESC LIMIT 10")
n5 = min(125_000_000, max_rows)
arrays, gkeys, aggs, _ = workloads.c5(n5)
host_arrays = []
for a in arrays:
    pb = engine.PinnedBuffer(a.shape, a.dtype)
    pb.array[:] = a
    host_arrays.append(pb)
cols = [p.array for p in host_arrays]


def plain():
    r = ctx.aggregate_host(cols, gkeys, aggs)
    r.free()


def top10():
    r = ctx.aggregate_host(cols, gkeys, aggs)
    s = ctx.sort(r, keys=[col(3), col(0)], desc=[True, False], limit=10)
    s.free()
    r.free()


for f in (plain, top10):
    f()
t = {plain: [], top10: []}
for _ in range(ROUNDS):
    for f in (plain, top10):
        ctx.sync()
        t0 = time.perf_counter()
        f()
        ctx.sync()
        t[f].append((time.perf_counter() - t0) * 1e3)
mp, mt = float(np.median(t[plain])), float(np.median(t[top10]))
print("rows %d: GROUP BY %.2f ms, + ORDER BY .. LIMIT 10 %.2f ms, difference %.2f ms (%.1f%%)" % (n5, mp, mt, mt - mp, 100 * (mt - mp) / mp))
print("  spread: GROUP BY %.2f-%.2f ms, with the clause %.2f-%.2f ms" % (min(t[plain]), max(t[plain]), min(t[top10]), max(t[top10])))
ctx.close()
