"""Utf8 predicate pre-pass (utf8_predicate.cu) on 1e8-row Utf8 columns in HBM.

Columns (seeded): "city" strings of 8-24 bytes built from a small set of shared prefixes and suffixes, and "exact", a set in
which about a third of the strings have the literal's length.  For `= 'lit'`, `< 'lit'`, `LIKE 'abc%'`, `LIKE '%abc%'` and
a general pattern it reports the pre-pass kernel's time (torch.profiler device time of the k_utf8_* launch, median over
the timed repetitions after warm-up), the selectivity, algorithmic bytes/s and the fraction of the H100 SXM data-sheet
3.35 TB/s.  Algorithmic bytes = 4*(n+1) offsets + the column's string bytes + n/8 output bits; a predicate that decides a
row on its length alone still counts the row's bytes.  It also times the whole dfgpu_filter_project call (CUDA events)
for `SELECT lat WHERE city LIKE ...` against `SELECT lat WHERE lat > x` at the same row count.

    python profiles/microbench_utf8_pred.py [--rows 100000000] [--reps 20]
"""
import argparse
import json
import statistics
import subprocess
import sys
import os

import numpy as np
import pyarrow as pa

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from datafusion_archive_b200 import engine  # noqa: E402
from datafusion_archive_b200.expr import col, lit  # noqa: E402

PEAK = 3.35e12


def make_strings(n, seed, exact):
    rng = np.random.default_rng(seed)
    heads = [b"Elgin, ", b"Leeds, ", b"London, ", b"Perth, ", b"Lee", b"Le", b"abcd", b"Xyz"]
    tails = [b"Scotland", b"the UK", b"UK", b"Wales", b"abc", b"x"]
    hi, ti = rng.integers(0, len(heads), n), rng.integers(0, len(tails), n)
    if exact:
        lens = np.where(rng.random(n) < 0.33, 12, rng.integers(8, 25, n))
    else:
        lens = rng.integers(8, 25, n)
    offs = np.zeros(n + 1, np.int64)
    np.cumsum(lens, out=offs[1:])
    data = np.frombuffer(rng.integers(97, 123, int(offs[-1]), dtype=np.uint8).tobytes(), np.uint8).copy()
    # write the head at the start and the tail at the end of each string (truncated to the string's length)
    for h in range(len(heads)):
        rows = np.nonzero(hi == h)[0]
        for j, ch in enumerate(heads[h]):
            r = rows[lens[rows] > j]
            data[offs[r] + j] = ch
    for t in range(len(tails)):
        rows = np.nonzero(ti == t)[0]
        tb = tails[t]
        for j, ch in enumerate(tb):
            r = rows[lens[rows] > len(tb) + 8]
            data[offs[r + 1] - len(tb) + j] = ch
    return pa.BinaryArray.from_buffers(pa.binary(), n, [None, pa.py_buffer(offs.astype(np.int32).tobytes()), pa.py_buffer(data.tobytes())]), int(offs[-1])


def kernel_ms(fn, reps):
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    times = [e.device_time for e in prof.events() if e.name.startswith("void dfgpu::") and "k_utf8_" in e.name]
    if not times:
        times = [e.device_time for e in prof.events() if "k_utf8_" in e.name]
    return statistics.median(times) / 1e3 if times else float("nan")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    n = a.rows
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": smi, "rows": n}))
    ctx = engine.GpuContext(0)
    lat = np.random.default_rng(3).random(n)
    for colname, exact in [("city", False), ("exact", True)]:
        arr, nbytes = make_strings(n, 1 if not exact else 2, exact)
        b = ctx.upload([arr, lat])
        algo = 4 * (n + 1) + nbytes + n / 8
        cases = [("= 'Leeds, abcxy'", col(0).eq(lit(b"Leeds, abcxy"))), ("< 'Lee'", col(0) < lit(b"Lee")),
                 ("LIKE 'Lee%'", col(0).like(lit(b"Lee%"))), ("LIKE '%Scotland%'", col(0).like(lit(b"%Scotland%"))),
                 ("LIKE 'L_e%a%UK'", col(0).like(lit(b"L_e%a%UK")))]
        for name, e in cases:
            def run():
                r = ctx.filter_project(b, None, [e])
                r.free()
            ms = kernel_ms(run, a.reps)
            r = ctx.filter_project(b, None, [e])
            (bits,) = r.columns()
            r.free()
            sel = float(np.count_nonzero(bits)) / n
            print(json.dumps({"column": colname, "predicate": name, "kernel_ms": round(ms, 4), "selectivity": round(sel, 4),
                              "GB_per_s": round(algo / (ms / 1e3) / 1e9, 1), "frac_peak": round(algo / (ms / 1e3) / PEAK, 3)}))
        if not exact:
            # whole operator: SELECT lat WHERE city LIKE ... against SELECT lat WHERE lat > x
            for name, pred in [("WHERE city LIKE '%Scotland%'", col(0).like(lit(b"%Scotland%"))), ("WHERE lat > 0.8", col(1) > 0.8)]:
                ts = []
                for i in range(a.reps + 3):
                    ctx.timer_start()
                    r = ctx.filter_project(b, pred, [col(1)])
                    t = ctx.timer_stop()
                    r.free()
                    if i >= 3:
                        ts.append(t)
                print(json.dumps({"query": "SELECT lat " + name, "filter_project_ms": round(statistics.median(ts), 3)}))
        b.free()
    ctx.close()


if __name__ == "__main__":
    main()
