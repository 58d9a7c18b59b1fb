"""Utf8 functions (utf8_function.cu) on a 1e8-row Utf8 column of 8-24-byte strings in HBM, built as in
microbench_utf8_pred.py.

For `WHERE length(s) > 16`, `SELECT upper(s) WHERE x > 0.5` and `WHERE lower(s) LIKE 'abc%'` it reports the whole
dfgpu_filter_project call (CUDA events, median over the timed repetitions after warm-up), the device time of the
k_utf8_view_* launches (torch.profiler), the selectivity, and algorithmic bytes/s as a fraction of the H100 SXM
data-sheet 3.35 TB/s.  Algorithmic bytes of the view kernels: 4*(n+1) offsets + the string bytes read + what they write
(8 bytes per row for a length; for a Utf8 result, the selected rows' offsets and bytes).

    python profiles/microbench_utf8_fn.py [--rows 100000000] [--reps 10]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from datafusion_archive_b200 import engine  # noqa: E402
from datafusion_archive_b200.expr import col, lit, utf8_fn  # noqa: E402
from microbench_utf8_pred import make_strings  # noqa: E402

PEAK = 3.35e12


def view_ms(fn, reps):
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    per = [e.device_time for e in prof.events() if "k_utf8_" in e.name]
    return sum(per) / reps / 1e3 if per else float("nan")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    n = a.rows
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": smi, "rows": n}))
    ctx = engine.GpuContext(0)
    arr, nbytes = make_strings(n, 1, False)
    x = np.random.default_rng(3).random(n)
    ids = np.arange(n, dtype=np.int64)
    b = ctx.upload([arr, x, ids])
    cases = [("SELECT id WHERE length(s) > 16", utf8_fn("length", col(0)) > lit(16), [col(2)]),
             ("SELECT upper(s) WHERE x > 0.5", col(1) > lit(0.5), [utf8_fn("upper", col(0))]),
             ("SELECT id WHERE lower(s) LIKE 'abc%'", utf8_fn("lower", col(0)).like(lit(b"abc%")), [col(2)])]
    for name, pred, proj in cases:
        def run():
            r = ctx.filter_project(b, pred, proj)
            r.free()
        ts = []
        for i in range(a.reps + 2):
            ctx.timer_start()
            r = ctx.filter_project(b, pred, proj)
            t = ctx.timer_stop()
            if i == 0:
                nsel = r.nrows
            r.free()
            if i >= 2:
                ts.append(t)
        ms = view_ms(run, a.reps)
        sel = nsel / n
        if "upper" in name:  # the selected rows' offsets, bytes and row numbers in, their offsets and bytes out
            algo = 2 * (4 + 8) * nsel + 2 * nbytes * sel + 8 * nsel
        elif "lower" in name:  # every row's view: offsets and bytes in, offsets, begins and bytes out
            algo = 4 * (n + 1) + 2 * nbytes + 8 * n
        else:
            algo = 4 * (n + 1) + nbytes + 8 * n
        print(json.dumps({"query": name, "filter_project_ms": round(statistics.median(ts), 3), "view_kernels_ms": round(ms, 3),
                          "selectivity": round(sel, 4), "frac_peak": round(algo / (ms / 1e3) / PEAK, 3)}))
    b.free()
    ctx.close()


if __name__ == "__main__":
    main()
