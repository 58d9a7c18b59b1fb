"""Inner equi-join (join.cu): kernel time of dfgpu_join_build and dfgpu_join_probe, from the CUDA events recorded around
every join launch (dfgpu_profile_*), median over the timed repetitions after one warm-up.

Cases: a 1e8-row probe (Int64 key, Float64 payload) against unique-key builds of 1e3, 1e6 and 1e7 rows (Int64 key,
Float64 payload), at 100 % and 10 % match rates; the output is both payloads.  Then the skewed build: one key repeated
4 Mi times, probed by 4 rows of which 2 match (8 Mi output rows), against 4 Mi unique keys probed once each.

Algorithmic bytes: the keys read (8 per probe row; 8 per build row for the build), plus the output columns written
(16 per output row), plus their source values read (16 per output row).  Fraction of the H100 SXM data-sheet 3.35 TB/s.

    python profiles/microbench_join.py [--probe-rows 100000000] [--reps 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from datafusion_archive_b200 import engine  # noqa: E402
from datafusion_archive_b200.expr import col  # noqa: E402

PEAK = 3.35e12


def timed(ctx, fn, reps):
    """(median kernel ms, last result) of fn() over `reps` runs after a warm-up; fn returns an object with .free()"""
    fn().free()
    ms, out = [], None
    for i in range(reps):
        ctx.profile_enable(True)
        out = fn()
        ms.append(ctx.profile_get()[0])
        ctx.profile_enable(False)
        if i < reps - 1:
            out.free()
    return statistics.median(ms), out


def case(ctx, name, bkeys, pkeys, reps):
    bb = ctx.upload([bkeys, np.ones(len(bkeys))])
    pb = ctx.upload([pkeys, np.ones(len(pkeys))])
    build_ms, j = timed(ctx, lambda: ctx.join_build(bb, [col(0)], keep_cols=[1]), reps)
    probe_ms, r = timed(ctx, lambda: j.probe(pb, [col(0)], probe_cols=[1], build_cols=[1]), reps)
    m = r.nrows
    r.free(); j.free(); bb.free(); pb.free()
    probe_bytes = 8 * len(pkeys) + 32 * m
    print(json.dumps({"case": name, "build_rows": len(bkeys), "probe_rows": len(pkeys), "output_rows": m,
                      "build_ms": round(build_ms, 3), "build_rows_per_s": round(len(bkeys) / (build_ms / 1e3)),
                      "build_frac_peak": round(8 * len(bkeys) / (build_ms / 1e3) / PEAK, 3),
                      "probe_ms": round(probe_ms, 3), "probe_rows_per_s": round(len(pkeys) / (probe_ms / 1e3)),
                      "probe_frac_peak": round(probe_bytes / (probe_ms / 1e3) / PEAK, 3)}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--probe-rows", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": smi, "probe_rows": a.probe_rows}), flush=True)
    ctx = engine.GpuContext(0)
    rng = np.random.default_rng(5)
    for b in (1_000, 1_000_000, 10_000_000):
        bkeys = rng.permutation(b).astype(np.int64)
        for rate in (1.0, 0.1):
            pkeys = rng.integers(0, int(b / rate), a.probe_rows, dtype=np.int64)
            case(ctx, "unique build %d, match %d%%" % (b, round(rate * 100)), bkeys, pkeys, a.reps)
    n = 4 << 20
    case(ctx, "skewed build: one key x 4Mi, 2 of 4 probe rows match", np.full(n, 7, np.int64), np.array([7, 8, 7, 1], np.int64), a.reps)
    case(ctx, "uniform: 4Mi unique keys, each probed once", np.arange(n, dtype=np.int64), rng.permutation(n).astype(np.int64), a.reps)
    ctx.close()


if __name__ == "__main__":
    main()
