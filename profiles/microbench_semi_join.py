"""Semi / anti join (join.cu): kernel time of dfgpu_join_semi against dfgpu_join_probe on the same data, from the CUDA
events recorded around every join launch (dfgpu_profile_*), median over the timed repetitions after one warm-up.

Cases: a 1e8-row probe (Int64 key, Float64 payload) against unique-key builds of 1e3, 1e6 and 1e7 rows (Int64 key),
for a semi and an anti join at 100 % and 10 % pass rates (a semi join passes the matching rows, an anti join the
others).  Both operators output the probe payload only, so the inner probe is timed without a build column.

Algorithmic bytes: the key read (8 per probe row), plus the payload read and written (16 per output row).  Fraction of
the H100 SXM data-sheet 3.35 TB/s.

    python profiles/microbench_semi_join.py [--probe-rows 100000000] [--reps 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from datafusion_archive_b200 import _abi as A  # noqa: E402
from datafusion_archive_b200 import engine  # noqa: E402
from datafusion_archive_b200.expr import col  # noqa: E402

PEAK = 3.35e12


def timed(ctx, fn, reps):
    """(median kernel ms, output rows) of fn() over `reps` runs after a warm-up; fn returns a result"""
    fn().free()
    ms, rows = [], 0
    for _ in range(reps):
        ctx.profile_enable(True)
        r = fn()
        ms.append(ctx.profile_get()[0])
        ctx.profile_enable(False)
        rows = r.nrows
        r.free()
    return statistics.median(ms), rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--probe-rows", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": smi, "probe_rows": a.probe_rows}), flush=True)
    ctx = engine.GpuContext(0)
    rng = np.random.default_rng(5)
    pay = np.ones(a.probe_rows)
    for b in (1_000, 1_000_000, 10_000_000):
        bb = ctx.upload([rng.permutation(b).astype(np.int64)])
        j = ctx.join_build(bb, [col(0)], keep_cols=[])
        bb.free()
        for kind, name in ((A.JOIN_SEMI, "semi"), (A.JOIN_ANTI, "anti")):
            for rate in (1.0, 0.1):
                match = rate if kind == A.JOIN_SEMI else 1.0 - rate
                pkeys = rng.integers(0, int(b / match), a.probe_rows, dtype=np.int64) if match > 0 else \
                    rng.integers(b, 2 * b, a.probe_rows, dtype=np.int64)
                pb = ctx.upload([pkeys, pay])
                semi_ms, m = timed(ctx, lambda: j.semi(pb, [col(0)], kind, probe_cols=[1]), a.reps)
                probe_ms, pm = timed(ctx, lambda: j.probe(pb, [col(0)], probe_cols=[1], build_cols=[]), a.reps)
                pb.free()
                print(json.dumps({"case": "%s, build %d, pass %d%%" % (name, b, round(rate * 100)), "build_rows": b, "probe_rows": a.probe_rows,
                                  "output_rows": m, "semi_ms": round(semi_ms, 3),
                                  "semi_frac_peak": round((8 * a.probe_rows + 16 * m) / (semi_ms / 1e3) / PEAK, 3),
                                  "inner_probe_rows": pm, "inner_probe_ms": round(probe_ms, 3),
                                  "inner_probe_frac_peak": round((8 * a.probe_rows + 16 * pm) / (probe_ms / 1e3) / PEAK, 3)}), flush=True)
        j.free()
    ctx.close()


if __name__ == "__main__":
    main()
