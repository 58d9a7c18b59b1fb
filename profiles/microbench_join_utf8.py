"""Inner equi-join on a Utf8 key (join.cu, k_join_utf8_*): kernel time of dfgpu_join_build and dfgpu_join_probe, from
the CUDA events recorded around every join launch (dfgpu_profile_*), median over the timed repetitions after one
warm-up — the method of microbench_join.py, whose Int64-key cases run first in the same process as the baseline.

Cases: a 1e8-row probe (Utf8 key of 8 to 24 bytes, Float64 payload) against builds of 1e3, 1e6 and 1e7 distinct
strings (Float64 payload), at 100 % and 10 % match rates; the output is both payloads.  Then the skewed build: one
string repeated 4 Mi times, probed by 4 rows of which 2 match (8 Mi output rows), against 4 Mi distinct strings probed
once each.  String i is its number in base 26 (6 letters) followed by letters that depend on i, 8 + (i mod 17) bytes
in all, so equal numbers give equal strings and a probe number past the build's count misses.

Algorithmic bytes: per probe row its 4-byte offset and its string's bytes (per build row the same for the build), plus
per output row the payloads read and written (32 bytes).  Fraction of the H100 SXM data-sheet 3.35 TB/s.

    python profiles/microbench_join_utf8.py [--probe-rows 100000000] [--reps 5] [--no-baseline]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import pyarrow as pa

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from datafusion_archive_b200 import engine  # noqa: E402
from datafusion_archive_b200.expr import col  # noqa: E402
import microbench_join as base  # noqa: E402

PEAK = base.PEAK
HI = 24


def strings(ids, chunk=10_000_000):
    """the Utf8 array of string number ids[i], built a chunk at a time"""
    ids = np.asarray(ids, np.int64)
    lens = (8 + ids % 17).astype(np.int32)
    off = np.zeros(len(ids) + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    if off[-1] >= 1 << 31:
        raise ValueError("more than 2 GiB of strings")
    data = np.empty(int(off[-1]), np.uint8)
    pos = np.arange(HI, dtype=np.uint8)
    step = (pos.astype(np.int64) * 7 % 26).astype(np.uint8)
    for c0 in range(0, len(ids), chunk):
        i = ids[c0:c0 + chunk]
        mat = np.empty((len(i), HI), np.uint8)
        mat[:, 6:] = 97 + ((i * 31 % 26).astype(np.uint8)[:, None] + step[None, 6:]) % 26
        for d in range(6):
            mat[:, d] = 97 + (i // 26 ** d) % 26
        data[off[c0]:off[c0 + len(i)]] = mat[pos[None, :] < lens[c0:c0 + chunk, None]]
    return pa.StringArray.from_buffers(len(ids), pa.py_buffer(off.astype(np.int32)), pa.py_buffer(data))


def case(ctx, name, bkeys, pkeys, reps):
    bb = ctx.upload([bkeys, np.ones(len(bkeys))])
    pb = ctx.upload([pkeys, np.ones(len(pkeys))])
    build_ms, j = base.timed(ctx, lambda: ctx.join_build(bb, [col(0)], keep_cols=[1]), reps)
    probe_ms, r = base.timed(ctx, lambda: j.probe(pb, [col(0)], probe_cols=[1], build_cols=[1]), reps)
    m = r.nrows
    r.free(); j.free(); bb.free(); pb.free()
    build_bytes = 4 * len(bkeys) + len(bkeys.buffers()[2])
    probe_bytes = 4 * len(pkeys) + len(pkeys.buffers()[2]) + 32 * m
    print(json.dumps({"case": name, "key": "utf8", "build_rows": len(bkeys), "probe_rows": len(pkeys), "output_rows": m,
                      "build_ms": round(build_ms, 3), "build_rows_per_s": round(len(bkeys) / (build_ms / 1e3)),
                      "build_frac_peak": round(build_bytes / (build_ms / 1e3) / PEAK, 3),
                      "probe_ms": round(probe_ms, 3), "probe_rows_per_s": round(len(pkeys) / (probe_ms / 1e3)),
                      "probe_frac_peak": round(probe_bytes / (probe_ms / 1e3) / PEAK, 3)}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--probe-rows", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-baseline", action="store_true", help="skip the Int64-key cases of microbench_join.py")
    a = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": smi, "probe_rows": a.probe_rows}), flush=True)
    ctx = engine.GpuContext(0)
    rng = np.random.default_rng(5)
    sizes = (1_000, 1_000_000, 10_000_000)
    if not a.no_baseline:
        for b in sizes:
            bkeys = rng.permutation(b).astype(np.int64)
            for rate in (1.0, 0.1):
                pkeys = rng.integers(0, int(b / rate), a.probe_rows, dtype=np.int64)
                base.case(ctx, "int64: unique build %d, match %d%%" % (b, round(rate * 100)), bkeys, pkeys, a.reps)
    for b in sizes:
        bkeys = strings(rng.permutation(b))
        for rate in (1.0, 0.1):
            pkeys = strings(rng.integers(0, int(b / rate), a.probe_rows))
            case(ctx, "utf8: distinct build %d, match %d%%" % (b, round(rate * 100)), bkeys, pkeys, a.reps)
            del pkeys
    n = 4 << 20
    case(ctx, "utf8 skewed build: one string x 4Mi, 2 of 4 probe rows match", strings(np.full(n, 7)), strings([7, 8, 7, 1]), a.reps)
    case(ctx, "utf8 uniform: 4Mi distinct strings, each probed once", strings(np.arange(n)), strings(rng.permutation(n)), a.reps)
    ctx.close()


if __name__ == "__main__":
    main()
