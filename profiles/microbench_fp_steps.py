#!/usr/bin/env python
"""Step time against kernel time of the filter/project operator, C2 and C3 shapes, data resident in HBM.

A step is one whole dfgpu_filter_project call, timed over K back-to-back calls with CUDA events (each step frees the
previous step's result, as bench.py does); the kernel is timed with the events dfgpu_profile_* records around each
launch.  step - kernel is the time per step the GPU spends outside the kernel.

  microbench_fp_steps.py [--rows N] [--steps K] [--warmup W]
      one run of the library engine.lib_path() names (DFGPU_LIB selects another build); prints one JSON line
  microbench_fp_steps.py --ab LIB_A LIB_B [--rounds R] [--rows N] [--steps K] [--warmup W]
      R rounds of each library, alternating A, B, A, B, ... in separate processes; prints the median and the range
      of every number per library, with the card's name and power limit
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def one_run(args):
    from datafusion_archive_b200 import engine, workloads
    ctx = engine.GpuContext(0)
    out = {"lib": engine.lib_path(), "rows": args.rows, "steps": args.steps}
    a2, pred2, proj2 = workloads.c2(args.rows, seed=42)
    a3, pred3, proj3 = workloads.c3(args.rows, seed=142)
    shapes = {"c2": (a2, pred2, proj2, int(np.count_nonzero(a2[0] > 0.5))),
              "c3": (a3[:2], pred3, proj3, int(np.count_nonzero(a3[1] < a3[0])))}
    for name, (arrays, pred, proj, nsel) in shapes.items():
        batch = ctx.upload(arrays)
        held = [None]

        def step():
            r = ctx.filter_project(batch, pred, proj)
            if held[0] is not None:
                held[0].free()
            held[0] = r
        for _ in range(args.warmup):
            step()
        ctx.sync()
        ctx.profile_enable(True)
        ctx.timer_start()
        for _ in range(args.steps):
            step()
        ms = ctx.timer_stop()
        kms, kn = ctx.profile_get()
        ctx.profile_enable(False)
        assert held[0].nrows == nsel, "%s: %d rows, expected %d" % (name, held[0].nrows, nsel)
        held[0].free()
        batch.free()
        out[name] = {"step_ms": ms / args.steps, "kernel_ms": kms / kn, "gap_ms": ms / args.steps - kms / kn, "launches": kn}
    ctx.close()
    print(json.dumps(out))


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # pragma: no cover
        return "nvidia-smi failed: %r" % e


def ab(args):
    libs = args.ab
    runs = {lib: [] for lib in libs}
    base = [sys.executable, os.path.abspath(__file__), "--rows", str(args.rows), "--steps", str(args.steps), "--warmup", str(args.warmup)]
    for rnd in range(args.rounds):
        for lib in libs:
            env = dict(os.environ, DFGPU_LIB=os.path.abspath(lib))
            line = subprocess.run(base, env=env, capture_output=True, text=True, check=True).stdout.strip().splitlines()[-1]
            runs[lib].append(json.loads(line))
            print("round %d %s: %s" % (rnd, lib, line), file=sys.stderr, flush=True)
    summary = {"gpu": gpu_info(), "rows": args.rows, "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds, "libs": {}}
    for lib in libs:
        s = {}
        for shape in ("c2", "c3"):
            s[shape] = {}
            for key in ("step_ms", "kernel_ms", "gap_ms"):
                v = [r[shape][key] for r in runs[lib]]
                s[shape][key] = {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))}
        summary["libs"][lib] = s
    print(json.dumps(summary, indent=1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--ab", nargs=2, metavar="LIB", default=None)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if args.ab:
        ab(args)
    else:
        one_run(args)


if __name__ == "__main__":
    main()
