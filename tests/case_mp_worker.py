"""Worker for tests/test_case_mp.py (launched by torch.distributed.run, NCCL, one H100 per rank).
Each rank aggregates its own rows with a communicator attached; every rank must get bit-identical results equal to the
single-GPU aggregate of all ranks' rows, for conditional aggregation (CASE arguments, with and without ELSE, under a
fused WHERE and without one), with and without GROUP BY, also when one rank has no rows.  Values are multiples of 1/8
so every f64 sum is exact in any order."""
import ctypes as C
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from datafusion_archive_b200 import _abi as A  # noqa: E402
from datafusion_archive_b200 import engine  # noqa: E402
from datafusion_archive_b200.expr import AggregateFunction, case, col  # noqa: E402

SCHEMA = [A.INT64, A.FLOAT64, A.INT64]


def rank_data(r, n):
    rng = np.random.default_rng(200 + r)
    k = rng.integers(0, 3000, n).astype(np.int64)
    v = (rng.integers(-4000, 4000, n) / 8).astype(np.float64)
    q = rng.integers(0, 50, n).astype(np.int64)
    q[k == 7 + r] = 0  # the CASE is null for this key on this rank only
    return [k, v, q]


def aggregate(ctx, arrays, keys, aggs, pred):
    """create -> (update) -> finish through the C ABI; arrays=None: a rank with no batch."""
    L = engine.lib()
    keep = []
    kptrs, klens, nk = A.make_programs([k.program(SCHEMA) for k in keys], keep)
    aggarr = A.make_aggs([a.lower(SCHEMA) for a in aggs], keep)
    st = C.c_void_p()
    engine.check(L.dfgpu_aggregate_create(ctx.h, kptrs, klens, nk, aggarr, len(aggs), 0, C.byref(st)))
    b = None
    try:
        if pred is not None:
            pprog = pred.program(SCHEMA)
            parr = (A.Insn * len(pprog))(*pprog)
            engine.check(L.dfgpu_aggregate_set_predicate(st, parr, len(pprog)))
        if arrays is not None:
            b = ctx.upload(arrays)
            engine.check(L.dfgpu_aggregate_update(st, b.h))
        out = C.c_void_p()
        engine.check(L.dfgpu_aggregate_finish(st, C.byref(out)))
        r = engine.Result(ctx, out)
        cols = r.columns()
        r.free()
        return cols
    finally:
        if b is not None:
            b.free()
        L.dfgpu_aggregate_free(st)


def canonical(cols, nkeys):
    """Rows sorted by key, as bytes: values and validity."""
    keys = [np.asarray(c) for c in cols[:nkeys]]
    order = np.argsort(keys[0], kind="stable") if nkeys else np.arange(1)
    out = [k[order].tobytes() for k in keys]
    for c in cols[nkeys:]:
        vals, valid = c if isinstance(c, tuple) else (c, np.ones(len(c), bool))
        out.append(np.asarray(vals)[order].tobytes())
        out.append(np.asarray(valid, bool)[order].tobytes())
    return b"".join(out)


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    pos = case([(col(2) > 0, col(1))])  # null where q = 0
    big = case([(col(1) > 100.0, col(1)), (col(1) < -100.0, col(1) * 2.0)], 0.0)
    aggs = [AggregateFunction("sum", big), AggregateFunction("sum", pos), AggregateFunction("count", pos),
            AggregateFunction("min", pos), AggregateFunction("max", pos), AggregateFunction("avg", pos)]
    shapes = {"scalar": [], "narrow": [col(0)], "bucket": [case([(col(1) < 0.0, col(2))], col(2) + case([(col(0) > 10, col(0))], 0))]}
    preds = {"no WHERE": None, "WHERE": col(1) > -300.0}

    # the single-GPU references over every rank's rows, computed before a communicator exists
    ctx = engine.GpuContext(local)
    n = 150_000
    variants = {v: [rank_data(r, 0 if (v == "rank 1 empty" and r == 1) else n) for r in range(world)]
                for v in ("all ranks", "rank 1 empty")}
    single = {}
    for variant, parts in variants.items():
        whole = [np.concatenate([p[j] for p in parts]) for j in range(3)]
        for name, keys in shapes.items():
            for pname, pred in preds.items():
                single[variant, name, pname] = canonical(aggregate(ctx, whole, keys, aggs, pred), len(keys))

    uid = [engine.comm_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(uid, src=0)
    ctx.comm_init(rank, world, uid[0])
    for variant, parts in variants.items():
        mine_rows = parts[rank] if len(parts[rank][0]) else None
        for name, keys in shapes.items():
            for pname, pred in preds.items():
                mine = canonical(aggregate(ctx, mine_rows, keys, aggs, pred), len(keys))
                assert mine == single[variant, name, pname], (variant, name, pname)
                every = [None] * world
                dist.all_gather_object(every, mine)
                assert all(e == mine for e in every), (variant, name, pname)
    dist.barrier()
    if rank == 0:
        print("MP_CASE_OK world=%d" % world)
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
