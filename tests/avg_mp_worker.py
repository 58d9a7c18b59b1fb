"""Worker for tests/test_avg_mp.py (launched by torch.distributed.run, NCCL, one H100 per rank).
Each rank aggregates its own rows with a communicator attached; every rank must get bit-identical AVG results equal to
the single-GPU AVG of all ranks' rows concatenated, for the scalar all-reduce, the narrow-key exchange and the
regroup merge of a Utf8 key.  Values are multiples of 1/8 so every f64 sum is exact in any order."""
import os
import sys

import numpy as np
import pyarrow as pa
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from datafusion_archive_b200 import engine  # noqa: E402
from datafusion_archive_b200.expr import AggregateFunction, col  # noqa: E402

WORDS = ["w%03d" % i for i in range(150)]


def rank_data(r):
    rng = np.random.default_rng(100 + r)
    n = 200_000
    k = rng.integers(0, 5000, n).astype(np.int64)
    v = (rng.integers(-4000, 4000, n) / 8).astype(np.float64)
    i = rng.integers(-1000, 1000, n).astype(np.int32)
    valid = rng.random(n) < 0.8
    valid[k == 11 + r] = False  # all null on this rank only: the group's AVG comes from the other rank
    valid[k == 42] = False      # all null everywhere: null
    s = [WORDS[j] for j in rng.integers(0, len(WORDS), n)]
    return k, v, i, valid, s


def query(ctx, arrays, keys, aggs):
    b = ctx.upload(arrays)
    try:
        r = ctx.aggregate(b, keys, aggs)
        try:
            return r.columns()
        finally:
            r.free()
    finally:
        b.free()


def canonical(cols, nkeys):
    """Rows sorted by key, as bytes: values and validity, for a bit-exact comparison across ranks and runs."""
    keys = [np.asarray(c) for c in cols[:nkeys]]
    order = np.argsort(keys[0], kind="stable") if nkeys else np.arange(1)
    out = [k[order].tobytes() for k in keys]
    for c in cols[nkeys:]:
        vals, valid = c if isinstance(c, tuple) else (c, np.ones(len(c), bool))
        out.append(np.asarray(vals)[order].tobytes())
        out.append(np.asarray(valid, bool)[order].tobytes())
    return b"".join(out)


def masked(vals, valid):
    vals = np.where(valid, vals, 0)  # null rows hold 0, as the engine's nullable columns do
    return pa.array(vals, mask=~valid)


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    avg = lambda c: AggregateFunction("avg", c)  # noqa: E731
    aggs = [avg(col(1)), avg(col(2)), AggregateFunction("count", col(1))]
    shapes = {"scalar": [], "narrow": [col(0)], "utf8": [col(3)]}

    # the single-GPU reference over every rank's rows, computed before a communicator exists
    ctx = engine.GpuContext(local)
    parts = [rank_data(r) for r in range(world)]
    k = np.concatenate([p[0] for p in parts])
    v = np.concatenate([p[1] for p in parts])
    i = np.concatenate([p[2] for p in parts])
    valid = np.concatenate([p[3] for p in parts])
    s = sum((p[4] for p in parts), [])
    single = {}
    for name, keys in shapes.items():
        single[name] = query(ctx, [k, masked(v, valid), i, s], keys, aggs)

    uid = [engine.comm_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(uid, src=0)
    ctx.comm_init(rank, world, uid[0])
    k, v, i, valid, s = parts[rank]
    for name, keys in shapes.items():
        got = query(ctx, [k, masked(v, valid), i, s], keys, aggs)
        mine = canonical(got, len(keys))
        assert mine == canonical(single[name], len(keys)), name
        every = [None] * world
        dist.all_gather_object(every, mine)
        assert all(e == mine for e in every), name
        if name == "narrow":
            key = np.asarray(got[0])
            a, ok = got[1]
            assert not ok[key == 42].any() and ok[(key == 11) | (key == 12)].all()
    dist.barrier()
    if rank == 0:
        print("MP_AVG_OK world=%d" % world)
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
