"""Worker for tests/test_sort_mp.py (launched by torch.distributed.run, NCCL, one H100 per rank).
Each rank runs HAVING / ORDER BY / LIMIT queries through SQL over its row range of one table, with a communicator
attached; every rank's rows must equal, in order and bit for bit, what one GPU returns over all the rows.  Covers a
narrow Int64 GROUP BY key, a Utf8 key (the regroup merge), and a table whose rows all fall to rank 0 (rank 1 has none)."""
import os
import sys

import numpy as np
import pyarrow as pa
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from datafusion_archive_b200 import engine, host  # noqa: E402

QUERIES = [
    "SELECT k, SUM(v), COUNT(v) FROM t GROUP BY k ORDER BY SUM(v) DESC LIMIT 25",
    "SELECT k, MIN(v) FROM t GROUP BY k HAVING CAST(COUNT(v) AS BIGINT) > 40 ORDER BY MAX(v), k DESC",
    "SELECT s, SUM(v) FROM t GROUP BY s ORDER BY s DESC LIMIT 7",
    "SELECT s, k, AVG(v) FROM t GROUP BY s, k HAVING AVG(v) > 0 ORDER BY AVG(v) DESC LIMIT 30",
    "SELECT COUNT(v) FROM t HAVING CAST(COUNT(v) AS BIGINT) > 0",
]


def table(n):
    rng = np.random.default_rng(7)
    k = rng.integers(0, 500, n).astype(np.int64)
    v = (rng.integers(-4000, 4000, n) / 8).astype(np.float64)  # multiples of 1/8: every sum is exact in any order
    s = ["city%d" % (x % 37) for x in rng.integers(0, 10_000, n)]
    return [("k", k), ("v", v), ("s", pa.array(s))]


def run(ctx, n):
    out = []
    for q in QUERIES:
        ctx.register_memory("t", table(n))  # a DataSource is read once
        rows = []
        for batch in ctx.sql(q).collect():
            cols = [[(x, bool(m)) for x, m in zip(*c)] if isinstance(c, tuple) else list(c) for c in batch]
            rows.extend(repr(r) for r in zip(*cols))
        out.append(rows)
    return out


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    sizes = [50_000, 1]  # with 1 row, rank 0 holds it and rank 1 has none
    single = {}
    for n in sizes:
        c = host.ExecutionContext(local)
        single[n] = run(c, n)
        c.close()
    for n in sizes:
        uid = [engine.comm_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(uid, src=0)
        c = host.ExecutionContext(local)
        c.set_partition(rank, world, uid[0])
        got = run(c, n)
        c.close()
        assert got == single[n], (n, rank)
        every = [None] * world
        dist.all_gather_object(every, got)
        assert all(e == got for e in every), n
    dist.barrier()
    if rank == 0:
        print("MP_SORT_OK world=%d" % world)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
