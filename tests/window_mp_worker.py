"""Worker for tests/test_window_mp.py (launched by torch.distributed.run, NCCL, one H100 per rank).
Each rank runs window queries through SQL over its row range of one table, with a communicator attached; the rank-ordered
concatenation of every rank's rows must equal, bit for bit, what one GPU returns over all the rows.  Covers float SUM /
AVG with rounding (the same association on any number of ranks), Utf8 and nullable keys, a WHERE, and a table whose
rows all fall to rank 0 (rank 1 has none)."""
import os
import sys

import numpy as np
import pyarrow as pa
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from datafusion_archive_b200 import engine, host  # noqa: E402

QUERIES = [
    "SELECT k, ROW_NUMBER() OVER (PARTITION BY k ORDER BY v DESC), RANK() OVER (ORDER BY s, k), SUM(x) OVER (PARTITION BY k ORDER BY v), "
    "AVG(x) OVER (PARTITION BY s), MIN(v) OVER (), COUNT(x) OVER (PARTITION BY s ORDER BY k DESC) FROM t",
    "SELECT v, DENSE_RANK() OVER (PARTITION BY s ORDER BY x), SUM(x) OVER () FROM t WHERE v > 0",
]


def table(n):
    rng = np.random.default_rng(7)
    k = rng.integers(0, 500, n).astype(np.int64)
    v = rng.integers(-4000, 4000, n).astype(np.int32)
    x = rng.standard_normal(n) * 10.0 ** rng.integers(-6, 6, n)  # sums round: the association must match
    xvalid = rng.random(n) < 0.9
    s = pa.array(["city%d" % (i % 37) for i in rng.integers(0, 10_000, n)], mask=rng.random(n) < 0.05)
    bits = np.packbits(xvalid, bitorder="little")
    xa = pa.Array.from_buffers(pa.float64(), n, [pa.py_buffer(bits.tobytes()), pa.py_buffer(x.tobytes())])
    return [("k", k), ("v", v), ("x", xa), ("s", s)]


def run(ctx, n):
    out = []
    for q in QUERIES:
        ctx.register_memory("t", table(n))  # a DataSource is read once
        rows = []
        for batch in ctx.sql(q).collect():
            cols = [[(x.tobytes() if hasattr(x, "tobytes") else x, bool(m)) for x, m in zip(*c)] if isinstance(c, tuple)
                    else [x.tobytes() if hasattr(x, "tobytes") else x for x in c] for c in batch]
            rows.extend(repr(r) for r in zip(*cols))
        out.append(rows)
    return out


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    sizes = [60_001, 1]  # with 1 row, rank 0 holds it and rank 1 has none
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
        every = [None] * world
        dist.all_gather_object(every, got)
        for q in range(len(QUERIES)):
            assert sum((e[q] for e in every), []) == single[n][q], (n, q, rank)
    dist.barrier()
    if rank == 0:
        print("MP_WINDOW_OK world=%d" % world)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
