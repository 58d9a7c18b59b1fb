"""Worker for tests/test_join_mp.py (launched by torch.distributed.run, NCCL, one H100 per rank).
Every rank registers the WHOLE tables; with a partition set, the join probes this rank's row range of the left table
against the whole right table (a broadcast join).  An aggregate over a join must give every rank the one-GPU result, and
the projected rows of all ranks together must be the one-GPU rows, also when a rank's range is empty.  Values are
multiples of 1/8 so every f64 sum is exact in any order."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from datafusion_archive_b200 import engine, host  # noqa: E402

# COUNT(DISTINCT) is refused with a communicator attached (tests/test_count_distinct_mp.py); SUM, COUNT and AVG cover
# the exchange
AGG = "SELECT region, SUM(salary), COUNT(id), AVG(salary) FROM people JOIN dept ON dept = dept_id GROUP BY region"
SCALAR = "SELECT COUNT(id), SUM(salary) FROM people JOIN dept ON dept = dept_id WHERE salary > 0"
PROJ = "SELECT id, name, salary FROM people JOIN dept ON dept = dept_id WHERE region <> 3"


def tables(n_people):
    rng = np.random.default_rng(7)
    people = [("id", np.arange(n_people, dtype=np.int64)), ("dept", rng.integers(0, 60, n_people).astype(np.int32)),
              ("salary", (rng.integers(-800, 8000, n_people) / 8).astype(np.float64))]
    dept_id = np.concatenate([np.arange(50, dtype=np.int32), np.arange(10, dtype=np.int32)])  # ids 0..9 twice, 50..59 absent
    dept = [("dept_id", dept_id), ("region", (dept_id % 7).astype(np.int64)), ("name", ["d%d" % d for d in dept_id])]
    return people, dept


def run(ctx, people, dept, sql):
    ctx.register_memory("people", people, batch_size=30_000)
    ctx.register_memory("dept", dept, batch_size=16)
    return ctx.sql(sql).collect()


def rows(batches):
    out = []
    for b in batches:
        cols = [c if isinstance(c, list) else np.asarray(c).tolist() for c in b]
        out.extend(zip(*cols))
    return sorted(out)


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    for n_people in (200_000, 1):  # 1 row: rank 1's range of the left table is empty
        people, dept = tables(n_people)
        single = host.ExecutionContext(local)
        exp = {q: rows(run(single, people, dept, q)) for q in (AGG, SCALAR, PROJ)}
        single.close()
        ctx = host.ExecutionContext(local)
        uid = [engine.comm_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(uid, src=0)
        ctx.set_partition(rank, world, uid[0])
        for q in (AGG, SCALAR):
            got = rows(run(ctx, people, dept, q))
            assert got == exp[q], (n_people, q, got[:5], exp[q][:5])
        mine = rows(run(ctx, people, dept, PROJ))
        every = [None] * world
        dist.all_gather_object(every, mine)
        assert sorted(sum(every, [])) == exp[PROJ], n_people
        if n_people == 1 and rank == 1:
            assert mine == []
        ctx.close()
    dist.barrier()
    if rank == 0:
        print("MP_JOIN_OK world=%d" % world)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
