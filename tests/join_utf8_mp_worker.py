"""Worker for tests/test_join_utf8_mp.py (launched by torch.distributed.run, NCCL, one H100 per rank).
Every rank registers the WHOLE tables and joins on a Utf8 key; with a partition set, the join probes this rank's row
range of the left table against the whole right table (a broadcast join).  An aggregate over the join must give every
rank the one-GPU result, and the projected rows of all ranks together must be the one-GPU rows, also when a rank's
range is empty.  Values are multiples of 1/8 so every f64 sum is exact in any order."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from datafusion_archive_b200 import engine, host  # noqa: E402

AGG = "SELECT region, SUM(salary), COUNT(id), AVG(salary) FROM people JOIN dept ON dname = dept_name GROUP BY region"
PROJ = "SELECT id, name, salary FROM people JOIN dept ON dname = dept_name AND grade = dept_grade WHERE region <> 3"


def tables(n_people):
    rng = np.random.default_rng(7)
    people = [("id", np.arange(n_people, dtype=np.int64)), ("dname", ["dept-%d" % d for d in rng.integers(0, 60, n_people)]),
              ("grade", rng.integers(0, 2, n_people).astype(np.int32)),
              ("salary", (rng.integers(-800, 8000, n_people) / 8).astype(np.float64))]
    ids = np.concatenate([np.arange(50), np.arange(10)])  # names 0..9 twice, 50..59 absent
    dept = [("dept_name", ["dept-%d" % d for d in ids]), ("dept_grade", (ids % 2).astype(np.int32)),
            ("region", (ids % 7).astype(np.int64)), ("name", ["d%d" % d for d in ids])]
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
        exp = {q: rows(run(single, people, dept, q)) for q in (AGG, PROJ)}
        single.close()
        if n_people > 1:
            assert exp[AGG] and exp[PROJ]
        ctx = host.ExecutionContext(local)
        uid = [engine.comm_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(uid, src=0)
        ctx.set_partition(rank, world, uid[0])
        got = rows(run(ctx, people, dept, AGG))
        assert got == exp[AGG], (n_people, got[:5], exp[AGG][:5])
        mine = rows(run(ctx, people, dept, PROJ))
        every = [None] * world
        dist.all_gather_object(every, mine)
        assert sorted(sum(every, [])) == exp[PROJ], n_people
        if n_people == 1 and rank == 1:
            assert mine == []
        ctx.close()
    dist.barrier()
    if rank == 0:
        print("MP_JOIN_UTF8_OK world=%d" % world)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
