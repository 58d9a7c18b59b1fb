"""Worker for tests/test_semi_join_mp.py (launched by torch.distributed.run, NCCL, one H100 per rank).
Every rank registers the WHOLE tables; with a partition set, the outer query reads this rank's row range of its table and
the subquery the whole of its own (a broadcast semi join), so each outer row is decided on exactly one rank.  An
aggregate over a semi join must give every rank the one-GPU result, and the projected rows of all ranks together must be
the one-GPU rows, also when a rank's range is empty.  Values are multiples of 1/8 so every f64 sum is exact in any
order."""
import os
import sys

import numpy as np
import pyarrow as pa
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from datafusion_archive_b200 import engine, host  # noqa: E402

AGG = [
    "SELECT region, SUM(salary), COUNT(id) FROM people WHERE dept IN (SELECT dept_id FROM dept WHERE region > 3) GROUP BY region",
    "SELECT COUNT(id), SUM(salary) FROM people WHERE dept NOT IN (SELECT dept_id FROM dept WHERE region > 3)",
    "SELECT COUNT(id), SUM(salary) FROM people WHERE dept NOT IN (SELECT dept_id FROM dept)",  # holds a null: no row
    "SELECT COUNT(id), AVG(salary) FROM people p WHERE EXISTS (SELECT 1 FROM dept WHERE dept_id = p.dept AND region < 3)",
]
PROJ = [
    "SELECT id, salary FROM people WHERE dept IN (SELECT dept_id FROM dept WHERE region > 3)",
    "SELECT id FROM people WHERE dept NOT IN (SELECT dept_id FROM dept WHERE region > 3) AND salary > 100",
    "SELECT id FROM people p WHERE NOT EXISTS (SELECT 1 FROM dept WHERE dept_id = p.dept)",
]


def tables(n_people):
    rng = np.random.default_rng(7)
    people = [("id", np.arange(n_people, dtype=np.int64)),
              ("dept", pa.array(rng.integers(0, 60, n_people).astype(np.int32), mask=rng.random(n_people) < 0.05)),
              ("region", rng.integers(0, 7, n_people).astype(np.int64)),
              ("salary", (rng.integers(-800, 8000, n_people) / 8).astype(np.float64))]
    dept_id = list(range(50)) + list(range(10)) + [None]  # ids 0..9 twice, 50..59 absent, one null (region 3)
    dept = [("dept_id", pa.array(dept_id, type=pa.int32())), ("region", np.array([3 if d is None else d % 7 for d in dept_id], np.int64))]
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
    for n_people in (200_000, 1):  # 1 row: rank 1's range of the outer table is empty
        people, dept = tables(n_people)
        single = host.ExecutionContext(local)
        exp = {q: rows(run(single, people, dept, q)) for q in AGG + PROJ}
        single.close()
        assert exp[AGG[2]] in ([(0, None)], [(0, 0.0)]), exp[AGG[2]]
        ctx = host.ExecutionContext(local)
        uid = [engine.comm_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(uid, src=0)
        ctx.set_partition(rank, world, uid[0])
        for q in AGG:
            got = rows(run(ctx, people, dept, q))
            assert got == exp[q], (n_people, q, got[:5], exp[q][:5])
        for q in PROJ:
            mine = rows(run(ctx, people, dept, q))
            every = [None] * world
            dist.all_gather_object(every, mine)
            assert sorted(sum(every, [])) == exp[q], (n_people, q)
            if n_people == 1 and rank == 1:
                assert mine == []
        ctx.close()
    dist.barrier()
    if rank == 0:
        print("MP_SEMI_JOIN_OK world=%d" % world)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
