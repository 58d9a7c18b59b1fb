"""Worker for tests/test_count_distinct_mp.py (launched by torch.distributed.run, NCCL, one H100 per rank).
COUNT(DISTINCT) has no pair exchange across ranks yet: with a communicator attached, every rank must get
NotImplemented at dfgpu_aggregate_create, grouped and ungrouped, and the other aggregates must still merge."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from datafusion_archive_b200 import _abi as A, engine  # noqa: E402
from datafusion_archive_b200.expr import AggregateFunction, col  # noqa: E402


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    ctx = engine.GpuContext(local)
    uid = [engine.comm_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(uid, src=0)
    ctx.comm_init(rank, world, uid[0])
    rng = np.random.default_rng(5 + rank)
    k = rng.integers(0, 100, 10_000).astype(np.int64)
    v = rng.integers(0, 20, 10_000).astype(np.int64)
    b = ctx.upload([k, v])
    for keys in ([col(0)], []):
        try:
            ctx.aggregate(b, keys, [AggregateFunction("count", col(1), distinct=True)])
            raise AssertionError("COUNT(DISTINCT) with a communicator attached did not fail")
        except engine.DfGpuError as e:
            assert e.code == A.ERR_NOT_IMPLEMENTED and "communicator attached" in e.msg, e.msg
    r = ctx.aggregate(b, [col(0)], [AggregateFunction("count", col(1))])  # every rank: the global counts
    got = r.columns()
    r.free()
    assert int(got[1].sum()) == 10_000 * world
    dist.barrier()
    if rank == 0:
        print("MP_COUNT_DISTINCT_OK world=%d" % world)
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
