"""Worker for the world_size>1 tests (launched by torch.distributed.run).
  mode gloo : CPU.  A numpy MODEL of the multi-GPU protocol (datafusion_archive_b200/parallel.py), not the
              product's merge: each rank computes its shard with the ORACLE (test infrastructure), splits
              its partial aggregate by owner rank, the segments travel over gloo, every rank merges only
              the keys it owns, the owned segments are gathered, and the result is checked against the
              oracle on the full data.  Exercises row ranges, the owner function and the merge algebra
              without a GPU; likewise a model of the regroup merge used for Utf8 / wide keys.
  mode nccl : GPUs.  Each rank drives its own H100 through the C ABI with a communicator attached;
              every rank must end with the SAME global result (dfgpu_aggregate_finish: owner-partitioned
              exchange over NCCL), also when one rank saw no rows at all.
"""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import oracle_lib as O  # noqa: E402
from datafusion_archive_b200 import _abi as A, parallel, workloads  # noqa: E402
from datafusion_archive_b200.expr import AggregateFunction, col, lit  # noqa: E402


def sort_by_key(cols):
    o = np.argsort(cols[0], kind="stable")
    return [c[o] for c in cols]


def aggregate_maybe_empty(ctx, engine, batch, schema, keys, aggs):
    """ctx.aggregate for a rank that may have no batch: create -> (update) -> finish through the C ABI."""
    import ctypes as C
    L = engine.lib()
    keep = []
    kptrs, klens, nk = A.make_programs([k.program(schema) for k in keys], keep)
    aggarr = A.make_aggs([a.lower(schema) for a in aggs], keep)
    st = C.c_void_p()
    engine.check(L.dfgpu_aggregate_create(ctx.h, kptrs, klens, nk, aggarr, len(aggs), 0, C.byref(st)))
    try:
        if batch is not None:
            engine.check(L.dfgpu_aggregate_update(st, batch.h))
        out = C.c_void_p()
        engine.check(L.dfgpu_aggregate_finish(st, C.byref(out)))
        r = engine.Result(ctx, out)
        cols = r.columns()
        r.free()
        return cols
    finally:
        L.dfgpu_aggregate_free(st)


def main():
    mode = sys.argv[1]
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    n = 400_000
    arrays, keys, aggs, _ = workloads.c5(n, nkeys=3000)
    aggs = aggs + [AggregateFunction("count", col(1))]
    funcs = [A.AGG_MIN, A.AGG_MAX, A.AGG_SUM, A.AGG_COUNT]
    full = sort_by_key(O.aggregate(arrays, keys, aggs))
    mine = parallel.shard(arrays, rank, world)
    fa, fpred, fproj = workloads.c2(n)
    fmine = parallel.shard(fa, rank, world)
    if mode == "gloo":
        dist.init_process_group("gloo")
        part = O.aggregate(mine, keys, aggs)
        segs = parallel.partition_by_owner(part, world)       # what this rank sends to every owner
        everyone = [None] * world
        dist.all_gather_object(everyone, segs)                 # (an all-to-all: rank r keeps everyone[s][r])
        owned = parallel.merge_partials([everyone[s][rank] for s in range(world)], funcs)
        assert np.all(parallel.owner_of(owned[0], world) == rank)
        gathered = [None] * world
        dist.all_gather_object(gathered, owned)
        merged = sort_by_key([np.concatenate([g[i] for g in gathered]) for i in range(len(owned))])
        fpart = O.filter_project(fmine, fpred, fproj)
        fg = [None] * world
        dist.all_gather_object(fg, fpart)
        fout = parallel.concat_in_rank_order(fg)
        # regroup merge (Utf8 / wide keys, aggregate.cu finish_regroup), MODEL: every rank's LOCAL RESULT is gathered and
        # aggregated once more with each aggregate's merge function (COUNT -> SUM of the counts)
        rng = np.random.default_rng(99)
        wn = 60_000
        wk1 = workloads.mix_keys(rng.integers(0, 150, wn, dtype=np.int64))
        wk2 = rng.integers(-(2 ** 62), 2 ** 62, 20, dtype=np.int64)[rng.integers(0, 20, wn)]
        ws = ["s%03d" % i for i in rng.integers(0, 40, wn)]
        wv = rng.random(wn)
        wlo, whi = parallel.row_range(rank, world, wn)
        for cols_, nk in (([wk1, wk2, wv], 2), ([ws, wv], 1)):
            wkeys = [col(i) for i in range(nk)]
            wa = [AggregateFunction("min", col(nk)), AggregateFunction("max", col(nk)), AggregateFunction("sum", col(nk)), AggregateFunction("count", col(nk))]
            local = O.aggregate([c[wlo:whi] for c in cols_], wkeys, wa)
            allres = [None] * world
            dist.all_gather_object(allres, [c if isinstance(c, list) else np.asarray(c) for c in local])
            cat = [sum((r[i] for r in allres), []) if isinstance(allres[0][i], list) else np.concatenate([r[i] for r in allres]) for i in range(nk + 4)]
            merge = [AggregateFunction("min", col(nk)), AggregateFunction("max", col(nk + 1)), AggregateFunction("sum", col(nk + 2)), AggregateFunction("sum", col(nk + 3))]
            got = O.aggregate(cat, wkeys, merge)
            exp = O.aggregate(cols_, wkeys, wa)
            rows = lambda cs: sorted(zip(*[c if isinstance(c, list) else c.tolist() for c in cs]), key=lambda r: r[:nk])  # noqa: E731
            g, e = rows(got), rows(exp)
            assert len(g) == len(e)
            for rg, re_ in zip(g, e):
                assert rg[:nk + 2] == re_[:nk + 2] and rg[nk + 3] == re_[nk + 3], (rg, re_)
                assert abs(rg[nk + 2] - re_[nk + 2]) <= 1e-9 * abs(re_[nk + 2]), (rg, re_)
        # no GROUP BY: scalars combine with the same algebra
        spart = O.aggregate(mine, [], aggs)
        sg = [None] * world
        dist.all_gather_object(sg, [np.zeros(1, dtype=np.int64)] + [np.asarray(c) for c in spart])
        smerged = parallel.merge_partials(sg, funcs)[1:]
    else:
        from datafusion_archive_b200 import engine
        local = int(os.environ.get("LOCAL_RANK", rank))
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
        ctx = engine.GpuContext(local)
        uid = [engine.comm_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(uid, src=0)
        ctx.comm_init(rank, world, uid[0])
        b = ctx.upload(mine)
        merged = sort_by_key(ctx.aggregate(b, keys, aggs).columns())  # every rank: the GLOBAL result
        smerged = ctx.aggregate(b, [], aggs).columns()
        # nullable no-GROUP-BY inputs: the non-null counts are summed over ranks, so an aggregate is null
        # only when NO rank saw a non-null input (array_from_scalar!, aggregate.rs:641-643)
        import pyarrow as pa
        lo, hi = parallel.row_range(rank, world, n)
        v = arrays[1]
        valid_some = np.zeros(n, dtype=bool)
        valid_some[: n // (2 * world)] = np.arange(n // (2 * world)) % 3 != 0  # non-null values on rank 0 only
        valid_none = np.zeros(n, dtype=bool)

        def nullable(values, valid):
            bits = np.packbits(valid, bitorder="little")
            return pa.Array.from_buffers(pa.float64(), len(values), [pa.py_buffer(bits.tobytes()), pa.py_buffer(np.ascontiguousarray(values).tobytes())])
        naggs = [AggregateFunction("min", col(0)), AggregateFunction("sum", col(0)), AggregateFunction("count", col(0)),
                 AggregateFunction("max", col(1)), AggregateFunction("count", col(1))]
        nb = ctx.upload([nullable(v[lo:hi], valid_some[lo:hi]), nullable(v[lo:hi], valid_none[lo:hi])])
        got = ctx.aggregate(nb, [], naggs).columns()
        exp = O.aggregate([nullable(v, valid_some), nullable(v, valid_none)], [], naggs)
        unp = lambda c: c if isinstance(c, tuple) else (c, np.ones(len(c), dtype=bool))  # noqa: E731
        for j, (g, e) in enumerate(zip(got, exp)):
            (gv, gm), (ev, em) = unp(g), unp(e)
            assert np.array_equal(gm, em), "validity of aggregate %d differs: %r vs %r" % (j, gm, em)
            if em[0]:
                assert gv[0] == ev[0] or abs(gv[0] - ev[0]) <= 1e-9 * abs(ev[0]), (j, gv, ev)
        # the same nullable columns under a fused WHERE that passes rows on rank 0 only: the aggregate sees the
        # filter's bitmap-free output, so every surviving row counts (values under nulls included) and the merged
        # scalars are non-null although rank 1 passed nothing
        w = (np.arange(n) < n // (4 * world)).astype(np.int32)
        wpred = col(2) > lit(0, A.INT32)
        wb = ctx.upload([nullable(v[lo:hi], valid_some[lo:hi]), nullable(v[lo:hi], valid_none[lo:hi]), w[lo:hi]])
        got = ctx.aggregate(wb, [], naggs, pred=wpred).columns()
        keep = w > 0
        exp = O.aggregate([v[keep], v[keep]], [], naggs)
        assert int(unp(got[2])[0][0]) == int(keep.sum()) and int(unp(got[4])[0][0]) == int(keep.sum())
        for j, (g, e) in enumerate(zip(got, exp)):
            (gv, gm), (ev, em) = unp(g), unp(e)
            assert gm[0] and em[0], "aggregate %d under the WHERE is null" % j
            assert gv[0] == ev[0] or abs(gv[0] - ev[0]) <= 1e-9 * abs(ev[0]), (j, gv, ev)
        wb.free()
        # every rank must hold bit-identical columns (same rows decoded in the same order)
        import hashlib
        digest = hashlib.sha256(b"".join(np.ascontiguousarray(c).tobytes() for c in merged)).hexdigest()
        digs = [None] * world
        dist.all_gather_object(digs, digest)
        assert len(set(digs)) == 1, "ranks hold different global results"
        # one rank contributes no batch at all: it still joins the exchange and gets the global result
        st_cols = aggregate_maybe_empty(ctx, engine, b if rank == 0 else None, [A.INT64, A.FLOAT64], keys, aggs)
        exp0 = sort_by_key(O.aggregate(parallel.shard(arrays, 0, world), keys, aggs))
        got0 = sort_by_key(st_cols)
        assert np.array_equal(got0[0], exp0[0]) and np.array_equal(got0[1], exp0[1]) and np.array_equal(got0[2], exp0[2])
        np.testing.assert_allclose(got0[3], exp0[3], rtol=1e-9)
        assert np.array_equal(got0[4], exp0[4])
        # fused WHERE under the communicator
        pred = col(1) < lit(0.5)
        gotp = sort_by_key(ctx.aggregate(b, keys, aggs, pred=pred).columns())
        keep = arrays[1] < 0.5
        expp = sort_by_key(O.aggregate([a[keep] for a in arrays], keys, aggs))
        assert np.array_equal(gotp[0], expp[0]) and np.array_equal(gotp[1], expp[1]) and np.array_equal(gotp[4], expp[4])
        np.testing.assert_allclose(gotp[3], expp[3], rtol=1e-9)
        # the same through the reference-shaped host API: every rank registers the WHOLE table, the
        # ExecutionContext works on its row range, ctx.sql() returns the global aggregate on every rank
        from datafusion_archive_b200 import host
        hctx = host.ExecutionContext(local)
        uid2 = [engine.comm_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(uid2, src=0)
        hctx.set_partition(rank, world, uid2[0])
        hctx.register_memory("t", [("k", arrays[0]), ("v", arrays[1])], batch_size=150_000)
        hk, hmn, hmx, hsm = hctx.sql("SELECT k, MIN(v), MAX(v), SUM(v) FROM t WHERE v < 0.5 GROUP BY k").collect()[0]
        ho, eo = np.argsort(hk), np.argsort(expp[0])
        assert np.array_equal(hk[ho], expp[0][eo]) and np.array_equal(hmn[ho], expp[1][eo]) and np.array_equal(hmx[ho], expp[2][eo])
        np.testing.assert_allclose(hsm[ho], expp[3][eo], rtol=1e-9)
        hctx.register_memory("t", [("k", arrays[0]), ("v", arrays[1])], batch_size=150_000)  # data sources are one-pass readers
        hpart = [np.concatenate([b[0] for b in hctx.sql("SELECT v FROM t WHERE v > 0.75").collect()] or [np.zeros(0)])]
        hg = [None] * world
        dist.all_gather_object(hg, hpart)
        # (per-batch row ranges: the concatenation in (batch, rank) order is the global output; compare as multisets per batch boundary-free)
        assert np.array_equal(np.sort(np.concatenate([g[0] for g in hg])), np.sort(arrays[1][arrays[1] > 0.75]))
        hctx.close()
        # key shapes that do not travel as packed 64-bit keys — wide composites and Utf8 — merge by regrouping the
        # gathered local results (aggregate.cu finish_regroup); every rank ends with the global result
        rng = np.random.default_rng(99)
        wn = 120_000
        wk1 = workloads.mix_keys(rng.integers(0, 200, wn, dtype=np.int64))
        wk2 = rng.integers(-(2 ** 62), 2 ** 62, 30, dtype=np.int64)[rng.integers(0, 30, wn)]
        wk3 = rng.integers(0, 5, wn, dtype=np.int32)
        vocab = ["", "a", "ab", "London, UK", "y" * 40] + ["s%03d" % i for i in range(50)]
        ws = [vocab[i] for i in rng.integers(0, len(vocab), wn)]
        wv = rng.random(wn)
        wi = rng.integers(-9, 9, wn, dtype=np.int64)

        def wide_aggs(cv, ci):
            return [AggregateFunction("min", col(cv)), AggregateFunction("max", col(cv)), AggregateFunction("sum", col(ci)),
                    AggregateFunction("count", col(cv)), AggregateFunction("sum", col(cv))]

        def rows(cols, nk):
            cols = [c if isinstance(c, list) else c.tolist() for c in cols]
            return sorted(zip(*cols), key=lambda r: r[:nk])

        wlo, whi = parallel.row_range(rank, world, wn)
        for cols_, wkeys, cv, ci, schema in [([wk1, wk2, wv, wi], [col(0), col(1)], 2, 3, [A.INT64, A.INT64, A.FLOAT64, A.INT64]),
                                             ([ws, wv, wi], [col(0)], 1, 2, [A.UTF8, A.FLOAT64, A.INT64]),
                                             ([ws, wk3, wv, wi], [col(0), col(1)], 2, 3, [A.UTF8, A.INT32, A.FLOAT64, A.INT64])]:
            nk = len(wkeys)
            wa = wide_aggs(cv, ci)
            wexp = rows(O.aggregate(cols_, wkeys, wa), nk)
            wb = ctx.upload([c[wlo:whi] for c in cols_])
            for variant in ("all ranks", "rank 1 empty"):
                if variant == "all ranks":
                    wgot = rows(ctx.aggregate(wb, wkeys, wa).columns(), nk)
                    want = wexp
                else:
                    wgot = rows(aggregate_maybe_empty(ctx, engine, wb if rank != 1 else None, schema, wkeys, wa), nk)
                    keep_rows = np.ones(wn, dtype=bool)
                    l1, h1 = parallel.row_range(1, world, wn)
                    keep_rows[l1:h1] = False
                    sel = [([x for x, k in zip(c, keep_rows) if k] if isinstance(c, list) else c[keep_rows]) for c in cols_]
                    want = rows(O.aggregate(sel, wkeys, wa), nk)
                assert len(wgot) == len(want), (variant, nk, len(wgot), len(want))
                for rg, re_ in zip(wgot, want):
                    for i, (x, y) in enumerate(zip(rg, re_)):
                        if i == nk + 4:
                            assert x == y or abs(x - y) <= 1e-9 * abs(y), (variant, rg, re_)
                        else:
                            assert x == y, (variant, rg, re_)
        fb = ctx.upload(fmine)
        fpart = ctx.filter_project(fb, fpred, fproj).columns()
        fg = [None] * world
        dist.all_gather_object(fg, fpart)
        fout = parallel.concat_in_rank_order(fg)
    assert np.array_equal(merged[0], full[0]), "keys differ"
    assert np.array_equal(merged[1], full[1]) and np.array_equal(merged[2], full[2]), "min/max differ"
    np.testing.assert_allclose(merged[3], full[3], rtol=1e-9)
    assert np.array_equal(merged[4], full[4]), "counts differ"
    sfull = O.aggregate(arrays, [], aggs)
    assert smerged[0][0] == sfull[0][0] and smerged[1][0] == sfull[1][0] and smerged[3][0] == sfull[3][0] == n
    assert abs(smerged[2][0] - sfull[2][0]) <= 1e-9 * abs(sfull[2][0])
    assert np.array_equal(fout[0], fa[0][fa[0] > 0.5]), "rank-ordered concatenation is not the global filter output"
    dist.barrier()
    if rank == 0:
        print("MP_OK mode=%s world=%d groups=%d" % (mode, world, len(merged[0])))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
