"""CASE on the GPU against a numpy reference that follows the contract of include/dfgpu.h: the WHENs' masks in order, the
chosen branch's validity, and each row's pending DivideByZero bits (a row raises only from the conditions up to the first
true one and the value chosen).  Every site: projections without and with a WHERE (TMA, direct and NULLS kernels), WHERE,
GROUP BY keys (narrow and wide), every aggregate's argument with and without GROUP BY and under a fused WHERE,
COUNT(DISTINCT), a join key and a semi-join key, the depth limit, and SQL over memory and CSV tables."""
import os

import numpy as np
import pyarrow as pa
import pytest

from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import engine, host
from datafusion_archive_b200.expr import AggregateFunction, case, col, lit
import expr_ref
from groupby_ref import arrow_nullable
from kernel_trace import traced_set as traced
from test_avg_gpu import rows

pytestmark = pytest.mark.gpu

DATA = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "data")
N = 100_003


@pytest.fixture(scope="module")
def ctx():
    c = engine.GpuContext(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def dctx():
    """A context whose filter/project always takes the direct kernel (DFGPU_FP_KERNEL=direct, read at creation)."""
    old = os.environ.get("DFGPU_FP_KERNEL")
    os.environ["DFGPU_FP_KERNEL"] = "direct"
    try:
        c = engine.GpuContext(0)
    finally:
        if old is None:
            del os.environ["DFGPU_FP_KERNEL"]
        else:
            os.environ["DFGPU_FP_KERNEL"] = old
    yield c
    c.close()


# ---- reference --------------------------------------------------------------------------------------------------
def ref(e, arrays, nulls):
    """(values, valid, err) of `e` per row, as the extended interpreter computes them.  `nulls`: the input columns'
    bitmaps are read (no WHERE above the expression); else every input slot reads as valid."""
    return expr_ref.evaluate(e, arrays, read_bitmaps=nulls)


def project(c, arrays, exprs, pred=None):
    b = c.upload(arrays)
    try:
        r = c.filter_project(b, pred, exprs)
        try:
            return r.columns()
        finally:
            r.free()
    finally:
        b.free()


def split(got):
    return got if isinstance(got, tuple) else (got, np.ones(len(got), bool))


def assert_column(got, v, valid):
    gv, gvalid = split(got)
    assert len(gv) == len(v)
    assert np.array_equal(gvalid, valid), (np.flatnonzero(gvalid != valid)[:8])
    gv, v = np.asarray(gv), np.asarray(v)
    if gv.dtype.kind == "f":
        assert np.array_equal(gv.view(np.uint8).reshape(len(gv), -1)[valid], v.astype(gv.dtype).view(np.uint8).reshape(len(v), -1)[valid])
    else:
        assert np.array_equal(gv[valid], v.astype(gv.dtype)[valid])


def check_projection(c, arrays, e, pred=None):
    """Project `e` (under `pred`) and compare it, and whether the call raised DivideByZero, with the reference."""
    v, valid, err = ref(e, arrays, nulls=pred is None)
    keep = np.ones(len(v), bool)
    if pred is not None:
        pv, pvalid, perr = ref(pred, arrays, nulls=True)
        keep = pv.astype(bool) & pvalid
        err = (err & keep) | perr
    if err.any():
        with pytest.raises(engine.DfGpuError) as ei:
            project(c, arrays, [e], pred)
        assert ei.value.code == A.ERR_ARROW and "DivideByZero" in ei.value.msg
        return
    (got,) = project(c, arrays, [e], pred)
    assert_column(got, v[keep], valid[keep])


def data(seed=1, n=N, null_rate=0.1):
    rng = np.random.default_rng(seed)
    x = rng.uniform(0, 1, n)
    k = rng.integers(-20, 20, n).astype(np.int64)
    y = rng.normal(0, 10, n)
    # null slots store 0: under a WHERE a surviving null slot is read as its stored value, and the reference reads 0
    m = rng.random(n) < null_rate
    yn = pa.array(np.where(m, 0.0, y), mask=m)
    mk = rng.random(n) < null_rate
    kn = pa.array(np.where(mk, 0, k), mask=mk)
    return [x, k, y, yn, kn]


NUMERIC = [A.INT8, A.INT16, A.INT32, A.INT64, A.UINT8, A.UINT16, A.UINT32, A.UINT64, A.FLOAT32, A.FLOAT64]


# ---- values of every dtype, nullable inputs, with and without ELSE -------------------------------------------------------
@pytest.mark.parametrize("dt", NUMERIC + [A.BOOL])
@pytest.mark.parametrize("nullable", [False, True])
def test_every_result_dtype(ctx, dctx, dt, nullable):
    rng = np.random.default_rng(dt)
    n = N
    x = rng.uniform(0, 1, n)
    if dt == A.BOOL:
        raw = rng.random(n) < 0.5
        other = col(0) < 0.3
    else:
        info = np.iinfo(A.NP_OF[dt]) if dt not in (A.FLOAT32, A.FLOAT64) else None
        raw = (rng.integers(info.min, info.max, n, endpoint=True, dtype=A.NP_OF[dt]) if info is not None
               else rng.normal(0, 1e6, n).astype(A.NP_OF[dt]))
        other = lit(7, dt)
    m = rng.random(n) < 0.2
    v = pa.array(np.where(m, np.zeros_like(raw), raw), mask=m) if nullable else pa.array(raw)
    arrays = [x, v]
    exprs = [case([(col(0) > 0.6, col(1)), (col(0) < 0.2, other)], col(1)),  # ELSE a column
             case([(col(0) > 0.5, col(1))], other),
             case([(col(0) > 0.5, col(1)), (col(0) > 0.25, other)])]  # no ELSE: null where no WHEN is taken
    for e in exprs:
        for c in (ctx, dctx):
            check_projection(c, arrays, e)
            check_projection(c, arrays, e, pred=col(0) < 0.9)


def test_kernels(ctx):
    x = np.random.default_rng(2).uniform(0, 1, 1_000_000)
    # with ELSE over null-free columns: the TMA interpreter; without ELSE: the NULLS kernel, with a WHERE too
    _, k = traced(lambda: project(ctx, [x], [case([(col(0) > 0.5, col(0))], 0.0)]))
    assert k == {"k_filter_project_tma<kCaseDepth,4,1,0,0>"}
    _, k = traced(lambda: project(ctx, [x], [case([(col(0) > 0.5, col(0))])]))
    assert k == {"k_filter_project<kCaseDepth,1>"}
    _, k = traced(lambda: project(ctx, [x], [case([(col(0) > 0.5, col(0))])], pred=col(0) < 0.7))
    assert k == {"k_filter_project<kCaseDepth,1>", "k_pack_bits"}
    (got,) = project(ctx, [x], [case([(col(0) > 0.5, col(0))])], pred=col(0) < 0.7)
    sel = x < 0.7
    assert_column(got, np.where(x[sel] > 0.5, x[sel], 0), x[sel] > 0.5)


def test_nulls_under_a_where_come_from_case_only(ctx):
    x, k, y, yn, kn = data(3)
    # the input bitmap of yn is dropped under the WHERE, the CASE's own null is kept
    e = case([(col(0) > 0.3, col(3))])
    check_projection(ctx, [x, k, y, yn, kn], e, pred=col(1) > 0)
    check_projection(ctx, [x, k, y, yn, kn], e)
    # a null condition is not taken
    e = case([(col(3) > 0.0, col(0)), (col(3).eq(col(3)), 2.0)], 3.0)
    check_projection(ctx, [x, k, y, yn, kn], e)
    # nested, in a condition and under arithmetic
    e = case([(case([(col(0) > 0.5, col(3))]) > 1.0, col(2) + case([(col(1) > 0, col(2))]))], col(0))
    check_projection(ctx, [x, k, y, yn, kn], e)
    check_projection(ctx, [x, k, y, yn, kn], e, pred=col(1) < 5)


# ---- laziness --------------------------------------------------------------------------------------------------------
def test_division_in_a_branch_not_taken_never_raises(ctx, dctx):
    x, k, y, yn, kn = data(4)
    arrays = [x, k, y, yn, kn]
    guarded = [
        case([(col(1).not_eq(0), col(2) / col(1).cast(A.FLOAT64))], 0.0),
        case([(col(1).not_eq(0), lit(100) / col(1))], 0),
        case([(col(1).eq(0), lit(0))], lit(100) / col(1)),
        case([(col(1).eq(0), 0.0), (col(2) / col(1).cast(A.FLOAT64) > 1.0, 1.0)], 2.0),  # a condition after the one taken
        case([(col(1).not_eq(0), case([(col(1) > 0, lit(7) / col(1))], lit(-7) / col(1)))]),  # nested
    ]
    for e in guarded:
        for c in (ctx, dctx):
            check_projection(c, arrays, e)
            check_projection(c, arrays, e, pred=col(0) < 0.5)
        b = ctx.upload(arrays)
        try:
            r = ctx.aggregate(b, [], [AggregateFunction("count", e)])
            assert r.columns()[0][0] == np.count_nonzero(ref(e, arrays, True)[1])
        finally:
            b.free()
        assert_where(ctx, arrays, e.eq(e))


def assert_where(c, arrays, p):
    (got,) = project(c, arrays, [col(0)], pred=p)
    pv, pvalid, perr = ref(p, arrays, True)
    assert not perr.any()
    assert np.array_equal(got, arrays[0][pv.astype(bool) & pvalid])


def test_division_taken_raises(ctx, dctx):
    x, k, y, yn, kn = data(5)
    arrays = [x, k, y, yn, kn]
    raising = [
        case([(col(1).eq(0), lit(100) / col(1))], 0),  # the THEN taken divides by zero
        case([(col(1).not_eq(0), 0)], lit(100) / col(1)),  # the ELSE chosen
        case([(lit(100) / col(1) > 1, 1)], 0),  # the first condition is always reached
        case([(col(1) > 100, 1), (lit(100) / col(1) > 1, 2)], 3),  # reached when the first is false
        case([(col(1).eq(0), case([(col(0) < 2.0, lit(1) / col(1))], 0))], 5),  # nested, taken
    ]
    for e in raising:
        for c in (ctx, dctx):
            check_projection(c, arrays, e)
        b = ctx.upload(arrays)
        try:
            with pytest.raises(engine.DfGpuError) as ei:
                ctx.aggregate(b, [col(1)], [AggregateFunction("sum", e)]).columns()
            assert ei.value.code == A.ERR_ARROW
        finally:
            b.free()
    # only rows that survive the WHERE raise
    check_projection(ctx, arrays, raising[0], pred=col(1).not_eq(0))


def test_aggregate_raises_only_for_rows_that_survive_the_where(ctx):
    x, k, y, yn, kn = data(12)
    arrays = [x, k, y, yn, kn]
    e = case([(col(0) < 2.0, lit(100) / col(1))])  # always taken: raises exactly where k = 0
    for keys in ([], [col(1)]):
        got = run_agg(ctx, arrays, keys, [AggregateFunction("sum", e), AggregateFunction("count", e)], pred=col(1).not_eq(0))
        assert int(np.asarray(split(got[-1])[0]).sum()) == np.count_nonzero(k != 0)
        with pytest.raises(engine.DfGpuError) as ei:
            run_agg(ctx, arrays, keys, [AggregateFunction("sum", e)], pred=col(1) > -100)
        assert ei.value.code == A.ERR_ARROW and "DivideByZero" in ei.value.msg


# ---- sites -----------------------------------------------------------------------------------------------------------
def test_where(ctx, dctx):
    x, k, y, yn, kn = data(6)
    arrays = [x, k, y, yn, kn]
    for p in [case([(col(1) > 0, col(0) > 0.5)], col(0) < 0.1), case([(col(3) > 0.0, col(0) > 0.5)]),
              case([(col(1) < 0, 1.0)], 0.0) > 0.5]:
        for c in (ctx, dctx):
            assert_where(c, arrays, p)


def agg_ref(func, v, valid, keep, groups=None):
    """One aggregate over the rows `keep`, per group when `groups` is given: COUNT / AVG / COUNT(DISTINCT) skip nulls, a
    reduction without GROUP BY skips them, GROUP BY SUM / MIN / MAX read the value 0 under a null."""
    def one(sel, grouped):
        use = sel & valid if (func in ("count", "avg", "distinct") or not grouped) else sel
        vals = v[use]
        if func == "count":
            return int(use.sum())
        if func == "distinct":
            return len(np.unique(vals))
        if len(vals) == 0:
            return None
        return {"sum": vals.sum(), "min": vals.min(), "max": vals.max(), "avg": vals.astype(np.float64).sum() / len(vals)}[func]
    if groups is None:
        return one(keep, False)
    return {int(g): one(keep & (groups == g), True) for g in np.unique(groups[keep])}


def run_agg(c, arrays, keys, aggs, pred=None):
    b = c.upload(arrays)
    try:
        r = c.aggregate(b, keys, aggs, pred=pred)
        try:
            return r.columns()
        finally:
            r.free()
    finally:
        b.free()


def val_or_none(col_, i):
    if isinstance(col_, tuple):
        return col_[0][i] if col_[1][i] else None
    return col_[i]


@pytest.mark.parametrize("with_pred", [False, True])
def test_aggregate_arguments(ctx, with_pred):
    x, k, y, yn, kn = data(7)
    arrays = [x, k, y, yn, kn]
    pred = col(0) < 0.8 if with_pred else None
    keep = x < 0.8 if with_pred else np.ones(len(x), bool)
    e_int = case([(col(0) > 0.5, col(1))])
    e_flt = case([(col(0) > 0.7, col(2)), (col(0) > 0.2, col(3))], 0.5)
    e_rare = case([(col(0) > 2.0, col(2))])  # never taken: every value is null
    funcs = ["sum", "min", "max", "count", "avg"]
    for e in (e_int, e_flt, e_rare):
        v, valid, _ = ref(e, arrays, nulls=not with_pred)
        # no GROUP BY
        got = run_agg(ctx, arrays, [], [AggregateFunction(f, e) for f in funcs] + [AggregateFunction("count", e, distinct=True)], pred)
        for f, g in zip(funcs + ["distinct"], got):
            exp = agg_ref(f, v, valid, keep)
            gv = val_or_none(g, 0)
            if exp is None or gv is None:
                assert gv is None and exp is None, (f, gv, exp)
            elif f == "avg" or v.dtype.kind == "f":
                assert np.isclose(gv, exp, rtol=1e-12), (f, gv, exp)
            else:
                assert gv == exp, (f, gv, exp)
        # GROUP BY k
        got = run_agg(ctx, arrays, [col(1)], [AggregateFunction(f, e) for f in funcs] + [AggregateFunction("count", e, distinct=True)], pred)
        keys = got[0]
        for j, f in enumerate(funcs + ["distinct"]):
            exp = agg_ref(f, v, valid, keep, groups=k)
            for i, kk in enumerate(keys):
                gv, ev = val_or_none(got[1 + j], i), exp[int(kk)]
                if ev is None or gv is None:
                    assert gv is None and ev is None, (f, kk, gv, ev)
                elif f == "avg" or v.dtype.kind == "f":
                    assert np.isclose(gv, ev, rtol=1e-12), (f, kk, gv, ev)
                else:
                    assert gv == ev, (f, kk, gv, ev)


def test_a_case_passes_the_value_stored_under_a_selected_null_through(ctx):
    """GROUP BY SUM / MIN / MAX and a GROUP BY key read the value stored under a null that a CASE selects, as they read
    a null column's own; COUNT skips the null."""
    n = 1_000
    v = np.arange(n, dtype=np.int64) + 100
    valid = np.arange(n) % 3 != 0
    y = arrow_nullable(v, valid)  # the stored values stay under the nulls
    k = (np.arange(n) % 4).astype(np.int64)
    x = np.linspace(0, 1, n)
    e = case([(col(2) < 2.0, col(0))], lit(0))  # always taken
    got = run_agg(ctx, [y, k, x], [col(1)], [AggregateFunction(f, e) for f in ("sum", "min", "max", "count")])
    for g, s, mn, mx, c in zip(*[split(c_)[0] for c_ in got]):
        sel = k == g
        assert (s, mn, mx, c) == (v[sel].sum(), v[sel].min(), v[sel].max(), valid[sel].sum()), g
    got = run_agg(ctx, [y, k, x], [case([(col(2) < 2.0, col(0))])], [AggregateFunction("count", col(2))])
    assert sorted(got[0].tolist()) == v.tolist() and (got[1] == 1).all()


def test_group_by_keys(ctx):
    x, k, y, yn, kn = data(8)
    arrays = [x, k, y, yn, kn]
    bucket = case([(col(2) < -10.0, lit(0)), (col(2) < 10.0, lit(1))], lit(2))
    got = run_agg(ctx, arrays, [bucket], [AggregateFunction("count", col(0)), AggregateFunction("sum", col(2))])
    b = np.where(y < -10, 0, np.where(y < 10, 1, 2))
    assert dict(zip(got[0], got[1])) == {g: int((b == g).sum()) for g in range(3)}
    # a null key (no ELSE) is its value 0
    nk = case([(col(0) > 0.5, col(1))])
    got = run_agg(ctx, arrays, [nk], [AggregateFunction("count", col(0))], pred=col(2) > 0.0)
    kv = np.where(x > 0.5, k, 0)[y > 0]
    assert dict(zip(got[0], got[1])) == {int(g): int((kv == g).sum()) for g in np.unique(kv)}
    # a wide composite key: two 64-bit parts
    got = run_agg(ctx, arrays, [bucket, case([(col(0) > 0.5, col(1))], col(1) * lit(1 << 40))], [AggregateFunction("count", col(0))])
    k2 = np.where(x > 0.5, k, k * (1 << 40))
    exp = {}
    for a_, b_ in zip(b, k2):
        exp[(int(a_), int(b_))] = exp.get((int(a_), int(b_)), 0) + 1
    assert {(int(a_), int(b_)): int(c_) for a_, b_, c_ in zip(got[0], got[1], got[2])} == exp


def test_join_and_semi_join_keys(ctx):
    rng = np.random.default_rng(9)
    n = 50_000
    pk = rng.integers(0, 1000, n).astype(np.int64)
    px = rng.uniform(0, 1, n)
    bk = np.arange(0, 2000, 2, dtype=np.int64)
    build = ctx.upload([bk])
    probe = ctx.upload([pk, px])
    try:
        key = case([(col(1) > 0.5, col(0))], col(0) + lit(1))
        kv = np.where(px > 0.5, pk, pk + 1)
        j = ctx.join_build(build, [col(0)], keep_cols=[0])
        try:
            r = j.probe(probe, [key], probe_cols=[0, 1], build_cols=[0])
            got = r.columns()
            exp_rows = np.flatnonzero(np.isin(kv, bk))
            assert len(got[0]) == len(exp_rows)
            assert np.array_equal(got[2], kv[exp_rows])
            # a null key never matches, though its value 0 is a build key
            r = j.probe(probe, [case([(col(1) > 0.5, col(0))])], probe_cols=[0, 1], build_cols=[0])
            got = r.columns()
            exp_rows = np.flatnonzero((px > 0.5) & np.isin(pk, bk))
            assert 0 in bk and len(got[0]) == len(exp_rows) and np.array_equal(np.sort(got[0]), np.sort(pk[exp_rows]))
            r = j.semi(probe, [case([(col(1) > 0.5, col(0))])], probe_cols=[0])
            (g,) = r.columns()
            assert np.array_equal(g, pk[(px > 0.5) & np.isin(pk, bk)])
        finally:
            j.free()
    finally:
        build.free()
        probe.free()


def test_depth_limit(ctx):
    x = np.random.default_rng(10).uniform(0, 1, 1000)
    e = col(0)
    for _ in range(6):  # every level of nesting in the THEN of the last WHEN adds 1 to the stack depth
        e = case([(col(0) > 0.5, e + col(0) * (col(0) + col(0)))], col(0))
    with pytest.raises(engine.DfGpuError) as ei:
        project(ctx, [x], [e])
    assert ei.value.code == A.ERR_NOT_IMPLEMENTED and "too deep" in ei.value.msg


# ---- SQL -------------------------------------------------------------------------------------------------------------
# A registered table is read by one query, so each query below registers its own.
@pytest.mark.parametrize("batch", [1_000_000, 7_000])
def test_sql_conditional_aggregation_over_a_join(batch):
    hctx = host.ExecutionContext(0)
    try:
        rng = np.random.default_rng(11)
        n, m = 40_000, 500
        part = np.arange(m, dtype=np.int64)
        ptype = rng.integers(0, 5, m).astype(np.int64)
        lp = rng.integers(0, m, n).astype(np.int64)
        price = rng.uniform(1, 100, n)
        disc = rng.uniform(0, 0.1, n)
        mode = rng.integers(0, 4, n).astype(np.int64)

        def sql(q):
            sql.i += 1
            hctx.register_memory("lineitem%d" % sql.i, [("l_partkey", lp), ("l_price", price), ("l_disc", disc), ("l_mode", mode)],
                                 batch_size=batch)
            hctx.register_memory("part%d" % sql.i, [("p_partkey", part), ("p_type", ptype)])
            return rows(hctx.sql(q.replace("lineitem", "lineitem%d" % sql.i).replace("JOIN part", "JOIN part%d" % sql.i)))
        sql.i = 0
        got = sql("SELECT SUM(CASE WHEN p_type = 3 THEN l_price * (1 - l_disc) ELSE 0 END), SUM(l_price * (1 - l_disc)) "
                  "FROM lineitem JOIN part ON l_partkey = p_partkey WHERE l_disc < 0.05")
        sel = disc < 0.05
        rev = price * (1 - disc)
        assert np.isclose(got[0][0], rev[sel & (ptype[lp] == 3)].sum(), rtol=1e-9)
        assert np.isclose(got[0][1], rev[sel].sum(), rtol=1e-9)
        got = dict((r[0], r[1:]) for r in sql(
            "SELECT l_mode, SUM(CASE WHEN p_type = 1 OR p_type = 2 THEN 1 ELSE 0 END), COUNT(CASE WHEN p_type > 2 THEN 1 END) "
            "FROM lineitem JOIN part ON l_partkey = p_partkey GROUP BY l_mode"))
        for g in range(4):
            s = mode == g
            assert got[g] == (int(np.isin(ptype[lp[s]], [1, 2]).sum()), int((ptype[lp[s]] > 2).sum()))
        # a guarded division, and a CASE projection whose nulls survive the WHERE
        got = sql("SELECT CASE WHEN l_mode <> 0 THEN l_price / l_mode END FROM lineitem WHERE l_disc < 0.01")
        s = disc < 0.01
        exp = [None if md == 0 else p / md for p, md in zip(price[s], mode[s])]
        assert [r[0] for r in got] == exp
    finally:
        hctx.close()


def test_sql_csv_and_errors():
    hctx = host.ExecutionContext(0)
    try:
        d = np.genfromtxt(os.path.join(DATA, "aggregate_test_1.csv"), delimiter=",", skip_header=1)

        def sql(q):
            sql.i += 1
            hctx.register_csv("c%d" % sql.i, os.path.join(DATA, "aggregate_test_1.csv"), [("a", A.INT32), ("b", A.FLOAT64)], 1024)
            hctx.register_memory("t%d" % sql.i, [("a", np.arange(10, dtype=np.int64))])
            return rows(hctx.sql(q.replace("FROM c", "FROM c%d" % sql.i).replace("FROM t", "FROM t%d" % sql.i)))
        sql.i = 0

        got = sql("SELECT CASE a WHEN 1 THEN b WHEN 2 THEN 2 * b END FROM c")
        assert [r[0] for r in got] == [b if a == 1 else 2 * b if a == 2 else None for a, b in d]
        got = sql("SELECT COUNT(CASE WHEN b > 2 THEN a END), SUM(CASE WHEN a > 1 THEN b END) FROM c")
        assert got[0][0] == int((d[:, 1] > 2).sum())
        assert np.isclose(got[0][1], d[d[:, 0] > 1, 1].sum())
        # a coerced CASE (under arithmetic, as a function argument) has its values cast, not itself
        got = sql("SELECT CASE WHEN b > 2 THEN a END + 1, sqrt(CASE WHEN b > 2 THEN a ELSE 4 END) FROM c")
        assert [r[0] for r in got] == [int(a) + 1 if b > 2 else None for a, b in d]
        assert [r[1] for r in got] == [float(np.sqrt(a if b > 2 else 4.0)) for a, b in d]
        got = dict((r[0], r[1]) for r in sql("SELECT a, MIN(CASE WHEN b > 2 THEN b END) FROM c GROUP BY a"))
        # GROUP BY MIN reads 0 under the null of a row where no WHEN is taken
        assert got == {int(a): min(b if b > 2 else 0.0 for aa, b in d if aa == a) for a in np.unique(d[:, 0])}

        def err(q):
            with pytest.raises(host.ExecutionError) as ei:
                sql(q)
            return ei.value
        e = err("SELECT CASE WHEN SUM(a) > 0 THEN 1 ELSE 0 END FROM t")
        assert e.code == A.ERR_EXECUTION and "SUM(#0)" in str(e)
        assert "CASE WHEN condition did not evaluate to boolean" in str(err("SELECT CASE WHEN a THEN 1 END FROM t"))
        assert "DivideByZero" in str(err("SELECT a FROM t WHERE a > 0 AND 10 / a > 1"))  # a WHERE reads every row
        got = sql("SELECT a FROM t WHERE CASE WHEN a <> 0 THEN 10 / a > 1 ELSE a > 5 END")
        assert [r[0] for r in got] == [1, 2, 3, 4, 5]
    finally:
        hctx.close()
