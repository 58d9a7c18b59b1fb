"""Built-in scalar functions on the GPU.  The exact functions (sqrt abs floor ceil trunc round signum) must equal a numpy
restatement of the Rust f64 methods bit for bit; the transcendentals must give the C99 Annex F special values exactly and be
within 3 ulp of the same function evaluated in long double.  Functions are checked in every position an expression can
take: WHERE (TMA and direct filter kernels), projections, the aggregate's fused WHERE and every aggregate's argument, with
nulls, through SQL, and at 1e7 rows.  Under DFGPU_TRACE the routing to the function-bearing kernel instantiations is
asserted, and function-free queries keep their kernels."""
import math
import os

import numpy as np
import pyarrow as pa
import pytest

from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import engine, host
from datafusion_archive_b200.expr import AggregateFunction, col, fn
from expr_ref import EXACT_REF, LONG, LONG2, rust_abs, rust_round, rust_signum
from kernel_trace import traced_set as traced
from test_avg_gpu import rows

pytestmark = pytest.mark.gpu

DATA = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "data")
EXACT = ["sqrt", "abs", "floor", "ceil", "trunc", "round", "signum"]


@pytest.fixture(scope="module")
def ctx():
    c = engine.GpuContext(0)
    yield c
    c.close()


def bits_equal(got, exp):
    got, exp = np.asarray(got, np.float64), np.asarray(exp, np.float64)
    both_nan = np.isnan(got) & np.isnan(exp)
    ok = (got.view(np.uint64) == exp.view(np.uint64)) | both_nan
    assert ok.all(), list(zip(got[~ok][:8], exp[~ok][:8]))


def within_ulps(got, exp_long, ulps=3):
    """|got - f(x) in long double| <= ulps units in the last place of the rounded reference; specials must match."""
    exp = np.asarray(exp_long).astype(np.float64)
    got = np.asarray(got, np.float64)
    special = ~np.isfinite(exp) | ~np.isfinite(got) | (exp == 0)
    bits_equal(got[special], exp[special])
    g, e = got[~special], np.asarray(exp_long)[~special]
    err = np.abs(g.astype(np.longdouble) - e) / np.spacing(np.abs(e.astype(np.float64))).astype(np.longdouble)
    assert err.max(initial=0) <= ulps, (float(err.max()), g[np.argmax(err)], e[np.argmax(err)])


def project(ctx, arrays, exprs, pred=None):
    b = ctx.upload(arrays)
    try:
        r = ctx.filter_project(b, pred, exprs)
        try:
            return r.columns()
        finally:
            r.free()
    finally:
        b.free()


SPECIAL = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, -np.nan, 5e-324, -5e-324, 2.2250738585072009e-308, 1e-310, 0.5, -0.5,
                    1.5, -1.5, 2.5, -2.5, 0.49999999999999994, -0.49999999999999994, -0.4, 2.0**52 + 1, -(2.0**52 + 1), 2.0**52 - 0.5,
                    2.0**53, 1.0, -1.0, 1e300, -1e300, 4.0, 2.0, 3.5, -7.25, 1e-5, 0.9999999999999999])


def exact_inputs(n=200_000, seed=3):
    rng = np.random.default_rng(seed)
    x = np.concatenate([SPECIAL, rng.normal(0, 10, n // 2), rng.integers(-50, 50, n // 4) * 0.5,
                        rng.standard_normal(n // 4) * 10.0 ** rng.integers(-300, 300, n // 4)])
    return x.astype(np.float64)


# ---- values ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", EXACT)
def test_exact_functions_bit_for_bit(ctx, name):
    x = exact_inputs()
    (got,), kernels = traced(lambda: project(ctx, [x], [fn(name, col(0))]))
    bits_equal(got, EXACT_REF[name](x))
    assert kernels == {"k_filter_project_tma<kFnDepth,4,1,0,0>"}


def test_exact_function_edges():
    """The restatements themselves, at the values the issue names."""
    x = np.array([0.5, 2.5, -2.5, 0.49999999999999994, -0.4, 1.5, -0.5, 2.0**52 + 1])
    bits_equal(rust_round(x), [1.0, 3.0, -3.0, 0.0, -0.0, 2.0, -1.0, 2.0**52 + 1])
    bits_equal(rust_signum(np.array([0.0, -0.0, np.inf, -np.inf, np.nan, -3.0])), [1.0, -1.0, 1.0, -1.0, np.nan, -1.0])
    bits_equal(rust_abs(np.array([-0.0, -np.inf, -5e-324])), [0.0, np.inf, 5e-324])


def domain(name, rng, n):
    if name == "exp":
        return rng.uniform(-708, 709, n)  # normal results; the special values below cover under- and overflow
    if name in ("ln", "log2", "log10"):
        return np.abs(rng.standard_normal(n)) * 10.0 ** rng.integers(-307, 307, n)
    if name in ("asin", "acos"):
        return rng.uniform(-1, 1, n)
    if name in ("sin", "cos", "tan"):  # small, moderate and huge arguments (the slow argument reduction)
        return np.concatenate([rng.uniform(-10, 10, n // 2), rng.standard_normal(n // 2) * 10.0 ** rng.integers(0, 301, n // 2)])
    return rng.standard_normal(n) * 10.0 ** rng.integers(-20, 20, n)


@pytest.mark.parametrize("name", sorted(LONG))
def test_transcendental_within_3_ulp(ctx, name):
    rng = np.random.default_rng(sorted(LONG).index(name))
    x = domain(name, rng, 100_000)
    x = np.concatenate([x, [1e300, -1e300, 1e22, 2.0**1000, 0.0, -0.0, 1.0, -1.0]]) if name in ("sin", "cos", "tan") else x
    (got,) = project(ctx, [x], [fn(name, col(0))])
    with np.errstate(all="ignore"):
        within_ulps(got, LONG[name](x.astype(np.longdouble)))


SPECIAL_CASES = [  # (function, x, [y,] the C99 Annex F value; the exact functions: the Rust value)
    ("sqrt", -1.0, math.nan), ("sqrt", -0.0, -0.0), ("sqrt", math.inf, math.inf),
    ("exp", math.inf, math.inf), ("exp", -math.inf, 0.0), ("exp", 0.0, 1.0), ("exp", 1000.0, math.inf), ("exp", math.nan, math.nan),
    ("ln", 0.0, -math.inf), ("ln", -0.0, -math.inf), ("ln", -1.0, math.nan), ("ln", 1.0, 0.0), ("ln", math.inf, math.inf),
    ("log2", 0.0, -math.inf), ("log2", 1.0, 0.0), ("log2", -1.0, math.nan), ("log10", 0.0, -math.inf), ("log10", 1.0, 0.0),
    ("log10", -2.0, math.nan), ("sin", -0.0, -0.0), ("sin", math.inf, math.nan), ("cos", 0.0, 1.0), ("cos", -math.inf, math.nan),
    ("tan", -0.0, -0.0), ("tan", math.inf, math.nan), ("asin", 2.0, math.nan), ("asin", -0.0, -0.0), ("acos", 1.0, 0.0),
    ("acos", -1.5, math.nan), ("atan", math.inf, math.atan(math.inf)), ("atan", -0.0, -0.0),
    ("power", 2.0, 0.0, 1.0), ("power", math.nan, 0.0, 1.0), ("power", 1.0, math.nan, 1.0), ("power", -2.0, math.inf, math.inf),
    ("power", -2.0, 0.5, math.nan), ("power", 0.0, -1.0, math.inf), ("power", -0.0, -1.0, -math.inf), ("power", -0.0, 3.0, -0.0),
    ("power", -math.inf, 3.0, -math.inf), ("power", -1.0, math.inf, 1.0), ("power", 0.5, math.inf, 0.0), ("power", 2.0, -math.inf, 0.0),
    ("power", math.inf, -2.0, 0.0), ("atan2", 0.0, -0.0, math.pi), ("atan2", -0.0, -0.0, -math.pi), ("atan2", 0.0, 0.0, 0.0),
    ("atan2", -0.0, 1.0, -0.0), ("atan2", math.inf, math.inf, math.atan2(math.inf, math.inf)), ("atan2", 1.0, math.nan, math.nan),
    ("abs", -math.nan, math.nan), ("signum", -0.0, -1.0), ("round", -0.4, -0.0), ("floor", -0.5, -1.0), ("ceil", -0.5, -0.0),
    ("trunc", -0.7, -0.0),
]


def test_special_values_exact(ctx):
    for name in sorted({c[0] for c in SPECIAL_CASES}):
        cases = [c for c in SPECIAL_CASES if c[0] == name]
        args = [np.array([c[i] for c in cases]) for i in range(1, len(cases[0]) - 1)]
        (got,) = project(ctx, args, [fn(name, *[col(i) for i in range(len(args))])])
        bits_equal(got, [c[-1] for c in cases])


@pytest.mark.parametrize("name", sorted(LONG2))
def test_binary_functions_within_3_ulp_in_every_operand_mode(ctx, name):
    rng = np.random.default_rng(7)
    n = 100_000
    x = np.abs(rng.standard_normal(n)) * 10.0 ** rng.integers(-3, 3, n)
    y = rng.uniform(-20, 20, n)
    if name == "power":  # negative bases with integer exponents too
        x[: n // 4] = -x[: n // 4]
        y[: n // 4] = np.round(y[: n // 4])
    ref = LONG2[name]
    L = lambda a: np.asarray(a, np.longdouble)  # noqa: E731
    cases = [  # RHS_COL, RHS_IMM, RHS_STACK (exchanged operands), literal on the left
        (fn(name, col(0), col(1)), ref(L(x), L(y))),
        (fn(name, col(0), 3.0), ref(L(x), L(3.0))),
        (fn(name, col(0), col(1) + 0.0), ref(L(x), L(y))),
        (fn(name, col(1) * 1.0, fn("abs", col(0))), ref(L(y), L(np.abs(x)))),
        (fn(name, 1.5, col(1)), ref(L(1.5), L(y))),
    ]
    got = project(ctx, [x, y], [e for e, _ in cases])
    with np.errstate(all="ignore"):
        for g, (_, exp) in zip(got, cases):
            within_ulps(g, exp)


def test_projection_nesting_and_arithmetic(ctx):
    rng = np.random.default_rng(11)
    a = rng.integers(-1000, 1000, 300_000) * 0.25
    b = rng.integers(-1000, 1000, 300_000) * 0.125
    exprs = [fn("sqrt", fn("abs", col(0))), fn("power", col(0), 2.0) + fn("power", col(1), 2.0),
             fn("floor", fn("ceil", col(0) * 3.0) / 2.0), fn("round", col(1)) - fn("trunc", col(0)), fn("signum", col(0) - col(1))]
    got = project(ctx, [a, b], exprs)
    bits_equal(got[0], np.sqrt(np.abs(a)))
    # pow is within the device library's bound, not exact, even for integer powers (power(19, 2) = 361.00000000000006)
    within_ulps(got[1], np.asarray(a, np.longdouble) ** 2 + np.asarray(b, np.longdouble) ** 2)
    bits_equal(got[2], np.floor(np.ceil(a * 3.0) / 2.0))
    bits_equal(got[3], rust_round(b) - np.trunc(a))
    bits_equal(got[4], rust_signum(a - b))


# ---- positions and routing ------------------------------------------------------------------------------------------
def test_where_on_the_tma_kernel(ctx):
    rng = np.random.default_rng(5)
    a = rng.uniform(0, 10, 500_000)
    i = rng.integers(-100, 100, 500_000).astype(np.int32)
    (got,), k = traced(lambda: project(ctx, [a], [col(0)], pred=fn("sqrt", col(0)) > 2.0))
    bits_equal(got, a[np.sqrt(a) > 2.0])
    assert k == {"k_filter_project_tma<kFnDepth,4,1,0,0>"}
    # an integer column cast to Float64, as the planner casts it: the generic (not Float64-only) interpreter
    (g1, g2), k = traced(lambda: project(ctx, [a, i], [col(1), fn("abs", col(1).cast(A.FLOAT64))],
                                         pred=fn("power", col(1).cast(A.FLOAT64), 2.0) < 400.0))
    sel = i.astype(np.float64) ** 2 < 400.0
    assert np.array_equal(g1, i[sel])
    bits_equal(g2, np.abs(i[sel].astype(np.float64)))
    assert k == {"k_filter_project_tma<kFnDepth,4,0,0,0>"}


def test_where_and_projection_on_the_direct_kernel_with_nulls(ctx):
    rng = np.random.default_rng(6)
    n = 200_000
    v = rng.uniform(-4, 16, n)
    mask = rng.random(n) < 0.2
    w = rng.uniform(0.5, 2, n)
    pa_v = pa.array(v, mask=mask)
    pa_w = pa.array(w, mask=rng.random(n) < 0.1)
    # WHERE: a null predicate value reads as false
    (got,), k = traced(lambda: project(ctx, [pa_v], [col(0)], pred=fn("sqrt", col(0)) > 2.0))
    keep = ~mask & (np.sqrt(np.where(mask, 0, v)) > 2.0)
    bits_equal(got if not isinstance(got, tuple) else got[0], v[keep])
    assert k == {"k_filter_project<kFnDepth,1>"}
    # projections: null exactly where `arg + 0.0` is null, with value 0
    for e, plain in [(fn("sqrt", col(0)), col(0) + 0.0), (fn("power", col(0), col(1)), col(0) + col(1)),
                     (fn("atan2", col(1) + 0.0, col(0)), col(1) + col(0)), (fn("floor", fn("abs", col(0))), col(0) + 0.0)]:
        g, p = project(ctx, [pa_v, pa_w], [e, plain])
        assert isinstance(g, tuple) and isinstance(p, tuple)
        assert np.array_equal(g[1], p[1])
        assert (np.asarray(g[0])[~np.asarray(g[1], bool)] == 0).all()


def test_direct_kernel_without_nulls():
    os.environ["DFGPU_FP_KERNEL"] = "direct"
    try:
        c = engine.GpuContext(0)
    finally:
        del os.environ["DFGPU_FP_KERNEL"]
    try:
        a = np.random.default_rng(2).uniform(-3, 3, 100_000)
        (g,), k = traced(lambda: project(c, [a], [fn("exp", col(0))], pred=fn("abs", col(0)) < 1.0))
        with np.errstate(all="ignore"):
            within_ulps(g, np.exp(a[np.abs(a) < 1.0].astype(np.longdouble)))
        assert k == {"k_filter_project<kFnDepth,0>"}
    finally:
        c.close()


def agg(name, arg, distinct=False):
    return AggregateFunction(name, arg, distinct=distinct)


def aggregate(ctx, arrays, keys, aggs, pred=None):
    b = ctx.upload(arrays)
    try:
        r = ctx.aggregate([b], keys, aggs, 0, pred=pred)
        try:
            return r.columns()
        finally:
            r.free()
    finally:
        b.free()


def test_every_aggregate_argument_with_and_without_group_by(ctx):
    rng = np.random.default_rng(9)
    n = 400_000
    k = rng.integers(0, 300, n).astype(np.int64)
    v = rng.uniform(-100, 100, n)
    f = np.floor(v)  # integers: every sum is exact in any order
    aggs = [agg("min", fn("floor", col(1))), agg("max", fn("floor", col(1))), agg("sum", fn("floor", col(1))),
            agg("count", fn("sqrt", col(1))), agg("avg", fn("floor", col(1))), agg("count", fn("abs", fn("floor", col(1))), True)]
    got, kern = traced(lambda: aggregate(ctx, [k, v], [col(0)], aggs))
    assert kern & {"k_hash_agg<kFnDepth,0,0>", "k_hash_agg<kFnDepth,1,0>"} and "k_distinct_insert<kFnDepth,0>" in kern
    order = np.argsort(got[0])
    keys = np.unique(k)
    assert np.array_equal(got[0][order], keys)
    for g, red in zip(got[1:4], [np.minimum, np.maximum, np.add]):
        ref = red.reduceat(f[np.argsort(k, kind="stable")], np.searchsorted(np.sort(k), keys))
        bits_equal(np.asarray(g)[order], ref)
    assert np.array_equal(np.asarray(got[4])[order], np.bincount(k)[keys])
    sums = np.bincount(k, weights=f)[keys]
    bits_equal(np.asarray(got[5] if not isinstance(got[5], tuple) else got[5][0])[order], sums / np.bincount(k)[keys])
    dist = [len(np.unique(np.abs(f[k == g]))) for g in keys]
    assert np.array_equal(np.asarray(got[6])[order], dist)

    got, kern = traced(lambda: aggregate(ctx, [k, v], [], aggs))
    assert "k_reduce<kFnDepth,0>" in kern and "k_distinct_insert<kFnDepth,0>" in kern
    vals = [np.asarray(c if not isinstance(c, tuple) else c[0])[0] for c in got]
    bits_equal(vals[:3], [f.min(), f.max(), f.sum()])
    assert vals[3] == n and vals[4] == f.sum() / n and vals[5] == len(np.unique(np.abs(f)))


def test_fused_where_and_nulls_in_aggregates(ctx):
    rng = np.random.default_rng(10)
    n = 300_000
    k = rng.integers(0, 50, n).astype(np.int64)
    v = rng.uniform(-10, 10, n)
    mask = rng.random(n) < 0.3
    pv = pa.array(v, mask=mask)
    # fused WHERE with a function, over a null-free batch
    got, kern = traced(lambda: aggregate(ctx, [k, v], [col(0)], [agg("count", col(1))], pred=fn("sqrt", fn("abs", col(1))) > 2.0))
    keep = np.sqrt(np.abs(v)) > 2.0
    assert dict(zip(got[0].tolist(), got[1].tolist())) == {int(g): int(c) for g, c in zip(*np.unique(k[keep], return_counts=True))}
    assert kern & {"k_hash_agg<kFnDepth,0,0>", "k_hash_agg<kFnDepth,1,0>"}
    # nulls: COUNT and AVG of f(x) see what they see of x + 0.0
    with_fn = aggregate(ctx, [k, pv], [col(0)], [agg("count", fn("round", col(1))), agg("avg", fn("trunc", col(1)) * 0.0 + 1.0)])
    plain = aggregate(ctx, [k, pv], [col(0)], [agg("count", col(1) + 0.0), agg("avg", col(1) * 0.0 + 1.0)])
    a, b = dict(zip(with_fn[0].tolist(), with_fn[1].tolist())), dict(zip(plain[0].tolist(), plain[1].tolist()))
    assert a == b
    got, kern = traced(lambda: aggregate(ctx, [k, pv], [], [agg("count", fn("power", col(1), 2.0)), agg("max", fn("abs", col(1)))]))
    assert int(got[0][0]) == int((~mask).sum())
    assert "k_reduce<kFnDepth,1>" in kern


def test_aggregate_update_host(ctx):
    rng = np.random.default_rng(12)
    n = 3_000_000
    k = rng.integers(0, 1000, n).astype(np.int64)
    v = rng.integers(-1000, 1000, n).astype(np.float64) + 0.25
    r = ctx.aggregate_host([k, v], [col(0)], [agg("sum", fn("floor", col(1)))], chunk_rows=1 << 20)
    try:
        got = r.columns()
    finally:
        r.free()
    ref = np.bincount(k, weights=np.floor(v))
    bits_equal(np.asarray(got[1])[np.argsort(got[0])], ref[np.unique(k)])


def test_ten_million_rows_multi_wave(ctx):
    n = 12_000_000
    a = np.random.default_rng(13).uniform(0, 1, n)
    (got,), k = traced(lambda: project(ctx, [a], [fn("sqrt", col(0))], pred=fn("sin", col(0)) > 0.5))
    sel = np.sin(a) > 0.5  # sin is monotone on [0, 1]; rows within 3 ulp of the boundary may differ
    near = np.abs(np.sin(a) - 0.5) < 1e-15
    assert abs(len(got) - sel.sum()) <= near.sum()
    if not near.any():
        bits_equal(got, np.sqrt(a[sel]))
    assert k == {"k_filter_project_tma<kFnDepth,4,1,0,0>"}


def test_function_free_queries_keep_their_kernels(ctx):
    rng = np.random.default_rng(14)
    a = rng.uniform(0, 1, 1_000_000)
    k = rng.integers(0, 100, 1_000_000).astype(np.int64)
    _, kern = traced(lambda: project(ctx, [a], [col(0)], pred=col(0) > 0.5))
    assert kern == {"k_filter_project_tma<1,8,1,1,1>"}
    _, kern = traced(lambda: project(ctx, [a], [col(0) * 2.0 + 1.0], pred=col(0) > 0.5))
    assert kern == {"k_filter_project_tma<2,8,1,0,0>"}
    _, kern = traced(lambda: aggregate(ctx, [k, a], [col(0)], [agg("sum", col(1))]))
    assert not any("kFnDepth" in x for x in kern) and any(x.startswith("k_hash_agg_lean") for x in kern)
    _, kern = traced(lambda: aggregate(ctx, [k, a], [], [agg("sum", col(1) * 2.0)]))
    assert "k_reduce<1,0>" in kern and not any("kFnDepth" in x for x in kern)


# ---- SQL -------------------------------------------------------------------------------------------------------------
def test_sql_memory_and_csv():
    hctx = host.ExecutionContext(0)
    try:
        rng = np.random.default_rng(15)
        n = 100_000
        a = rng.integers(-50, 50, n).astype(np.int32)
        b = rng.uniform(0, 4, n)
        hctx.register_memory("t", [("a", a), ("b", b)], batch_size=30_000)
        rel = hctx.sql("SELECT SQRT(b), power(a, 2), Abs(a) FROM t WHERE signum(a) > 0")
        assert rel.schema() == [("SQRT", A.FLOAT64), ("power", A.FLOAT64), ("Abs", A.FLOAT64)]
        got = rows(rel)
        sel = a >= 0  # signum(+0.0) = 1.0
        bits_equal([r[0] for r in got], np.sqrt(b[sel]))
        within_ulps(np.array([r[1] for r in got]), a[sel].astype(np.longdouble) ** 2)
        bits_equal([r[2] for r in got], np.abs(a[sel]).astype(np.float64))
        hctx.register_memory("u", [("a", a), ("b", b)], batch_size=30_000)
        got = dict(rows(hctx.sql("SELECT a, SUM(floor(b)) FROM u WHERE ceil(b) >= 2 GROUP BY a")))
        keep = np.ceil(b) >= 2
        assert got == {int(g): float(np.floor(b[keep & (a == g)]).sum()) for g in np.unique(a[keep])}

        hctx.register_csv("c", os.path.join(DATA, "aggregate_test_1.csv"), [("a", A.INT32), ("b", A.FLOAT64)], 1024)
        data = np.genfromtxt(os.path.join(DATA, "aggregate_test_1.csv"), delimiter=",", skip_header=1)
        got = rows(hctx.sql("SELECT round(b), ln(a) FROM c WHERE a > 1"))
        sel = data[:, 0] > 1
        bits_equal([r[0] for r in got], rust_round(data[sel, 1]))
        within_ulps(np.array([r[1] for r in got]), np.log(data[sel, 0].astype(np.longdouble)))
    finally:
        hctx.close()


def test_sql_errors():
    hctx = host.ExecutionContext(0)
    try:
        for i in range(6):
            hctx.register_memory("t%d" % i, [("a", np.arange(10, dtype=np.int64)), ("b", np.arange(10, dtype=np.float64))])

        def err(sql):
            with pytest.raises(host.ExecutionError) as ei:
                rows(hctx.sql(sql))
            return ei.value

        e = err("SELECT foo(b) FROM t0")
        assert e.code == A.ERR_GENERAL and "Invalid function 'foo'" in str(e)
        e = err("SELECT power(b) FROM t1")
        assert e.code == A.ERR_EXECUTION and "'power' takes 2 arguments" in str(e)
        e = err("SELECT sqrt(SUM(b)) FROM t2")  # an aggregate inside a function is not planned as an aggregate
        assert e.code == A.ERR_EXECUTION and "SUM(#1)" in str(e)
        e = err("SELECT sqrt(b), COUNT(a) FROM t3 GROUP BY sqrt(b)")
        assert "Unsupported GROUP BY data type" in str(e)
        e = err("SELECT COUNT(a) FROM t4 GROUP BY CAST(sqrt(b) AS BIGINT)")
        assert "CAST not implemented for expression" in str(e)
        e = err("SELECT sqrt(9)")
        assert e.code == A.ERR_NOT_IMPLEMENTED
    finally:
        hctx.close()
