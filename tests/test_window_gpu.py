"""dfgpu_window through the C ABI and window functions through SQL, compared against the exact numpy reference of
tests/window_ref.py.  GPU required."""
import os

import numpy as np
import pyarrow as pa
import pytest

from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import engine, host
from datafusion_archive_b200.expr import BinaryExpr, col, lit

import groupby_ref as G
import window_ref as W

pytestmark = pytest.mark.gpu
DATA = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "data")
INTS = [A.INT8, A.INT16, A.INT32, A.INT64, A.UINT8, A.UINT16, A.UINT32, A.UINT64]
NUMERIC = INTS + [A.FLOAT32, A.FLOAT64]
AGGS = [W.MIN, W.MAX, W.SUM, W.COUNT, W.AVG]
RANKS = [W.ROW_NUMBER, W.RANK, W.DENSE_RANK]
TILE = 2048  # positions per tile of the segmented scan


@pytest.fixture(scope="module")
def ctx():
    c = engine.GpuContext(0)
    yield c
    c.close()


def values(rng, dtype, n, distinct=None):
    t = A.NP_OF[dtype]
    if dtype in (A.FLOAT32, A.FLOAT64):
        v = (rng.integers(0, distinct, n) if distinct else rng.standard_normal(n) * 1e3).astype(t)
        edges = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, np.finfo(t).max, np.finfo(t).min, np.finfo(t).tiny], dtype=t)
    else:
        info = np.iinfo(t)
        v = (rng.integers(0, distinct, n) if distinct else rng.integers(info.min, info.max, n, endpoint=True, dtype=t)).astype(t)
        edges = np.array([info.min, info.max, 0, 1, info.max - 1], dtype=t)
    k = min(n, len(edges), max(1, n // 8))
    v[rng.choice(n, size=k, replace=False)] = edges[:k]
    return v


def to_arrow(dtype, vals, valid):
    if dtype == A.UTF8:
        return pa.array(list(vals), type=pa.string(), mask=None if valid is None else ~np.asarray(valid, dtype=bool))
    return np.asarray(vals) if valid is None else G.arrow_nullable(np.asarray(vals), valid)


def run(ctx, cols, part, order, fns):
    """cols: [(dtype, values, valid)]; part: column indices; order: [(index, desc)]; fns: [(func, index or None)].
    Runs dfgpu_window over the uploaded columns and checks it against the reference."""
    n = len(cols[0][1])
    b = ctx.upload([to_arrow(*c) for c in cols])
    try:
        r = ctx.window(b, [(W.FUNC_CODE[f], col(a) if a is not None else None, 0) for f, a in fns], partition=[col(i) for i in part],
                       order=[col(i) for i, _ in order], desc=[d for _, d in order])
        got = r.columns()
        r.free()
    finally:
        b.free()
    exp = W.window(n, [cols[i] for i in part], [cols[i] + (d,) for i, d in order], [(f, cols[a] if a is not None else None) for f, a in fns])
    W.assert_matches(got, exp, "n=%d part=%s order=%s" % (n, part, order))
    return got


@pytest.mark.parametrize("kdt", NUMERIC + [A.UTF8])
@pytest.mark.parametrize("desc", [False, True])
def test_key_dtypes(ctx, kdt, desc):
    rng = np.random.default_rng(kdt * 2 + desc)
    n = 3 * TILE + 17
    if kdt == A.UTF8:
        pool = ["", "a", "a\0", "ab", "b", "é", "aaaaaaaa", "aaaaaaaab", "aaaaaaaa\0", "zz"]
        k = ([pool[i] for i in rng.integers(0, len(pool), n)], None)
        o = ([pool[i] for i in rng.integers(0, len(pool), n)], rng.random(n) < 0.8)
    else:
        k = (values(rng, kdt, n, distinct=7), None)
        o = (values(rng, kdt, n, distinct=50), rng.random(n) < 0.8)
    cols = [(kdt,) + k, (kdt,) + o, (A.INT64, values(rng, A.INT64, n), rng.random(n) < 0.9),
            (A.FLOAT64, rng.integers(-1000, 1000, n).astype(np.float64) / 8, None)]
    fns = [(f, None) for f in RANKS] + [(f, 2) for f in AGGS] + [(W.SUM, 3), (W.AVG, 3)]
    run(ctx, cols, [0], [(1, desc)], fns)
    run(ctx, cols, [1], [(0, not desc)], fns)  # a nullable partition key


@pytest.mark.parametrize("adt", NUMERIC)
def test_every_function_every_argument_dtype(ctx, adt):
    rng = np.random.default_rng(100 + adt)
    n = 2 * TILE + 3
    cols = [(A.INT32, rng.integers(0, 5, n).astype(np.int32), None), (A.INT16, rng.integers(0, 40, n).astype(np.int16), rng.random(n) < 0.9),
            (adt, values(rng, adt, n), rng.random(n) < 0.85)]
    fns = [(f, 2) for f in AGGS] + [(f, None) for f in RANKS]
    run(ctx, cols, [0], [(1, False)], fns)  # running frames
    run(ctx, cols, [0], [], fns)            # whole partitions
    run(ctx, cols, [], [], fns)             # OVER ()


@pytest.mark.parametrize("n", [0, 1, 2, TILE - 1, TILE, TILE + 1, 2 * TILE - 1, 2 * TILE + 1])
def test_sizes_and_tile_boundaries(ctx, n):
    rng = np.random.default_rng(n)
    cols = [(A.INT64, rng.integers(0, 3, n), None), (A.FLOAT64, rng.standard_normal(n), rng.random(n) < 0.7),
            (A.INT32, rng.integers(-5, 5, n).astype(np.int32), None)]
    fns = [(f, None) for f in RANKS] + [(f, 1) for f in AGGS] + [(W.SUM, 2)]
    run(ctx, cols, [0], [(2, False)], fns)
    run(ctx, cols, [], [(2, True)], fns)


def test_one_partition_many_tiles_and_singletons(ctx):
    rng = np.random.default_rng(7)
    n = 40 * TILE + 5
    cols = [(A.INT64, np.zeros(n, np.int64), None), (A.INT64, np.arange(n), None), (A.INT32, rng.integers(-9, 9, n).astype(np.int32), None),
            (A.FLOAT64, rng.integers(-99, 99, n).astype(np.float64) / 4, rng.random(n) < 0.5)]
    fns = [(f, None) for f in RANKS] + [(W.SUM, 2), (W.MIN, 2), (W.MAX, 3), (W.AVG, 3), (W.COUNT, 3), (W.SUM, 3)]
    run(ctx, cols, [0], [(2, False)], fns)  # one partition over 41 tiles, many peers
    run(ctx, cols, [1], [(2, False)], fns)  # every row its own partition


def test_all_null_frames_and_float_edges(ctx):
    n = 64
    v = np.array([np.nan, -0.0, 0.0, np.inf, -np.inf, 1.5, np.nan, -2.0] * 8)
    valid = np.ones(n, dtype=bool)
    valid[:8] = False  # partition 0 is all null
    k = np.repeat(np.arange(8), 8)
    cols = [(A.INT64, k, None), (A.FLOAT64, v, valid), (A.FLOAT32, v.astype(np.float32), valid), (A.INT64, np.arange(n) % 3, None)]
    fns = [(f, c) for f in AGGS for c in (1, 2)]
    run(ctx, cols, [0], [(3, False)], fns)
    run(ctx, cols, [0], [], fns)
    got = run(ctx, [(A.FLOAT64, np.full(9, np.nan), None), (A.INT64, np.zeros(9, np.int64), None)], [1], [], [(W.MIN, 0), (W.MAX, 0)])
    assert np.isnan(got[0]).all() and np.isnan(got[1]).all()


def test_float_keys_partition_by_encoding(ctx):
    k = np.array([0.0, -0.0, np.nan, -np.nan, np.inf, 0.0, -0.0, np.nan])
    cols = [(A.FLOAT64, k, np.array([1, 1, 1, 1, 1, 0, 0, 1], bool)), (A.INT64, np.arange(8), None)]
    got = run(ctx, cols, [0], [], [(W.COUNT, 1), (W.ROW_NUMBER, None)])
    # two nulls share a partition, all NaNs share one, -0.0 and +0.0 are two
    assert list(got[0]) == [1, 1, 3, 3, 1, 2, 2, 3]


def test_expression_keys_and_arguments(ctx):
    rng = np.random.default_rng(3)
    n = 5000
    a, b = rng.integers(-50, 50, n), rng.integers(0, 9, n)
    bt = ctx.upload([a, b])
    try:
        r = ctx.window(bt, [(A.AGG_SUM, BinaryExpr(col(0), A.OP_MUL, lit(2)), 0), (A.WIN_RANK, None, 0)],
                       partition=[BinaryExpr(col(1), A.OP_DIV, lit(3))], order=[BinaryExpr(col(0), A.OP_ADD, col(1))], desc=[True])
        got = r.columns()
        r.free()
    finally:
        bt.free()
    exp = W.window(n, [(A.INT64, b // 3, None)], [(A.INT64, a + b, None, True)], [(W.SUM, (A.INT64, a * 2, None)), (W.RANK, None)])
    W.assert_matches(got, exp)


def test_large_input(ctx):
    n = (1 << 24) + 1
    rng = np.random.default_rng(5)
    k = rng.integers(0, 1000, n)
    v = rng.integers(-1000, 1000, n).astype(np.int32)
    b = ctx.upload([k, v])
    try:
        r = ctx.window(b, [(A.WIN_ROW_NUMBER, None, 0), (A.AGG_SUM, col(1), 0), (A.AGG_COUNT, col(1), 0)], partition=[col(0)])
        got = r.columns()
        r.free()
    finally:
        b.free()
    order = np.lexsort([np.arange(n), k])
    sk = k[order]
    start = np.ones(n, dtype=bool)
    start[1:] = sk[1:] != sk[:-1]
    pf = np.maximum.accumulate(np.where(start, np.arange(n), 0))
    rn = np.empty(n, np.uint64)
    rn[order] = np.arange(n) - pf + 1
    assert np.array_equal(got[0], rn)
    tot = np.bincount(k, weights=v, minlength=1000).astype(np.int64)
    assert np.array_equal(got[1], tot[k].astype(np.int32))
    assert np.array_equal(got[2], np.bincount(k, minlength=1000)[k].astype(np.uint64))


def test_float_sum_is_deterministic(ctx):
    rng = np.random.default_rng(11)
    n = 300_000
    v = rng.standard_normal(n) * 10.0 ** rng.integers(-8, 8, n)
    b = ctx.upload([rng.integers(0, 3, n), v, rng.integers(0, 1000, n)])
    try:
        outs = []
        for _ in range(2):
            r = ctx.window(b, [(A.AGG_SUM, col(1), 0), (A.AGG_AVG, col(1), 0)], partition=[col(0)], order=[col(2)])
            outs.append(r.columns())
            r.free()
    finally:
        b.free()
    for x, y in zip(*outs):
        assert np.array_equal(x.view(np.uint64), y.view(np.uint64))


def test_refusals(ctx):
    b = ctx.upload([np.arange(4), np.array([True, False, True, True]), ["a", "b", "c", "d"]])
    try:
        with pytest.raises(engine.DfGpuError) as e:
            ctx.window(b, [(A.WIN_RANK, None, 0)], partition=[col(1)])
        assert e.value.code == A.ERR_NOT_IMPLEMENTED and "Boolean" in e.value.msg
        with pytest.raises(engine.DfGpuError) as e:
            ctx.window(b, [(A.AGG_COUNT_DISTINCT, col(0), 0)], partition=[col(0)])
        assert e.value.code == A.ERR_NOT_IMPLEMENTED
        for f in (A.AGG_SUM, A.AGG_MIN, A.AGG_AVG):
            with pytest.raises(engine.DfGpuError) as e:
                ctx.window(b, [(f, col(2), 0)])
            assert e.value.code == A.ERR_EXECUTION and e.value.msg == "Unsupported data type for aggregate: Utf8"
    finally:
        b.free()


def test_kernels_have_no_fallback(ctx):
    """The post-sort work runs in the window kernels (DFGPU_TRACE names every launch)."""
    import subprocess
    import sys
    code = ("from datafusion_archive_b200 import engine, _abi as A\nfrom datafusion_archive_b200.expr import col\nimport numpy as np\n"
            "c = engine.GpuContext(0)\nb = c.upload([np.arange(5000) % 7, np.arange(5000.0)])\n"
            "c.window(b, [(A.AGG_SUM, col(1), 0), (A.WIN_RANK, None, 0)], partition=[col(0)], order=[col(1)]).columns()\n")
    env = dict(os.environ, DFGPU_TRACE="1")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, cwd=os.path.dirname(os.path.dirname(__file__)))
    assert out.returncode == 0, out.stderr
    text = out.stdout + out.stderr
    for k in ("k_win_flags", "k_win_bounds", "k_win_tile_reduce", "k_win_carry", "k_win_tile_scan", "k_win_out", "k_sort_scatter"):
        assert k in text, k


# ---- SQL ---------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def sql():
    c = host.ExecutionContext(0)
    yield c
    c.close()


def collect(rel):
    """The relation's batches as whole columns, a nullable column as (values, valid)."""
    batches = rel.collect()
    if not batches:
        return None
    out = []
    for i in range(len(batches[0])):
        parts = [b[i] for b in batches]
        if any(isinstance(p, tuple) for p in parts):
            vals = np.concatenate([p[0] if isinstance(p, tuple) else p for p in parts])
            valid = np.concatenate([p[1] if isinstance(p, tuple) else np.ones(len(p), bool) for p in parts])
            out.append((vals, valid))
        else:
            out.append(np.concatenate(parts) if not isinstance(parts[0], list) else sum(parts, []))
    return out


def table(sql, n=30_000, seed=0):
    """Registers tables t and d (a DataSource is read once: each query registers them again, with the same rows)."""
    rng = np.random.default_rng(seed)
    k = rng.integers(0, 40, n)
    v = rng.integers(-1000, 1000, n).astype(np.int32)
    x = rng.integers(-4000, 4000, n) / 16.0
    xvalid = rng.random(n) < 0.9
    city = np.array(["Rome", "oslo", "Lima", "", "Bern", "rome"])[rng.integers(0, 6, n)]
    sql.register_memory("t", [("k", k), ("v", v), ("x", G.arrow_nullable(x, xvalid)), ("city", pa.array(list(city)))])
    sql.register_memory("d", [("dk", np.arange(0, 40, 3)), ("w", np.arange(0, 40, 3) * 10)])


def col_of(c):
    return (c[0], c[1]) if isinstance(c, tuple) else (c, None)


def test_sql_functions_and_specifications(sql):
    table(sql)
    inp = collect(sql.sql("SELECT k, v, x, city FROM t"))
    table(sql)
    got = collect(sql.sql(
        "SELECT ROW_NUMBER() OVER (PARTITION BY k ORDER BY v DESC), rank() OVER (PARTITION BY city ORDER BY k), "
        "DENSE_RANK() OVER (ORDER BY city DESC, k), SUM(v) OVER (PARTITION BY k ORDER BY v DESC), COUNT(x) OVER (PARTITION BY city), "
        "MIN(x) OVER (PARTITION BY k ORDER BY v DESC), MAX(v) OVER (), AVG(x) OVER (PARTITION BY city ORDER BY k), "
        "x - AVG(x) OVER (PARTITION BY city ORDER BY k), SUM(v) OVER (PARTITION BY k ORDER BY v DESC) * 2 FROM t"))
    k, v, (x, xv), city = inp[0], inp[1], col_of(inp[2]), inp[3]
    K, V, X, C = (A.INT64, k, None), (A.INT32, v, None), (A.FLOAT64, x, xv), (A.UTF8, city, None)
    n = len(k)
    checks = [
        (0, [K], [V + (True,)], W.ROW_NUMBER, None), (1, [C], [K + (False,)], W.RANK, None), (2, [], [C + (True,), K + (False,)], W.DENSE_RANK, None),
        (3, [K], [V + (True,)], W.SUM, V), (4, [C], [], W.COUNT, X), (5, [K], [V + (True,)], W.MIN, X), (6, [], [], W.MAX, V),
        (7, [C], [K + (False,)], W.AVG, X),
    ]
    for i, part, order, f, arg in checks:
        W.assert_matches([got[i]], W.window(n, part, order, [(f, arg)]), "column %d" % i)
    g8, m8 = col_of(got[8])
    g7, m7 = col_of(got[7])
    ok = np.ones(n, dtype=bool) if xv is None else xv.copy()
    for m in (m7, m8):
        if m is not None:
            ok &= m
    assert np.array_equal(g8[ok].view(np.uint64), (x[ok] - g7[ok]).view(np.uint64))
    assert np.array_equal(got[9], (got[3].astype(np.int64) * 2).astype(np.int64)) or np.array_equal(got[9], got[3] * np.int32(2))


def test_sql_where_join_and_in(sql):
    table(sql)
    where = "WHERE v > 0 AND city <> 'oslo'"
    inp = collect(sql.sql("SELECT k, v, x FROM t " + where))
    table(sql)
    got = collect(sql.sql("SELECT v, RANK() OVER (PARTITION BY k ORDER BY x), SUM(x) OVER (PARTITION BY k) FROM t " + where))
    k, v, (x, xv) = inp[0], inp[1], col_of(inp[2])
    assert np.array_equal(got[0], v)  # input order
    W.assert_matches(got[1:], W.window(len(k), [(A.INT64, k, None)], [(A.FLOAT64, x, xv, False)], [(W.RANK, None)]) +
                     W.window(len(k), [(A.INT64, k, None)], [], [(W.SUM, (A.FLOAT64, x, xv))]))
    table(sql)
    inp = collect(sql.sql("SELECT k, w FROM t JOIN d ON k = dk"))
    table(sql)
    got = collect(sql.sql("SELECT w, COUNT(*) OVER (PARTITION BY w), ROW_NUMBER() OVER (ORDER BY w DESC) FROM t JOIN d ON k = dk"))
    kk, w = inp[0], inp[1]
    assert np.array_equal(got[0], w)
    W.assert_matches(got[1:], W.window(len(w), [(A.INT64, w, None)], [], [(W.COUNT, (A.INT64, kk, None))]) +
                     W.window(len(w), [], [(A.INT64, w, None, True)], [(W.ROW_NUMBER, None)]))
    table(sql)
    inp = collect(sql.sql("SELECT k, v FROM t WHERE k IN (SELECT dk FROM d)"))
    table(sql)
    got = collect(sql.sql("SELECT MAX(v) OVER (PARTITION BY k), DENSE_RANK() OVER (ORDER BY k) FROM t WHERE k IN (SELECT dk FROM d)"))
    W.assert_matches(got, W.window(len(inp[0]), [(A.INT64, inp[0], None)], [], [(W.MAX, (A.INT32, inp[1], None))]) +
                     W.window(len(inp[0]), [], [(A.INT64, inp[0], None, False)], [(W.DENSE_RANK, None)]))


def test_sql_over_nothing_and_empty(sql):
    table(sql, n=5000)
    got = collect(sql.sql("SELECT ROW_NUMBER() OVER (), COUNT(1) OVER () FROM t"))
    assert np.array_equal(got[0], np.arange(1, 5001, dtype=np.uint64)) and (got[1] == 5000).all()
    table(sql, n=5000)
    assert collect(sql.sql("SELECT RANK() OVER (ORDER BY v) FROM t WHERE v > 100000")) is None


def test_sql_golden_csv(sql):
    sql.register_csv("t1", os.path.join(DATA, "aggregate_test_1.csv"), [("a", A.INT32), ("b", A.FLOAT64)], 1024)
    got = collect(sql.sql("SELECT a, b, RANK() OVER (PARTITION BY a ORDER BY b DESC), SUM(b) OVER (PARTITION BY a) FROM t1"))
    a, b = got[0], got[1]
    W.assert_matches(got[2:], W.window(len(a), [(A.INT32, a, None)], [(A.FLOAT64, b, None, True)], [(W.RANK, None)]) +
                     W.window(len(a), [(A.INT32, a, None)], [], [(W.SUM, (A.FLOAT64, b, None))]))


def test_sql_order_by_keeps_its_error(sql):
    table(sql, n=100)
    with pytest.raises(host.ExecutionError) as e:
        collect(sql.sql("SELECT k, RANK() OVER (ORDER BY v) FROM t ORDER BY k"))
    assert e.value.code == A.ERR_NOT_IMPLEMENTED
