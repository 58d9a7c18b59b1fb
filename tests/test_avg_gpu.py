"""AVG(x) on the GPU against the exact reference of tests/groupby_ref.py.  Inputs are integers or multiples of 1/8 small
enough that every f64 sum is exact in any order, so results must equal the f64 quotient of the sum of the non-null values
and their count; random floats are compared with math.fsum at rtol 1e-12.  Under DFGPU_TRACE each dispatch case asserts
the kernel that ran."""
import math
import os

import numpy as np
import pyarrow as pa
import pytest

import groupby_ref as G
from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import engine, host
from datafusion_archive_b200.expr import AggregateFunction, col, lit
from kernel_trace import traced_set as traced

pytestmark = pytest.mark.gpu

DATA = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "data")
INTS = [np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64]
ALL = INTS + [np.float32, np.float64]


@pytest.fixture(scope="module")
def ctx():
    c = engine.GpuContext(0)
    yield c
    c.close()


def avg(arg):
    return AggregateFunction("avg", arg)


def gpu(ctx, batches, keys, aggs, pred=None, expected=0):
    """Aggregate over `batches` (lists of columns); returns the result columns."""
    bs = [ctx.upload(b) for b in batches]
    try:
        r = ctx.aggregate(bs, keys, aggs, expected, pred=pred)
        try:
            return r.columns()
        finally:
            r.free()
    finally:
        for b in bs:
            b.free()


def run(ctx, batches, keys, aggs, pred=None, expected=0):
    return traced(lambda: gpu(ctx, batches, keys, aggs, pred, expected))


def check(got, keys, v, where=None):
    """`got` (the keys, then AVG(v)) against groupby_ref."""
    G.assert_matches(got, G.aggregate(keys, [(G.AVG, v)], where=where))


def values(dt, n, rng):
    """Values whose f64 sums are exact in any order: small integers, multiples of 1/8 for floats, plus the extremes for
    integers narrower than 32 bits."""
    if np.dtype(dt).kind == "f":
        return (rng.integers(-4000, 4000, n) / 8).astype(dt)
    info = np.iinfo(dt)
    if info.bits <= 16:
        v = rng.integers(info.min, info.max, n, endpoint=True).astype(dt)
    else:
        lo = 0 if info.min == 0 else -(1 << 20)
        v = rng.integers(lo, 1 << 20, n).astype(dt)
    return v


@pytest.mark.parametrize("kdt", INTS, ids=lambda d: np.dtype(d).name)
@pytest.mark.parametrize("vdt", ALL, ids=lambda d: np.dtype(d).name)
def test_key_by_argument_dtype(ctx, kdt, vdt):
    rng = np.random.default_rng(int(np.dtype(kdt).num) * 100 + np.dtype(vdt).num)
    n = 20_000
    k = rng.integers(0, 60, n).astype(kdt)
    v = values(vdt, n, rng)
    got, _ = run(ctx, [[k, v]], [col(0)], [avg(col(1))])
    check(got, [k], v)


def test_lean_equals_sum_over_count(ctx):
    rng = np.random.default_rng(1)
    n = 2_000_000
    k = rng.integers(0, 100_000, n).astype(np.int64)
    v = rng.random(n) * 100.0 - 50.0  # not exact: the lean kernel's sum order decides the last bits
    got, names = run(ctx, [[k, v]], [col(0)], [avg(col(1))])
    assert "k_hash_agg_lean<12,1>" in names, sorted(names)
    assert "k_avg_finish" in names
    sc, names2 = run(ctx, [[k, v]], [col(0)], [AggregateFunction("sum", col(1)), AggregateFunction("count", col(1))])
    assert "k_hash_agg_lean<12,1>" in names2
    o, so = np.argsort(got[0]), np.argsort(sc[0])
    assert np.array_equal(got[0][o], sc[0][so])
    assert got[1][o] == pytest.approx(sc[1][so] / sc[2][so], rel=1e-12)
    # exact data: the two queries agree bit for bit
    w = (rng.integers(-800, 800, n) / 8).astype(np.float64)
    got, _ = run(ctx, [[k, w]], [col(0)], [avg(col(1))])
    sc, _ = run(ctx, [[k, w]], [col(0)], [AggregateFunction("sum", col(1)), AggregateFunction("count", col(1))])
    o, so = np.argsort(got[0]), np.argsort(sc[0])
    assert np.array_equal(got[0][o], sc[0][so]) and np.array_equal(got[1][o], sc[1][so] / sc[2][so])
    check(got, [k], w)


@pytest.mark.parametrize("vdt", [np.int32, np.int64, np.float32], ids=lambda d: np.dtype(d).name)
def test_plain_kernel(ctx, vdt):
    rng = np.random.default_rng(2)
    n = 500_000
    k = rng.integers(0, 5000, n).astype(np.int64)
    v = values(vdt, n, rng)
    got, names = run(ctx, [[k, v]], [col(0)], [avg(col(1))])
    assert "k_hash_agg_plain<2,0>" in names and not any(x.startswith("k_hash_agg_lean") for x in names), sorted(names)
    check(got, [k], v)


def test_interpreter_expression_argument(ctx):
    rng = np.random.default_rng(3)
    n = 300_000
    k = rng.integers(0, 3000, n).astype(np.int64)
    a = rng.integers(-1000, 1000, n).astype(np.int64)
    b = rng.integers(-1000, 1000, n).astype(np.int64)
    got, names = run(ctx, [[k, a, b]], [col(0)], [avg(col(1) * lit(3, A.INT64) + col(2))])
    assert any(x.startswith("k_hash_agg<") and x.endswith(",0,0>") for x in names), sorted(names)
    check(got, [k], a * 3 + b)


def test_nulls_kernel_and_all_null_group(ctx):
    rng = np.random.default_rng(4)
    n = 200_000
    k = rng.integers(0, 500, n).astype(np.int32)
    v = rng.integers(-100, 100, n).astype(np.int64)
    valid = rng.random(n) < 0.6
    valid[k == 7] = False  # a group whose values are all null
    arr = pa.array(v, mask=~valid)
    got, names = run(ctx, [[k, arr]], [col(0)], [avg(col(1)), AggregateFunction("count", col(1))])
    assert "k_hash_agg<8,0,1>" in names, sorted(names)
    G.assert_matches(got, G.aggregate([k], [(G.AVG, (v, valid)), (G.COUNT, (v, valid))]))
    g7 = np.flatnonzero(got[0] == 7)[0]
    assert not got[1][1][g7] and got[2][g7] == 0
    # the result reports its null count
    bs = [ctx.upload([k, arr])]
    r = ctx.aggregate(bs, [col(0)], [avg(col(1))])
    nulls = engine.C.c_int64()
    engine.check(engine.lib().dfgpu_result_col_nulls(r.h, 1, engine.C.byref(nulls)))
    assert nulls.value == 1
    r.free()
    bs[0].free()
    # null-free groups under the same nullable column carry no extra nulls; without GROUP BY nulls are skipped too
    whole, names = run(ctx, [[arr]], [], [avg(col(0))])
    assert "k_reduce<8,1>" in names
    assert not isinstance(whole[0], tuple)  # a non-null AVG carries no bitmap
    assert float(whole[0][0]) == float(np.float64(v[valid].sum()) / valid.sum())


def test_front_table(ctx):
    rng = np.random.default_rng(5)
    n = 1_200_000
    batches = []
    for _ in range(2):  # the second batch sees <= 1024 groups after 2^20 rows: the shared-memory front table
        k = rng.integers(0, 300, n).astype(np.int64)
        v = rng.integers(-5000, 5000, n).astype(np.int32)
        batches.append([k, v])
    got, names = run(ctx, batches, [col(0)], [avg(col(1))])
    assert "k_hash_agg_plain<2,1>" in names, sorted(names)
    k = np.concatenate([b[0] for b in batches])
    v = np.concatenate([b[1] for b in batches])
    check(got, [k], v)


def test_wide_composite_key(ctx):
    rng = np.random.default_rng(6)
    n = 200_000
    k1 = rng.integers(-(1 << 40), 1 << 40, 40)[rng.integers(0, 40, n)].astype(np.int64)
    k2 = rng.integers(0, 30, n).astype(np.int64)
    v = (rng.integers(-800, 800, n) / 8).astype(np.float32)
    got, names = run(ctx, [[k1, k2, v]], [col(0), col(1)], [avg(col(2))])
    assert "k_hash_agg_wide<8,0>" in names, sorted(names)
    check(got, [k1, k2], v)


def test_utf8_key(ctx):
    rng = np.random.default_rng(7)
    n = 50_000
    words = ["w%d" % i for i in range(97)]
    idx = rng.integers(0, len(words), n)
    s = [words[i] for i in idx]
    v = rng.integers(-1000, 1000, n).astype(np.int16)
    got, names = run(ctx, [[s, v]], [col(0)], [avg(col(1))])
    assert "k_utf8_group_verify" in names
    index = {w: i for i, w in enumerate(words)}
    check([np.array([index[w] for w in got[0]])] + got[1:], [idx], v)


def test_table_growth_with_replay(ctx):
    rng = np.random.default_rng(8)
    per = 1_500_000
    keys = rng.permutation(3 * per).astype(np.int64)  # 4.5e6 distinct groups in batches too small for the prefix estimate
    batches = [[keys[i * per:(i + 1) * per], (keys[i * per:(i + 1) * per] % 1000).astype(np.int32)] for i in range(3)]
    extra = [[keys[:per], (keys[:per] % 1000 + 1).astype(np.int32)]]  # every group of the first batch gets a second value
    got, names = run(ctx, batches + extra, [col(0)], [avg(col(1)), AggregateFunction("count", col(1))])
    assert "k_merge" in names, sorted(names)
    k = np.concatenate([b[0] for b in batches + extra])
    v = np.concatenate([b[1] for b in batches + extra])
    g = got[0]
    order = np.argsort(g)
    vals = np.asarray(got[1])[order]
    kk = np.sort(keys)
    assert np.array_equal(g[order], kk)
    s = np.zeros(3 * per)
    c = np.zeros(3 * per)
    np.add.at(s, k, v.astype(np.float64))
    np.add.at(c, k, 1)
    assert np.array_equal(vals, s[kk] / c[kk])


def test_reduce_kernels(ctx):
    rng = np.random.default_rng(9)
    v = (rng.integers(-8000, 8000, 3_000_001) / 8).astype(np.float64)
    got, names = run(ctx, [[v]], [], [avg(col(0))])
    assert "k_reduce_f64" in names, sorted(names)
    assert float(got[0][0]) == float(np.float64(v.sum()) / len(v))
    i = rng.integers(-(1 << 20), 1 << 20, 3_000_001).astype(np.int32)
    got, names = run(ctx, [[i]], [], [avg(col(0))])
    assert "k_reduce<1,0>" in names, sorted(names)
    assert float(got[0][0]) == float(np.float64(i.astype(np.int64).sum()) / len(i))
    # random floats: against a correctly rounded sum
    w = rng.standard_normal(1_000_000) * 1e3
    got, _ = run(ctx, [[w]], [], [avg(col(0))])
    assert float(got[0][0]) == pytest.approx(math.fsum(w) / len(w), rel=1e-12)


@pytest.mark.parametrize("case", ["zero_rows", "no_row_passes", "all_null"])
def test_scalar_null(ctx, case):
    v = np.arange(1000, dtype=np.float64)
    where = None
    if case == "zero_rows":
        batches = [[v[:0]]]
    elif case == "no_row_passes":
        batches, where = [[v]], col(0) < -1.0
    else:
        batches = [[pa.array(v, mask=np.ones(len(v), bool))]]
    got, _ = run(ctx, batches, [], [avg(col(0)), AggregateFunction("count", col(0))], pred=where)
    assert isinstance(got[0], tuple) and not got[0][1][0]
    assert int(np.asarray(got[1] if not isinstance(got[1], tuple) else got[1][0])[0]) == 0


def test_no_batch(ctx):
    keep = []
    aggarr = A.make_aggs([(A.AGG_AVG, col(0).program([A.FLOAT64]), 0)], keep)
    st = engine.C.c_void_p()
    engine.check(engine.lib().dfgpu_aggregate_create(ctx.h, None, None, 0, aggarr, 1, 0, engine.C.byref(st)))
    try:
        out = engine.C.c_void_p()
        engine.check(engine.lib().dfgpu_aggregate_finish(st, engine.C.byref(out)))
        r = engine.Result(ctx, out)
        (val,) = r.columns()
        r.free()
    finally:
        engine.lib().dfgpu_aggregate_free(st)
    assert isinstance(val, tuple) and not val[1][0]


def test_float_edges(ctx):
    inf, nan = np.inf, np.nan
    groups = {0: [1.0, nan, 2.0], 1: [inf, -inf, 3.0], 2: [inf, 5.0], 3: [-inf, -inf], 4: [0.5, 0.25]}
    k = np.array([g for g, xs in groups.items() for _ in xs], dtype=np.int64)
    v = np.array([x for xs in groups.values() for x in xs], dtype=np.float64)
    for keys, arrays in (([col(0)], [k, v]), ([col(0)], [k.astype(np.int32), v])):
        got, _ = run(ctx, [arrays], keys, [avg(col(1))])
        check(got, arrays[:1], v)
    for g in (1, 2):
        whole, _ = run(ctx, [[v[k == g]]], [], [avg(col(0))])
        check(whole, [], v[k == g])


def test_float32_subnormals_are_kept(ctx):
    tiny = np.finfo(np.float32).smallest_subnormal
    v = np.array([tiny, 3 * tiny, tiny * 2, tiny], dtype=np.float32)
    k = np.zeros(len(v), np.int64)
    got, _ = run(ctx, [[k, v]], [col(0)], [avg(col(1))])
    assert got[1][0] == np.float64(tiny) * 7 / 4 != 0.0
    check(got, [k], v)
    whole, _ = run(ctx, [[v]], [], [avg(col(0))])
    check(whole, [], v)
    valid = np.array([1, 1, 0, 1], bool)
    nul, _ = run(ctx, [[k, pa.array(v, mask=~valid)]], [col(0)], [avg(col(1))])
    check(nul, [k], (v, valid))


def test_int64_extremes(ctx):
    lo, hi = np.iinfo(np.int64).min, np.iinfo(np.int64).max
    k = np.array([0, 0, 0, 1, 1, 2, 3], dtype=np.int64)
    v = np.array([hi, hi, lo, lo, lo, hi, (1 << 53) + 1], dtype=np.int64)
    got, _ = run(ctx, [[k, v]], [col(0)], [avg(col(1))])
    check(got, [k], v)  # each value rounded when widened: 2^63 / 3, -2^63, 2^63, 2^53
    u = np.array([np.iinfo(np.uint64).max, 1], dtype=np.uint64)
    whole, _ = run(ctx, [[u]], [], [avg(col(0))])
    assert float(whole[0][0]) == 2.0 ** 63  # 2^64 - 1 widens to 2^64, and 2^64 + 1 rounds to 2^64


def test_batches_where_and_mixed(ctx):
    rng = np.random.default_rng(10)
    n = 600_000
    k = rng.integers(0, 2000, n).astype(np.int64)
    v = rng.integers(-50, 50, n).astype(np.int32)
    w = (rng.integers(-80, 80, n) / 8).astype(np.float64)
    batches = [[k[i::3], v[i::3], w[i::3]] for i in range(3)]
    kk = np.concatenate([b[0] for b in batches])
    vv = np.concatenate([b[1] for b in batches])
    ww = np.concatenate([b[2] for b in batches])
    got, _ = run(ctx, batches, [col(0)], [avg(col(2))], pred=col(1) > lit(10, A.INT32))
    check(got, [kk], ww, where=vv > 10)
    mixed = [AggregateFunction("sum", col(1)), avg(col(1)), AggregateFunction("count", col(1), distinct=True), avg(col(2)),
             AggregateFunction("min", col(2))]
    got, _ = run(ctx, batches, [col(0)], mixed)
    base, _ = run(ctx, batches, [col(0)], [mixed[0], mixed[2], mixed[4]])
    o, ob = np.argsort(got[0]), np.argsort(base[0])
    for i, j in ((1, 1), (3, 2), (5, 3)):
        assert np.array_equal(np.asarray(got[i])[o], np.asarray(base[j])[ob])
    exp = [(G.SUM, vv), (G.AVG, vv), (G.COUNT_DISTINCT, vv), (G.AVG, ww), (G.MIN, ww)]
    G.assert_matches(got, G.aggregate([kk], exp))
    whole, _ = run(ctx, batches, [], mixed)
    G.assert_matches(whole, G.aggregate([], exp))


def test_update_host_chunks(ctx):
    rng = np.random.default_rng(11)
    n = 9_000_000
    k = rng.integers(0, 100_000, n).astype(np.int64)
    v = rng.integers(0, 100, n).astype(np.int64)
    r = ctx.aggregate_host([k, v], keys=[col(0)], aggs=[avg(col(1))], chunk_rows=4 << 20)
    chunked = r.columns()
    r.free()
    check(chunked, [k], v)


def test_errors(ctx):
    k = np.array([1, 2, 1], dtype=np.int64)
    for arg in (np.array([True, False, True]), ["a", "b", "c"]):
        errs = []
        for f in ("sum", "avg"):
            with pytest.raises(engine.DfGpuError) as e:
                gpu(ctx, [[k, arg]], [col(0)], [AggregateFunction(f, col(1))])
            errs.append((e.value.code, e.value.msg))
        assert errs[0] == errs[1], errs
    keep = []
    for odt in (A.INT64, A.FLOAT32, A.UINT64):
        aggarr = A.make_aggs([(A.AGG_AVG, col(0).program([A.FLOAT64]), odt)], keep)
        st = engine.C.c_void_p()
        rc = engine.lib().dfgpu_aggregate_create(ctx.h, None, None, 0, aggarr, 1, 0, engine.C.byref(st))
        assert rc == A.ERR_EXECUTION
        assert "unexpected type when creating array from aggregate map" in engine.lib().dfgpu_last_error().decode()
    # each AVG takes two of the 8 accumulator words
    with pytest.raises(engine.DfGpuError) as e:
        gpu(ctx, [[k, k.astype(np.float64)]], [col(0)], [avg(col(1))] * 4 + [AggregateFunction("sum", col(1))])
    assert e.value.code == A.ERR_NOT_IMPLEMENTED and "accumulator words" in e.value.msg
    got = gpu(ctx, [[k, k.astype(np.float64)]], [col(0)], [avg(col(1))] * 4)
    G.assert_matches(got, G.aggregate([k], [(G.AVG, k.astype(np.float64))] * 4))


def rows(rel):
    """The rows of a relation as tuples, None for a null."""
    out = []
    for batch in rel.collect():
        cols = []
        for c in batch:
            if isinstance(c, tuple):
                cols.append([x if ok else None for x, ok in zip(list(c[0]), c[1])])
            else:
                cols.append(list(c))
        out.extend(zip(*cols))
    return out


def test_sql(ctx):
    hctx = host.ExecutionContext(0)
    try:
        hctx.register_csv("t1", os.path.join(DATA, "aggregate_test_1.csv"), [("a", A.INT32), ("b", A.FLOAT64)], 1024)
        rel = hctx.sql("SELECT a, AVG(b), AVG(a) FROM t1 GROUP BY a")
        assert [dt for _, dt in rel.schema()][1:] == [A.FLOAT64, A.FLOAT64]
        got = sorted(rows(rel))
        data = np.genfromtxt(os.path.join(DATA, "aggregate_test_1.csv"), delimiter=",", skip_header=1)
        for a, m, ma in got:
            xs = data[data[:, 0] == a, 1]
            assert float(m) == pytest.approx(math.fsum(xs) / len(xs), rel=1e-12) and float(ma) == float(a)
        # a data source is read once: every query below scans a table of its own
        hctx.register_csv("t2", os.path.join(DATA, "aggregate_test_1.csv"), [("a", A.INT32), ("b", A.FLOAT64)], 1024)
        rel = hctx.sql("SELECT AVG(b) FROM t2 WHERE a > 2")
        (m,), = rows(rel)
        xs = data[data[:, 0] > 2, 1]
        assert float(m) == pytest.approx(math.fsum(xs) / len(xs), rel=1e-12)

        rng = np.random.default_rng(17)
        k = rng.integers(0, 50, 100_000).astype(np.int64)
        v = rng.integers(-20, 20, 100_000).astype(np.int32)
        hctx.register_memory("t", [("k", k), ("v", v)], batch_size=30_000)
        rel = hctx.sql("SELECT k, AVG(v) FROM t WHERE v > 3 GROUP BY k")
        assert [dt for _, dt in rel.schema()] == [A.INT64, A.FLOAT64]
        check([np.concatenate(c) for c in zip(*rel.collect())], [k], v, where=v > 3)
        hctx.register_memory("u", [("k", k), ("v", v)], batch_size=30_000)
        rel = hctx.sql("SELECT AVG(v), COUNT(v) FROM u WHERE v > 100")
        assert rows(rel) == [(None, 0)]
    finally:
        hctx.close()


def test_sql_nulls(ctx):
    """null_test.csv: AVG skips the nulls of its argument, with and without GROUP BY."""
    hctx = host.ExecutionContext(0)
    try:
        fields = [("c_int", A.INT32), ("c_float", A.FLOAT64), ("c_string", A.UTF8), ("c_bool", A.BOOL)]
        hctx.register_csv("t", os.path.join(DATA, "null_test.csv"), fields, 1024)
        hctx.register_csv("t2", os.path.join(DATA, "null_test.csv"), fields, 1024)  # a data source is read once
        c_float = [1.1, 2.2, 4.4, 6.6]  # row 3 is null
        rel = hctx.sql("SELECT AVG(c_float), AVG(c_int), COUNT(c_float) FROM t")
        assert [dt for _, dt in rel.schema()] == [A.FLOAT64, A.FLOAT64, A.UINT64]
        ((m, mi, c),) = rows(rel)
        assert m == pytest.approx(math.fsum(c_float) / 4, rel=1e-12) and mi == 3.0 and c == 4
        got = dict(rows(hctx.sql("SELECT c_int, AVG(c_float) FROM t2 GROUP BY c_int")))
        assert got == {1: 1.1, 2: 2.2, 3: None, 4: 4.4, 5: 6.6}
    finally:
        hctx.close()
