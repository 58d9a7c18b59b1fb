"""COUNT(DISTINCT x) on the GPU, exact against the reference of tests/groupby_ref.py: +0.0 and -0.0 are one value,
every NaN is one value, and nulls are skipped."""
import os

import numpy as np
import pyarrow as pa
import pytest

import groupby_ref as G
from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import engine, host
from datafusion_archive_b200.expr import AggregateFunction, col

pytestmark = pytest.mark.gpu

DATA = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "data")
INTS = [np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64]
ALL = INTS + [np.float32, np.float64]


@pytest.fixture(scope="module")
def ctx():
    c = engine.GpuContext(0)
    yield c
    c.close()


def cd(arg):
    return AggregateFunction("count", arg, distinct=True)


def check(got, keys, v, where=None):
    """`got` (the keys, then COUNT(DISTINCT v)) against groupby_ref."""
    G.assert_matches(got, G.aggregate(keys, [(G.COUNT_DISTINCT, v)], where=where))


def gpu(ctx, arrays, keys, aggs, pred=None, batches=1):
    bs = [ctx.upload([a[i::batches] if batches > 1 else a for a in arrays]) for i in range(batches)]
    try:
        r = ctx.aggregate(bs, keys=keys, aggs=aggs, pred=pred)
        try:
            return r.columns()
        finally:
            r.free()
    finally:
        for b in bs:
            b.free()


def values(dt, n, rng, distinct=50):
    if np.dtype(dt).kind == "f":
        base = rng.integers(-distinct // 2, distinct // 2, n).astype(dt) / dt(4)
        return base.astype(dt)
    info = np.iinfo(dt)
    pool = rng.integers(info.min, info.max, distinct, dtype=np.int64 if info.min < 0 else np.uint64, endpoint=True).astype(dt)
    pool[:2] = [info.min, info.max]
    return pool[rng.integers(0, distinct, n)]


@pytest.mark.parametrize("kdt", INTS, ids=lambda d: np.dtype(d).name)
@pytest.mark.parametrize("vdt", ALL, ids=lambda d: np.dtype(d).name)
def test_key_by_argument_dtype(ctx, kdt, vdt):
    rng = np.random.default_rng(int(np.dtype(kdt).num) * 100 + np.dtype(vdt).num)
    n = 30_000
    k = values(kdt, n, rng, distinct=40)
    v = values(vdt, n, rng, distinct=60)
    got = gpu(ctx, [k, v], [col(0)], [cd(col(1))])
    check(got, [k], v)


@pytest.mark.parametrize("vdt", [np.float32, np.float64], ids=lambda d: np.dtype(d).name)
def test_float_edges(ctx, vdt):
    specials = [0.0, -0.0, np.inf, -np.inf, np.finfo(vdt).tiny / 4, -np.finfo(vdt).tiny / 4, np.finfo(vdt).max, 1.5]
    v = np.array(specials * 50, dtype=vdt)
    nan_bits = [0x7FC00000, 0x7FC00001, 0xFFC00000, 0x7F800001] if vdt == np.float32 else \
        [0x7FF8000000000000, 0x7FF8000000000001, 0xFFF8000000000000, 0x7FF0000000000001]
    nans = np.array(nan_bits * 25, dtype=np.uint32 if vdt == np.float32 else np.uint64).view(vdt)
    v = np.concatenate([v, nans])
    k = np.arange(len(v), dtype=np.int64) % 3
    got = gpu(ctx, [k, v], [col(0)], [cd(col(1))])
    check(got, [k], v)
    # +0.0 and -0.0 are one value, and every NaN payload is one more
    assert got[1][np.flatnonzero(got[0] == 0)[0]] == len(specials)
    whole = gpu(ctx, [v], [], [cd(col(0))])
    assert int(whole[0][0]) == len(specials)


def test_nulls(ctx):
    rng = np.random.default_rng(7)
    n = 50_000
    k = rng.integers(0, 100, n).astype(np.int32)
    v = rng.integers(0, 30, n).astype(np.int64)
    valid = rng.random(n) < 0.7
    valid[k == 5] = False  # a group whose values are all null: present, count 0
    arr = pa.array(v, mask=~valid)
    got = gpu(ctx, [k, arr], [col(0)], [cd(col(1)), AggregateFunction("count", col(1))])
    G.assert_matches(got, G.aggregate([k], [(G.COUNT_DISTINCT, (v, valid)), (G.COUNT, (v, valid))]))
    g5 = np.flatnonzero(got[0] == 5)[0]
    assert got[1][g5] == 0 and got[2][g5] == 0
    whole = gpu(ctx, [arr], [], [cd(col(0))])
    assert int(whole[0][0]) == len(np.unique(v[valid]))


def count_and_distinct(ctx, batches, where=None):
    """(COUNT(x), COUNT(DISTINCT x)) without GROUP BY over `batches`, each a list of one column, as Result columns."""
    bs = [ctx.upload(b) for b in batches]
    try:
        r = ctx.aggregate(bs, keys=[], aggs=[AggregateFunction("count", col(0)), cd(col(0))], pred=where)
        try:
            return r.columns()
        finally:
            r.free()
    finally:
        for b in bs:
            b.free()


@pytest.mark.parametrize("case", ["zero_rows", "no_row_passes", "all_null", "distinct_values", "distinct_with_nulls"])
def test_matches_count_when_all_distinct(ctx, case):
    """On an input whose non-null values are all different, COUNT(DISTINCT x) equals COUNT(x) bit for bit, validity included."""
    v = np.arange(1000, dtype=np.float64)
    where = None
    if case == "zero_rows":
        batches = [[v[:0]]]
    elif case == "no_row_passes":
        batches, where = [[v]], col(0) < -1.0
    elif case == "all_null":
        batches = [[pa.array(v, mask=np.ones(len(v), bool))]]
    elif case == "distinct_values":
        batches = [[v[:500]], [v[500:]]]
    else:
        batches = [[pa.array(v, mask=(np.arange(len(v)) % 3) == 0)]]
    cnt, dis = count_and_distinct(ctx, batches, where)
    if isinstance(cnt, tuple):
        assert isinstance(dis, tuple)
        assert np.array_equal(cnt[0], dis[0]) and np.array_equal(cnt[1], dis[1])
    else:
        assert not isinstance(dis, tuple) and np.array_equal(cnt, dis)


def test_no_batch_matches_count(ctx):
    keep = []
    aggarr = A.make_aggs([(A.AGG_COUNT, col(0).program([A.FLOAT64]), A.UINT64), (A.AGG_COUNT_DISTINCT, col(0).program([A.FLOAT64]), A.UINT64)], keep)
    st = engine.C.c_void_p()
    engine.check(engine.lib().dfgpu_aggregate_create(ctx.h, None, None, 0, aggarr, 2, 0, engine.C.byref(st)))
    try:
        out = engine.C.c_void_p()
        engine.check(engine.lib().dfgpu_aggregate_finish(st, engine.C.byref(out)))
        r = engine.Result(ctx, out)
        cnt, dis = r.columns()
        r.free()
    finally:
        engine.lib().dfgpu_aggregate_free(st)
    assert np.array_equal(cnt[0], dis[0]) and np.array_equal(cnt[1], dis[1]) and not cnt[1][0]


def test_empty_marker_key_and_pair(ctx):
    # key -1 packs to EMPTY_KEY (the group table's sentinel slot); (-1, -1) equals the pair set's empty marker
    k = np.array([-1, -1, -1, -1, 0, 0, 7, -1], dtype=np.int64)
    v = np.array([-1, -1, 3, 4, -1, -1, -1, 3], dtype=np.int64)
    got = gpu(ctx, [k, v], [col(0)], [cd(col(1))])
    check(got, [k], v)
    assert sorted(zip(got[0].tolist(), got[1].tolist())) == [(-1, 3), (0, 1), (7, 1)]
    check(gpu(ctx, [k, v], [col(0)], [cd(col(1))], batches=3), [k], v)


def test_three_batches(ctx):
    rng = np.random.default_rng(3)
    k = rng.integers(0, 1000, 300_000).astype(np.int64)
    v = rng.integers(0, 100, 300_000).astype(np.int64)
    one = gpu(ctx, [k, v], [col(0)], [cd(col(1))])
    three = gpu(ctx, [k, v], [col(0)], [cd(col(1))], batches=3)
    check(one, [k], v)
    check(three, [k], v)


def test_set_growth(ctx, capfd, monkeypatch):
    """>= 1e7 distinct pairs arriving in batches too small for the prefix estimate: the sets grow x4 at least twice."""
    monkeypatch.setenv("DFGPU_TRACE", "1")
    n = 10_500_000
    rng = np.random.default_rng(11)
    v = rng.permutation(n).astype(np.int64)
    k = (v % 1000).astype(np.int32)
    got = gpu(ctx, [k, v], [col(0)], [cd(col(1))], batches=5)
    err = capfd.readouterr().err
    assert err.count("launch k_set_move") >= 2
    check(got, [k], v)  # every value is distinct: each group counts its rows
    monkeypatch.delenv("DFGPU_TRACE")
    whole = gpu(ctx, [v], [], [cd(col(0))])  # one big first batch: the prefix sizes the set
    assert int(whole[0][0]) == n


@pytest.mark.parametrize("ngroups", [1000, 1_000_000])
def test_front_and_line_tables(ctx, ngroups):
    rng = np.random.default_rng(ngroups)
    n = 6_000_000
    k = rng.integers(0, ngroups, n).astype(np.int64)
    v = rng.integers(0, 50, n).astype(np.int64)
    w = rng.random(n)
    plain = [AggregateFunction("min", col(2)), AggregateFunction("max", col(2)), AggregateFunction("sum", col(2)),
             AggregateFunction("count", col(2))]
    got = gpu(ctx, [k, v, w], [col(0)], plain + [cd(col(1))])
    base = gpu(ctx, [k, v, w], [col(0)], plain)
    o, ob = np.argsort(got[0]), np.argsort(base[0])
    assert np.array_equal(got[0][o], base[0][ob])
    for a in (1, 2, 4):
        assert np.array_equal(got[a][o], base[a][ob])
    np.testing.assert_allclose(got[3][o], base[3][ob], rtol=1e-9)
    check([got[0], got[5]], [k], v)


def test_where_and_expression_argument(ctx):
    rng = np.random.default_rng(5)
    n = 200_000
    k = rng.integers(0, 500, n).astype(np.int32)
    a = rng.integers(0, 40, n).astype(np.int64)
    b = rng.integers(0, 40, n).astype(np.int64)
    got = gpu(ctx, [k, a, b], [col(0)], [cd(col(1) + col(2))], pred=col(1) > 10)
    check(got, [k], a + b, where=a > 10)
    whole = gpu(ctx, [k, a, b], [], [cd(col(1) + col(2))], pred=col(1) > 10)
    check(whole, [], a + b, where=a > 10)


def test_several_distinct_and_mixed(ctx):
    rng = np.random.default_rng(9)
    n = 400_000
    k1 = rng.integers(-3, 3, n).astype(np.int16)
    k2 = rng.integers(0, 200, n).astype(np.uint32)
    a = rng.integers(0, 90, n).astype(np.int32)
    b = rng.integers(0, 7, n).astype(np.float64)
    keys = [col(0), col(1)]
    mixed = [AggregateFunction("sum", col(2)), cd(col(2)), AggregateFunction("max", col(3)), cd(col(3)), cd(col(2)),
             AggregateFunction("count", col(2))]
    got = gpu(ctx, [k1, k2, a, b], keys, mixed)
    base = gpu(ctx, [k1, k2, a, b], keys, [mixed[0], mixed[2], mixed[5]])
    o, ob = np.lexsort((got[1], got[0])), np.lexsort((base[1], base[0]))
    for i, j in ((2, 2), (4, 3), (7, 4)):
        assert np.array_equal(got[i][o], base[j][ob])
    G.assert_matches(got, G.aggregate([k1, k2], [(G.SUM, a), (G.COUNT_DISTINCT, a), (G.MAX, b), (G.COUNT_DISTINCT, b),
                                                  (G.COUNT_DISTINCT, a), (G.COUNT, a)]))


def test_update_host_chunks(ctx):
    rng = np.random.default_rng(13)
    n = 9_000_000
    k = rng.integers(0, 100_000, n).astype(np.int64)
    v = rng.integers(0, 100, n).astype(np.int64)
    aggs = [AggregateFunction("sum", col(1)), cd(col(1))]
    r = ctx.aggregate_host([k, v], keys=[col(0)], aggs=aggs, chunk_rows=4 << 20)
    chunked = r.columns()
    r.free()
    resident = gpu(ctx, [k, v], [col(0)], aggs)
    exp = G.aggregate([k], [(G.SUM, v), (G.COUNT_DISTINCT, v)])
    G.assert_matches(chunked, exp, "chunked")
    G.assert_matches(resident, exp, "resident")


def test_not_implemented_shapes(ctx):
    s = ["a", "b", "a"]
    k = np.array([1, 2, 1], dtype=np.int64)
    v = np.array([1.0, 2.0, 1.0])
    for arrays, keys, arg in (([s, v], [col(0)], col(1)),              # Utf8 key
                              ([k, k, v], [col(0), col(1)], col(2)),  # composite key wider than 64 bits
                              ([k, s], [col(0)], col(1))):           # Utf8 argument
        with pytest.raises(engine.DfGpuError) as e:
            gpu(ctx, arrays, keys, [cd(arg)])
        assert e.value.code == A.ERR_NOT_IMPLEMENTED and "COUNT(DISTINCT)" in e.value.msg
    with pytest.raises(engine.DfGpuError) as e:  # Boolean argument: as for the other aggregates
        gpu(ctx, [k, np.array([True, False, True])], [col(0)], [cd(col(1))])
    assert e.value.code == A.ERR_EXECUTION


def rows(rel):
    out = []
    for batch in rel.collect():
        out.extend(zip(*batch))
    return sorted(out)


def test_sql(ctx):
    hctx = host.ExecutionContext(0)
    try:
        hctx.register_csv("t1", os.path.join(DATA, "aggregate_test_1.csv"), [("a", A.INT32), ("b", A.FLOAT64)], 1024)
        got = rows(hctx.sql("SELECT a, COUNT(DISTINCT b), MIN(b) FROM t1 GROUP BY a"))
        data = np.genfromtxt(os.path.join(DATA, "aggregate_test_1.csv"), delimiter=",", skip_header=1)
        exp = sorted((int(a), len(np.unique(data[data[:, 0] == a, 1])), data[data[:, 0] == a, 1].min()) for a in np.unique(data[:, 0]))
        assert [(int(a), int(c), float(m)) for a, c, m in got] == exp
        rng = np.random.default_rng(17)
        k = rng.integers(0, 50, 100_000).astype(np.int64)
        v = rng.integers(0, 20, 100_000).astype(np.int32)
        hctx.register_memory("t", [("k", k), ("v", v)], batch_size=30_000)
        rel = hctx.sql("SELECT k, COUNT(DISTINCT v) FROM t WHERE v > 3 GROUP BY k")
        check([np.concatenate(c) for c in zip(*rel.collect())], [k], v, where=v > 3)
        hctx.register_memory("u", [("k", k), ("v", v)], batch_size=30_000)
        got = rows(hctx.sql("SELECT COUNT(DISTINCT v + v), COUNT(v) FROM u"))
        assert [(int(a), int(b)) for a, b in got] == [(len(np.unique(v + v)), len(v))]
    finally:
        hctx.close()
