"""CAST between the ten numeric dtypes on the GPU, against the exact Rust `as` reference of tests/cast_ref.py, at every
site that evaluates expressions: filter/project (TMA interpreter at K = 8 and 4, the direct kernel, the null-aware
direct kernel, the chunked host path), predicates, the aggregate's keys, arguments and fused WHERE, join keys, and
the SQL planner's implicit coercions.

Bit for bit unless noted; NaNs compare as a class.  Each ABI case runs with DFGPU_TRACE set and asserts the kernel it
is about, so a case cannot silently land on another instantiation."""

import numpy as np
import pytest

import cast_ref as CR
import groupby_ref as R
from kernel_trace import traced_set as traced
from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import engine, host
from datafusion_archive_b200.expr import AggregateFunction, col, lit, utf8_fn

pytestmark = pytest.mark.gpu

N = 1_000_003  # the last tile is ragged at every tile size
NUMERIC = CR.NUMERIC
NAME = {np.dtype(d): np.dtype(d).name for d in NUMERIC}
F32, F64, I64, U64 = np.float32, np.float64, np.int64, np.uint64


def code(dt):
    return CR.CODE[np.dtype(dt)]


@pytest.fixture(scope="module")
def ctx():
    c = engine.GpuContext(0)
    yield c
    c.close()


def launched(names, want):
    assert want in names, (want, sorted(names))


def assert_same(got, exp, what):
    bad = CR.same(got, exp)
    assert not len(bad), (what, len(bad), bad[:5], np.asarray(got)[bad[:5]], np.asarray(exp)[bad[:5]])


def deep(c, depth):
    """An Int64 expression equal to col(c) whose register stack depth is `depth` (>= 2): any program set holding it
    is too deep for the TMA kernel and runs in the direct one."""
    e = col(c) - col(c)
    for _ in range(depth - 2):
        e = (col(c) - col(c)) + e
    return col(c) + e


_SOURCES = {}


def source(src):
    """N values of dtype src with every edge of every target, and the exact cast of them to each target."""
    key = np.dtype(src)
    if key not in _SOURCES:
        rng = np.random.default_rng(100 + key.num)
        x = CR.fill(rng, src, None, N)
        _SOURCES[key] = (x, {np.dtype(d): CR.cast(x, d) for d in NUMERIC})
    return _SOURCES[key]


def fp(ctx, arrays, pred, proj):
    def go():
        b = ctx.upload(arrays)
        try:
            r = ctx.filter_project(b, pred, proj)
            try:
                return r.columns()
            finally:
                r.free()
        finally:
            b.free()
    return traced(go)


CASTS = [col(0).cast(code(d)) for d in NUMERIC]


# ---- a. the projection matrix: all 100 (source, target) pairs at every filter/project site --------------------------
@pytest.mark.parametrize("src", NUMERIC, ids=NAME.get)
def test_projection_tma_k8(ctx, src):
    # predicate over a Float32 column + the source: at most 12 bytes a row, 8 rows per lane
    x, exp = source(src)
    p = np.random.default_rng(1).random(N).astype(F32)
    got, names = fp(ctx, [x, p], col(1) < lit(0.75, A.FLOAT32), CASTS)
    launched(names, "k_filter_project_tma<2,8,0,0,0>")
    m = p < np.float32(0.75)
    for g, d in zip(got, NUMERIC):
        assert_same(g, exp[np.dtype(d)][m], ("k8", NAME[np.dtype(src)], NAME[np.dtype(d)]))


@pytest.mark.parametrize("src", NUMERIC, ids=NAME.get)
def test_projection_tma_k4(ctx, src):
    # predicate over two Float64 columns + the source: 17 to 24 bytes a row, 4 rows per lane
    x, exp = source(src)
    rng = np.random.default_rng(2)
    p, q = rng.random(N), rng.random(N)
    got, names = fp(ctx, [x, p, q], (col(1) < lit(0.75)) & (col(2) > lit(0.1)), CASTS)
    launched(names, "k_filter_project_tma<2,4,0,0,0>")
    m = (p < 0.75) & (q > 0.1)
    for g, d in zip(got, NUMERIC):
        assert_same(g, exp[np.dtype(d)][m], ("k4", NAME[np.dtype(src)], NAME[np.dtype(d)]))


@pytest.mark.parametrize("src", NUMERIC, ids=NAME.get)
def test_projection_direct(ctx, src):
    # a projection of stack depth 5 sends the whole program set to the direct kernel; no predicate
    x, exp = source(src)
    w = np.arange(N, dtype=I64)
    got, names = fp(ctx, [x, w], None, CASTS + [deep(1, 5)])
    launched(names, "k_filter_project<8,0>")
    assert np.array_equal(got[-1], w)
    for g, d in zip(got, NUMERIC):
        assert_same(g, exp[np.dtype(d)], ("direct", NAME[np.dtype(src)], NAME[np.dtype(d)]))


@pytest.mark.parametrize("src", NUMERIC, ids=NAME.get)
def test_projection_direct_nullable(ctx, src):
    x, exp = source(src)
    rng = np.random.default_rng(3)
    valid = rng.random(N) > 0.3
    # without a WHERE: a null row has value 0 and stays null
    got, names = fp(ctx, [R.arrow_nullable(x, valid)], None, CASTS)
    launched(names, "k_filter_project<8,1>")
    for g, d in zip(got, NUMERIC):
        assert isinstance(g, tuple), (NAME[np.dtype(d)], "lost its bitmap")
        v, m = g
        assert np.array_equal(m, valid)
        e = np.where(valid, exp[np.dtype(d)], np.zeros(1, dtype=d))
        assert_same(v, e, ("nulls", NAME[np.dtype(src)], NAME[np.dtype(d)]))
    # under a WHERE the bitmap is dropped and the value under a surviving null slot is cast like any other
    p = rng.random(N)
    got, names = fp(ctx, [R.arrow_nullable(x, valid), p], col(1) < lit(0.75), CASTS)
    launched(names, "k_filter_project<8,1>")
    sel = p < 0.75
    for g, d in zip(got, NUMERIC):
        assert not isinstance(g, tuple)
        assert_same(g, exp[np.dtype(d)][sel], ("nulls+where", NAME[np.dtype(src)], NAME[np.dtype(d)]))


@pytest.mark.parametrize("src", NUMERIC, ids=NAME.get)
def test_projection_host_chunks(ctx, src):
    x, exp = source(src)
    p = np.random.default_rng(4).random(N).astype(F32)

    def go():
        r = ctx.filter_project_host([x, p], col(1) < lit(0.75, A.FLOAT32), CASTS, chunk_rows=131_071)
        try:
            return [r.host_view(i).copy() for i in range(len(CASTS))]
        finally:
            r.free()
    got, names = traced(go)
    launched(names, "k_filter_project_tma<2,8,0,0,0>")
    m = p < np.float32(0.75)
    for g, d in zip(got, NUMERIC):
        assert_same(g, exp[np.dtype(d)][m], ("host", NAME[np.dtype(src)], NAME[np.dtype(d)]))


def test_casts_feeding_arithmetic(ctx):
    # arithmetic in the target type wraps (integers) or rounds (Float32) there
    rng = np.random.default_rng(5)
    n = 300_001
    a, b = CR.fill(rng, I64, np.int8, n), CR.fill(rng, F64, np.uint8, n)
    c8 = [col(0).cast(A.INT8) + col(1).cast(A.INT8), col(0).cast(A.UINT8) * col(1).cast(A.UINT8),
          col(0).cast(A.INT16) - col(1).cast(A.INT16), col(0).cast(A.FLOAT32) + col(1).cast(A.FLOAT32)]
    got, names = fp(ctx, [a, b, np.arange(n, dtype=I64)], None, c8 + [deep(2, 5)])
    launched(names, "k_filter_project<8,0>")
    ca = {d: CR.cast(a, d).astype(object) for d in (np.int8, np.uint8, np.int16)}
    cb = {d: CR.cast(b, d).astype(object) for d in (np.int8, np.uint8, np.int16)}
    assert_same(got[0], CR.wrap_int(ca[np.int8] + cb[np.int8], np.int8), "i8 +")
    assert_same(got[1], CR.wrap_int(ca[np.uint8] * cb[np.uint8], np.uint8), "u8 *")
    assert_same(got[2], CR.wrap_int(ca[np.int16] - cb[np.int16], np.int16), "i16 -")
    with np.errstate(all="ignore"):
        assert_same(got[3], CR.cast(a, F32) + CR.cast(b, F32), "f32 +")


def test_cast_of_a_synthetic_int64_column(ctx):
    # length(s) is an Int64 column the Utf8 function view computes; 2^24 + 1 characters round to 2^24 in Float32
    strs = ["", "a", "héllo", "x" * 300, "y" * ((1 << 24) + 1), "z" * ((1 << 24) + 3)] * 3 + ["w" * (k % 50) for k in range(20_000)]
    lens = np.array([len(s) for s in strs], dtype=I64)
    got, names = fp(ctx, [strs], None, [utf8_fn("length", col(0)).cast(A.FLOAT32), utf8_fn("length", col(0)).cast(A.UINT8)])
    assert any(n.startswith("k_filter_project") for n in names), sorted(names)
    assert_same(got[0], CR.cast(lens, F32), "length as f32")
    assert_same(got[1], CR.cast(lens, np.uint8), "length as u8")


# ---- b. predicates over casts ---------------------------------------------------------------------------------------
OPS = {"eq": (lambda e, r: e.eq(r), np.equal), "ne": (lambda e, r: e.not_eq(r), np.not_equal), "lt": (lambda e, r: e < r, np.less),
       "le": (lambda e, r: e <= r, np.less_equal), "gt": (lambda e, r: e > r, np.greater), "ge": (lambda e, r: e >= r, np.greater_equal)}
# (target, source): the sources that reach the target's edges (saturation from floats, wrap and rounding from integers)
PRED_PAIRS = [(t, s) for t in NUMERIC for s in ([F64, U64] if CR.is_float(t) else [F64, I64, U64])]


@pytest.mark.parametrize("t,s", PRED_PAIRS, ids=["%s_from_%s" % (NAME[np.dtype(t)], NAME[np.dtype(s)]) for t, s in PRED_PAIRS])
def test_predicates(ctx, t, s):
    rng = np.random.default_rng(np.dtype(t).num * 31 + np.dtype(s).num)
    n = 200_003
    x, y = CR.fill(rng, s, t, n), CR.fill(rng, s, t, n)
    cx, cy = CR.cast(x, t), CR.cast(y, t)
    fin = cx[~np.isnan(cx)] if CR.is_float(t) else cx
    v = np.unique(fin)[len(np.unique(fin)) // 3]  # a value the cast produces, so Eq finds rows
    rid = np.arange(n, dtype=np.int32)
    w = np.dtype(s).itemsize
    for direct in (False, True):
        for op, (mk, f) in OPS.items():
            for rhs_col in (False, True):
                pred = mk(col(0).cast(code(t)), col(1).cast(code(t)) if rhs_col else lit(v.item(), code(t)))
                proj = [col(2)] + ([deep(3, 5)] if direct else [])
                arrays = [x, y, rid] + ([np.zeros(n, dtype=I64)] if direct else [])
                got, names = fp(ctx, arrays, pred, proj)
                if direct:
                    launched(names, "k_filter_project<8,0>")
                else:
                    k = 8 if (2 * w if rhs_col else w) + 4 <= 16 else 4
                    launched(names, "k_filter_project_tma<2,%d,0,0,0>" % k)
                with np.errstate(invalid="ignore"):
                    m = f(cx, cy if rhs_col else np.dtype(t).type(v))
                assert np.array_equal(got[0], rid[m]), (op, rhs_col, direct, v)


# ---- c. aggregate sites -----------------------------------------------------------------------------------------------
def agg(ctx, arrays, keys, aggs, pred=None):
    def go():
        b = ctx.upload(arrays)
        try:
            r = ctx.aggregate([b], keys, aggs, 0, pred=pred)
            try:
                return r.columns()
            finally:
                r.free()
        finally:
            b.free()
    return traced(go)


INT_TARGETS = CR.INTS
KEY_PAIRS = [(t, s) for t in INT_TARGETS for s in [F64, F32, I64 if CR.is_signed(t) else U64]]


@pytest.mark.parametrize("t,s", KEY_PAIRS, ids=["%s_from_%s" % (NAME[np.dtype(t)], NAME[np.dtype(s)]) for t, s in KEY_PAIRS])
def test_group_by_cast_key(ctx, t, s):
    # saturated keys pack to the table's empty marker (CAST(1e300 AS UInt64), CAST(-1.0 AS Int64)); NaN merges with 0
    rng = np.random.default_rng(np.dtype(t).num * 7 + np.dtype(s).num)
    n = 300_001
    x = CR.fill(rng, s, t, n, pool=300)
    v = rng.integers(-1000, 1000, n).astype(I64)
    spec = [(R.COUNT, 1), (R.SUM, 1), (R.MIN, 1), (R.MAX, 1)]
    got, names = agg(ctx, [x, v], [col(0).cast(code(t))], [AggregateFunction(f, col(1)) for f, _ in spec])
    launched(names, "k_hash_agg<1,0,0>")
    k = CR.cast(x, t)
    R.assert_matches(got, R.aggregate([k], [(f, v) for f, _ in spec]), "key %s from %s" % (NAME[np.dtype(t)], NAME[np.dtype(s)]))


@pytest.mark.parametrize("pair", [(np.int16, np.uint8), (I64, U64)], ids=["narrow", "wide"])
def test_group_by_two_cast_keys(ctx, pair):
    rng = np.random.default_rng(8)
    n = 300_001
    x, y = CR.fill(rng, F64, pair[0], n, pool=200), CR.fill(rng, F32, pair[1], n, pool=200)
    v = rng.integers(-1000, 1000, n).astype(I64)
    spec = [(R.COUNT, 2), (R.SUM, 2), (R.MAX, 2)]
    got, names = agg(ctx, [x, y, v], [col(0).cast(code(pair[0])), col(1).cast(code(pair[1]))], [AggregateFunction(f, col(2)) for f, _ in spec])
    launched(names, "k_hash_agg<1,0,0>" if pair[0] == np.int16 else "k_hash_agg_wide<8,0>")
    R.assert_matches(got, R.aggregate([CR.cast(x, pair[0]), CR.cast(y, pair[1])], [(f, v) for f, _ in spec]), str(pair))


def _avg_check(got, vals, keys, what):
    """AVG = f64 sum / u64 count: within the f64 summation bound of the exact mean, plus the division's rounding."""
    f = CR.cast(vals, F64)
    e = R.aggregate(keys, [(R.SUM, f), (R.COUNT, f)])
    s, cnt = e.aggs[0], e.aggs[1]["values"].astype(np.float64)
    nk = len(keys)
    order = np.lexsort([np.asarray(got[k]) for k in reversed(range(nk))]) if nk else np.arange(1)
    g = np.asarray(got[nk] if not isinstance(got[nk], tuple) else got[nk][0])[order]
    sp = s["special"]
    assert np.array_equal(np.isnan(g), sp == 1), (what, "NaN")
    fin = sp == 0
    mean = (s["exact"][fin] / cnt[fin].astype(np.longdouble))
    err = np.abs(g[fin].astype(np.longdouble) - mean).astype(np.float64)
    bound = s["bound"][fin] / cnt[fin] + np.abs(mean.astype(np.float64)) * 2.0 ** -52
    assert (err <= bound).all(), (what, "AVG", np.flatnonzero(err > bound)[:5])


@pytest.mark.parametrize("t", NUMERIC, ids=NAME.get)
def test_aggregates_of_a_cast(ctx, t):
    # integer SUM wraps in t; Float32 SUM is checked against the groupby_ref bound.  Sources that cannot overflow a
    # float SUM in any order: UInt64 (values >= 2^63 too) for the float targets, Float64 (saturating) for the others
    s = U64 if CR.is_float(t) else F64
    rng = np.random.default_rng(np.dtype(t).num + 50)
    n = 400_001
    x = CR.fill(rng, s, t, n)
    k = rng.integers(0, 97, n).astype(np.int32)
    ct = CR.cast(x, t)
    arg = col(1).cast(code(t))
    spec = [R.SUM, R.MIN, R.MAX, R.COUNT]
    for keys, kv, kern in (([col(0)], [k], "k_hash_agg<1,0,0>"), ([], [], "k_reduce<1,0>")):
        got, names = agg(ctx, [k, x], keys, [AggregateFunction(f, arg) for f in spec])
        launched(names, kern)
        R.assert_matches(got, R.aggregate(kv, [(f, ct) for f in spec]), "aggs of %s (%d keys)" % (NAME[np.dtype(t)], len(keys)))
        got, names = agg(ctx, [k, x], keys, [AggregateFunction("avg", arg)])
        assert any(nm.startswith("k_hash_agg") or nm.startswith("k_reduce") for nm in names), sorted(names)
        _avg_check(got, ct, kv, "avg of %s" % NAME[np.dtype(t)])


@pytest.mark.parametrize("t", INT_TARGETS + [F32], ids=NAME.get)
def test_fused_where_over_a_cast(ctx, t):
    rng = np.random.default_rng(np.dtype(t).num + 70)
    n = 300_001
    x = CR.fill(rng, F64, t, n)
    k = rng.integers(0, 50, n).astype(np.int32)
    v = rng.integers(-1000, 1000, n).astype(I64)
    ct = CR.cast(x, t)
    fin = ct[~np.isnan(ct)] if CR.is_float(t) else ct
    lim = np.unique(fin)[len(np.unique(fin)) // 2]
    spec = [R.SUM, R.COUNT, R.MIN]
    pred = col(1).cast(code(t)) >= lit(lim.item(), code(t))
    m = ct >= lim
    got, names = agg(ctx, [k, x, v], [col(0)], [AggregateFunction(f, col(2)) for f in spec], pred=pred)
    launched(names, "k_hash_agg<1,0,0>")
    R.assert_matches(got, R.aggregate([k[m]], [(f, v[m]) for f in spec]), "where %s" % NAME[np.dtype(t)])
    got, names = agg(ctx, [k, x, v], [], [AggregateFunction(f, col(2)) for f in spec], pred=pred)
    launched(names, "k_reduce<1,0>")
    R.assert_matches(got, R.aggregate([], [(f, v[m]) for f in spec]), "reduce where %s" % NAME[np.dtype(t)])


@pytest.mark.parametrize("s", [F64, F32, I64, U64, np.int32], ids=NAME.get)
def test_count_distinct_of_a_cast(ctx, s):
    rng = np.random.default_rng(np.dtype(s).num + 90)
    n = 300_001
    x = CR.fill(rng, s, np.int16, n)
    k = rng.integers(0, 20, n).astype(np.int32)
    c = CR.cast(x, np.int16)
    got, names = agg(ctx, [k, x], [], [AggregateFunction("count", col(1).cast(A.INT16), distinct=True)])
    launched(names, "k_distinct_insert<2,0>")
    assert int(got[0][0]) == len(np.unique(c))
    got, names = agg(ctx, [k, x], [col(0)], [AggregateFunction("count", col(1).cast(A.INT16), distinct=True)])
    launched(names, "k_distinct_insert<2,0>")
    order = np.argsort(got[0])
    want = [len(np.unique(c[k == g])) for g in np.sort(got[0])]
    assert np.array_equal(got[1][order], np.array(want, dtype=np.uint64))


# ---- d. join keys ---------------------------------------------------------------------------------------------------
def test_join_probe_cast_key(ctx):
    # NaN -> 0, ±inf and out-of-range values saturate: they match the build keys 0, INT32_MIN and INT32_MAX
    bk = np.array([0, -(2 ** 31), 2 ** 31 - 1, 5, -7], dtype=np.int32)
    rng = np.random.default_rng(12)
    pk = CR.fill(rng, F64, np.int32, 100_003)
    c = CR.cast(pk, np.int32)

    def go():
        pb = ctx.upload([pk, np.arange(len(pk), dtype=I64)])
        bb = ctx.upload([bk, np.arange(len(bk), dtype=I64)])
        j = ctx.join_build(bb, [col(0)], keep_cols=[1])
        try:
            r = j.probe(pb, [col(0).cast(A.INT32)], probe_cols=[1], build_cols=[1])
            try:
                return r.columns()
            finally:
                r.free()
        finally:
            j.free(); pb.free(); bb.free()
    got, names = traced(go)
    assert any(nm.startswith("k_join") for nm in names), sorted(names)
    pos = {int(v): i for i, v in enumerate(bk)}
    exp = sorted((i, pos[int(v)]) for i, v in enumerate(c) if int(v) in pos)
    assert sorted(zip(got[0].tolist(), got[1].tolist())) == exp
    assert {0, -(2 ** 31), 2 ** 31 - 1} <= {int(c[i]) for i, _ in exp}
    assert np.isnan(pk[[i for i, _ in exp]]).any() and np.isinf(pk[[i for i, _ in exp]]).any()


def sql_batches(hctx, tables, sql):
    """Registers the in-memory tables ({name: {column: array}}) afresh, since a scan drains them, and runs sql."""
    for name, cols in tables.items():
        hctx.register_memory(name, list(cols.items()))
    return hctx.sql(sql).collect()


def sql_rows(hctx, tables, sql):
    out = []
    for b in sql_batches(hctx, tables, sql):
        cols = [c if isinstance(c, list) else np.asarray(c).tolist() for c in b]
        out.extend(zip(*cols))
    return sorted(out, key=repr)


def test_sql_join_and_in_over_mixed_types():
    # the planner coerces both key sides to their supertype.  Widening casts are exact; where the supertype needs a
    # cast the planner does not insert implicitly (UInt64 -> Int64, UInt8 -> Int8) the query is refused
    a = {"u8": np.array([0, 1, 127, 128, 200, 255], dtype=np.uint8), "u64": np.array([0, 5, 2 ** 63, 2 ** 64 - 1, 7, 1], dtype=U64),
         "i16": np.array([-1, 1, 127, -32768, 200, 255], dtype=np.int16), "f32": np.array([0.0, 1.0, 16777216.0, 2.5, 200.0, 255.0], dtype=F32)}
    b = {"i8": np.array([-56, 1, 127, -1, 0, -128], dtype=np.int8), "i64": np.array([-1, 5, -(2 ** 63), 1, 16777217, 255], dtype=I64),
         "u16": np.array([200, 1, 255, 65535, 0, 128], dtype=np.uint16)}
    hctx = host.ExecutionContext(0)
    try:
        tabs = {"a": a, "b": b}
        for on in ("a.u64 = b.i64", "a.u8 = b.i8"):
            with pytest.raises(host.ExecutionError) as e:
                sql_batches(hctx, tabs, "SELECT a.u8 FROM a JOIN b ON " + on)
            assert "Cannot automatically convert" in e.value.msg, e.value.msg
        # Int16 = Int64 (the Int16 side widens), UInt8 = UInt16 (UInt8 widens); float keys are refused
        for on, x, y, st in (("a.i16 = b.i64", a["i16"], b["i64"], I64), ("a.u8 = b.u16", a["u8"], b["u16"], np.uint16)):
            cx, cy = CR.coerce(x, y, st)
            exp = sorted((i, j) for i in range(6) for j in range(6) if cx[i] == cy[j])
            got = sql_rows(hctx, tabs, "SELECT a.u8, b.i8 FROM a JOIN b ON " + on)
            assert got == sorted((int(a["u8"][i]), int(b["i8"][j])) for i, j in exp), on
        with pytest.raises(host.ExecutionError) as e:
            sql_batches(hctx, tabs, "SELECT a.u8 FROM a JOIN b ON a.f32 = b.i64")
        assert "JOIN keys of type Float32 are not supported" in e.value.msg
        got = sql_rows(hctx, tabs, "SELECT i16 FROM a WHERE u8 IN (SELECT u16 FROM b)")
        assert got == sorted(((int(a["i16"][i]),) for i in range(6) if (a["u8"][i].astype(np.uint16) == b["u16"]).any()), key=repr)
        got = sql_rows(hctx, tabs, "SELECT u8 FROM a WHERE i16 NOT IN (SELECT i8 FROM b)")
        assert got == sorted((int(a["u8"][i]),) for i in range(6) if not (a["i16"][i] == b["i8"].astype(np.int16)).any())
        with pytest.raises(host.ExecutionError) as e:
            sql_batches(hctx, tabs, "SELECT u8 FROM a WHERE u64 IN (SELECT i64 FROM b)")
        assert "Cannot automatically convert" in e.value.msg
    finally:
        hctx.close()


# ---- e. SQL over one column of each numeric dtype --------------------------------------------------------------------
SQL_TYPES = {"SMALLINT": np.int16, "INT": np.int32, "BIGINT": I64, "FLOAT": F64, "REAL": F64, "DOUBLE": F64}


@pytest.fixture(scope="module")
def typed():
    rng = np.random.default_rng(14)
    n = 20_011
    cols = {"c_" + NAME[np.dtype(d)]: CR.fill(rng, d, None, n, pool=500) for d in NUMERIC}
    hctx = host.ExecutionContext(0)
    yield hctx, cols
    hctx.close()


def one_col(hctx, cols, sql):
    bs = sql_batches(hctx, {"t": cols}, sql)
    return np.concatenate([np.asarray(b[0]) for b in bs]) if bs else None


@pytest.mark.parametrize("src", NUMERIC, ids=NAME.get)
def test_sql_explicit_casts(typed, src):
    hctx, cols = typed
    name = "c_" + NAME[np.dtype(src)]
    x = cols[name]
    for sqlt, dt in SQL_TYPES.items():
        got = one_col(hctx, cols, "SELECT CAST(%s AS %s) FROM t" % (name, sqlt))
        assert_same(got, CR.cast(x, dt), (name, sqlt))


def test_sql_mixed_type_arithmetic_and_comparisons(typed):
    hctx, cols = typed
    planned = refused = 0
    for a in NUMERIC:
        for b in NUMERIC:
            na, nb = "c_" + NAME[np.dtype(a)], "c_" + NAME[np.dtype(b)]
            st = host.supertype(code(a), code(b))
            sql = "SELECT %s + %s, %s * %s FROM t WHERE %s < %s" % (na, nb, na, nb, na, nb)
            ops = CR.coerce(cols[na], cols[nb], CR.DTYPE[st]) if st else None
            if ops is None:
                with pytest.raises(host.ExecutionError) as e:
                    sql_batches(hctx, {"t": cols}, sql)
                assert ("No common supertype" if st is None else "Cannot automatically convert") in e.value.msg, (na, nb, e.value.msg)
                refused += 1
                continue
            x, y = ops
            bs = sql_batches(hctx, {"t": cols}, sql)
            got = [np.concatenate([np.asarray(bt[i]) for bt in bs]) for i in range(2)]
            with np.errstate(all="ignore"):
                m = x < y
                xs, ys = x[m], y[m]
                if CR.is_float(x.dtype):
                    s, p = xs + ys, xs * ys
                else:
                    s = CR.wrap_int(xs.astype(object) + ys.astype(object), x.dtype)
                    p = CR.wrap_int(xs.astype(object) * ys.astype(object), x.dtype)
            assert_same(got[0], s, (na, nb, "+"))
            assert_same(got[1], p, (na, nb, "*"))
            planned += 1
    assert planned > 30 and refused > 10, (planned, refused)


@pytest.mark.parametrize("src", NUMERIC, ids=NAME.get)
def test_sql_literal_comparisons(typed, src):
    hctx, cols = typed
    name = "c_" + NAME[np.dtype(src)]
    x = cols[name]
    if np.dtype(src) == np.dtype(U64):
        # UInt64 vs an Int64 literal has the supertype Int64, but the planner does not cast UInt64 to Int64
        with pytest.raises(host.ExecutionError) as e:
            one_col(hctx, cols, "SELECT %s FROM t WHERE %s > 5" % (name, name))
        assert "Cannot automatically convert UInt64 to Int64" in e.value.msg
        return
    for litx in ("5", "-3", "9007199254740993", "-9223372036854775807", "2.5", "-0.5", "1000000000000000000000.0", "9007199254740993.0"):
        is_f = "." in litx or "e" in litx
        st = CR.DTYPE[host.supertype(code(src), A.FLOAT64 if is_f else A.INT64)]
        if not is_f and st == np.dtype(F32):
            # Float32 vs an Int64 literal casts the literal to Float32: only Int64 -> Float64 literals are folded
            with pytest.raises(host.ExecutionError) as e:
                one_col(hctx, cols, "SELECT %s FROM t WHERE %s > %s" % (name, name, litx))
            assert "CAST from Int64 to Float32" in e.value.msg
            continue
        if not CR.can_coerce_from(st, src):
            with pytest.raises(host.ExecutionError):
                one_col(hctx, cols, "SELECT %s FROM t WHERE %s > %s" % (name, name, litx))
            continue
        # the literal is an Int64 or Float64; CAST(Int64 literal AS Float64) is folded on the host, correctly rounded
        lv = float(litx) if is_f else int(litx)
        lc = CR.cast(np.array([lv], dtype=F64 if is_f else I64), st)[0] if (is_f and st != F64) or (not is_f and st != I64) else lv
        cx = CR.cast(x, st) if np.dtype(st) != x.dtype else x
        for op, f in (("<", np.less), (">=", np.greater_equal), ("=", np.equal)):
            got = one_col(hctx, cols, "SELECT %s FROM t WHERE %s %s %s" % (name, name, op, litx))
            with np.errstate(invalid="ignore"):
                m = f(cx, np.dtype(st).type(lc))
            assert_same(got if got is not None else x[:0], x[m], (name, op, litx))


# ---- f. refusals ------------------------------------------------------------------------------------------------------
def test_refusals_through_the_abi(ctx):
    b = ctx.upload([np.arange(4, dtype=I64), np.array([1.5, 2, 3, 4]), ["a", "b", "c", "d"], np.array([True, False, True, True])])
    try:
        for e, code_, msg in [
            (col(0).cast(A.UTF8), A.ERR_NOT_IMPLEMENTED, "CAST column from Int64 to Utf8"),
            (col(0).cast(A.BOOL), A.ERR_NOT_IMPLEMENTED, "CAST column from Int64 to Boolean"),
            (col(2).cast(A.INT64), A.ERR_NOT_IMPLEMENTED, "CAST column from Utf8 to Int64"),
            (col(3).cast(A.INT32), A.ERR_NOT_IMPLEMENTED, "CAST column from Boolean to Int32"),
            ((col(0) + lit(1)).cast(A.FLOAT64), A.ERR_GENERAL, "CAST not implemented for expression"),
            (lit(1.5).cast(A.INT32), A.ERR_NOT_IMPLEMENTED, "CAST from Float64 to Int32"),
            (lit(7).cast(A.INT32), A.ERR_NOT_IMPLEMENTED, "CAST from Int64 to Int32"),
            (lit(7, A.INT32).cast(A.FLOAT64), A.ERR_NOT_IMPLEMENTED, "CAST from Int32 to Float64"),
        ]:
            with pytest.raises(engine.DfGpuError) as ex:
                ctx.filter_project(b, None, [e])
            assert ex.value.code == code_ and msg in ex.value.msg, (e, ex.value.code, ex.value.msg)
            with pytest.raises(engine.DfGpuError) as ex:
                ctx.aggregate([b], [], [AggregateFunction("count", e)])
            assert msg in ex.value.msg, (e, ex.value.msg)
        # the one literal cast there is: Int64 -> Float64, folded on the host and correctly rounded
        r = ctx.filter_project(b, None, [lit(9007199254740993).cast(A.FLOAT64) + col(1)])
        assert r.columns()[0].tolist() == [9007199254740992.0 + v for v in (1.5, 2, 3, 4)]
        r.free()
    finally:
        b.free()


def test_refusals_through_sql(typed):
    hctx, cols = typed
    for sql, msg in [
        ("SELECT CAST(c_int64 AS VARCHAR) FROM t", "CAST column from Int64 to Utf8"),
        ("SELECT CAST(c_int64 AS BOOLEAN) FROM t", "CAST column from Int64 to Boolean"),
        ("SELECT CAST(c_int64 + 1 AS DOUBLE) FROM t", "CAST not implemented for expression"),
        ("SELECT c_int32 FROM t WHERE c_int32 > CAST(2.5 AS INT)", "CAST from Float64 to Int32"),
        ("SELECT c_int16 FROM t WHERE c_int16 > CAST(7 AS SMALLINT)", "CAST from Int64 to Int16"),
    ]:
        with pytest.raises(host.ExecutionError) as e:
            sql_batches(hctx, {"t": cols}, sql)
        assert msg in e.value.msg, (sql, e.value.msg)
