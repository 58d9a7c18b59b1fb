"""Utf8 functions on the GPU, byte-exact against the Python reference of utf8_fn_ref: projections of every function and of
nests under a WHERE of selectivity 0, ~1 % and 1; nullable, all-null, sliced and empty columns; strings straddling
16-byte words and longer than 4 KiB; 2^20 random rows; predicates over functions under AND / OR; Int64 lengths as
aggregate arguments, GROUP BY keys and in the fused WHERE, on the resident and the chunked host paths; SQL over the
golden CSV files; and the refusals."""
import ctypes as C
import os

import numpy as np
import pyarrow as pa
import pytest

from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import engine, host
from datafusion_archive_b200.expr import AggregateFunction, col, lit, utf8_fn
from kernel_trace import traced_set as traced
from test_avg_gpu import rows
from utf8_fn_ref import NESTS, build, ev, is_int, random_strings

pytestmark = pytest.mark.gpu

DATA = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "data")


@pytest.fixture(scope="module")
def ctx():
    c = engine.GpuContext(0)
    yield c
    c.close()


def fetch(r):
    """Result columns as numpy arrays, Utf8 ones as lists of bytes (the bytes need not be UTF-8); a nullable column as
    (values, valid), a nullable Utf8 column with None where null."""
    L = engine.lib()
    nrows, ncols = C.c_int64(), C.c_int()
    L.dfgpu_result_shape(r.h, C.byref(nrows), C.byref(ncols))
    n = nrows.value
    out = []
    for i in range(ncols.value):
        dt, nulls = C.c_int32(), C.c_int64()
        engine.check(L.dfgpu_result_col_dtype(r.h, i, C.byref(dt)))
        engine.check(L.dfgpu_result_col_nulls(r.h, i, C.byref(nulls)))
        validity = np.zeros(max(1, (n + 7) // 8), np.uint8) if nulls.value else None
        vptr = validity.ctypes.data if validity is not None else None
        ok = None
        if dt.value == A.UTF8:
            nb = C.c_int64()
            engine.check(L.dfgpu_result_col_bytes(r.h, i, C.byref(nb)))
            data = np.zeros(max(1, nb.value), np.uint8)
            offs = np.zeros(n + 1, np.int32)
            engine.check(L.dfgpu_result_copy_col(r.h, i, data.ctypes.data, vptr, offs.ctypes.data))
            raw = data.tobytes()
            ok = np.unpackbits(validity, bitorder="little")[:n].astype(bool) if validity is not None else np.ones(n, bool)
            out.append([raw[offs[k]:offs[k + 1]] if ok[k] else None for k in range(n)])
            continue
        if dt.value == A.BOOL:
            packed = np.zeros(max(1, (n + 7) // 8), np.uint8)
            engine.check(L.dfgpu_result_copy_col(r.h, i, packed.ctypes.data, vptr, None))
            vals = np.unpackbits(packed, bitorder="little")[:n].astype(bool)
        else:
            vals = np.zeros(max(1, n), A.NP_OF[dt.value])
            engine.check(L.dfgpu_result_copy_col(r.h, i, vals.ctypes.data, vptr, None))
            vals = vals[:n]
        out.append((vals, np.unpackbits(validity, bitorder="little")[:n].astype(bool)) if validity is not None else vals)
    return out


def project(ctx, arrays, exprs, pred=None):
    b = ctx.upload(arrays)
    try:
        r = ctx.filter_project(b, pred, exprs)
        try:
            return fetch(r)
        finally:
            r.free()
    finally:
        b.free()


def binary(vals):
    return pa.array(vals, type=pa.binary())


def ints(got):
    """An Int64 result column as a list with None where null."""
    if isinstance(got, tuple):
        return [int(v) if ok else None for v, ok in zip(got[0], got[1])]
    return [int(v) for v in got]


@pytest.mark.parametrize("nest", NESTS, ids=[repr(n) for n in NESTS])
def test_projection_under_where(ctx, nest):
    vals = random_strings(3000, 1)
    x = np.random.default_rng(2).random(len(vals))
    for thr in (2.0, 0.99, -1.0):  # selectivity 0, ~1 %, 1
        sel = [v for v, xi in zip(vals, x) if xi > thr]
        (got,), k = traced(lambda: project(ctx, [binary(vals), x], [build(nest)], pred=col(1) > lit(float(thr))))
        exp = [ev(nest, v) for v in sel]
        assert (ints(got) if is_int(nest) else got) == exp, (nest, thr)
        assert "k_utf8_view_len" in k or (not sel and not is_int(nest))  # a Utf8 projection runs over the selected rows only


@pytest.mark.parametrize("nest", NESTS, ids=[repr(n) for n in NESTS])
def test_nullable_sliced_and_no_where(ctx, nest):
    vals = random_strings(2500, 3, null_frac=0.2)
    arr = binary(vals).slice(37, 2000)
    (got,), _ = traced(lambda: project(ctx, [arr], [build(nest)]))
    exp = [ev(nest, v) for v in vals[37:2037]]
    assert (ints(got) if is_int(nest) else got) == exp


def test_case_only_view_reuses_offsets(ctx):
    vals = random_strings(5000, 4)
    (u, l), k = traced(lambda: project(ctx, [binary(vals)], [utf8_fn("upper", col(0)), utf8_fn("lower", col(0))]))
    assert u == [ev(("upper", "s"), v) for v in vals] and l == [ev(("lower", "s"), v) for v in vals]
    assert "k_utf8_view_copy" in k and "k_utf8_view_len" not in k


def test_edge_columns(ctx):
    long = b"ab\xc3\xa9 " * 1500 + b"x"  # > 4 KiB
    for vals in ([None] * 50, [b""] * 50, [], [long, b" " * 5000, None, long[:4097], b"   "],
                 [b"q" * n for n in range(1, 40)], [b" " * n + b"x" + b" " * n for n in range(0, 40)]):
        for nest in NESTS:
            (got,), _ = traced(lambda: project(ctx, [binary(vals)], [build(nest)]))
            assert (ints(got) if is_int(nest) else got) == [ev(nest, v) for v in vals], (nest, len(vals))


def test_large_random(ctx):
    n = 1 << 20
    vals = random_strings(n, 5, null_frac=0.05, max_pieces=6)
    x = np.random.default_rng(6).random(n)
    nests = [("upper", ("trim", ("substr", "s", 2))), ("length", "s"), ("substr", "s", 2, 3)]
    got = project(ctx, [binary(vals), x], [build(t) for t in nests], pred=col(1) > lit(0.5))
    sel = [v for v, xi in zip(vals, x) if xi > 0.5]
    assert got[0] == [ev(nests[0], v) if v is not None else b"" for v in sel]  # under a WHERE a null row is ''
    assert ints(got[1]) == [ev(nests[1], v) if v is not None else 0 for v in sel]  # under a WHERE a result has no validity
    assert got[2] == [ev(nests[2], v) if v is not None else b"" for v in sel]


def like_prefix(s, p):
    return s is not None and s.startswith(p)


def test_predicates_over_functions(ctx):
    vals = random_strings(4000, 7, null_frac=0.1)
    x = np.random.default_rng(8).integers(0, 10, len(vals)).astype(np.int64)
    low, up = [ev(("lower", "s"), v) for v in vals], [ev(("upper", "s"), v) for v in vals]
    ln = [ev(("length", "s"), v) for v in vals]
    cases = [
        (utf8_fn("lower", col(0)).like(lit(b"ab%")), [like_prefix(v, b"ab") for v in low]),
        (utf8_fn("upper", col(0)).eq(lit(b"Z")), [v == b"Z" for v in up]),
        (utf8_fn("length", col(0)) > lit(3), [v is not None and v > 3 for v in ln]),
        (utf8_fn("lower", col(0)).like(lit(b"ab%")) & (col(1) > lit(4)), [like_prefix(v, b"ab") and xi > 4 for v, xi in zip(low, x)]),
        ((col(1) < lit(2)) | utf8_fn("upper", col(0)).eq(lit(b"Z")), [xi < 2 or v == b"Z" for v, xi in zip(up, x)]),
        ((utf8_fn("length", col(0)) > lit(5)) | (col(1).eq(lit(3))), [(v is not None and v > 5) or xi == 3 for v, xi in zip(ln, x)]),
        (utf8_fn("trim", col(0)).eq(utf8_fn("rtrim", utf8_fn("ltrim", col(0)))), [True for v in vals]),
    ]
    ids = np.arange(len(vals), dtype=np.int64)
    for e, exp in cases:
        (got,), k = traced(lambda: project(ctx, [binary(vals), x, ids], [col(2)], pred=e))
        assert list(got) == [i for i, m in enumerate(exp) if m]
        assert "k_utf8_view_len" in k or "k_utf8_view_copy" in k


def agg(ctx, arrays, keys, aggs, pred=None, nb=2):
    n = len(arrays[0])
    bounds = [int(v) for v in np.linspace(0, n, nb + 1)]
    bs = [ctx.upload([a[bounds[i]:bounds[i + 1]] for a in arrays]) for i in range(nb)]
    try:
        r = ctx.aggregate(bs, keys, aggs, 0, pred=pred)
        try:
            return r.columns()
        finally:
            r.free()
    finally:
        for b in bs:
            b.free()


def test_aggregates_of_lengths(ctx):
    vals = random_strings(20000, 9, null_frac=0.1)
    arr = binary(vals)
    lens = np.array([ev(("length", "s"), v) if v is not None else -1 for v in vals])
    ok = lens >= 0
    L = utf8_fn("length", col(0))
    got = agg(ctx, [arr], [], [AggregateFunction("sum", L), AggregateFunction("min", L), AggregateFunction("max", L),
                               AggregateFunction("avg", L), AggregateFunction("count", L, distinct=True), AggregateFunction("count", L)])
    vals_ = [g[0][0] if isinstance(g, tuple) else g[0] for g in got]
    assert int(vals_[0]) == lens[ok].sum() and int(vals_[1]) == lens[ok].min() and int(vals_[2]) == lens[ok].max()
    assert float(vals_[3]) == pytest.approx(lens[ok].mean(), rel=1e-12)
    assert int(vals_[4]) == len(np.unique(lens[ok])) and int(vals_[5]) == ok.sum()
    # GROUP BY length(s): a null key is its own group
    x = np.random.default_rng(10).random(len(vals))
    got = agg(ctx, [arr, x], [L], [AggregateFunction("count", col(1)), AggregateFunction("sum", col(1))])
    keys = ints(got[0])
    exp = {}
    for l, xi in zip(lens, x):
        kk = max(int(l), 0)  # a null key is read as its value, 0, as for any nullable integer key
        c, s = exp.get(kk, (0, 0.0))
        exp[kk] = (c + 1, s + xi)
    assert sorted(keys) == sorted(exp)
    for kk, c, s in zip(keys, ints(got[1]), got[2]):
        assert c == exp[kk][0] and s == pytest.approx(exp[kk][1], rel=1e-9)
    # a fused WHERE on a view, grouped by octet_length(trim(s))
    O = utf8_fn("octet_length", utf8_fn("trim", col(0)))
    got = agg(ctx, [arr, x], [O], [AggregateFunction("count", col(1))], pred=utf8_fn("lower", col(0)).like(lit(b"%a%")))
    exp = {}
    for v in vals:
        if v is not None and b"a" in ev(("lower", "s"), v):
            kk = len(v.strip(b" "))
            exp[kk] = exp.get(kk, 0) + 1
    assert dict(zip(ints(got[0]), ints(got[1]))) == exp


def test_chunked_host_aggregate(ctx):
    vals = random_strings(300_000, 11)
    arr = binary(vals)
    lens = np.array([ev(("length", "s"), v) for v in vals])
    x = np.ones(len(vals))
    r = ctx.aggregate_host([arr, x], [utf8_fn("length", col(0))], [AggregateFunction("count", col(1))], chunk_rows=70_000)
    try:
        k, c = r.columns()
    finally:
        r.free()
    u, cnt = np.unique(lens, return_counts=True)
    assert dict(zip(ints(k), ints(c))) == dict(zip(u.tolist(), cnt.tolist()))


def test_sql_over_golden_csv(ctx):
    hctx = host.ExecutionContext(0)
    tables = iter(range(100))

    def sql(name, fields, query):  # a CSV data source is read once: every query gets its own registration
        t = "%s%d" % (name, next(tables))
        hctx.register_csv(t, os.path.join(DATA, name + ".csv"), fields, 1024)
        return rows(hctx.sql(query.replace("{t}", t)))

    try:
        people = [("id", A.INT32), ("name", A.UTF8)]
        plain = sql("people", people, "SELECT id, name FROM {t}")
        assert plain
        got = sql("people", people, "SELECT id, upper(name), length(name), substr(name, 2, 3), lower(trim(name)) FROM {t}")
        assert got == [(i, n.upper(), len(n), n[1:4], n.strip(" ").lower()) for i, n in plain]
        got = sql("people", people, "SELECT id FROM {t} WHERE lower(name) LIKE '%a%'")
        assert got == [(i,) for i, n in plain if "a" in n.lower()]
        got = sql("people", people, "SELECT id FROM {t} WHERE length(name) > 4")
        assert got == [(i,) for i, n in plain if len(n) > 4]
        cities_t = [("city", A.UTF8), ("lat", A.FLOAT64), ("lng", A.FLOAT64)]
        cities = sql("uk_cities", cities_t, "SELECT city, lat FROM {t}")
        assert cities
        got = sorted(sql("uk_cities", cities_t, "SELECT length(city), COUNT(lat) FROM {t} GROUP BY length(city)"))
        u, cnt = np.unique([len(c) for c, _ in cities], return_counts=True)
        assert got == list(zip(u.tolist(), cnt.tolist()))
        got = sql("uk_cities", cities_t, "SELECT upper(city), octet_length(trim(city)) FROM {t} WHERE lat > 53")
        assert got == [(c.upper(), len(c.strip(" ").encode())) for c, lat in cities if lat > 53]
    finally:
        hctx.close()


def test_refusals(ctx):
    vals = random_strings(100, 12)
    b = ctx.upload([binary(vals), np.arange(100, dtype=np.int32)])
    try:
        for keys, aggs, code, msg in [
            ([utf8_fn("upper", col(0))], [AggregateFunction("count", col(1))], A.ERR_NOT_IMPLEMENTED, "Utf8 GROUP BY keys must be plain columns"),
            ([], [AggregateFunction("sum", utf8_fn("trim", col(0)))], A.ERR_EXECUTION, "Unsupported data type for aggregate: Utf8"),
            ([], [AggregateFunction("sum", col(0))], A.ERR_EXECUTION, "Unsupported data type for aggregate: Utf8"),
        ]:
            with pytest.raises(engine.DfGpuError) as ei:
                r = ctx.aggregate([b], keys, aggs, 0)
                r.free()
            assert ei.value.code == code and msg in ei.value.msg, ei.value.msg
        for e, code, msg in [(utf8_fn("upper", col(1)), A.ERR_EXECUTION, "function 'upper' takes a Utf8 argument, not Int32"),
                             (utf8_fn("upper", lit("x")), A.ERR_NOT_IMPLEMENTED, "over a Utf8 literal"),
                             (utf8_fn("substr", col(0), 1, -1), A.ERR_EXECUTION, "negative substring length not allowed"),
                             (utf8_fn("substr", col(0), col(1)), A.ERR_NOT_IMPLEMENTED, "Int64 literals")]:
            with pytest.raises(engine.DfGpuError) as ei:
                r = ctx.filter_project(b, None, [e])
                r.free()
            assert ei.value.code == code and msg in ei.value.msg, ei.value.msg
    finally:
        b.free()
