"""Inner equi-join on the GPU (dfgpu_join_build / dfgpu_join_probe and JOIN through ctx.sql()), compared with the
exact join of tests/join_ref.py.  Rows are compared as sorted multisets: the order of one probe row's matches is
unspecified."""
import numpy as np
import pyarrow as pa
import pytest

from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import engine, host
from datafusion_archive_b200.expr import col, lit
from join_ref import inner as ref_join, same_pairs

pytestmark = pytest.mark.gpu

INTS = [np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64]


@pytest.fixture(scope="module")
def ctx():
    c = engine.GpuContext(0)
    yield c
    c.close()


def valid_of(a):
    if isinstance(a, (pa.Array, pa.ChunkedArray)):
        return np.asarray(a.is_valid())
    return np.ones(len(a), dtype=bool)


def values_of(a, dtype=None):
    if isinstance(a, (pa.Array, pa.ChunkedArray)):
        return np.asarray(a.fill_null(0).to_numpy(zero_copy_only=False), dtype=dtype)
    return np.asarray(a, dtype=dtype)


def gpu_pairs(ctx, probe_arrays, pkeys, build_arrays, bkeys):
    """Join with a row-number column appended to each side; returns (probe rows, build rows)."""
    pa_ = list(probe_arrays) + [np.arange(len(values_of(probe_arrays[0])), dtype=np.int64)]
    ba_ = list(build_arrays) + [np.arange(len(values_of(build_arrays[0])), dtype=np.int64)]
    pb, bb = ctx.upload(pa_), ctx.upload(ba_)
    j = ctx.join_build(bb, bkeys, keep_cols=[len(ba_) - 1])
    bb.free()
    r = j.probe(pb, pkeys, probe_cols=[len(pa_) - 1], build_cols=[len(ba_) - 1])
    got = r.columns()
    r.free(); j.free(); pb.free()
    return got[0], got[1]


def nullable(vals, valid, dtype):
    return pa.array(np.asarray(vals, dtype=dtype), mask=~np.asarray(valid, bool))


@pytest.mark.parametrize("dt", INTS, ids=lambda d: np.dtype(d).name)
def test_every_integer_key_dtype(ctx, dt):
    rng = np.random.default_rng(1)
    info = np.iinfo(dt)
    special = [0, info.max, info.min, -1 if info.min < 0 else info.max - 1, 1]
    pk = np.concatenate([np.array(special, dtype=dt), rng.integers(-3 if info.min < 0 else 0, 6, 3000).astype(dt)])
    bk = np.concatenate([np.array(special * 2, dtype=dt), rng.integers(-3 if info.min < 0 else 0, 6, 500).astype(dt)])
    pvalid = rng.random(len(pk)) > 0.1
    bvalid = rng.random(len(bk)) > 0.1
    pcol, bcol = nullable(pk, pvalid, dt), nullable(bk, bvalid, dt)
    same_pairs(gpu_pairs(ctx, [pcol], [col(0)], [bcol], [col(0)]), ref_join([pcol], [bcol]))


def test_key_minus_one_and_zero(ctx):
    # -1 packs to the empty-slot marker; 0 is an ordinary key
    for dt in (np.int64, np.int32, np.uint64):
        pk = np.array([-1, 0, 5, -1, 0], dtype=np.int64).astype(dt)
        bk = np.array([0, -1, -1, 7, 0, 0], dtype=np.int64).astype(dt)
        same_pairs(gpu_pairs(ctx, [pk], [col(0)], [bk], [col(0)]), ref_join([pk], [bk]))


def test_composite_keys(ctx):
    rng = np.random.default_rng(2)
    a = rng.integers(-2, 3, 5000).astype(np.int32)
    b = rng.integers(-2, 3, 5000).astype(np.int32)
    c = rng.integers(-2, 3, 800).astype(np.int32)
    d = rng.integers(-2, 3, 800).astype(np.int32)
    same_pairs(gpu_pairs(ctx, [a, b], [col(0), col(1)], [c, d], [col(0), col(1)]), ref_join([a, b], [c, d]))
    x = [rng.integers(-3, 3, 4000).astype(np.int16), rng.integers(-3, 3, 4000).astype(np.int32), rng.integers(0, 4, 4000).astype(np.uint8)]
    x[0] = nullable(x[0], rng.random(4000) > 0.05, np.int16)
    y = [rng.integers(-3, 3, 700).astype(np.int16), rng.integers(-3, 3, 700).astype(np.int32), rng.integers(0, 4, 700).astype(np.uint8)]
    y[2] = nullable(y[2], rng.random(700) > 0.05, np.uint8)
    keys = [col(0), col(1), col(2)]
    same_pairs(gpu_pairs(ctx, x, keys, y, keys), ref_join(x, y))


def test_null_keys_duplicates_no_match_and_empty_sides(ctx):
    pk = nullable([1, 1, 2, 3, 0], [True, True, True, False, False], np.int64)
    bk = nullable([1, 1, 1, 3, 0, 9], [True, True, True, False, False, True], np.int64)
    same_pairs(gpu_pairs(ctx, [pk], [col(0)], [bk], [col(0)]), ref_join([pk], [bk]))  # 2 x 3 pairs for key 1
    none = np.array([100, 200], dtype=np.int64)
    got = gpu_pairs(ctx, [none], [col(0)], [np.array([1, 2], dtype=np.int64)], [col(0)])
    assert len(got[0]) == 0
    empty = np.zeros(0, dtype=np.int64)
    assert len(gpu_pairs(ctx, [none], [col(0)], [empty], [col(0)])[0]) == 0
    assert len(gpu_pairs(ctx, [empty], [col(0)], [none], [col(0)])[0]) == 0


def test_empty_result_keeps_dtypes(ctx):
    pb = ctx.upload([np.array([1, 2], np.int64), pa.array(["a", None]), np.array([True, False])])
    bb = ctx.upload([np.array([5], np.int64), np.array([1.5]), pa.array(["x"])])
    j = ctx.join_build(bb, [col(0)])
    r = j.probe(pb, [col(0)])
    assert r.nrows == 0
    assert [r.dtype(i) for i in range(6)] == [A.INT64, A.UTF8, A.BOOL, A.INT64, A.FLOAT64, A.UTF8]
    r.columns()
    r.free(); j.free(); pb.free(); bb.free()


def test_large_random(ctx):
    rng = np.random.default_rng(3)
    bk = rng.integers(0, 2_000_000, 1_000_000, dtype=np.int64)
    pk = rng.integers(0, 2_000_000, 10_000_000, dtype=np.int64)
    same_pairs(gpu_pairs(ctx, [pk], [col(0)], [bk], [col(0)]), ref_join([pk], [bk]))


def _probe_kernel_ms(ctx, build_keys, probe_keys):
    bb, pb = ctx.upload([build_keys]), ctx.upload([probe_keys])
    j = ctx.join_build(bb, [col(0)], keep_cols=[0])
    j.probe(pb, [col(0)], probe_cols=[0], build_cols=[0]).free()  # warm-up
    ctx.profile_enable(True)
    r = j.probe(pb, [col(0)], probe_cols=[0], build_cols=[0])
    ms, _ = ctx.profile_get()
    ctx.profile_enable(False)
    n = r.nrows
    r.free(); j.free(); bb.free(); pb.free()
    return ms, n


def test_skewed_build_key(ctx):
    n = 4 << 20
    skew_ms, skew_rows = _probe_kernel_ms(ctx, np.full(n, 7, np.int64), np.array([7, 8, 7, 1], np.int64))
    uni_ms, uni_rows = _probe_kernel_ms(ctx, np.arange(n, dtype=np.int64), np.arange(n, dtype=np.int64))
    assert skew_rows == 2 * n and uni_rows == n
    # the skewed probe writes twice the rows of the uniform one: it must take time of the same order
    assert skew_ms < 10 * uni_ms + 1.0, (skew_ms, uni_ms)
    # and the pairs are right
    got = gpu_pairs(ctx, [np.array([7, 8, 7, 1], np.int64)], [col(0)], [np.full(n, 7, np.int64)], [col(0)])
    assert sorted(set(got[0].tolist())) == [0, 2]
    assert np.array_equal(np.sort(got[1][got[0] == 0]), np.arange(n))


def test_payload_columns_with_nulls(ctx):
    rng = np.random.default_rng(4)
    n_p, n_b = 3000, 400
    pk = rng.integers(0, 50, n_p).astype(np.int32)
    bk = rng.integers(0, 50, n_b).astype(np.int32)
    f64 = nullable(rng.random(n_p), rng.random(n_p) > 0.2, np.float64)
    i8 = nullable(rng.integers(-100, 100, n_b), rng.random(n_b) > 0.2, np.int8)
    bools = pa.array(rng.random(n_b) > 0.5, mask=rng.random(n_b) < 0.2)
    strs = pa.array(["s%d" % (i * 7 % 13) * (i % 4) for i in range(n_p)], mask=rng.random(n_p) < 0.2)
    pb = ctx.upload([pk, f64, strs])
    bb = ctx.upload([bk, i8, bools])
    j = ctx.join_build(bb, [col(0)], keep_cols=[1, 2])
    bb.free()
    r = j.probe(pb, [col(0)], probe_cols=[1, 2], build_cols=[2, 1])
    got = r.columns()
    r.free(); j.free(); pb.free()
    prow, brow = ref_join([pk], [bk])
    assert r.nrows == len(prow)

    def rows(c):  # (valid, value or None) per output row, as python values
        v, m = c if isinstance(c, tuple) else (c, np.ones(len(c), bool))
        v = v if isinstance(v, list) else np.asarray(v).tolist()
        return [(bool(ok), x if ok else None) for x, ok in zip(v, m.tolist())]

    def expect(arr, idx):
        py = arr.to_pylist()
        return [(py[i] is not None, py[i]) for i in idx]

    got_rows = sorted(zip(rows(got[0]), rows(got[1]), rows(got[2]), rows(got[3])), key=repr)
    exp_rows = sorted(zip(expect(f64, prow), expect(strs, prow), expect(bools, brow), expect(i8, brow)), key=repr)
    bad = [k for k, (g, e) in enumerate(zip(got_rows, exp_rows)) if g != e]
    assert not bad, (len(bad), got_rows[bad[0]], exp_rows[bad[0]])


def test_cast_key_program(ctx):
    # CAST(UInt32 AS Int32) wraps: 4294967295 becomes -1 and matches the build key -1
    pk = np.array([4294967295, 5, 2147483648, 7], dtype=np.uint32)
    bk = np.array([-1, 5, -2147483648, 8], dtype=np.int32)
    got = gpu_pairs(ctx, [pk], [col(0).cast(A.INT32)], [bk], [col(0)])
    same_pairs(got, (np.array([0, 1, 2]), np.array([0, 1, 2])))
    # an arithmetic key program, evaluated as a projection
    same_pairs(gpu_pairs(ctx, [np.arange(10, dtype=np.int64)], [col(0) + lit(1)], [np.arange(10, dtype=np.int64)], [col(0)]),
               (np.arange(9), np.arange(1, 10)))


def test_refusals(ctx):
    i32 = np.array([1, 2], np.int32)
    i64 = np.array([1, 2], np.int64)
    f64 = np.array([1.0, 2.0])
    bb = ctx.upload([i32, i64, f64])
    pb = ctx.upload([i64, i32])
    j = ctx.join_build(bb, [col(0)], keep_cols=[0])
    with pytest.raises(engine.DfGpuError) as e:
        j.probe(pb, [col(0)])
    assert e.value.code == A.ERR_EXECUTION and "JOIN key types differ: Int64 and Int32" in e.value.msg
    with pytest.raises(engine.DfGpuError) as e:
        j.probe(pb, [col(1)], build_cols=[1])
    assert e.value.code == A.ERR_GENERAL and "not kept" in e.value.msg
    j.free()
    with pytest.raises(engine.DfGpuError) as e:
        ctx.join_build(bb, [col(2)])
    assert e.value.code == A.ERR_NOT_IMPLEMENTED and "Float64" in e.value.msg
    with pytest.raises(engine.DfGpuError) as e:
        ctx.join_build(bb, [col(1), col(0)])
    assert e.value.code == A.ERR_NOT_IMPLEMENTED and "wider than 64 bits" in e.value.msg
    with pytest.raises(engine.DfGpuError) as e:
        ctx.join_build(bb, [col(1) / lit(0)])
    assert e.value.code == A.ERR_ARROW and "DivideByZero" in e.value.msg
    bb.free(); pb.free()


# ---- through ctx.sql() ------------------------------------------------------------------------------------------------
def sql_rows(hctx, sql):
    out = []
    for b in hctx.sql(sql).collect():
        cols = [c if isinstance(c, list) else np.asarray(c).tolist() for c in b]
        out.extend(zip(*cols))
    return sorted(out, key=repr)


@pytest.fixture(scope="module")
def tables():
    rng = np.random.default_rng(11)
    n = 50_000
    orders = {"oid": np.arange(n, dtype=np.int64), "cust": rng.integers(0, 1200, n).astype(np.int32),
              "prod": rng.integers(0, 40, n).astype(np.int16), "amount": (rng.integers(0, 8000, n) / 8).astype(np.float64)}
    cust = {"cid": np.arange(1000, dtype=np.int32), "region": rng.integers(0, 9, 1000).astype(np.int64),
            "cname": ["c%d" % i for i in range(1000)]}
    prod = {"pid": np.arange(50, dtype=np.int16), "price": (rng.integers(1, 100, 50) / 8).astype(np.float64)}
    return orders, cust, prod


def register(hctx, tables, batch_size=0):
    orders, cust, prod = tables
    hctx.register_memory("orders", list(orders.items()), batch_size=batch_size)
    hctx.register_memory("cust", list(cust.items()), batch_size=batch_size // 7 if batch_size else 0)
    hctx.register_memory("prod", list(prod.items()), batch_size=batch_size // 100 if batch_size else 0)


def py_join(tables):
    """orders JOIN cust ON cust = cid JOIN prod ON prod = pid as python dict rows"""
    orders, cust, prod = tables
    out = []
    for i in range(len(orders["oid"])):
        c, p = int(orders["cust"][i]), int(orders["prod"][i])
        if c < 1000 and p < 50:
            out.append(dict(oid=int(orders["oid"][i]), cust=c, prod=p, amount=float(orders["amount"][i]), region=int(cust["region"][c]),
                            cname=cust["cname"][c], price=float(prod["price"][p])))
    return out


@pytest.mark.parametrize("batch_size", [0, 7000], ids=["one-batch", "multi-batch"])
def test_sql_projection_where_residual(tables, batch_size):
    hctx = host.ExecutionContext(0)
    try:
        ref = py_join(tables)
        register(hctx, tables, batch_size)
        got = sql_rows(hctx, "SELECT o.oid, c.cname, amount FROM orders o JOIN cust c ON o.cust = c.cid AND amount > region "
                             "WHERE amount < 500")
        exp = sorted([(r["oid"], r["cname"], r["amount"]) for r in ref if r["amount"] > r["region"] and r["amount"] < 500], key=repr)
        assert got == exp
        register(hctx, tables, batch_size)
        got = sql_rows(hctx, "SELECT oid, cname, price FROM orders JOIN cust ON cust = cid JOIN prod ON prod = pid")
        assert got == sorted([(r["oid"], r["cname"], r["price"]) for r in ref], key=repr)
    finally:
        hctx.close()


@pytest.mark.parametrize("batch_size", [0, 7000], ids=["one-batch", "multi-batch"])
def test_sql_group_by_over_join(tables, batch_size):
    hctx = host.ExecutionContext(0)
    try:
        ref = py_join(tables)
        register(hctx, tables, batch_size)
        got = sql_rows(hctx, "SELECT region, SUM(amount), COUNT(oid), AVG(amount), COUNT(DISTINCT prod) FROM orders JOIN cust "
                             "ON cust = cid GROUP BY region")
        groups = {}
        for r in ref:
            groups.setdefault(r["region"], []).append(r)
        exp = sorted([(k, sum(r["amount"] for r in g), len(g), sum(r["amount"] for r in g) / len(g), len({r["prod"] for r in g}))
                      for k, g in groups.items()], key=repr)
        assert got == exp
        # a star join under a scalar aggregate
        register(hctx, tables, batch_size)
        got = sql_rows(hctx, "SELECT SUM(price), COUNT(oid) FROM orders JOIN cust ON cust = cid JOIN prod ON prod = pid WHERE region > 2")
        sel = [r for r in ref if r["region"] > 2]
        assert got == [(sum(r["price"] for r in sel), len(sel))]
    finally:
        hctx.close()


def test_relation_outliving_its_context(tables):
    # a join relation still holding its hash table when the context closes: the context releases it first
    hctx = host.ExecutionContext(0)
    register(hctx, tables, 7000)
    rel = hctx.sql("SELECT oid, cname FROM orders JOIN cust ON cust = cid")
    assert rel.next() is not None
    hctx.close()
    del rel
    # and a drained one released its table already; a fresh context still works
    hctx = host.ExecutionContext(0)
    register(hctx, tables, 7000)
    rel = hctx.sql("SELECT COUNT(oid) FROM orders JOIN cust ON cust = cid")
    assert int(rel.collect()[0][0][0]) == len(py_join(tables))
    hctx.close()
