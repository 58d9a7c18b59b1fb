"""Inner equi-join on keys with Utf8 parts, alone or mixed with integer parts (dfgpu_join_build / dfgpu_join_probe and
JOIN through ctx.sql()), compared with the exact join of tests/join_ref.py.  Utf8 parts compare byte for byte, a null part
never matches, and two keys that share a hash tag must not match: DFGPU_JOIN_TAG_BITS cuts the tag to force that.
Rows are compared as sorted multisets: the order of one probe row's matches is unspecified."""
import time

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import engine, host
from datafusion_archive_b200.expr import col, utf8_fn
from join_ref import inner as ref_join, same_pairs

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = engine.GpuContext(0)
    yield c
    c.close()


def as_arrow(a):
    return a if isinstance(a, pa.Array) else pa.array(a)


def gpu_pairs(ctx, probe_arrays, pkeys, build_arrays, bkeys):
    """Join with a row-number column appended to each side; returns (probe rows, build rows)."""
    pa_ = list(probe_arrays) + [np.arange(len(probe_arrays[0]), dtype=np.int64)]
    ba_ = list(build_arrays) + [np.arange(len(build_arrays[0]), dtype=np.int64)]
    pb, bb = ctx.upload(pa_), ctx.upload(ba_)
    j = ctx.join_build(bb, bkeys, keep_cols=[len(ba_) - 1])
    bb.free()
    r = j.probe(pb, pkeys, probe_cols=[len(pa_) - 1], build_cols=[len(ba_) - 1])
    got = r.columns()
    r.free(); j.free(); pb.free()
    return got[0], got[1]


def check(ctx, probe, pkeys, build, bkeys, ref_p=None, ref_b=None):
    """Join column lists on keys (a column number or a key program); the reference joins the arrays ref_p / ref_b
    (default: the key columns).  Returns the number of pairs."""
    ref_p = ref_p if ref_p is not None else [probe[k] for k in pkeys]
    ref_b = ref_b if ref_b is not None else [build[k] for k in bkeys]
    prog = lambda ks: [col(k) if isinstance(k, int) else k for k in ks]
    exp = ref_join(ref_p, ref_b)
    same_pairs(gpu_pairs(ctx, probe, prog(pkeys), build, prog(bkeys)), exp)
    return len(exp[0])


def strings(rng, n, pool, lo=8, hi=24):
    """n strings drawn from `pool` distinct random lowercase strings of lo..hi bytes, built without a Python loop per row"""
    lens = rng.integers(lo, hi + 1, pool)
    mat = rng.integers(97, 123, (pool, hi), dtype=np.uint8)
    pick = rng.integers(0, pool, n)
    ln = lens[pick]
    data = mat[pick][np.arange(hi)[None, :] < ln[:, None]]
    off = np.zeros(n + 1, np.int32)
    np.cumsum(ln, out=off[1:])
    return pa.StringArray.from_buffers(n, pa.py_buffer(off), pa.py_buffer(data.tobytes()))


# ---- key shapes ---------------------------------------------------------------------------------------------------------
def test_duplicates_nulls_and_empty_string(ctx):
    p = pa.array(["a", "", "b", None, "a", "", "zz", "a ", "A", None, "b"])
    b = pa.array(["", "a", "a", None, "b", "", "a ", "q", None])
    assert check(ctx, [p], [0], [b], [0]) > 0


def test_strings_differing_in_length_last_byte_or_far_in(ctx):
    long16 = "x" * 16
    kib4 = "y" * 4096
    vals = ["ab", "abc", "abd", "abcd", long16 + "a", long16 + "b", long16, long16 + "ab", kib4 + "0", kib4 + "1", kib4, "p" * 37,
            "p" * 36 + "q", "q" + "p" * 36]
    rng = np.random.default_rng(1)
    # rows at every alignment: the strings before a row shift where its bytes start
    p = pa.array([vals[i] for i in rng.integers(0, len(vals), 500)])
    b = pa.array([vals[i] for i in rng.integers(0, len(vals), 120)] + vals)
    assert check(ctx, [p], [0], [b], [0]) > 0


def test_non_ascii_bytes(ctx):
    vals = ["é", "e", "été", "ete", "中文", "中", "😀", "😀😀", "ß", "ss", "naïve", "naive"]
    rng = np.random.default_rng(2)
    p = pa.array([vals[i] for i in rng.integers(0, len(vals), 800)])
    b = pa.array([vals[i] for i in rng.integers(0, len(vals), 90)])
    assert check(ctx, [p], [0], [b], [0]) > 0


def test_empty_side_and_all_null(ctx):
    some = pa.array(["a", "b", "a"])
    empty = pa.array([], type=pa.string())
    nulls = pa.array([None, None, None], type=pa.string())
    assert check(ctx, [some], [0], [empty], [0]) == 0
    assert check(ctx, [empty], [0], [some], [0]) == 0
    assert check(ctx, [nulls], [0], [some], [0]) == 0
    assert check(ctx, [some], [0], [nulls], [0]) == 0


# ---- mixed keys -----------------------------------------------------------------------------------------------------------
def nullable(vals, valid):
    return pa.array(vals, mask=~np.asarray(valid, bool))


def mixed_case(rng, n):
    words = ["k%d" % i for i in range(7)] + [""]
    s = nullable([words[i] for i in rng.integers(0, len(words), n)], rng.random(n) > 0.1)
    i32 = nullable(rng.integers(-2, 3, n).astype(np.int32), rng.random(n) > 0.1)
    i64 = nullable(rng.integers(-2, 3, n).astype(np.int64), rng.random(n) > 0.1)
    t = nullable([words[i] for i in rng.integers(0, len(words), n)], rng.random(n) > 0.1)
    i16 = rng.integers(0, 2, n).astype(np.int16)
    return [s, i32, i64, t, i16]


@pytest.mark.parametrize("parts", [(0, 1), (2, 0), (0, 3), (1, 0, 3), (3, 4, 0, 1)], ids=["utf8+i32", "i64+utf8", "utf8+utf8",
                                                                                          "i32+utf8+utf8", "four-parts"])
def test_mixed_keys(ctx, parts):
    rng = np.random.default_rng(3)
    p, b = mixed_case(rng, 4000), mixed_case(rng, 600)
    keys = list(parts)
    assert check(ctx, p, keys, b, keys) > 0


def test_refusals(ctx):
    bb = ctx.upload([pa.array(["a", "b"]), np.array([1, 2], np.int64), np.array([1, 2], np.int32), np.array([1.0, 2.0])])
    with pytest.raises(engine.DfGpuError) as e:
        ctx.join_build(bb, [col(1), col(2), col(0)])
    assert e.value.code == A.ERR_NOT_IMPLEMENTED and "wider than 64 bits" in e.value.msg
    with pytest.raises(engine.DfGpuError) as e:
        ctx.join_build(bb, [col(0), col(3)])
    assert e.value.code == A.ERR_NOT_IMPLEMENTED and "Float64" in e.value.msg
    j = ctx.join_build(bb, [col(0)])
    pb = ctx.upload([np.array([1, 2], np.int64), pa.array(["a", "b"])])
    with pytest.raises(engine.DfGpuError) as e:
        j.probe(pb, [col(0)])
    assert e.value.code == A.ERR_EXECUTION and "JOIN key types differ: Int64 and Utf8" in e.value.msg
    j.free()
    j = ctx.join_build(bb, [col(1)])
    with pytest.raises(engine.DfGpuError) as e:
        j.probe(pb, [col(1)])
    assert e.value.code == A.ERR_EXECUTION and "JOIN key types differ: Utf8 and Int64" in e.value.msg
    j.free(); pb.free(); bb.free()


# ---- key expressions --------------------------------------------------------------------------------------------------------
def test_key_expressions(ctx):
    rng = np.random.default_rng(4)
    names = ["Alpha", "beta", "GAMMA", "Delta", "alpha", "BETA", "x" * 20 + "Y"]
    p = nullable([names[i] for i in rng.integers(0, len(names), 2000)], rng.random(2000) > 0.05)
    b = pa.array([n.lower() for n in names] + ["delta", "gamma"])
    low = pa.array([None if v is None else v.lower() for v in p.to_pylist()])
    assert check(ctx, [p], [utf8_fn("lower", col(0))], [b], [0], ref_p=[low]) > 0
    codes_ = pa.array(["ab%d-%d" % (i % 13, i) for i in range(3000)])
    prefix = pa.array(["ab%d-" % i for i in range(0, 20, 2)])
    sub = pc.utf8_slice_codeunits(codes_, 0, 4)
    assert check(ctx, [prefix], [0], [codes_], [utf8_fn("substr", col(0), 1, 4)], ref_b=[sub]) > 0


# ---- payloads -------------------------------------------------------------------------------------------------------------
def test_payloads_and_key_outputs(ctx):
    rng = np.random.default_rng(5)
    n_p, n_b = 3000, 500
    words = ["w%d" % i for i in range(60)]
    pk = nullable([words[i] for i in rng.integers(0, 60, n_p)], rng.random(n_p) > 0.1)
    bk = nullable([words[i] for i in rng.integers(0, 60, n_b)], rng.random(n_b) > 0.1)
    f64 = nullable(rng.random(n_p), rng.random(n_p) > 0.2)
    pstr = pa.array(["s%d" % (i * 7 % 13) * (i % 4) for i in range(n_p)], mask=rng.random(n_p) < 0.2)
    i8 = nullable(rng.integers(-100, 100, n_b).astype(np.int8), rng.random(n_b) > 0.2)
    bools = pa.array(rng.random(n_b) > 0.5, mask=rng.random(n_b) < 0.2)
    bstr = pa.array(["t%d" % i for i in range(n_b)], mask=rng.random(n_b) < 0.2)
    pb = ctx.upload([pk, f64, pstr])
    bb = ctx.upload([bk, i8, bools, bstr])
    j = ctx.join_build(bb, [col(0)], keep_cols=[0, 1, 2, 3])
    bb.free()
    r = j.probe(pb, [col(0)], probe_cols=[0, 1, 2], build_cols=[3, 2, 1, 0])
    got = r.columns()
    r.free(); j.free(); pb.free()
    prow, brow = ref_join([pk], [bk])

    def rows(c):
        v, m = c if isinstance(c, tuple) else (c, np.ones(len(c), bool))
        v = v if isinstance(v, list) else np.asarray(v).tolist()
        return [x if ok else None for x, ok in zip(v, m.tolist())]

    def expect(arr, idx):
        py = arr.to_pylist()
        return [py[i] for i in idx]

    got_rows = sorted(zip(*[rows(c) for c in got]), key=repr)
    exp_rows = sorted(zip(expect(pk, prow), expect(f64, prow), expect(pstr, prow), expect(bstr, brow), expect(bools, brow),
                          expect(i8, brow), expect(bk, brow)), key=repr)
    assert len(got_rows) == len(exp_rows) > 0
    assert got_rows == exp_rows


# ---- forced collisions --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", [4, 1])
def test_forced_tag_collisions(ctx, monkeypatch, bits):
    monkeypatch.setenv("DFGPU_JOIN_TAG_BITS", str(bits))
    rng = np.random.default_rng(6)
    distinct = ["key-%d" % i for i in range(3000)]
    # many distinct build strings, most of them repeated, so that many share a tag and the rounds run
    b = nullable([distinct[i] for i in rng.integers(0, 2000, 6000)], rng.random(6000) > 0.02)
    p = pa.array([distinct[i] for i in rng.integers(0, 3000, 20000)])
    assert check(ctx, [p], [0], [b], [0]) > 0
    i32b, i32p = rng.integers(0, 3, 6000).astype(np.int32), rng.integers(0, 3, 20000).astype(np.int32)
    assert check(ctx, [p, i32p], [0, 1], [b, i32b], [0, 1]) > 0


def test_tag_bits_out_of_range(ctx, monkeypatch):
    monkeypatch.setenv("DFGPU_JOIN_TAG_BITS", "0")
    bb = ctx.upload([pa.array(["a"])])
    with pytest.raises(engine.DfGpuError) as e:
        ctx.join_build(bb, [col(0)])
    assert "DFGPU_JOIN_TAG_BITS" in e.value.msg
    bb.free()


# ---- scale ------------------------------------------------------------------------------------------------------------------
def test_large_random(ctx):
    rng = np.random.default_rng(7)
    b = strings(rng, 1_000_000, 2_000_000)
    p = strings(np.random.default_rng(7), 10_000_000, 2_000_000)  # the same pool: about half the probe rows match
    assert check(ctx, [p], [0], [b], [0]) > 1_000_000


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
    hot = pa.array(["the hot key"] * n)
    probe = pa.array(["the hot key", "cold", "the hot key", "the hot ke"])
    t0 = time.perf_counter()
    skew_ms, skew_rows = _probe_kernel_ms(ctx, hot, probe)
    assert time.perf_counter() - t0 < 60
    uniq = pa.array(["u%08d" % i for i in range(n)])
    uni_ms, uni_rows = _probe_kernel_ms(ctx, uniq, uniq)
    assert skew_rows == 2 * n and uni_rows == n
    assert skew_ms < 10 * uni_ms + 1.0, (skew_ms, uni_ms)
    got = gpu_pairs(ctx, [probe], [col(0)], [hot], [col(0)])
    assert sorted(set(got[0].tolist())) == [0, 2]
    assert np.array_equal(np.sort(got[1][got[0] == 0]), np.arange(n))


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
    cust_of = rng.integers(0, 1200, n)
    orders = {"oid": np.arange(n, dtype=np.int64), "cname": ["cust-%d" % c for c in cust_of],
              "ucname": ["CUST-%d" % c for c in cust_of], "prod": rng.integers(0, 40, n).astype(np.int16),
              "amount": (rng.integers(0, 8000, n) / 8).astype(np.float64)}
    cust = {"cname": ["cust-%d" % i for i in range(1000)], "region": rng.integers(0, 9, 1000).astype(np.int64),
            "city": ["city%d" % (i % 17) for i in range(1000)]}
    prod = {"pid": np.arange(50, dtype=np.int16), "price": (rng.integers(1, 100, 50) / 8).astype(np.float64)}
    return orders, cust, prod, cust_of


def register(hctx, tables, batch_size=0):
    orders, cust, prod, _ = tables
    hctx.register_memory("orders", list(orders.items()), batch_size=batch_size)
    hctx.register_memory("cust", list(cust.items()), batch_size=batch_size // 7 if batch_size else 0)
    hctx.register_memory("prod", list(prod.items()), batch_size=batch_size // 100 if batch_size else 0)


def py_join(tables):
    orders, cust, prod, cust_of = tables
    out = []
    for i in range(len(orders["oid"])):
        c, p = int(cust_of[i]), int(orders["prod"][i])
        if c < 1000:
            out.append(dict(oid=int(orders["oid"][i]), cname=orders["cname"][i], prod=p, amount=float(orders["amount"][i]),
                            region=int(cust["region"][c]), city=cust["city"][c], price=float(prod["price"][p]) if p < 50 else None))
    return out


@pytest.mark.parametrize("batch_size", [0, 7000], ids=["one-batch", "multi-batch"])
def test_sql_projection_where_residual(tables, batch_size):
    hctx = host.ExecutionContext(0)
    try:
        ref = py_join(tables)
        register(hctx, tables, batch_size)
        got = sql_rows(hctx, "SELECT o.oid, c.city, o.cname, amount FROM orders o JOIN cust c ON o.cname = c.cname AND amount > region "
                             "WHERE amount < 500")
        exp = sorted([(r["oid"], r["city"], r["cname"], r["amount"]) for r in ref if r["amount"] > r["region"] and r["amount"] < 500], key=repr)
        assert got == exp and len(exp) > 0
        register(hctx, tables, batch_size)
        got = sql_rows(hctx, "SELECT oid, city, price FROM orders o JOIN cust c ON o.cname = c.cname JOIN prod ON prod = pid")
        assert got == sorted([(r["oid"], r["city"], r["price"]) for r in ref if r["price"] is not None], key=repr)
        register(hctx, tables, batch_size)
        got = sql_rows(hctx, "SELECT oid, region FROM orders o JOIN cust c ON lower(o.ucname) = c.cname")
        assert got == sorted([(r["oid"], r["region"]) for r in ref], key=repr)
    finally:
        hctx.close()


@pytest.mark.parametrize("batch_size", [0, 7000], ids=["one-batch", "multi-batch"])
def test_sql_group_by_over_join(tables, batch_size):
    hctx = host.ExecutionContext(0)
    try:
        ref = py_join(tables)
        register(hctx, tables, batch_size)
        got = sql_rows(hctx, "SELECT region, SUM(amount), COUNT(oid), AVG(amount), COUNT(DISTINCT prod) FROM orders o JOIN cust c "
                             "ON o.cname = c.cname GROUP BY region")
        groups = {}
        for r in ref:
            groups.setdefault(r["region"], []).append(r)
        exp = sorted([(k, sum(r["amount"] for r in g), len(g), sum(r["amount"] for r in g) / len(g), len({r["prod"] for r in g}))
                      for k, g in groups.items()], key=repr)
        assert len(got) == len(exp)
        for g, e in zip(got, exp):
            assert g[0] == e[0] and g[2] == e[2] and g[4] == e[4]
            assert g[1] == pytest.approx(e[1], rel=1e-12) and g[3] == pytest.approx(e[3], rel=1e-12)
        # a Utf8 GROUP BY key over the join
        register(hctx, tables, batch_size)
        got = sql_rows(hctx, "SELECT city, SUM(amount), COUNT(oid) FROM orders o JOIN cust c ON o.cname = c.cname GROUP BY city")
        by_city = {}
        for r in ref:
            by_city.setdefault(r["city"], []).append(r)
        exp = sorted([(k, sum(r["amount"] for r in g), len(g)) for k, g in by_city.items()], key=repr)
        assert [(g[0], g[2]) for g in got] == [(e[0], e[2]) for e in exp]
        assert all(g[1] == pytest.approx(e[1], rel=1e-12) for g, e in zip(got, exp))
    finally:
        hctx.close()
