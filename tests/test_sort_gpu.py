"""dfgpu_sort through the C ABI and HAVING / ORDER BY / LIMIT through SQL, compared exactly against the numpy reference
order of tests/sort_ref.py (np.lexsort over each key's encoding, the row number last).  GPU required."""
import os

import numpy as np
import pyarrow as pa
import pytest

from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import engine, host
from datafusion_archive_b200.expr import Utf8Function, col, lit

import sort_ref as R

pytestmark = pytest.mark.gpu
DATA = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "data")
INTS = [A.INT8, A.INT16, A.INT32, A.INT64, A.UINT8, A.UINT16, A.UINT32, A.UINT64]


@pytest.fixture(scope="module")
def ctx():
    c = engine.GpuContext(0)
    yield c
    c.close()


def int_values(rng, dtype, n):
    info = np.iinfo(A.NP_OF[dtype])
    v = rng.integers(info.min, info.max, size=n, dtype=A.NP_OF[dtype], endpoint=True)
    edges = np.array([info.min, info.max, 0, 1, info.max - 1], dtype=A.NP_OF[dtype])
    v[:len(edges)] = edges[:n]
    return v


def float_values(rng, dtype, n):
    t = A.NP_OF[dtype]
    bits = np.uint32 if dtype == A.FLOAT32 else np.uint64
    v = rng.standard_normal(n).astype(t) * t(1e3)
    info = np.finfo(t)
    nan_payloads = np.array([0x7fc00001, 0xffc00002, 0x7f800001] if dtype == A.FLOAT32 else
                            [0x7ff8000000000001, 0xfff8000000000002, 0x7ff0000000000001], dtype=bits).view(t)
    edges = np.concatenate([np.array([0.0, -0.0, np.inf, -np.inf, info.max, info.min, info.tiny, -info.tiny, info.smallest_subnormal,
                                      -info.smallest_subnormal], dtype=t), nan_payloads])
    k = min(n, len(edges))
    v[rng.choice(n, size=k, replace=False)] = edges[:k]
    return v


def strings(rng, n):
    pool = ["", "a", "a\0", "a\0b", "ab", "b", "é", "€x", "ÿ", "aaaaaaaa", "aaaaaaaab", "aaaaaaaa\0", "aaaaaaaaaaaaaaaaX",
            "aaaaaaaaaaaaaaaaY", "aaaaaaaaaaaaaaaa", "aaaaaaaaaaaaaaaaaaaaaaaaZ", "zz"]
    return [pool[i] for i in rng.integers(0, len(pool), size=n)]


def to_arrow(dtype, vals, valid):
    mask = None if valid is None else ~np.asarray(valid, dtype=bool)
    if dtype == A.UTF8:
        return pa.array(list(vals), type=pa.string(), mask=mask)
    return pa.array(np.asarray(vals), mask=mask)


def run(ctx, arrays, keys, desc, keep=None, limit=-1):
    b = ctx.upload(arrays)
    try:
        r = ctx.sort(b, keys=keys, desc=desc, keep=keep, limit=limit)
        try:
            return r.columns()
        finally:
            r.free()
    finally:
        b.free()


def check(ctx, specs, keep_valid=None, keep_null=None, limit=-1, extra=()):
    """Sort by the key columns `specs` [(dtype, vals, valid, desc)], with an Int64 row-number payload and the `extra`
    columns [(dtype, vals, valid)]; compare every output column with the reference."""
    n = len(specs[0][1]) if specs else len(extra[0][1])
    arrays = [to_arrow(dt, v, ok) for dt, v, ok, _ in specs] + [np.arange(n, dtype=np.int64)] + [to_arrow(dt, v, ok) for dt, v, ok in extra]
    keep = None
    kept = None
    if keep_valid is not None:
        arrays.append(pa.array(np.asarray(keep_valid, dtype=bool), mask=None if keep_null is None else np.asarray(keep_null, dtype=bool)))
        keep = col(len(arrays) - 1)
        kept = np.asarray(keep_valid, dtype=bool) & (True if keep_null is None else ~np.asarray(keep_null, dtype=bool))
    got = run(ctx, arrays, [col(i) for i in range(len(specs))], [d for *_, d in specs], keep=keep, limit=limit)
    want = R.order(n, specs, kept)
    if limit >= 0:
        want = want[:limit]
    assert np.array_equal(got[len(specs)], want)
    if len(want) == 0:
        assert all(len(c[0] if isinstance(c, tuple) else c) == 0 for c in got)
        return want
    for i, (dt, v, ok) in enumerate([(dt, v, ok) for dt, v, ok, _ in specs] + list(extra)):
        g = got[i if i < len(specs) else i + 1]
        if isinstance(g, tuple):
            g, gmask = g
            assert ok is not None and np.array_equal(gmask, np.asarray(ok, dtype=bool)[want])
        else:
            assert ok is None or np.asarray(ok, dtype=bool)[want].all()
        if dt == A.UTF8:
            exp = [v[j] for j in want]
            okw = [True] * len(want) if ok is None else list(np.asarray(ok, dtype=bool)[want])
            assert [x for x, o in zip(g, okw) if o] == [x for x, o in zip(exp, okw) if o]
        elif dt == A.BOOL:
            assert np.array_equal(np.asarray(g, dtype=bool), np.asarray(v, dtype=bool)[want])
        else:
            exp = np.asarray(v)[want]
            okw = np.ones(len(want), bool) if ok is None else np.asarray(ok, dtype=bool)[want]
            assert np.array_equal(np.asarray(g).view(np.uint8).reshape(len(want), -1)[okw], exp.view(np.uint8).reshape(len(want), -1)[okw])
    return want


@pytest.mark.parametrize("desc", [False, True])
@pytest.mark.parametrize("dtype", INTS + [A.FLOAT32, A.FLOAT64, A.UTF8])
def test_every_key_dtype(ctx, dtype, desc):
    rng = np.random.default_rng(dtype * 2 + desc)
    n = 20_000
    if dtype == A.UTF8:
        v = strings(rng, n)
    elif dtype in (A.FLOAT32, A.FLOAT64):
        v = float_values(rng, dtype, n)
    else:
        v = int_values(rng, dtype, n)
    check(ctx, [(dtype, v, None, desc)])


@pytest.mark.parametrize("desc", [False, True])
@pytest.mark.parametrize("dtype", [A.INT32, A.UINT64, A.FLOAT64, A.UTF8])
def test_nullable_keys(ctx, dtype, desc):
    rng = np.random.default_rng(100 + dtype)
    n = 10_000
    v = strings(rng, n) if dtype == A.UTF8 else (float_values(rng, dtype, n) if dtype == A.FLOAT64 else int_values(rng, dtype, n) % 7)
    valid = rng.random(n) > 0.3
    check(ctx, [(dtype, v, valid, desc)])


@pytest.mark.parametrize("seed", range(4))
def test_mixed_keys(ctx, seed):
    rng = np.random.default_rng(seed)
    n = 50_000
    pool = [(A.INT8, lambda: rng.integers(-3, 3, n).astype(np.int8)), (A.UINT32, lambda: rng.integers(0, 5, n).astype(np.uint32)),
            (A.FLOAT32, lambda: rng.choice(np.array([0.0, -0.0, 1.0, np.nan, -np.inf], np.float32), n)),
            (A.UTF8, lambda: strings(rng, n)), (A.INT64, lambda: rng.integers(-2, 2, n))]
    nk = 2 + seed % 3
    specs = []
    for i in rng.choice(len(pool), size=nk, replace=False):
        dt, gen = pool[i]
        specs.append((dt, gen(), (rng.random(n) > 0.1) if rng.random() < 0.5 else None, bool(rng.random() < 0.5)))
    check(ctx, specs)


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 2047, 2048, 2049, 4095, 4096, 4097, 1_000_000, (1 << 24) + 1])
def test_sizes(ctx, n):
    rng = np.random.default_rng(n)
    check(ctx, [(A.INT64, rng.integers(-50, 50, n), None, False), (A.FLOAT64, rng.standard_normal(n), None, True)])


def test_all_equal_keys_keep_input_order(ctx):
    n = 100_000
    want = check(ctx, [(A.INT32, np.full(n, 7, np.int32), None, False), (A.UTF8, ["same"] * n, None, True)])
    assert np.array_equal(want, np.arange(n))


def test_constant_high_digits_skip_passes(ctx):
    rng = np.random.default_rng(5)
    n = 200_000
    before = ctx.kernel_launches()
    check(ctx, [(A.INT64, rng.integers(0, 1000, n), None, False)])  # 2 live digits of 8
    narrow = ctx.kernel_launches() - before
    before = ctx.kernel_launches()
    check(ctx, [(A.INT64, rng.integers(-(1 << 62), 1 << 62, n), None, False)])
    wide = ctx.kernel_launches() - before
    assert wide - narrow == 6 * 5  # six more passes of count + three scan kernels + scatter


def test_utf8_edges(ctx):
    edge = ["", "", "a", "a\0", "\0", "\0\0", "a\0\0", "ab", "aaaaaaaa", "aaaaaaaa\0", "aaaaaaaaa", "aaaaaaaaaaaaaaaa", "aaaaaaaaaaaaaaaa\0",
            "aaaaaaaaaaaaaaaab", "aaaaaaaaaaaaaaaaaaaaaaaaa", "aaaaaaaaaaaaaaaaaaaaaaaab", "é", "ÿ", "€", "\U0001F600", "z" * 40]
    rng = np.random.default_rng(9)
    v = [edge[i] for i in rng.integers(0, len(edge), 5000)]
    for desc in (False, True):
        check(ctx, [(A.UTF8, v, None, desc)])


def test_utf8_random_million(ctx):
    rng = np.random.default_rng(11)
    n = 1_000_000
    lens = rng.integers(0, 41, n)
    raw = rng.integers(97, 101, int(lens.sum()), dtype=np.uint8).tobytes().decode()
    ends = np.cumsum(lens)
    v = [raw[e - l:e] for e, l in zip(ends, lens)]
    check(ctx, [(A.UTF8, v, None, False)])


@pytest.mark.parametrize("limit", [0, 1, 9_999, 10_000, 10_005])
def test_limit(ctx, limit):
    rng = np.random.default_rng(limit)
    n = 10_000
    check(ctx, [(A.INT16, rng.integers(-5, 5, n).astype(np.int16), None, True)], limit=limit,
          extra=[(A.UTF8, strings(rng, n), rng.random(n) > 0.5), (A.BOOL, rng.random(n) > 0.5, None)])


def test_keep_mask_with_nulls(ctx):
    rng = np.random.default_rng(3)
    n = 30_000
    check(ctx, [(A.UINT8, rng.integers(0, 256, n).astype(np.uint8), None, False)], keep_valid=rng.random(n) > 0.4,
          keep_null=rng.random(n) < 0.2, limit=1000, extra=[(A.FLOAT64, rng.standard_normal(n), rng.random(n) > 0.5)])


def test_keep_without_keys_keeps_row_order(ctx):
    rng = np.random.default_rng(4)
    n = 10_000
    kv = rng.random(n) > 0.5
    b = ctx.upload([np.arange(n, dtype=np.int64), pa.array(kv)])
    r = ctx.sort(b, keep=col(1))
    assert np.array_equal(r.columns()[0], np.flatnonzero(kv))
    r.free()
    b.free()


def test_expression_keys(ctx):
    rng = np.random.default_rng(6)
    n = 20_000
    a, b = rng.integers(-100, 100, n), rng.integers(-100, 100, n)
    s = [x.upper() if i % 2 else x for i, x in enumerate(strings(rng, n))]
    bt = ctx.upload([a, b, pa.array(s), np.arange(n, dtype=np.int64)])
    r = ctx.sort(bt, keys=[Utf8Function("lower", col(2)), col(0) + col(1)], desc=[True, False], keep=col(0) > lit(-50))
    got = r.columns()[3]
    r.free()
    bt.free()
    low = [x.lower() if x.isascii() else "".join(c.lower() if c.isascii() else c for c in x) for x in s]
    want = R.order(n, [(A.UTF8, low, None, True), (A.INT64, a + b, None, False)], a > -50)
    assert np.array_equal(got, want)


def test_sort_a_device_result_in_place(ctx):
    rng = np.random.default_rng(8)
    n = 50_000
    k = rng.integers(0, 1000, n)
    v = rng.integers(0, 10, n)
    from datafusion_archive_b200.expr import AggregateFunction
    b = ctx.upload([k, v])
    agg = ctx.aggregate(b, keys=[col(0)], aggs=[AggregateFunction("SUM", col(1))])
    r = ctx.sort(agg, keys=[col(1), col(0)], desc=[True, False], limit=10)
    keys, sums = r.columns()
    r.free()
    agg.free()
    b.free()
    ref = {}
    for x, y in zip(k, v):
        ref[x] = ref.get(x, 0) + y
    want = sorted(ref.items(), key=lambda t: (-t[1], t[0]))[:10]
    assert list(zip(keys.tolist(), sums.tolist())) == want


def test_refusals(ctx):
    b = ctx.upload([np.arange(10, dtype=np.int64), np.ones(10, bool)])
    with pytest.raises(engine.DfGpuError) as ei:
        ctx.sort(b, keys=[col(1)])
    assert ei.value.code == A.ERR_NOT_IMPLEMENTED and "Boolean" in ei.value.msg
    with pytest.raises(engine.DfGpuError) as ei:
        ctx.sort(b, keys=[col(0)], keep=col(0))
    assert ei.value.code == A.ERR_EXECUTION and "not Boolean" in ei.value.msg
    b.free()


# ---- SQL ---------------------------------------------------------------------------------------------------------------
@pytest.fixture()
def sql():
    c = host.ExecutionContext(0)
    yield c
    c.close()


def rows(rel):
    out = []
    for batch in rel.collect():
        cols = [[v if m else None for v, m in zip(*c)] if isinstance(c, tuple) else list(c) for c in batch]
        out.extend(zip(*cols))
    return [tuple(x.item() if hasattr(x, "item") else x for x in r) for r in out]


def test_golden_group_by_order_by(sql):
    sql.register_csv("t1", os.path.join(DATA, "aggregate_test_1.csv"), [("a", A.INT32), ("b", A.FLOAT64)], 1024)
    assert rows(sql.sql("SELECT a, MIN(b), MAX(b) FROM t1 GROUP BY a ORDER BY a")) == [(1, 1.1, 2.2), (2, 3.3, 5.5), (3, 1.0, 2.0)]
    sql.register_csv("t2", os.path.join(DATA, "aggregate_test_2.csv"), [("a", A.UTF8), ("b", A.FLOAT64)], 1024)
    assert [r[0] for r in rows(sql.sql("SELECT a, MIN(b), MAX(b) FROM t2 GROUP BY a ORDER BY a"))] == ["one", "three", "two"]


def memory_table(sql, n=20_000, seed=0):
    """Registers table t (a DataSource is read once: a second query over it registers it again)."""
    rng = np.random.default_rng(seed)
    k = rng.integers(0, 300, n)
    v = rng.integers(-5, 6, n)
    x = rng.standard_normal(n)
    xvalid = ~np.isin(k % 17, [3])  # groups with k % 17 == 3 have no x at all
    city = np.array(["Rome", "oslo", "Lima", "kyiv", "Bern", "rome"])[k % 6]
    sql.register_memory("t", [("k", k), ("v", v), ("x", pa.array(x, mask=~xvalid)), ("city", pa.array(list(city)))])
    return k, v, x, xvalid, city


def groups(k, *cols):
    out = {}
    for i, key in enumerate(k.tolist()):
        out.setdefault(key, []).append(i)
    return out


def test_top_n_with_a_tie_at_the_limit(sql):
    k, v, *_ = memory_table(sql)
    g = groups(k)
    sums = {key: int(v[ix].sum()) for key, ix in g.items()}
    want = sorted(sums.items(), key=lambda t: (-t[1], t[0]))
    cut = 7
    while want[cut - 1][1] != want[cut][1]:  # put the limit inside a run of equal sums
        cut += 1
    assert rows(sql.sql("SELECT k, SUM(v) FROM t GROUP BY k ORDER BY SUM(v) DESC LIMIT %d" % cut)) == want[:cut]


def test_having_on_a_hidden_count_and_limit_without_order(sql):
    k, v, *_ = memory_table(sql)
    g = groups(k)
    want = sorted((key, int(v[ix].sum())) for key, ix in g.items() if len(ix) > 70)
    assert rows(sql.sql("SELECT k, SUM(v) FROM t GROUP BY k HAVING CAST(COUNT(v) AS BIGINT) > 70 ORDER BY k")) == want
    memory_table(sql)  # a DataSource is read once
    assert rows(sql.sql("SELECT k, SUM(v) FROM t GROUP BY k HAVING CAST(COUNT(v) AS BIGINT) > 70 LIMIT 5")) == want[:5]


def test_order_by_avg_with_null_groups_and_having_keeps_the_null(sql):
    k, v, x, xvalid, _ = memory_table(sql)
    g = groups(k)
    avg = {}
    for key, ix in g.items():
        ok = [i for i in ix if xvalid[i]]
        avg[key] = float(np.sum(x[ok])) / len(ok) if ok else None
    got = rows(sql.sql("SELECT k, AVG(x) FROM t GROUP BY k HAVING CAST(COUNT(v) AS BIGINT) > 0 ORDER BY AVG(x) DESC, k"))
    nonnull = sorted(((a, b) for a, b in avg.items() if b is not None), key=lambda t: (-t[1], t[0]))
    nulls = sorted((a, b) for a, b in avg.items() if b is None)
    assert nulls and [r[0] for r in got] == [a for a, _ in nonnull + nulls]
    assert [r[1] is None for r in got] == [b is None for _, b in nonnull + nulls]
    np.testing.assert_allclose([r[1] for r in got if r[1] is not None], [b for _, b in nonnull], rtol=1e-12)


def test_order_by_utf8_key_and_lower(sql):
    k, v, _, _, city = memory_table(sql)
    got = rows(sql.sql("SELECT city, COUNT(v) FROM t GROUP BY city ORDER BY city"))
    cnt = {c: int((city == c).sum()) for c in set(city.tolist())}
    assert got == sorted(cnt.items())
    memory_table(sql)
    got = rows(sql.sql("SELECT city, COUNT(v) FROM t GROUP BY city ORDER BY lower(city) DESC"))
    want = sorted(cnt.items())
    want.sort(key=lambda t: t[0].lower().encode(), reverse=True)  # stable: equal lower-case names stay in name order
    assert got == want


def test_count_distinct_order_by(sql):
    k, v, *_ = memory_table(sql)
    g = groups(k)
    d = {key: len(set(v[ix].tolist())) for key, ix in g.items()}
    want = sorted(d.items(), key=lambda t: (-t[1], t[0]))[:12]
    assert rows(sql.sql("SELECT k, COUNT(DISTINCT v) FROM t GROUP BY k ORDER BY COUNT(DISTINCT v) DESC LIMIT 12")) == want


def test_join_group_by_order_by(sql):
    k, v, *_ = memory_table(sql)
    dim_k = np.arange(0, 300, 2, dtype=np.int64)
    dim_w = (dim_k % 5).astype(np.int64)
    sql.register_memory("d", [("dk", dim_k), ("w", dim_w)])
    got = rows(sql.sql("SELECT w, SUM(v) FROM t JOIN d ON k = dk GROUP BY w ORDER BY SUM(v) DESC, w"))
    s = {}
    for key, val in zip(k.tolist(), v.tolist()):
        if key % 2 == 0:
            s[key % 5] = s.get(key % 5, 0) + val
    assert got == sorted(s.items(), key=lambda t: (-t[1], t[0]))


def test_order_by_a_case_made_null(sql):
    k, v, *_ = memory_table(sql)
    g = groups(k)
    sums = {key: int(v[ix].sum()) for key, ix in g.items()}
    got = rows(sql.sql("SELECT k, SUM(v) FROM t GROUP BY k ORDER BY CASE WHEN SUM(v) > 0 THEN SUM(v) END DESC"))
    pos = sorted(((a, b) for a, b in sums.items() if b > 0), key=lambda t: (-t[1], t[0]))
    rest = sorted((a, b) for a, b in sums.items() if b <= 0)
    assert got == pos + rest


def test_no_group_by_having(sql):
    memory_table(sql)
    assert rows(sql.sql("SELECT COUNT(v) FROM t HAVING CAST(COUNT(v) AS BIGINT) > 1000000")) == []
    memory_table(sql)
    assert rows(sql.sql("SELECT COUNT(v) FROM t HAVING CAST(COUNT(v) AS BIGINT) > 10")) == [(20_000,)]
    sql.register_memory("e", [("a", np.zeros(0, np.int64))])
    assert rows(sql.sql("SELECT MIN(a) FROM e HAVING MIN(a) > 0")) == []
    # the one row of nulls of an empty input goes through HAVING too, and keeps its null (a null is below every value)
    assert rows(sql.sql("SELECT MIN(a) FROM e HAVING MIN(a) < 1")) == [(None,)]


def test_non_aggregate_order_by_keeps_its_error(sql):
    memory_table(sql)
    with pytest.raises(host.ExecutionError) as ei:
        sql.sql("SELECT k FROM t ORDER BY k").collect()
    assert ei.value.code == A.ERR_NOT_IMPLEMENTED and "unimplemented!()" in ei.value.msg
