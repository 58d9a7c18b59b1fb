"""The exact GROUP BY reference (tests/groupby_ref.py) against the CPU oracle, on small inputs with edge values, with and
without a WHERE; and its AVG, COUNT(DISTINCT) and no-row rules, which the oracle does not have, worked by hand.

The oracle restates the reference's `f64::min` / `f64::max`, which return whichever zero came first, so float
MIN / MAX are compared with -0.0 and +0.0 as equal here; the reference's own ±0 order is checked directly."""
import numpy as np
import pytest

import groupby_ref as R
import oracle_lib as O
from datafusion_archive_b200.expr import AggregateFunction, col, lit

FUNCS = [R.MIN, R.MAX, R.SUM, R.COUNT]


def oracle_cols(arrays, nkeys, aggs):
    """Oracle result of GROUP BY col(0..nkeys) with aggs = [(func, column index)]."""
    return O.aggregate(arrays, [col(i) for i in range(nkeys)], [AggregateFunction(f, col(c)) for f, c in aggs])


def zeros_equal(got, exp):
    """Copies of got / exp in which float MIN / MAX results carry +0.0 for either zero."""
    nk = len(exp.keys)
    got = list(got)
    for i, e in enumerate(exp.aggs):
        if e["func"] in (R.MIN, R.MAX) and np.issubdtype(e["dtype"], np.floating):
            e["values"] = e["values"] + e["dtype"].type(0)
            c = got[nk + i]
            got[nk + i] = (c[0] + c[0].dtype.type(0), c[1]) if isinstance(c, tuple) else c + c.dtype.type(0)
    return got, exp


def data(rng, n, kdt, vdt, for_sum):
    k = rng.integers(-3, 20, n).astype(kdt)
    k[::7] = np.array(-1).astype(kdt)  # the key that packs to the empty marker
    if np.issubdtype(kdt, np.integer):
        k[3::11] = np.iinfo(kdt).min
        k[5::13] = np.iinfo(kdt).max
    v = R.sprinkle(rng, R.random_values(rng, vdt, n), R.edges(vdt, for_sum), frac=0.2)
    return k, v


@pytest.mark.parametrize("kdt", [np.int64, np.uint64, np.int32, np.int8])
@pytest.mark.parametrize("vdt", [np.float64, np.float32, np.int64, np.uint64, np.int32, np.uint16])
def test_reference_matches_oracle_groupby(kdt, vdt):
    rng = np.random.default_rng(int(np.dtype(kdt).num) * 100 + np.dtype(vdt).num)
    n = 3001
    k, v = data(rng, n, kdt, vdt, for_sum=False)
    _, s = data(rng, n, kdt, vdt, for_sum=True)
    aggs = [(R.MIN, 1), (R.MAX, 1), (R.SUM, 2), (R.COUNT, 1), (R.SUM, 1) if not np.issubdtype(vdt, np.floating) else (R.COUNT, 2)]
    exp = R.aggregate([k], [(f, [None, v, s][c]) for f, c in aggs])
    got, exp = zeros_equal(oracle_cols([k, v, s], 1, aggs), exp)
    R.assert_matches(got, exp, "oracle")


def test_reference_matches_oracle_composite_keys():
    rng = np.random.default_rng(5)
    n = 2003
    cases = [[np.int32, np.int32], [np.int16, np.int16, np.int32], [np.uint8, np.int8, np.uint16, np.int32]]
    for dts in cases:
        keys = [rng.integers(-3, 3, n).astype(dt) for dt in dts]
        for k in keys:
            k[::5] = np.array(-1).astype(k.dtype)  # (-1, -1, ...) packs to all ones
        v = R.sprinkle(rng, R.random_values(rng, np.int64, n), R.edges(np.int64))
        aggs = [(R.MIN, 0), (R.MAX, 0), (R.SUM, 0), (R.COUNT, 0)]
        exp = R.aggregate(keys, [(f, v) for f, _ in aggs])
        got = O.aggregate(keys + [v], [col(i) for i in range(len(keys))], [AggregateFunction(f, col(len(keys))) for f, _ in aggs])
        R.assert_matches(got, exp, str(dts))


def test_reference_matches_oracle_nulls():
    rng = np.random.default_rng(6)
    n = 2500
    k, v = data(rng, n, np.int32, np.float64, for_sum=False)
    _, s = data(rng, n, np.int32, np.float64, for_sum=True)
    vk, vv, vs = rng.random(n) > 0.2, rng.random(n) > 0.3, rng.random(n) > 0.5
    aggs = [(R.MIN, 1), (R.MAX, 1), (R.SUM, 2), (R.COUNT, 1), (R.COUNT, 2)]
    arrays = [R.arrow_nullable(k, vk), R.arrow_nullable(v, vv), R.arrow_nullable(s, vs)]
    exp = R.aggregate([(k, vk)], [(f, [None, (v, vv), (s, vs)][c]) for f, c in aggs])
    got, exp = zeros_equal(oracle_cols(arrays, 1, aggs), exp)
    R.assert_matches(got, exp, "nulls")
    # no GROUP BY: null values are skipped (the oracle's NaN-first quirk of DESIGN §7 is kept out: row 0 is 1.0)
    s[0], vs[0] = 1.0, True
    aggs0 = [AggregateFunction(f, col(0)) for f in FUNCS]
    got = O.aggregate([R.arrow_nullable(s, vs)], [], aggs0)
    exp = R.aggregate([], [(f, (s, vs)) for f in FUNCS])
    got, exp = zeros_equal(got, exp)
    R.assert_matches(got, exp, "reduce")


def test_reference_semantics_by_hand():
    nan, inf = np.nan, np.inf
    k = np.array([1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 7], dtype=np.int64)
    v = np.array([0.0, -0.0, -0.0, 0.0, nan, nan, inf, 1.0, inf, -inf, nan, 5e-324])
    exp = R.aggregate([k], [(R.MIN, v), (R.MAX, v), (R.SUM, v), (R.COUNT, v)])
    mn, mx, sm, ct = exp.aggs
    assert np.array_equal(exp.keys[0], np.arange(1, 8))
    bits = lambda a: a.view(np.uint64).tolist()  # noqa: E731
    assert bits(mn["values"][:2]) == bits(np.array([-0.0, -0.0])) and bits(mx["values"][:2]) == bits(np.array([0.0, 0.0]))
    assert mn["isnan"].tolist() == [False, False, True, False, False, True, False]
    assert mn["values"][3] == 1.0 and mx["values"][3] == inf and mn["values"][4] == -inf and mx["values"][4] == inf
    assert sm["special"].tolist() == [0, 0, 1, 2, 1, 1, 0]
    assert ct["values"].tolist() == [2, 2, 2, 2, 2, 1, 1]
    # integer SUM wraps at the output width
    iv = np.array([2 ** 31 - 1, 1, 5], dtype=np.int32)
    e = R.aggregate([np.zeros(3, dtype=np.int64)], [(R.SUM, iv)])
    assert e.aggs[0]["values"].dtype == np.int32 and e.aggs[0]["values"][0] == np.int32(-2 ** 31 + 5)
    # the SUM bound catches one lost row of a large sum
    big = np.full(100_000, 1.0) + np.arange(100_000) * 1e-6
    e = R.aggregate([np.zeros(len(big), dtype=np.int64)], [(R.SUM, big)])
    lost = float(np.sum(big[1:]))
    with pytest.raises(AssertionError):
        R.assert_matches([np.zeros(1, dtype=np.int64), np.array([lost])], e)
    R.assert_matches([np.zeros(1, dtype=np.int64), np.array([float(np.sum(big))])], e)


def test_reference_matches_oracle_where():
    """A WHERE: the reference over the rows the mask passes, reading the values under a column's nulls as FilterRelation's
    bitmap-free output does, equals the oracle's filter-then-aggregate."""
    rng = np.random.default_rng(7)
    n = 2500
    k, v = data(rng, n, np.int32, np.float64, for_sum=False)
    _, s = data(rng, n, np.int32, np.int64, for_sum=True)
    w = rng.random(n)
    arrays = [k, R.arrow_nullable(v, rng.random(n) > 0.3), s, w]
    aggs = [(R.MIN, 1), (R.MAX, 1), (R.SUM, 2), (R.COUNT, 1)]
    pred = col(3) < lit(0.5)
    got = O.filtered_aggregate(arrays, pred, [col(0)], [AggregateFunction(f, col(c)) for f, c in aggs])
    got, exp = zeros_equal(got, R.aggregate([k], [(f, [None, v, s][c]) for f, c in aggs], where=w < 0.5))
    R.assert_matches(got, exp, "where")
    aggs0 = [AggregateFunction("sum", col(2)), AggregateFunction("count", col(1))]
    R.assert_matches(O.filtered_aggregate(arrays, pred, [], aggs0), R.aggregate([], [(R.SUM, s), (R.COUNT, v)], where=w < 0.5))


def test_avg_and_count_distinct_by_hand():
    nan, inf = np.nan, np.inf
    k = np.array([1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7], dtype=np.int64)
    v = np.array([1.0, 2.0, nan, nan, inf, 1.0, inf, -inf, 0.0, -0.0, 5.0, 6.0, 3.0])
    valid = np.ones(len(v), dtype=bool)
    valid[10:12] = False  # group 6: every value is null
    avg, cd = R.aggregate([k], [(R.AVG, (v, valid)), (R.COUNT_DISTINCT, (v, valid))]).aggs
    assert avg["dtype"] == np.float64 and cd["dtype"] == np.uint64
    assert np.flatnonzero(avg["null"]).tolist() == [5] and not cd["null"].any()
    assert avg["special"].tolist() == [0, 1, 2, 1, 0, 0, 0]  # NaN, +inf, and NaN for +inf with -inf
    assert avg["exact"][[0, 4, 6]].tolist() == [1.5, 0.0, 3.0] and not avg["bound"][[0, 4, 6]].any()
    assert cd["values"].tolist() == [2, 1, 2, 2, 1, 0, 1]  # every NaN one value, +0.0 and -0.0 one value
    f32 = np.array([np.float32(-0.0), 0.0, nan, -nan, 1.5, 1.5], dtype=np.float32)
    assert R.aggregate([], [(R.COUNT_DISTINCT, f32)]).aggs[0]["values"].tolist() == [3]
    # integers are rounded to f64 before they are added: here every partial sum is exact, and so is the quotient
    lo, hi = np.iinfo(np.int64).min, np.iinfo(np.int64).max
    i = np.array([hi, hi, lo, (1 << 53) + 1], dtype=np.int64)
    e = R.aggregate([np.array([0, 0, 0, 1], dtype=np.int64)], [(R.AVG, i)])
    assert not e.aggs[0]["bound"].any()
    R.assert_matches([np.array([0, 1], dtype=np.int64), np.array([2.0 ** 63 / 3, 2.0 ** 53])], e)
    with pytest.raises(AssertionError):
        R.assert_matches([np.array([0, 1], dtype=np.int64), np.array([np.nextafter(2.0 ** 63 / 3, 0), 2.0 ** 53])], e)
    u = np.array([np.iinfo(np.uint64).max, 1], dtype=np.uint64)
    R.assert_matches([np.array([2.0 ** 63])], R.aggregate([], [(R.AVG, u)]))
    # a sum that is not exact: the SUM bound over the count catches one lost row
    big = np.full(100_000, 1.0) + np.arange(100_000) * 1e-6
    e = R.aggregate([], [(R.AVG, big)])
    assert e.aggs[0]["bound"][0] > 0
    R.assert_matches([np.array([float(np.sum(big)) / len(big)])], e)
    with pytest.raises(AssertionError):
        R.assert_matches([np.array([float(np.sum(big[1:])) / len(big)])], e)


def test_no_row_and_all_null():
    """Without GROUP BY the result is one row: over zero rows, all-null values or a WHERE that passes nothing, COUNT and
    COUNT(DISTINCT) are 0 and MIN / MAX / SUM / AVG are null.  With GROUP BY such an input has no group."""
    v = np.array([1.0, 2.0, 3.0])
    funcs = [R.COUNT, R.COUNT_DISTINCT, R.MIN, R.MAX, R.SUM, R.AVG]
    none = np.zeros(3, dtype=bool)
    null = (np.zeros(1), np.zeros(1, dtype=bool))
    want = [np.zeros(1, dtype=np.uint64)] * 2 + [null] * 4
    for exp in (R.aggregate([], [(f, v[:0]) for f in funcs]), R.aggregate([], [(f, (v, none)) for f in funcs]),
                R.aggregate([], [(f, v) for f in funcs], where=none)):
        R.assert_matches(want, exp)
    exp = R.aggregate([np.arange(3)], [(f, v) for f in funcs], where=none)
    assert len(exp.keys[0]) == 0
    R.assert_matches([np.zeros(0, dtype=np.int64)] + [np.zeros(0, dtype=d["dtype"]) for d in exp.aggs], exp)
    # a WHERE that passes some rows: only those are aggregated
    R.assert_matches([np.array([2], dtype=np.uint64), np.array([2.5])], R.aggregate([], [(R.COUNT, v), (R.AVG, v)], where=v > 1.5))
