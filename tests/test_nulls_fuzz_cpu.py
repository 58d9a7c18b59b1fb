"""The nullable-table generator of tests/fuzz_exprs.py and its queries, on the CPU oracle alone (no GPU): the invariants
the GPU fuzz relies on (every dtype occurs, garbage sits under the nulls, each divisor placement occurs, queries fit the
engine's limits and never divide by zero unless asked to), the oracle's filter-then-aggregate against groupby_ref on the
same rows, and the worked example of a WHERE over nulls."""
import numpy as np

import fuzz_exprs as F
import groupby_ref as G
import oracle_lib as O
from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200.expr import AggregateFunction, col, lit


def test_table_invariants():
    rng = np.random.default_rng(1)
    n = 5_000
    t = F.gen_table(rng, n, surviving_zero=True)
    assert set(F.NUMERIC) <= set(t.dtype) and t.dtype.count(A.BOOL) == 2
    gate = t.hidden[t.gate] > 0
    for i, (v, valid) in enumerate(zip(t.hidden, t.valid)):
        assert len(t.arrays[i]) == n
        if valid is None:
            assert t.arrays[i].buffers()[0] is None and t.profile[i] == "nobitmap"
            continue
        mask = np.unpackbits(np.frombuffer(t.arrays[i].buffers()[0], dtype=np.uint8), bitorder="little")[:n].astype(bool)
        assert np.array_equal(mask, valid)
        if t.profile[i] == "allnull":
            assert not valid.any()
        if t.profile[i] == "bitmap":
            assert valid.all()
        if not (~valid).any():
            continue
        if t.dtype[i] == A.BOOL:
            assert v[~valid].all()  # a hidden 1 under every Boolean null
            continue
        hidden = v[~valid]
        garbage = F.garbage(t.dtype[i])
        if i in t.values.values():
            # only garbage under the nulls of a value column (NaN compares unequal: test it apart)
            ok = np.isin(hidden, garbage) | (np.isnan(hidden) if hidden.dtype.kind == "f" else False)
            assert ok.all(), i
        else:
            assert not (hidden == -1).any() if hidden.dtype.kind == "i" else True
    for d in F.NUMERIC:
        s, g = t.safe[d], t.gated[d]
        assert not (t.hidden[g] == 0)[gate].any(), d  # a gated divisor's zeros are in rows every WHERE drops
        if d in F.FLOATS or np.iinfo(A.NP_OF[d]).min < 0:
            assert not (t.hidden[s] == -1).any() and not (t.hidden[g] == -1).any(), d
        if t.valid[s] is not None:
            valid = t.valid[s]
            assert not ((t.hidden[s] == 0) & valid).any(), d  # a safe divisor's zeros are under nulls only
    # f32 data is clear of subnormals
    for i, d in enumerate(t.dtype):
        if d == A.FLOAT32:
            v = t.hidden[i]
            assert not ((v != 0) & (np.abs(v) < np.finfo(np.float32).tiny)).any()


def test_each_divisor_placement_occurs():
    """Zeros under nulls, in rows the WHERE drops, and (asked for) under nulls in surviving rows."""
    rng = np.random.default_rng(2)
    seen = set()
    for surviving in (False, True):
        t = F.gen_table(rng, 4_000, profiles="nulls", surviving_zero=surviving)
        gate = t.hidden[t.gate] > 0
        for d in F.NUMERIC:
            for role in ("safe", "gated"):
                i = getattr(t, role)[d]
                zero = t.hidden[i] == 0
                null = ~t.valid[i]
                if (zero & null).any():
                    seen.add("under null")
                if (zero & ~gate).any():
                    seen.add("dropped row")
                if (zero & null & gate).any():
                    seen.add("surviving row")
    assert seen == {"under null", "dropped row", "surviving row"}


def test_generated_queries_run_on_the_oracle():
    """Filter / project queries with and without a predicate: the oracle accepts all of them and none divides by zero;
    trees reach depth 8 and CASTs and Boolean leaves occur."""
    rng = np.random.default_rng(3)
    t = F.gen_table(rng, 3_000)
    depth8 = casts = bool_leaves = 0
    for q in range(120):
        pred, proj = F.gen_fp_query(rng, t, with_pred=q % 2 == 0)
        O.rows(t.arrays, pred, proj)
        progs = [e.program(t.dtype) for e in proj + ([pred] if pred is not None else [])]
        casts += any(i.op == A.OP_CAST for p in progs for i in p)
        bool_leaves += any(i.op == A.OP_COL and t.dtype[i.col] == A.BOOL for p in progs for i in p)
        depth8 += any(F._cap(e)[1] >= 8 for e in proj + ([pred] if pred is not None else []))
    assert casts >= 10 and bool_leaves >= 10 and depth8 >= 5, (casts, bool_leaves, depth8)


def test_surviving_zero_divisor_raises_on_the_oracle():
    rng = np.random.default_rng(4)
    t = F.gen_table(rng, 2_000, profiles="nulls", surviving_zero=True, dtypes=[A.INT32])
    gate = col(t.gate) > lit(0, A.INT32)
    e = col(t.values[A.INT32]) / col(t.safe[A.INT32])
    O.rows(t.arrays, None, [e])  # null-aware without a predicate: no error
    try:
        O.rows(t.arrays, gate, [e])
        raise AssertionError("a zero divisor in a surviving row must raise")
    except O.OracleError as err:
        assert "DivideByZero" in err.msg


def test_oracle_filtered_aggregate_vs_groupby_ref():
    """The oracle's filter-then-aggregate equals groupby_ref over the rows the oracle evaluated, the comparison the GPU
    fuzz makes (without GROUP BY float MIN / MAX are left out: arrow 0.12 returns NaN when a batch starts with NaN)."""
    rng = np.random.default_rng(5)
    for qi in range(12):
        n = 2_000
        t = F.gen_table(rng, n)
        kc = F.add_keys(rng, t, [[A.INT32], [A.INT64, A.UINT64], [], [A.INT8, A.UINT16, A.INT32]][qi % 4], n)
        pred, keys, aggs = F.gen_agg_query(rng, t, kc, with_pred=qi % 3 != 0, plain_args=qi % 2 == 0)
        if not keys:
            aggs = [a for a in aggs if not (a.name in ("min", "max") and A.NP_OF.get(a.arg.get_type(t.dtype), np.int8)().dtype.kind == "f")]
            if not aggs:
                continue
        got = O.filtered_aggregate(t.arrays, pred, keys, aggs)
        r = O.rows(t.arrays, pred, keys + [a.arg for a in aggs])
        if not keys and pred is not None and len(np.asarray(r[0][0] if isinstance(r[0], tuple) else r[0])) == 0:
            continue  # nothing passed: the oracle's COUNT is null, the engine's 0 (the GPU fuzz compares that case)
        G.assert_matches(got, G.aggregate(r[:len(keys)], [(G.func_of(a), r[len(keys) + i]) for i, a in enumerate(aggs)]), ctx=str(qi))


def test_worked_example_on_the_oracle():
    """v = [1, null (100 under it), 3, null (-50 under it)], k = [0, 0, 1, 1], WHERE w > 0 passes every row."""
    v = F.column(np.array([1.0, 100.0, 3.0, -50.0]), np.array([1, 0, 1, 0], dtype=bool))
    k = np.array([0, 0, 1, 1], dtype=np.int64)
    w = np.array([1.0, 1.0, 1.0, 1.0])
    pred = col(2) > lit(0.0)
    out = O.filtered_aggregate([v, k, w], pred, [], [AggregateFunction(f, col(0)) for f in ("min", "max", "sum", "count")])
    assert [float(np.asarray(c)[0]) for c in out] == [-50.0, 100.0, 54.0, 4.0]
    out = O.filtered_aggregate([v, k, w], pred, [col(1)], [AggregateFunction("count", col(0)), AggregateFunction("sum", col(0) * lit(2.0))])
    order = np.argsort(out[0])
    assert out[1][order].tolist() == [2, 2] and out[2][order].tolist() == [202.0, -94.0]
    # without the WHERE: no-GROUP-BY reductions skip the nulls
    out = O.aggregate([v, k, w], [], [AggregateFunction(f, col(0)) for f in ("min", "max", "sum", "count")])
    assert [float(np.asarray(c[0] if isinstance(c, tuple) else c)[0]) for c in out] == [1.0, 3.0, 4.0, 2.0]
