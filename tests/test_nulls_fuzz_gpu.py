"""Randomized parity of the null-aware kernels with the CPU oracle: nullable columns of all ten numeric dtypes and
Boolean columns, with deliberate garbage under every null slot (tests/fuzz_exprs.py), through filter / project, GROUP BY
(narrow and wide keys), the reduction without GROUP BY, COUNT(DISTINCT) and AVG, with and without a fused WHERE.

A WHERE under an aggregate is compared with filter-then-aggregate, the reference's wiring: FilterRelation copies values
and drops the bitmaps, so the aggregate sees the surviving rows with no nulls.  Every aggregate result is checked by
`groupby_ref` over the rows the oracle evaluated; MIN / MAX / SUM / COUNT are compared with the oracle's own aggregate
too.  Every case runs under DFGPU_TRACE and asserts that the NULLS instantiation it is about was launched."""
import numpy as np
import pyarrow as pa
import pytest

import fuzz_exprs as F
import groupby_ref as G
import oracle_lib as O
from kernel_trace import capfd_launched
from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import engine, host
from datafusion_archive_b200.expr import AggregateFunction, col, lit

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = engine.GpuContext(0)
    yield c
    c.close()


@pytest.fixture
def launched(monkeypatch, capfd):
    """Returns a function that yields the canonical names of the kernels launched since the last call:
    `k_hash_agg<8, false, true>` -> `k_hash_agg<8,0,1>`."""
    return capfd_launched(monkeypatch, capfd)


def unpack(c):
    if isinstance(c, tuple):
        return np.asarray(c[0]), np.asarray(c[1], dtype=bool)
    return (np.asarray(c) if not isinstance(c, list) else c), np.ones(len(c), dtype=bool)


def same(g, e):
    """Bit-exact, except that any NaN equals any NaN."""
    g, e = np.asarray(g), np.asarray(e)
    if g.dtype != e.dtype or g.shape != e.shape:
        return False
    if np.issubdtype(g.dtype, np.floating):
        gn, en = np.isnan(g), np.isnan(e)
        if not np.array_equal(gn, en):
            return False
        g, e = g[~gn], e[~en]
    if g.dtype == np.bool_:
        return np.array_equal(g, e)
    u = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[g.dtype.itemsize]
    return np.array_equal(g.view(u), e.view(u))


def same_value(g, e):
    """Equal as values (+0.0 equals -0.0: MIN / MAX may meet either zero first), any NaN equals any NaN."""
    g, e = np.asarray(g), np.asarray(e)
    if g.dtype != e.dtype or g.shape != e.shape:
        return False
    return np.array_equal(g, e, equal_nan=np.issubdtype(g.dtype, np.floating))


def upload_all(ctx, batches):
    return [ctx.upload(b) for b in batches]


def concat(batches):
    """One array per column over every batch (the oracle's input for a state fed batch by batch)."""
    arrow = lambda x: pa.array(x) if isinstance(x, np.ndarray) else x  # noqa: E731
    return [pa.concat_arrays([arrow(b[i]) for b in batches]) if len(batches) > 1 else batches[0][i] for i in range(len(batches[0]))]


def both(oracle_fn, gpu_fn):
    """(expected, got), or (None, None) when the oracle raises: then the engine must raise the same Arrow error."""
    try:
        exp = oracle_fn()
    except O.OracleError as e:
        assert "DivideByZero" in e.msg, e.msg
        with pytest.raises(engine.DfGpuError) as ei:
            gpu_fn()
        assert "DivideByZero" in str(ei.value)
        return None, None
    return exp, gpu_fn()


def gpu_fp(ctx, batch, pred, proj):
    r = ctx.filter_project(batch, pred, proj)
    try:
        return r.columns()
    finally:
        r.free()


def gpu_agg(ctx, batches, keys, aggs, pred=None):
    r = ctx.aggregate(batches, keys, aggs, 0, pred=pred)
    try:
        return r.columns()
    finally:
        r.free()


def assert_fp_equal(got, exp, what):
    assert len(got) == len(exp), what
    for i, (g, e) in enumerate(zip(got, exp)):
        (gv, gm), (ev, em) = unpack(g), unpack(e)
        assert np.array_equal(gm, em), (what, i, "validity")
        assert same(gv[gm], ev[em]), (what, i, "values")


# ---------------------------------------------------------------------------------------------------------------
# filter / project
# ---------------------------------------------------------------------------------------------------------------
def test_fuzz_filter_project_nullable(ctx, launched):
    """Random predicates and projections (depth <= 8, CAST, Boolean leaves) over nullable tables: the same rows in the
    same order, bit for bit, validity included; without a predicate the projections keep their nulls, with one they
    are evaluated as over bitmap-free arrays."""
    rng = np.random.default_rng(20261017)
    ran = raised = 0
    for n, profiles in [(20_011, None), (50_000, "nulls"), (3_001, None), (20_011, None)]:
        t = F.gen_table(rng, n, profiles=profiles)
        b = ctx.upload(t.arrays)
        try:
            for q in range(30):
                with_pred = q % 3 != 0
                pred, proj = F.gen_fp_query(rng, t, with_pred=with_pred)
                exp, got = both(lambda: O.rows(t.arrays, pred, proj), lambda: gpu_fp(ctx, b, pred, proj))
                if exp is None:
                    raised += 1
                    continue
                assert_fp_equal(got, exp, (n, q, pred, proj))
                ran += 1
        finally:
            b.free()
    assert ran >= 100 and raised <= 10, (ran, raised)
    assert "k_filter_project<8,1>" in launched()


def test_filter_project_zero_divisor_in_surviving_row(ctx):
    """A zero under a null is no error without a predicate; under one, the projections see the values under the
    nulls, and a zero divisor in a surviving row raises DivideByZero on both sides (and one in a dropped row does not)."""
    rng = np.random.default_rng(5)
    for d in F.NUMERIC:
        t = F.gen_table(rng, 4_000, profiles="nulls", surviving_zero=True, dtypes=[d])
        num, safe, gated = col(t.values[d]), col(t.safe[d]), col(t.gated[d])
        gate = col(t.gate) > lit(0, A.INT32)
        b = ctx.upload(t.arrays)
        try:
            assert_fp_equal(gpu_fp(ctx, b, None, [num / safe]), O.rows(t.arrays, None, [num / safe]), d)
            assert_fp_equal(gpu_fp(ctx, b, gate, [num / gated]), O.rows(t.arrays, gate, [num / gated]), d)
            exp, got = both(lambda: O.rows(t.arrays, gate, [num / safe]), lambda: gpu_fp(ctx, b, gate, [num / safe]))
            assert exp is None, d
        finally:
            b.free()


# ---------------------------------------------------------------------------------------------------------------
# aggregates
# ---------------------------------------------------------------------------------------------------------------
def expected(rows, nkeys, aggs):
    """groupby_ref's expectation from the per-row values the oracle evaluated (keys first, then one column per
    aggregate argument)."""
    return G.aggregate(rows[:nkeys], [(G.func_of(a), rows[nkeys + i]) for i, a in enumerate(aggs)])


def sorted_result(cols, nkeys):
    cols = [unpack(c) for c in cols]
    if not nkeys:
        return cols
    order = np.lexsort([cols[k][0] for k in reversed(range(nkeys))])
    return [(v[order], m[order]) for v, m in cols]


def check_aggregate(arrays, pred, keys, aggs, got_fn, what):
    """GPU vs the oracle's filter-then-aggregate: keys, COUNT, integer aggregates and (with GROUP BY) float MIN / MAX
    exact; float SUM to the gamma bound of groupby_ref, from the oracle's per-row values.  Without
    GROUP BY, float MIN / MAX come from groupby_ref too: arrow 0.12's scan returns NaN when the first value of a batch
    is NaN while the engine skips NaN, a documented deviation (DESIGN §7)."""
    nk = len(keys)
    exp, got = both(lambda: O.filtered_aggregate(arrays, pred, keys, aggs), got_fn)
    if exp is None:
        return "raised"
    rows = O.rows(arrays, pred, keys + [a.arg for a in aggs])
    G.assert_matches(got, expected(rows, nk, aggs), ctx=str(what))
    g, e = sorted_result(got, nk), sorted_result(exp, nk)
    assert len(g) == len(e) and len(g[0][0]) == len(e[0][0]), what
    for i, ((gv, gm), (ev, em)) in enumerate(zip(g, e)):
        if i >= nk and aggs[i - nk].name == "count" and not len(unpack(rows[0])[0]):
            continue  # the oracle's COUNT over no row is null; groupby_ref's 0 was checked above
        assert np.array_equal(gm, em), (what, i, "validity")
        if i >= nk:
            a = aggs[i - nk]
            floating = np.issubdtype(ev.dtype, np.floating)
            if floating and (a.name == "sum" or (a.name in ("min", "max") and nk == 0)):
                continue  # checked against groupby_ref above
        assert same_value(gv[gm], ev[em]), (what, i)
    return "ok"


def test_fuzz_groupby_nullable(ctx, launched):
    """GROUP BY 1-3 integer keys (plain columns and expressions; two 64-bit keys take the wide-key kernel) with
    MIN / MAX / SUM / COUNT over nullable columns and expressions, with and without a fused WHERE."""
    rng = np.random.default_rng(71)
    key_sets = [[A.INT32], [A.INT8, A.UINT16], [A.INT64, A.UINT64], [A.INT16, A.INT64, A.UINT32], [A.UINT8]]
    outcomes = []
    seen = set()
    for qi in range(20):
        plain = qi % 4 == 3
        n = 200_000 if plain else 3_000
        kd = key_sets[qi % len(key_sets)]
        t = F.gen_table(rng, n)
        kc = F.add_keys(rng, t, kd, n)
        pred, keys, aggs = F.gen_agg_query(rng, t, kc, with_pred=qi % 3 != 0, plain_args=plain)
        b = upload_all(ctx, [t.arrays])
        try:
            outcomes.append(check_aggregate(t.arrays, pred, keys, aggs, lambda: gpu_agg(ctx, b, keys, aggs, pred), (qi, pred, keys)))
        finally:
            for x in b:
                x.free()
        seen |= launched()
    assert outcomes.count("ok") >= 16, outcomes
    assert "k_hash_agg<8,0,1>" in seen and "k_hash_agg_wide<8,1>" in seen, sorted(seen)


def test_fuzz_no_groupby_nullable(ctx, launched):
    """The reduction without GROUP BY: MIN / MAX / SUM / COUNT over nullable columns and expressions; without a WHERE
    nulls are skipped and an aggregate with no valid value is null, under one every surviving row counts."""
    rng = np.random.default_rng(72)
    outcomes = []
    seen = set()
    for qi in range(16):
        plain = qi % 4 == 3
        n = 1_000_000 if qi == 15 else 200_000 if plain else 4_000
        t = F.gen_table(rng, n, dtypes=[A.INT32, A.UINT64, A.FLOAT32, A.FLOAT64] if n == 1_000_000 else F.NUMERIC)
        pred, keys, aggs = F.gen_agg_query(rng, t, [], with_pred=qi % 2 == 0, plain_args=plain or qi == 15)
        b = upload_all(ctx, [t.arrays])
        try:
            outcomes.append(check_aggregate(t.arrays, pred, keys, aggs, lambda: gpu_agg(ctx, b, keys, aggs, pred), (qi, pred)))
        finally:
            for x in b:
                x.free()
        seen |= launched()
    assert outcomes.count("ok") >= 12, outcomes
    assert "k_reduce<8,1>" in seen, sorted(seen)


def test_fuzz_multibatch_mixed_nulls(ctx, launched):
    """1-3 batches per aggregate state, some null-free (the plain and lean kernels) and some nullable (the NULLS
    kernels), the same query over all of them."""
    rng = np.random.default_rng(73)
    outcomes = []
    seen = set()
    for qi in range(12):
        nb = 1 + qi % 3
        grouped = qi % 2 == 0
        plain = qi % 4 < 2
        n = 100_000 if plain else 2_000
        kd = [A.INT64] if qi % 4 == 0 else [A.INT16, A.INT32]
        batches, proto = [], None
        for j in range(nb):
            t = F.gen_table(rng, n, profiles="nobitmap" if j % 2 == 1 else None)
            kc = F.add_keys(rng, t, kd, n) if grouped else []
            batches.append(t)
            proto = proto or (t, kc)
        t, kc = proto
        pred, keys, aggs = F.gen_agg_query(rng, t, kc, with_pred=qi % 3 != 2, plain_args=plain)
        arrays = concat([x.arrays for x in batches])
        b = upload_all(ctx, [x.arrays for x in batches])
        try:
            outcomes.append(check_aggregate(arrays, pred, keys, aggs, lambda: gpu_agg(ctx, b, keys, aggs, pred), (qi, nb, pred)))
        finally:
            for x in b:
                x.free()
        seen |= launched()
    assert outcomes.count("ok") >= 9, outcomes
    assert "k_reduce<8,1>" in seen and "k_hash_agg<8,0,1>" in seen, sorted(seen)


@pytest.mark.parametrize("with_pred", [False, True])
def test_one_state_mixes_lean_plain_and_nulls_kernels(ctx, launched, with_pred):
    """One GROUP BY state fed null-free, nullable and null-free batches: the null-free ones take the interpreter-free
    kernels (without a WHERE, SUM and COUNT of one Int64-keyed Float64 column: the lean kernel; with a column-comparison
    WHERE: the plain kernel), the nullable one the NULLS kernel, and all of them fold into the same table."""
    rng = np.random.default_rng(76)
    n = 200_000
    batches = []
    for j in range(3):
        k = rng.integers(0, 1000, n, dtype=np.int64)
        v = rng.random(n) * 4 - 2
        w = rng.integers(0, 2, n, dtype=np.int32)
        if j == 1:
            valid = rng.random(n) >= 0.3
            g = F.garbage(A.FLOAT64)
            v = F.column(np.where(valid, v, g[rng.integers(0, len(g), n)]), valid)
        batches.append([k, v, w])
    keys = [col(0)]
    if with_pred:
        pred = col(2) > lit(0, A.INT32)
        aggs = [AggregateFunction(f, col(1)) for f in ("min", "max", "sum", "count")]
        fast = "k_hash_agg_plain<"
    else:
        pred = None
        aggs = [AggregateFunction("sum", col(1)), AggregateFunction("count", col(1))]
        fast = "k_hash_agg_lean<"
    b = upload_all(ctx, batches)
    try:
        assert check_aggregate(concat(batches), pred, keys, aggs, lambda: gpu_agg(ctx, b, keys, aggs, pred), with_pred) == "ok"
    finally:
        for x in b:
            x.free()
    seen = launched()
    assert "k_hash_agg<8,0,1>" in seen and any(s.startswith(fast) for s in seen), sorted(seen)


@pytest.mark.parametrize("kernel", ["k_hash_agg<8,0,1>", "k_hash_agg_wide<8,1>", "k_reduce<8,1>", "k_distinct_insert<8,1>"])
def test_aggregate_zero_divisor_in_surviving_row(ctx, launched, kernel):
    """Under a WHERE the keys and arguments see the values under the nulls: a zero there, in a row that passes, raises
    DivideByZero on both sides, as an argument and as a key.  The same division over divisors whose zeros sit only in
    rows the WHERE drops does not raise, and neither does it without a WHERE, where the null quotient is null."""
    rng = np.random.default_rng(81)
    n = 4_000
    raised = 0
    for d in (A.INT32, A.UINT64, A.FLOAT64):
        t = F.gen_table(rng, n, profiles="nulls", surviving_zero=True, dtypes=[d])
        gate = col(t.gate) > lit(0, A.INT32)
        num = col(t.values[d])
        bad, good = num / col(t.safe[d]), num / col(t.gated[d])
        if kernel == "k_hash_agg<8,0,1>" or kernel == "k_distinct_insert<8,1>":
            keys = [col(F.add_keys(rng, t, [A.INT32], n)[0])]
        elif kernel == "k_hash_agg_wide<8,1>":
            keys = [col(k) for k in F.add_keys(rng, t, [A.INT64, A.INT64], n)]
        else:
            keys = []
        b = upload_all(ctx, [t.arrays])
        try:
            if kernel == "k_distinct_insert<8,1>":
                # the oracle has no COUNT(DISTINCT): its filter-then-project raises for the same argument
                distinct = lambda e: [AggregateFunction("count", e, distinct=True)]  # noqa: E731
                exp, _ = both(lambda: O.rows(t.arrays, gate, [bad]), lambda: gpu_agg(ctx, b, keys, distinct(bad), gate))
                assert exp is None, d
                raised += 1
                gpu_agg(ctx, b, keys, distinct(good), gate)
                gpu_agg(ctx, b, keys, distinct(bad))
                continue
            cases = [(gate, keys, [AggregateFunction("sum", bad), AggregateFunction("count", num)], "raised"),
                     (gate, keys, [AggregateFunction("sum", good), AggregateFunction("count", num)], "ok"),
                     (None, keys, [AggregateFunction("sum", bad), AggregateFunction("count", bad)], "ok")]
            if keys and d != A.FLOAT64:  # the division as a GROUP BY key
                cases.append((gate, keys[:-1] + [bad], [AggregateFunction("count", num)], "raised"))
                cases.append((gate, keys[:-1] + [good], [AggregateFunction("count", num)], "ok"))
            for pred, ks, aggs, want in cases:
                got = check_aggregate(t.arrays, pred, ks, aggs, lambda: gpu_agg(ctx, b, ks, aggs, pred), (kernel, d, pred, ks))
                assert got == want, (kernel, d, pred, ks, got)
                raised += got == "raised"
        finally:
            for x in b:
                x.free()
    assert raised >= 3
    assert kernel in launched()


def test_aggregate_host_nullable_where(ctx):
    """aggregate_host (one host batch, chunked inside the library) with a fused WHERE over nullable columns."""
    rng = np.random.default_rng(74)
    for qi, kd in enumerate([[A.INT32], [], [A.INT64, A.INT64]]):
        n = 300_000
        t = F.gen_table(rng, n, profiles="nulls", dtypes=[A.INT16, A.INT64, A.FLOAT32, A.FLOAT64])
        kc = F.add_keys(rng, t, kd, n)
        pred, keys, aggs = F.gen_agg_query(rng, t, kc, with_pred=True, plain_args=True)

        def run():
            r = ctx.aggregate_host(t.arrays, keys, aggs, pred=pred, chunk_rows=70_000)
            try:
                return r.columns()
            finally:
                r.free()
        assert check_aggregate(t.arrays, pred, keys, aggs, run, (qi, pred)) == "ok"


def nullable(values, valid):
    return F.column(np.asarray(values), np.asarray(valid, dtype=bool))


def test_where_over_nulls_worked_example(ctx):
    """v = [1, null (100 under it), 3, null (-50 under it)], k = [0, 0, 1, 1], WHERE w > 0 passes every row: the
    aggregate sees FilterRelation's output, in which the values under the nulls are ordinary values."""
    v = nullable(np.array([1.0, 100.0, 3.0, -50.0]), [1, 0, 1, 0])
    k = np.array([0, 0, 1, 1], dtype=np.int64)
    w = np.array([1.0, 1.0, 1.0, 1.0])
    arrays = [v, k, w]
    pred = col(2) > lit(0.0)
    b = upload_all(ctx, [arrays])
    try:
        got = gpu_agg(ctx, b, [], [AggregateFunction(f, col(0)) for f in ("min", "max", "sum", "count")], pred)
        assert [float(unpack(c)[0][0]) for c in got] == [-50.0, 100.0, 54.0, 4.0]
        got = sorted_result(gpu_agg(ctx, b, [col(1)], [AggregateFunction("count", col(0)), AggregateFunction("sum", col(0) * lit(2.0))], pred), 1)
        assert got[1][0].tolist() == [2, 2] and got[2][0].tolist() == [202.0, -94.0]
        # without the WHERE the nulls are skipped (no GROUP BY) or counted out (COUNT)
        got = gpu_agg(ctx, b, [], [AggregateFunction(f, col(0)) for f in ("min", "max", "sum", "count")])
        assert [float(unpack(c)[0][0]) for c in got] == [1.0, 3.0, 4.0, 2.0]
        # AVG and COUNT(DISTINCT) count every surviving row too
        got = gpu_agg(ctx, b, [], [AggregateFunction("avg", col(0)), AggregateFunction("count", col(0), distinct=True)], pred)
        assert float(unpack(got[0])[0][0]) == 13.5 and int(unpack(got[1])[0][0]) == 4
        # a WHERE that passes nothing: MIN / MAX / SUM null, COUNT 0
        got = gpu_agg(ctx, b, [], [AggregateFunction(f, col(0)) for f in ("min", "sum", "count")], col(2) < lit(0.0))
        assert not unpack(got[0])[1][0] and not unpack(got[1])[1][0] and int(unpack(got[2])[0][0]) == 0
    finally:
        for x in b:
            x.free()


def test_avg_count_distinct_nullable(ctx, launched):
    """AVG and COUNT(DISTINCT) with and without GROUP BY and WHERE: without a WHERE the nulls are skipped, under one
    every surviving row counts, its value being the one under the null."""
    rng = np.random.default_rng(75)
    seen = set()
    for qi in range(10):
        n = 20_000
        t = F.gen_table(rng, n)
        kc = F.add_keys(rng, t, [A.INT32] if qi % 2 == 0 else [A.INT8, A.UINT32], n) if qi % 5 != 4 else []
        with_pred = qi % 3 != 1
        cands = [t.values[d] for d in F.NUMERIC] + [t.safe[d] for d in F.NUMERIC]
        args = [col(int(rng.choice(cands))) for _ in range(3)]
        args.append(col(t.values[A.INT32]) * lit(2, A.INT32))
        while True:
            g = F.QueryGen(rng, t, set(rng.choice(cands, 5, replace=False).tolist()) | {t.gate} | set(t.bools))
            pred = g.predicate() if with_pred else None
            if F.fits([col(k) for k in kc] + args + ([pred] if pred is not None else []), t.dtype):
                break
        funcs = ["avg", "distinct", "avg" if qi % 2 else "distinct", "distinct"]
        aggs = [AggregateFunction("count", a, distinct=True) if f == "distinct" else AggregateFunction("avg", a) for f, a in zip(funcs, args)]
        keys = [col(k) for k in kc]
        b = upload_all(ctx, [t.arrays])
        try:
            got = gpu_agg(ctx, b, keys, aggs, pred)
        finally:
            for x in b:
                x.free()
        seen |= launched()
        G.assert_matches(got, expected(O.rows(t.arrays, pred, keys + args), len(keys), aggs), ctx=str(qi))
    assert "k_distinct_insert<8,1>" in seen, sorted(seen)


# ---------------------------------------------------------------------------------------------------------------
# SQL
# ---------------------------------------------------------------------------------------------------------------
def test_sql_where_over_nullable_memory_table():
    """SELECT k, COUNT(v), SUM(v * 2) FROM t WHERE w > 0 GROUP BY k over a nullable in-memory table, and its form
    without GROUP BY: the values under the nulls of v are ordinary values after the WHERE."""
    v = nullable(np.array([1, 100, 3, -50], dtype=np.int64), [1, 0, 1, 0])
    k = np.array([0, 0, 1, 1], dtype=np.int64)
    w = np.array([1, 1, 1, 1], dtype=np.int64)
    hctx = host.ExecutionContext(0)
    try:
        for name in ("t", "u", "x"):  # a registered in-memory table is read once
            hctx.register_memory(name, [("k", k), ("v", v), ("w", w)])
        rows = []
        for batch in hctx.sql("SELECT k, COUNT(v), SUM(v * 2) FROM t WHERE w > 0 GROUP BY k").collect():
            rows.extend(zip(*[unpack(c)[0].tolist() for c in batch]))
        assert sorted(rows) == [(0, 2, 202), (1, 2, -94)]
        rows = []
        for batch in hctx.sql("SELECT COUNT(v), SUM(v * 2) FROM u WHERE w > 0").collect():
            rows.extend(zip(*[unpack(c)[0].tolist() for c in batch]))
        assert rows == [(4, 108)]
        rows = []
        for batch in hctx.sql("SELECT COUNT(v), SUM(v) FROM x").collect():
            rows.extend(zip(*[unpack(c)[0].tolist() for c in batch]))
        assert rows == [(2, 4)]
    finally:
        hctx.close()
