"""GPU parity tests: the sm_90a path through the C ABI vs the CPU oracle on the same seeded inputs
(bit-exact for integer/index/ordering work and every non-reduced f64, 1e-9 relative for f64 SUM) or vs the exact
GROUP BY reference of tests/groupby_ref.py, the reference's golden vectors, edge cases, and size-independent properties
at BASELINE sizes."""
import numpy as np
import pytest

import groupby_ref as G
import oracle_lib as O
from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import engine, workloads
from datafusion_archive_b200.expr import AggregateFunction, case, col, lit
from kernel_trace import traced

pytestmark = pytest.mark.gpu

SUM_RTOL = 1e-9  # north_star tolerance for Float64 aggregates


@pytest.fixture(scope="module")
def ctx():
    c = engine.GpuContext(0)
    yield c
    c.close()


def gpu_fp(ctx, arrays, pred, proj):
    b = ctx.upload(arrays)
    try:
        r = ctx.filter_project(b, pred, proj)
        try:
            return r.columns()
        finally:
            r.free()
    finally:
        b.free()


def gpu_agg(ctx, arrays, keys, aggs, nbatches=1, expected=0, pred=None):
    n = len(arrays[0])
    bounds = [int(x) for x in np.linspace(0, n, nbatches + 1)]
    batches = [ctx.upload([a[bounds[i]:bounds[i + 1]] for a in arrays]) for i in range(nbatches)]
    try:
        r = ctx.aggregate(batches, keys, aggs, expected, pred=pred)
        try:
            return r.columns()
        finally:
            r.free()
    finally:
        for b in batches:
            b.free()


def assert_cols_bit_equal(got, exp):
    assert len(got) == len(exp)
    for g, e in zip(got, exp):
        assert g.dtype == e.dtype
        assert g.shape == e.shape
        assert np.array_equal(g.view(np.uint8), e.view(np.uint8))


def sort_by_key(cols, nkeys=1):
    order = np.lexsort([cols[k] for k in reversed(range(nkeys))])
    return [c[order] for c in cols]


# ---------------------------------------------------------------------------------------------
# golden vectors of the reference (tests/golden/reference_vectors.json)
# ---------------------------------------------------------------------------------------------
def test_golden_csv_query_with_predicate(ctx, golden, fmt_f64):
    # tests/sql.rs:30-37 minus the Utf8 column (Utf8 gather is a "next" row, SURVEY §8f-3)
    c = golden["uk_cities"]
    arrays = [np.array(c["lat"]), np.array(c["lng"])]
    pred = (col(0) > lit(51.0)) & (col(0) < lit(53).cast(A.FLOAT64))
    out = gpu_fp(ctx, arrays, pred, [col(0), col(1), col(0) + col(1)])
    exp_lines = golden["csv_query_with_predicate"]["expected"].splitlines()
    got = ["%s\t%s\t%s" % tuple(fmt_f64(x) for x in row) for row in zip(*out)]
    assert got == [l.split("\t", 1)[1] for l in exp_lines]


def test_golden_csv_query_with_predicate_full(ctx, golden, fmt_f64):
    # tests/sql.rs:30-37 including the Utf8 column (GPU Utf8 gather, filter.rs:93-103)
    c = golden["uk_cities"]
    arrays = [c["city"], np.array(c["lat"]), np.array(c["lng"])]
    pred = (col(1) > lit(51.0)) & (col(1) < lit(53).cast(A.FLOAT64))
    out = gpu_fp(ctx, arrays, pred, [col(0), col(1), col(2), col(1) + col(2)])
    s = "".join('"%s"\t%s\t%s\t%s\n' % (a, fmt_f64(b), fmt_f64(c_), fmt_f64(d)) for a, b, c_, d in zip(*out))
    assert s == golden["csv_query_with_predicate"]["expected"]


def test_utf8_gather_vs_oracle(ctx):
    rng = np.random.default_rng(17)
    n = 200_000
    words = ["", "a", "bc", "déjà vu", "x" * 40, "London, UK", "\"quoted\""]
    strs = [words[i] + str(i % 977) * (i % 3) for i in rng.integers(0, len(words), n)]
    v = rng.random(n)
    for pred in [col(1) > lit(0.5), col(1) > lit(0.999), col(1) > lit(-1.0), col(1) > lit(2.0), None]:
        got = gpu_fp(ctx, [strs, v], pred, [col(0), col(1) * col(1), col(0)])
        exp = O.filter_project([strs, v], pred, [col(0), col(1) * col(1), col(0)])
        assert got[0] == exp[0] and got[2] == exp[2]
        assert np.array_equal(got[1], exp[1])
    # FilterRelation alone: every input column, Utf8 included (filter.rs:55-57)
    got = gpu_fp(ctx, [strs, v], col(1) < lit(0.25), [])
    exp = O.filter_project([strs, v], col(1) < lit(0.25), [])
    assert got[0] == exp[0] and np.array_equal(got[1], exp[1])


def test_golden_cast(ctx, golden):
    c = golden["uk_cities"]
    out = gpu_fp(ctx, [np.array(c["lat"])], None, [col(0).cast(A.INT32)])
    assert out[0].dtype == np.int32
    assert "".join("%d\n" % v for v in out[0]) == golden["csv_query_cast"]["expected"]


def test_golden_min_max_lat(ctx, golden):
    c = golden["uk_cities"]
    out = gpu_agg(ctx, [np.array(c["lat"])], [], [AggregateFunction("min", col(0)), AggregateFunction("max", col(0))])
    assert out[0][0] == golden["min_lat"] and out[1][0] == golden["max_lat"]


def test_golden_min_max_sum_group_by(ctx, golden):
    t = golden["aggregate_test_1"]
    arrays = [np.array(t["a"], dtype=np.int32), np.array(t["b"])]
    aggs = [AggregateFunction("min", col(1)), AggregateFunction("max", col(1)), AggregateFunction("sum", col(1))]
    out = sort_by_key(gpu_agg(ctx, arrays, [col(0)], aggs))
    exp = sorted(tuple(r) for r in golden["test_min_max_sum_group_by"])
    assert out[0].dtype == np.int32
    for i, (a, mn, mx, sm) in enumerate(exp):
        assert out[0][i] == a and out[1][i] == mn and out[2][i] == mx  # bit-exact
        assert abs(out[3][i] - sm) <= SUM_RTOL * abs(sm)


# ---------------------------------------------------------------------------------------------
# filter + project vs oracle
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 2047, 2048, 2049, 4096, 100_003, 1_000_000])
def test_c2_filter_sizes(ctx, n):
    arrays, pred, proj = workloads.c2(n, seed=42 + n)
    got = gpu_fp(ctx, arrays, pred, proj)
    if n == 0:
        assert len(got[0]) == 0
        return
    exp = O.filter_project(arrays, pred, proj)
    assert_cols_bit_equal(got, exp)


def test_c2_selectivities(ctx):
    a = np.random.default_rng(7).random(300_000)
    for thr in [-1.0, 0.0, 0.001, 0.5, 0.999, 1.0, 2.0]:
        got = gpu_fp(ctx, [a], col(0) > lit(thr), [col(0)])
        assert np.array_equal(got[0], a[a > thr])


def test_c3_fused_expr_filter(ctx):
    arrays, pred, proj = workloads.c3(500_000)
    got = gpu_fp(ctx, arrays, pred, proj)
    exp = O.filter_project(arrays, pred, proj)
    assert_cols_bit_equal(got, exp)
    a, b = arrays[0], arrays[1]
    m = b < a
    assert np.array_equal(got[0], (a + b)[m]) and np.array_equal(got[1], (a * b)[m])


def test_host_pipelined_matches_resident_path(ctx):
    # dfgpu_filter_project_host: chunked upload / kernel / download; same rows, same order, same bits
    arrays, pred, proj = workloads.c3(3_000_017)
    exp = O.filter_project(arrays, pred, proj)
    for chunk in [0, 1 << 20, 999_983, 4_000_000]:
        r = ctx.filter_project_host(arrays, pred, proj, chunk_rows=chunk)
        got = [r.host_view(i).copy() for i in range(r.ncols)]
        r.free()
        assert_cols_bit_equal(got, exp)
    # pinned inputs, unreferenced Utf8 column present, no predicate, empty input
    pin = engine.PinnedBuffer((1_000_000,), np.float64)
    pin.array[:] = np.random.default_rng(2).random(1_000_000)
    strs = ["x"] * 1_000_000
    r = ctx.filter_project_host([strs, pin.array], None, [col(1) * lit(2.0)], chunk_rows=300_000)
    assert np.array_equal(r.host_view(0), pin.array * 2.0)
    r.free()
    r = ctx.filter_project_host([np.array([], dtype=np.float64)], col(0) > lit(0.5), [col(0)])
    assert r.nrows == 0
    r.free()
    # referenced Utf8 / nullable / Boolean columns, and a numeric projection with a CASE without ELSE: the same entry
    # point runs the resident operator (device result)
    import pyarrow as pa
    rng = np.random.default_rng(5)
    m = 200_000
    x = rng.random(m)
    names = ["n%05d" % (i % 977) for i in range(m)]
    xn = pa.array(x, mask=rng.random(m) < 0.1)
    flag = rng.random(m) < 0.5
    for arrs, p_, pr in [([names, x], col(1) > lit(0.5), [col(0), col(1)]),
                         ([xn, x], col(1) < lit(0.25), [col(0), col(0) + col(1)]),
                         ([flag, x], col(0) & (col(1) > lit(0.5)), [col(1)]),
                         ([x], col(0) < lit(0.9), [col(0), case([(col(0) > lit(0.5), col(0) * lit(2.0))])])]:
        r = ctx.filter_project_host(arrs, p_, pr)
        assert not r.on_host
        got = r.columns()
        r.free()
        exp = gpu_fp(ctx, arrs, p_, pr)
        assert len(got) == len(exp)
        for g, e in zip(got, exp):
            if isinstance(g, tuple):
                assert np.array_equal(g[1], e[1]) and np.array_equal(g[0][g[1]], e[0][e[1]])
            elif isinstance(g, list):
                assert g == e
            else:
                assert np.array_equal(g, e)
    r = ctx.filter_project_host(arrays, pred, proj)
    assert r.on_host
    r.free()
    # a Boolean projection: the resident operator runs once, and no chunk runs before it
    r, k = traced(lambda: ctx.filter_project_host([x], col(0) > lit(0.5), [col(0), col(0) < lit(0.75)], chunk_rows=50_000))
    assert not r.on_host
    assert sum(n.startswith("k_filter_project") for n in k) == 1 and k.count("k_pack_bits") == 1
    got = r.columns()
    r.free()
    assert np.array_equal(got[0], x[x > 0.5]) and np.array_equal(got[1], x[x > 0.5] < 0.75)
    with pytest.raises(engine.DfGpuError) as e:
        ctx.filter_project_host([pin.array], None, [col(0) / lit(0.0)])
    assert e.value.code == A.ERR_ARROW
    pin.free()


def test_filter_emits_all_columns_when_no_projection(ctx):
    # FilterRelation alone gathers every input column (filter.rs:55-57)
    arrays, pred, _ = workloads.c3(50_000)
    got = gpu_fp(ctx, arrays, pred, [])
    exp = O.filter_project(arrays, pred, [])
    assert len(got) == 4
    assert_cols_bit_equal(got, exp)


def test_projection_without_filter(ctx):
    arrays, _, proj = workloads.c3(70_001)
    got = gpu_fp(ctx, arrays, None, proj)
    exp = O.filter_project(arrays, None, proj)
    assert_cols_bit_equal(got, exp)


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 100_003])
def test_boolean_projection_outputs(ctx, n):
    # ProjectRelation evaluates any expression (projection.rs:50-58); a comparison or AND / OR yields a
    # bit-packed BooleanArray (expression.rs:212-224,236-290)
    rng = np.random.default_rng(5)
    a, b = rng.random(n), rng.random(n)
    i = rng.integers(-5, 5, n, dtype=np.int64)
    arrays = [a, b, i]
    proj = [col(0) < col(1), (col(0) > lit(0.5)) & (col(2) >= lit(0)), col(0), (col(2).eq(lit(0))) | (col(1) <= lit(0.1)), col(0) + col(1)]
    if n == 0:
        got = gpu_fp(ctx, arrays, None, proj)
        assert [g.dtype for g in got] == [np.dtype(bool), np.dtype(bool), np.dtype("f8"), np.dtype(bool), np.dtype("f8")]
        assert all(len(g) == 0 for g in got)
        return
    assert_cols_bit_equal(gpu_fp(ctx, arrays, None, proj), O.filter_project(arrays, None, proj))
    pred = col(1) > lit(0.3)
    assert_cols_bit_equal(gpu_fp(ctx, arrays[:2], pred, proj[:1] + [col(1) >= col(0)]), O.filter_project(arrays[:2], pred, proj[:1] + [col(1) >= col(0)]))


def test_boolean_input_columns(ctx):
    # BooleanArray inputs (bit-packed): boolean_ops! takes any BooleanArray operand (expression.rs:212-224),
    # a Boolean column can be the whole predicate, be projected, and carry nulls
    import pyarrow as pa
    rng = np.random.default_rng(21)
    for n in [0, 1, 7, 8, 9, 100_003]:
        a = rng.random(n)
        f = rng.random(n) < 0.4
        g = rng.random(n) < 0.7
        cases = [(col(1), [col(0)]), (col(1) & (col(0) > lit(0.5)), [col(0), col(1)]), ((col(1) | col(2)) & (col(0) < lit(0.9)), [col(2), col(0) * lit(2.0)]),
                 (None, [col(1) | (col(0) > lit(0.5)), col(1) & col(2)])]
        for pred, proj in cases:
            got = gpu_fp(ctx, [a, f, g], pred, proj)
            if n == 0:  # (the oracle's relation yields no batch at all for an empty input)
                assert all(len(x) == 0 for x in got)
                continue
            exp = O.rows([a, f, g], pred, proj)
            assert len(got) == len(exp)
            for x, y in zip(got, exp):
                assert np.array_equal(np.asarray(x), np.asarray(y))
    # nullable Boolean column next to a nullable Float64 column (arrow 0.12 and / or: null if either side is null)
    n = 50_000
    a = rng.random(n)
    f = rng.random(n) < 0.5
    fa = pa.array(f, mask=rng.random(n) < 0.2)
    na = pa.array(a, mask=rng.random(n) < 0.1)
    for pred, proj in [(col(1) & (col(0) > lit(0.3)), [col(0), col(1)]), (None, [col(1) | (col(0) < lit(0.5))])]:
        assert_nullable_equal(gpu_fp(ctx, [na, fa], pred, proj), O.rows([na, fa], pred, proj))
    # fused WHERE with a Boolean column under an aggregate
    k = rng.integers(0, 50, n, dtype=np.int64)
    exp = O.filtered_aggregate([k, a, f], col(2) & (col(1) < lit(0.8)), [col(0)], [AggregateFunction("max", col(1)), AggregateFunction("count", col(1))])
    got = gpu_agg(ctx, [k, a, f], [col(0)], [AggregateFunction("max", col(1)), AggregateFunction("count", col(1))], pred=col(2) & (col(1) < lit(0.8)))
    check_groupby(got, exp, 1, exact_cols={0, 1, 2}, sum_cols=set())
    with pytest.raises(engine.DfGpuError) as ei:  # aggregate.rs:848-850
        gpu_agg(ctx, [k, a, f], [col(2)], [AggregateFunction("max", col(1))])
    assert "Unsupported GROUP BY data type" in str(ei.value)


def test_compound_predicates_and_nested_expressions(ctx):
    rng = np.random.default_rng(3)
    a, b, c = rng.random(200_000), rng.random(200_000), rng.random(200_000) + 0.5
    arrays = [a, b, c]
    pred = ((col(0) > lit(0.25)) & (col(1) <= col(0))) | ((col(2) * col(2)) < (col(0) + lit(1.0)))
    proj = [(col(0) + col(1)) * (col(2) - col(0)), col(0) / col(2), (col(0) - lit(0.5)) * ((col(1) + col(2)) / (col(2) + lit(1.0)))]
    got = gpu_fp(ctx, arrays, pred, proj)
    exp = O.filter_project(arrays, pred, proj)
    assert_cols_bit_equal(got, exp)


@pytest.mark.parametrize("np_dt", [np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64, np.float32, np.float64])
def test_all_numeric_dtypes(ctx, np_dt):
    # expression.rs:136-165,176-206 dispatch ten numeric types; wrap-around integer arithmetic
    rng = np.random.default_rng(11)
    n = 100_000
    if np.issubdtype(np_dt, np.integer):
        info = np.iinfo(np_dt)
        x = rng.integers(info.min, info.max, n, dtype=np_dt, endpoint=True)
        y = rng.integers(info.min, info.max, n, dtype=np_dt, endpoint=True)
        y[y == 0] = 1
    else:
        x = (rng.random(n) * 200 - 100).astype(np_dt)
        y = (rng.random(n) * 200 - 100).astype(np_dt)
        y[y == 0] = 1
    dt = A.DTYPE_OF_NP[np.dtype(np_dt)]
    arrays = [x, y]
    pred = (col(0) < col(1)) | (col(0).eq(col(1)))
    proj = [col(0) + col(1), col(0) - col(1), col(0) * col(1), col(0) / col(1), col(0)]
    exp = O.rows(arrays, pred, proj)
    got = gpu_fp(ctx, arrays, pred, proj)
    assert_cols_bit_equal(got, exp)
    lt = lit(int(x[5]) if np.issubdtype(np_dt, np.integer) else float(x[5]), dt)
    for p in [col(0) >= lt, col(0).not_eq(lt), col(0) > lt, col(0) <= lt]:
        assert_cols_bit_equal(gpu_fp(ctx, arrays, p, [col(1)]), O.rows(arrays, p, [col(1)]))


def test_lean_filter_shapes_all_operators(ctx):
    # the lean consumer loop of k_filter_project_tma is instantiated per comparison operator and operand kind
    # (column / literal) for one or two copy / arithmetic projections: every instantiation against the oracle,
    # NaN, +-0, infinities and a zero divisor among the rows, tile-ragged sizes
    rng = np.random.default_rng(77)
    for n in [4095, 70_001]:
        a = rng.random(n)
        b = rng.random(n)
        special = np.array([np.nan, 0.0, -0.0, np.inf, -np.inf, 5e-324, 0.5])
        a[rng.integers(0, n, 300)] = special[rng.integers(0, len(special), 300)]
        b[rng.integers(0, n, 300)] = special[rng.integers(0, len(special), 300)]
        b[::7] = a[::7]  # equal pairs
        preds = []
        for rhs in (col(1), lit(0.5)):
            preds += [col(0) < rhs, col(0) <= rhs, col(0) > rhs, col(0) >= rhs, col(0).eq(rhs), col(0).not_eq(rhs)]
        projs = [[col(0)], [col(1), col(0)], [col(0) + col(1), col(0) * col(1)], [col(0) - col(1)], [col(1) * lit(3.0), col(0) - lit(0.25)],
                 [col(0) + lit(1.0)]]
        for i, p in enumerate(preds):
            pr = projs[i % len(projs)]
            assert_cols_bit_equal(gpu_fp(ctx, [a, b], p, pr), O.filter_project([a, b], p, pr))
        # six referenced columns: the 1024-row tile (K = 2) instantiation; four: the 2048-row one
        c, d2, e, f = rng.random(n), rng.random(n), rng.random(n), rng.random(n)
        for arrs, p_, pr in [([a, b, c, d2, e, f], col(0) < col(1), [col(2) + col(3), col(4) * col(5)]),
                             ([a, b, c, d2], col(0) >= col(1), [col(2) - col(3), col(3)])]:
            assert_cols_bit_equal(gpu_fp(ctx, arrs, p_, pr), O.filter_project(arrs, p_, pr))
        # division: fine while no surviving row divides by zero; DivideByZero otherwise (like the generic path)
        d = np.where(b == 0.0, 1.0, b)
        assert_cols_bit_equal(gpu_fp(ctx, [a, d], col(0) > lit(0.25), [col(0) / col(1)]), O.filter_project([a, d], col(0) > lit(0.25), [col(0) / col(1)]))
        assert_cols_bit_equal(gpu_fp(ctx, [a, d], col(0) > lit(0.25), [col(0) / lit(4.0), col(1)]), O.filter_project([a, d], col(0) > lit(0.25), [col(0) / lit(4.0), col(1)]))
        z = d.copy()
        z[n // 2] = 0.0
        a2 = a.copy()
        a2[n // 2] = 0.75  # the row survives the filter
        with pytest.raises(Exception):
            gpu_fp(ctx, [a2, z], col(0) > lit(0.25), [col(0) / col(1)])
        a2[n // 2] = 0.1   # filtered out: no error
        assert_cols_bit_equal(gpu_fp(ctx, [a2, z], col(0) > lit(0.25), [col(0) / col(1)]), O.filter_project([a2, z], col(0) > lit(0.25), [col(0) / col(1)]))


@pytest.mark.parametrize("np_dt", [np.int64, np.uint64])
def test_lean_filter_shapes_integer_operands(ctx, np_dt):
    # the same loop with Int64 / UInt64 comparisons (signed vs unsigned order at the extremes), 64-bit wrap-around
    # arithmetic in the projections, and a predicate over an integer column projecting a Float64 column
    rng = np.random.default_rng(78)
    n = 66_000
    info = np.iinfo(np_dt)
    a = rng.integers(info.min, info.max, n, dtype=np_dt, endpoint=True)
    b = rng.integers(info.min, info.max, n, dtype=np_dt, endpoint=True)
    a[::5] = rng.integers(0, 50, len(a[::5])).astype(np_dt)
    b[::5] = rng.integers(0, 50, len(b[::5])).astype(np_dt)
    a[::11] = info.max
    b[::13] = info.min
    f = rng.random(n)
    dt = A.INT64 if np_dt == np.int64 else A.UINT64
    preds = []
    for rhs in (col(1), lit(25, dt)):
        preds += [col(0) < rhs, col(0) <= rhs, col(0) > rhs, col(0) >= rhs, col(0).eq(rhs), col(0).not_eq(rhs)]
    projs = [[col(0)], [col(2), col(1)], [col(0) + col(1), col(0) * col(1)], [col(0) - col(1)], [col(1) * lit(3, dt), col(2) * lit(0.5)],
             [col(0) + lit(7, dt)]]
    for i, p in enumerate(preds):
        pr = projs[i % len(projs)]
        assert_cols_bit_equal(gpu_fp(ctx, [a, b, f], p, pr), O.rows([a, b, f], p, pr))


def test_nan_and_signed_zero_compare(ctx):
    a = np.array([np.nan, 0.0, -0.0, 1.0, -np.inf, np.inf, np.nan, 5e-324] * 100)
    b = np.roll(a, 3)
    for p in [col(0) < col(1), col(0) >= col(1), col(0).eq(col(1)), col(0).not_eq(col(1))]:
        got = gpu_fp(ctx, [a, b], p, [col(0), col(1)])
        exp = O.filter_project([a, b], p, [col(0), col(1)])
        assert_cols_bit_equal(got, exp)


def test_error_behaviour_matches_reference(ctx):
    a = np.arange(100, dtype=np.int64)
    f = np.arange(100, dtype=np.float64)
    b = ctx.upload([a, f])
    cases = [
        (lambda: ctx.filter_project(b, None, [col(0) + col(1)]), A.ERR_EXECUTION, "math_ops"),
        (lambda: ctx.filter_project(b, col(1) > lit(1), [col(1)]), A.ERR_EXECUTION, "comparison_ops"),
        (lambda: ctx.filter_project(b, col(1) + col(1), [col(1)]), A.ERR_EXECUTION, "did not evaluate to boolean"),
        (lambda: ctx.filter_project(b, None, [col(1) / lit(0.0)]), A.ERR_ARROW, "DivideByZero"),
        (lambda: ctx.filter_project(b, None, [col(0) / lit(0)]), A.ERR_ARROW, "DivideByZero"),
        (lambda: ctx.filter_project(b, None, [col(7)]), A.ERR_INVALID_COLUMN, "out of range"),
        (lambda: ctx.aggregate(b, [col(1)], [AggregateFunction("sum", col(1))]), A.ERR_EXECUTION, "Unsupported GROUP BY data type"),
        (lambda: ctx.filter_project(b, None, [(col(1) + col(1)).cast(A.INT32)]), A.ERR_GENERAL, "CAST not implemented for expression"),
        (lambda: ctx.filter_project(b, None, [lit(1.5).cast(A.INT32)]), A.ERR_NOT_IMPLEMENTED, "CAST from Float64"),
    ]
    for fn, code, msg in cases:
        with pytest.raises(engine.DfGpuError) as e:
            fn()
        assert e.value.code == code, e.value.msg
        assert msg in e.value.msg
    # a divide by zero on a row the filter drops is NOT an error (projection runs on the filtered batch)
    r = ctx.filter_project(b, col(1) > lit(0.5), [col(1) / col(1)])
    assert r.nrows == 99
    r.free()
    with pytest.raises(engine.DfGpuError):
        ctx.filter_project(b, None, [col(1) / col(1)])
    b.free()


# ---------------------------------------------------------------------------------------------
# aggregates vs oracle
# ---------------------------------------------------------------------------------------------
def check_groupby(got, exp, nkeys, exact_cols, sum_cols):
    got, exp = sort_by_key(got, nkeys), sort_by_key(exp, nkeys)
    assert len(got) == len(exp)
    for i in range(len(got)):
        assert got[i].dtype == exp[i].dtype and got[i].shape == exp[i].shape
        if i in sum_cols:
            np.testing.assert_allclose(got[i], exp[i], rtol=SUM_RTOL, atol=0)
        else:
            assert np.array_equal(got[i].view(np.uint8), exp[i].view(np.uint8)), "column %d" % i


def test_c4_sum_count(ctx):
    arrays, keys, aggs, _ = workloads.c4(1_000_000, nkeys=10_000)
    got = gpu_agg(ctx, arrays, keys, aggs)
    exp = O.aggregate(arrays, keys, aggs)
    assert got[2].dtype == np.uint64
    check_groupby(got, exp, 1, exact_cols={0, 2}, sum_cols={1})


def test_c5_min_max_sum_multibatch(ctx):
    arrays, keys, aggs, _ = workloads.c5(800_000, nkeys=50_000)
    got = gpu_agg(ctx, arrays, keys, aggs, nbatches=3)
    exp = O.aggregate(arrays, keys, aggs, batch_size=1024)
    check_groupby(got, exp, 1, exact_cols={0, 1, 2}, sum_cols={3})


def test_groupby_table_growth_all_distinct_keys(ctx):
    # more distinct keys than the initial table admits: exercises the overflow-replay + grow path
    n = 2_600_000
    k = workloads.mix_keys(np.arange(n, dtype=np.int64))
    v = np.random.default_rng(5).random(n)
    aggs = [AggregateFunction("sum", col(1)), AggregateFunction("count", col(1)), AggregateFunction("max", col(1))]
    got = sort_by_key(gpu_agg(ctx, [k, v], [col(0)], aggs))
    order = np.argsort(k)
    assert np.array_equal(got[0], k[order])
    assert np.array_equal(got[1], v[order]) and np.array_equal(got[3], v[order])
    assert np.all(got[2] == 1)


def test_groupby_low_cardinality_front_table(ctx):
    # few groups in a big batch: the sampled prefix routes the bulk through the shared-memory front table
    n = 6_000_000
    rng = np.random.default_rng(31)
    for ngroups in [1, 7, 900]:
        k = workloads.mix_keys(rng.integers(0, ngroups, n, dtype=np.int64))
        k[::1000] = -1  # the key that equals the empty marker takes the global path
        v = rng.random(n)
        iv = rng.integers(-50, 50, n, dtype=np.int64)
        aggs = [AggregateFunction("sum", col(1)), AggregateFunction("count", col(1)), AggregateFunction("min", col(1)),
                AggregateFunction("max", col(1)), AggregateFunction("sum", col(2))]
        got = gpu_agg(ctx, [k, v, iv], [col(0)], aggs)
        G.assert_matches(got, G.aggregate([k], [(G.SUM, v), (G.COUNT, v), (G.MIN, v), (G.MAX, v), (G.SUM, iv)]), ngroups)


def test_groupby_high_cardinality_layouts(ctx):
    # (a) cardinality hint -> AoS table from the start; (b) no hint: the sampled prefix switches layouts
    n = 5_000_000
    rng = np.random.default_rng(33)
    k = workloads.mix_keys(rng.integers(0, 1_500_000, n, dtype=np.int64))
    v = rng.random(n)
    aggs = [AggregateFunction("min", col(1)), AggregateFunction("max", col(1)), AggregateFunction("sum", col(1)), AggregateFunction("count", col(1))]
    exp = G.aggregate([k], [(G.MIN, v), (G.MAX, v), (G.SUM, v), (G.COUNT, v)])
    for hint in [2_000_000, 0]:
        G.assert_matches(gpu_agg(ctx, [k, v], [col(0)], aggs, expected=hint), exp, hint)
    # two batches: the second one finds the table already converted
    G.assert_matches(gpu_agg(ctx, [k, v], [col(0)], aggs, nbatches=2), exp, "two batches")


def test_groupby_fused_where_vs_oracle(ctx):
    # SELECT k, MIN(v), MAX(v), SUM(v), COUNT(v) FROM g WHERE <pred> GROUP BY k: the predicate runs inside the
    # scan kernel.  Comparison chains take the interpreter-free kernel, arithmetic predicates the interpreter.
    n = 1_000_000
    arrays, keys, aggs, _ = workloads.c5(n, nkeys=20_000)
    aggs = aggs + [AggregateFunction("count", col(1))]
    preds = [col(1) < lit(0.25),
             (col(1) > lit(0.1)) & (col(1) < lit(0.9)),
             (col(1) < lit(0.05)) | (col(1) >= lit(0.95)),
             (col(1) * lit(2.0)) < lit(0.5),
             col(1) < lit(-1.0)]  # nothing passes: empty result
    for pred in preds:
        exp = O.filtered_aggregate(arrays, pred, keys, aggs)
        for nb in [1, 3]:
            got = gpu_agg(ctx, arrays, keys, aggs, nbatches=nb, pred=pred)
            check_groupby(got, exp, 1, exact_cols={0, 1, 2, 4}, sum_cols={3})
    # expression keys and arguments (interpreter path) under a predicate on another column.  Small: the oracle
    # restates the reference's per-row re-evaluation of an aggregate's argument expression (aggregate.rs:559),
    # which is quadratic in the batch size
    rng = np.random.default_rng(77)
    m = 20_000
    k = rng.integers(0, 500, m, dtype=np.int64)
    w = rng.integers(-100, 100, m, dtype=np.int64)
    v = rng.random(m)
    keys2 = [col(0) + lit(7)]
    aggs2 = [AggregateFunction("sum", col(2) * lit(3.0)), AggregateFunction("max", col(1)), AggregateFunction("count", col(2))]
    pred2 = (col(1) > lit(-20)) & (col(2) < lit(0.75))
    exp = O.filtered_aggregate([k, w, v], pred2, keys2, aggs2)
    got = gpu_agg(ctx, [k, w, v], keys2, aggs2, pred=pred2)
    check_groupby(got, exp, 1, exact_cols={0, 2, 3}, sum_cols={1})
    # Int32 keys / Float32 arguments through the plain kernel's 4-byte loads, odd row count
    k32 = rng.integers(0, 3000, n - 1, dtype=np.int32)
    v32 = rng.random(n - 1).astype(np.float32)
    aggs3 = [AggregateFunction("min", col(1)), AggregateFunction("max", col(1)), AggregateFunction("count", col(1))]
    pred3 = col(1) >= lit(0.5, A.FLOAT32)
    exp = O.filtered_aggregate([k32, v32], pred3, [col(0)], aggs3)
    got = gpu_agg(ctx, [k32, v32], [col(0)], aggs3, pred=pred3)
    check_groupby(got, exp, 1, exact_cols={0, 1, 2, 3}, sum_cols=set())


def test_no_groupby_fused_where_vs_oracle(ctx):
    n = 700_001
    rng = np.random.default_rng(78)
    v = rng.random(n)
    w = rng.integers(0, 1000, n, dtype=np.int64)
    aggs = [AggregateFunction("min", col(0)), AggregateFunction("max", col(0)), AggregateFunction("sum", col(0)), AggregateFunction("count", col(0)),
            AggregateFunction("sum", col(1))]
    for pred in [col(0) < lit(0.3), (col(1) >= lit(500)) & (col(0) > lit(0.5))]:
        exp = O.filtered_aggregate([v, w], pred, [], aggs)
        got = gpu_agg(ctx, [v, w], [], aggs, nbatches=2, pred=pred)
        for i, (g, e) in enumerate(zip(got, exp)):
            if i == 2:
                np.testing.assert_allclose(g, e, rtol=SUM_RTOL)
            else:
                assert np.array_equal(g, e), i
    # nothing passes: MIN / MAX / SUM are null, exactly as over an empty input
    got = gpu_agg(ctx, [v, w], [], aggs[:3], pred=col(0) < lit(-1.0))
    exp = O.filtered_aggregate([v, w], col(0) < lit(-1.0), [], aggs[:3])
    for g, e in zip(got, exp):
        assert isinstance(g, tuple) == isinstance(e, tuple)
        if isinstance(g, tuple):
            assert np.array_equal(g[1], e[1])
    # a predicate that is not Boolean is the reference's FilterRelation error
    with pytest.raises(engine.DfGpuError) as ei:
        gpu_agg(ctx, [v, w], [], aggs[:1], pred=col(0) + lit(1.0))
    assert "did not evaluate to boolean" in str(ei.value)



def test_golden_group_by_string_min_max(ctx, golden, fmt_f64):
    # tests/sql.rs:55-67: GROUP BY a Utf8 column
    t = golden["aggregate_test_2"]
    out = gpu_agg(ctx, [t["a"], np.array(t["b"])], [col(0)], [AggregateFunction("min", col(1)), AggregateFunction("max", col(1))])
    got = sorted('"%s"\t%s\t%s\n' % (a, fmt_f64(b), fmt_f64(c)) for a, b, c in zip(*out))
    assert got == sorted(golden["csv_query_group_by_string_min_max"]["expected"].splitlines(True))


def test_groupby_utf8_keys_vs_oracle(ctx):
    rng = np.random.default_rng(51)
    n = 120_000
    vocab = ["", "a", "b", "ab", "ba", "London, UK", "x" * 33] + ["k%05d" % i for i in range(3000)]
    ks = [vocab[i] for i in rng.integers(0, len(vocab), n)]
    v = rng.random(n)
    iv = rng.integers(-9, 9, n, dtype=np.int64)
    aggs = [AggregateFunction("min", col(1)), AggregateFunction("max", col(1)), AggregateFunction("sum", col(2)), AggregateFunction("count", col(1))]
    exp = O.aggregate([ks, v, iv], [col(0)], aggs)
    for nb in [1, 4]:
        got = gpu_agg(ctx, [ks, v, iv], [col(0)], aggs, nbatches=nb)
        assert len(got) == 5 and len(got[0]) == len(exp[0])
        go = sorted(range(len(got[0])), key=lambda i: got[0][i])
        eo = sorted(range(len(exp[0])), key=lambda i: exp[0][i])
        assert [got[0][i] for i in go] == [exp[0][i] for i in eo]
        for c in range(1, 5):
            assert np.array_equal(np.asarray(got[c])[go], np.asarray(exp[c])[eo])


def sorted_rows(cols, nkeys):
    """Rows of a GROUP BY result as tuples, sorted by the key tuple (keys may be strings or numbers)."""
    cols = [c if isinstance(c, list) else c.tolist() for c in cols]
    return sorted(zip(*cols), key=lambda r: r[:nkeys])


def check_wide(got, exp, nkeys, sum_cols=()):
    g, e = sorted_rows(got, nkeys), sorted_rows(exp, nkeys)
    assert len(g) == len(e)
    for rg, re_ in zip(g, e):
        for i, (x, y) in enumerate(zip(rg, re_)):
            if i in sum_cols:
                assert x == y or abs(x - y) <= SUM_RTOL * abs(y), (rg, re_)
            else:
                assert x == y or (x != x and y != y), (rg, re_)


def test_groupby_wide_composite_keys(ctx):
    # GROUP BY k1, k2 with two Int64 columns (128 key bits), three keys of mixed widths, (Utf8, Int32) and
    # (Int64, Utf8, Utf8): the reference takes any Vec<GroupByScalar> (aggregate.rs:65-76, 807-852)
    rng = np.random.default_rng(61)
    n = 300_000
    k1 = workloads.mix_keys(rng.integers(0, 300, n, dtype=np.int64))
    k2 = rng.integers(-(2 ** 62), 2 ** 62, 40, dtype=np.int64)[rng.integers(0, 40, n)]
    k3 = rng.integers(0, 7, n, dtype=np.int32)
    vocab = ["", "a", "ab", "London, UK", "y" * 40] + ["s%03d" % i for i in range(60)]
    s1 = [vocab[i] for i in rng.integers(0, len(vocab), n)]
    s2 = [vocab[i] for i in rng.integers(0, 5, n)]
    v = rng.random(n)
    iv = rng.integers(-9, 9, n, dtype=np.int64)
    aggs = lambda c_v, c_i: [AggregateFunction("min", col(c_v)), AggregateFunction("max", col(c_v)), AggregateFunction("sum", col(c_i)),  # noqa: E731
                             AggregateFunction("count", col(c_v)), AggregateFunction("sum", col(c_v))]
    cases = [([k1, k2, v, iv], [col(0), col(1)], 2, 3),
             ([k1, k2, k3, v, iv], [col(0), col(1), col(2)], 3, 4),
             ([s1, k3, v, iv], [col(0), col(1)], 2, 3),
             ([k1, s1, s2, v, iv], [col(0), col(1), col(2)], 3, 4)]
    for arrays, keys, c_v, c_i in cases:
        nk = len(keys)
        ag = aggs(c_v, c_i)
        exp = O.aggregate(arrays, keys, ag)
        for nb in [1, 3]:
            got = gpu_agg(ctx, arrays, keys, ag, nbatches=nb)
            check_wide(got, exp, nk, sum_cols={nk + 4})
    # fused WHERE with wide keys
    pred = col(2) < lit(0.5)
    exp = O.filtered_aggregate([k1, k2, v, iv], pred, [col(0), col(1)], aggs(2, 3))
    check_wide(gpu_agg(ctx, [k1, k2, v, iv], [col(0), col(1)], aggs(2, 3), pred=pred), exp, 2, sum_cols={6})


def test_groupby_wide_keys_growth_and_contention(ctx):
    # (a) more distinct 128-bit keys than the initial table admits: growth by moving the slots; (b) a handful of
    # hot wide keys over many rows: thousands of rows meet a slot while its creator is still publishing it
    n = 2_300_000
    a = workloads.mix_keys(np.arange(n, dtype=np.int64))
    b = a[::-1].copy()
    v = np.random.default_rng(3).random(n)
    ag = [AggregateFunction("sum", col(2)), AggregateFunction("count", col(2)), AggregateFunction("max", col(2))]
    got = gpu_agg(ctx, [a, b, v], [col(0), col(1)], ag)
    o = np.lexsort([got[1], got[0]])
    oe = np.lexsort([b, a])
    assert np.array_equal(got[0][o], a[oe]) and np.array_equal(got[1][o], b[oe])
    assert np.array_equal(got[2][o], v[oe]) and np.all(got[3] == 1) and np.array_equal(got[4][o], v[oe])
    n = 3_000_000
    rng = np.random.default_rng(4)
    hot1 = rng.integers(0, 3, n, dtype=np.int64) * (2 ** 40)
    hot2 = rng.integers(0, 2, n, dtype=np.int64) - 1
    w = rng.random(n)
    got = gpu_agg(ctx, [hot1, hot2, w], [col(0), col(1)], ag)
    assert len(got[0]) == 6 and int(got[3].sum()) == n
    for i in range(6):
        m = (hot1 == got[0][i]) & (hot2 == got[1][i])
        assert got[3][i] == int(m.sum()) and got[4][i] == w[m].max()
        assert abs(got[2][i] - w[m].sum()) <= 1e-9 * w[m].sum()


def test_groupby_sentinel_and_extreme_keys(ctx):
    k = np.array([-1, -1, 0, np.iinfo(np.int64).min, np.iinfo(np.int64).max, -1, 0, 7], dtype=np.int64)
    v = np.arange(8, dtype=np.float64) + 0.5
    aggs = [AggregateFunction("sum", col(1)), AggregateFunction("min", col(1)), AggregateFunction("count", col(1))]
    got = gpu_agg(ctx, [k, v], [col(0)], aggs)
    exp = O.aggregate([k, v], [col(0)], aggs)
    check_groupby(got, exp, 1, set(), {1})


@pytest.mark.parametrize("kdt", [np.int8, np.uint8, np.int16, np.uint16, np.int32, np.uint32, np.uint64])
def test_groupby_key_dtypes(ctx, kdt):
    rng = np.random.default_rng(9)
    info = np.iinfo(kdt)
    k = rng.integers(info.min, min(info.max, info.min + 5000), 200_000, dtype=kdt, endpoint=True)
    v = rng.random(200_000)
    iv = rng.integers(-1000, 1000, 200_000, dtype=np.int64)
    aggs = [AggregateFunction("min", col(1)), AggregateFunction("max", col(1)), AggregateFunction("sum", col(2)),
            AggregateFunction("min", col(2)), AggregateFunction("max", col(2)), AggregateFunction("count", col(2))]
    got = gpu_agg(ctx, [k, v, iv], [col(0)], aggs)
    exp = O.aggregate([k, v, iv], [col(0)], aggs)
    check_groupby(got, exp, 1, set(), set())  # everything here is exact (int SUM wraps identically)


def test_groupby_two_keys_and_expression_args(ctx):
    rng = np.random.default_rng(13)
    n = 150_000
    k1 = rng.integers(-50, 50, n, dtype=np.int32)
    k2 = rng.integers(0, 40, n, dtype=np.uint16)
    a, b = rng.random(n), rng.random(n)
    aggs = [AggregateFunction("sum", col(2) * col(3)), AggregateFunction("max", col(2) + col(3)), AggregateFunction("count", col(2))]
    got = gpu_agg(ctx, [k1, k2, a, b], [col(0), col(1)], aggs)
    # the reference re-evaluates aggregate arguments per row (aggregate.rs:559): keep the oracle input small
    m = 4000
    got_small = gpu_agg(ctx, [k1[:m], k2[:m], a[:m], b[:m]], [col(0), col(1)], aggs)
    exp_small = O.aggregate([k1[:m], k2[:m], a[:m], b[:m]], [col(0), col(1)], aggs)
    check_groupby(got_small, exp_small, 2, set(), {2})
    # full size against the exact reference
    G.assert_matches(got, G.aggregate([k1, k2], [(G.SUM, a * b), (G.MAX, a + b), (G.COUNT, a)]), "full size")


@pytest.mark.parametrize("np_dt", [np.int32, np.int64, np.uint16, np.float32, np.float64])
def test_no_groupby_reduce(ctx, np_dt):
    rng = np.random.default_rng(21)
    n = 777_777
    x = (rng.random(n) * 1000 - 500).astype(np_dt)
    aggs = [AggregateFunction("min", col(0)), AggregateFunction("max", col(0)), AggregateFunction("sum", col(0)), AggregateFunction("count", col(0))]
    got = gpu_agg(ctx, [x], [], aggs, nbatches=2)
    exp = O.aggregate([x], [], aggs, batch_size=100_000)
    assert [len(g) for g in got] == [1, 1, 1, 1]
    assert got[0][0] == exp[0][0] and got[1][0] == exp[1][0] and got[3][0] == exp[3][0] == n
    if np.issubdtype(np_dt, np.integer):
        assert got[2][0] == exp[2][0]
    else:
        # f32 sums: the reference folds sequentially in f32; tolerance scaled to the type
        rtol = SUM_RTOL if np_dt == np.float64 else 1e-3
        ref = float(np.sum(x.astype(np.float64)))
        assert abs(float(got[2][0]) - ref) <= rtol * max(1.0, abs(ref)) + (0 if np_dt == np.float64 else 50.0)
        if np_dt == np.float64:
            assert abs(float(got[2][0]) - float(exp[2][0])) <= SUM_RTOL * abs(float(exp[2][0])) + 1e-6


def test_no_groupby_empty_input_is_null(ctx):
    got = gpu_agg(ctx, [np.array([], dtype=np.float64)], [], [AggregateFunction("sum", col(0)), AggregateFunction("min", col(0))])
    for c in got:
        vals, mask = c
        assert len(vals) == 1 and not mask[0]


# ---------------------------------------------------------------------------------------------
# BASELINE sizes: size-independent properties (the oracle is too slow here)
# ---------------------------------------------------------------------------------------------
def test_c2_full_size_properties(ctx):
    n = 100_000_000
    arrays, pred, proj = workloads.c2(n)
    a = arrays[0]
    b = ctx.upload(arrays)
    r = ctx.filter_project(b, pred, proj)
    out = r.columns()[0]
    r.free()
    m = a > 0.5
    assert len(out) == int(m.sum())
    assert np.array_equal(out, a[m])  # order-preserving, bit-exact
    # idempotence: filtering the output again keeps everything
    b2 = ctx.upload([out])
    r2 = ctx.filter_project(b2, pred, proj)
    assert r2.nrows == len(out)
    r2.free(); b2.free(); b.free()


def test_c4_full_size_properties(ctx):
    n = 100_000_000
    arrays, keys, aggs, k_raw = workloads.c4(n)
    got = gpu_agg(ctx, arrays, keys, aggs)
    assert len(got[0]) == len(np.unique(k_raw[:1_000_000])) or len(got[0]) == 100_000
    assert int(got[2].sum()) == n  # checksum of counts
    cnt = np.bincount(k_raw, minlength=100_000)
    sm = np.bincount(k_raw, weights=arrays[1], minlength=100_000)
    inv = workloads.mix_keys(np.arange(100_000, dtype=np.int64))
    order = np.argsort(inv)
    got = sort_by_key(got)
    assert np.array_equal(got[0], inv[order])
    assert np.array_equal(got[2], cnt[order].astype(np.uint64))
    np.testing.assert_allclose(got[1], sm[order], rtol=SUM_RTOL)


def test_c3_full_size_parity(ctx):
    # BASELINE configs[2] at its stated size: 1e8 rows x 4 Float64 columns, fused expr + filter, bit-exact vs numpy
    n = 100_000_000
    arrays, pred, proj = workloads.c3(n)
    a, b = arrays[0], arrays[1]
    bt = ctx.upload(arrays)
    r = ctx.filter_project(bt, pred, proj)
    out = r.columns()
    r.free(); bt.free()
    m = b < a
    assert len(out[0]) == int(m.sum())
    assert np.array_equal(out[0], (a + b)[m])  # one IEEE add / multiply per element: bit-exact, order-preserving
    assert np.array_equal(out[1], (a * b)[m])


def test_c5_full_size_parity(ctx):
    # BASELINE configs[4] per-GPU shard at its stated size (1e9 rows / 8 GPUs = 1.25e8 rows, 1e6 keys):
    # keys / MIN / MAX bit-exact, SUM within 1e-9 relative.  Checker: numpy bincount for SUM and torch
    # scatter_reduce (amin / amax, an independent library implementation) for MIN / MAX on the same rows.
    import torch
    n = 125_000_000
    arrays, keys, aggs, k_raw = workloads.c5(n)
    got = sort_by_key(gpu_agg(ctx, arrays, keys, aggs))
    v = arrays[1]
    kt, vt = torch.from_numpy(k_raw).cuda(), torch.from_numpy(v).cuda()
    mn = torch.full((1_000_000,), float("inf"), dtype=torch.float64, device="cuda").scatter_reduce_(0, kt, vt, "amin").cpu().numpy()
    mx = torch.full((1_000_000,), float("-inf"), dtype=torch.float64, device="cuda").scatter_reduce_(0, kt, vt, "amax").cpu().numpy()
    del kt, vt
    torch.cuda.empty_cache()
    cnt = np.bincount(k_raw, minlength=1_000_000)
    present = np.nonzero(cnt)[0]
    sm = np.bincount(k_raw, weights=v, minlength=1_000_000)[present]
    mixed = workloads.mix_keys(present.astype(np.int64))
    order = np.argsort(mixed)
    assert np.array_equal(got[0], mixed[order])
    assert np.array_equal(got[1], mn[present][order]) and np.array_equal(got[2], mx[present][order])
    np.testing.assert_allclose(got[3], sm[order], rtol=SUM_RTOL)


# ---------------------------------------------------------------------------------------------
# nulls: arrow 0.12 array_ops semantics as the reference's operators see them (oracle restates them)
# ---------------------------------------------------------------------------------------------
def nullable(values, valid):
    """pyarrow array over OUR buffers, so the bytes under null slots are known to both sides."""
    import pyarrow as pa
    values = np.ascontiguousarray(values)
    bits = np.packbits(np.asarray(valid, dtype=bool), bitorder="little")
    return pa.Array.from_buffers(pa.from_numpy_dtype(values.dtype), len(values), [pa.py_buffer(bits.tobytes()), pa.py_buffer(values.tobytes())])


def unpack(c):
    return c if isinstance(c, tuple) else (c, np.ones(len(c), dtype=bool))


def assert_nullable_equal(got, exp):
    assert len(got) == len(exp)
    for g, e in zip(got, exp):
        (gv, gm), (ev, em) = unpack(g), unpack(e)
        assert gv.dtype == ev.dtype and np.array_equal(gm, em)
        assert np.array_equal(gv[gm].view(np.uint8), ev[em].view(np.uint8))


def test_nulls_filter_and_projection(ctx):
    rng = np.random.default_rng(41)
    n = 150_001
    a, b = rng.random(n), rng.random(n)
    i = rng.integers(-100, 100, n, dtype=np.int64)
    va, vb, vi = rng.random(n) > 0.2, rng.random(n) > 0.3, rng.random(n) > 0.1
    arrays = [nullable(a, va), nullable(b, vb), nullable(i, vi), a.copy()]
    preds = [col(0) > lit(0.5), col(0) < lit(0.5), col(0) < col(1), col(0) >= col(1), col(0).eq(col(1)), col(0).not_eq(col(1)),
             (col(0) > lit(0.3)) & (col(1) < lit(0.6)), (col(0) > lit(0.9)) | (col(1) <= col(0)), (col(0) + col(1)) > lit(1.0),
             col(2) > lit(0)]
    O.set_extensions(filter_all_primitives=True)
    try:
        for pred in preds:
            proj = [col(0), col(1), col(0) * col(1), col(2), col(3)]
            assert_nullable_equal(gpu_fp(ctx, arrays, pred, proj), O.filter_project(arrays, pred, proj))
        # no predicate: projections keep / produce nulls
        proj = [col(0), col(0) + col(1), col(0) * lit(2.0), col(2) - col(2), col(0) < col(1), col(3), col(2).cast(A.INT32)]
        assert_nullable_equal(gpu_fp(ctx, arrays, None, proj), O.filter_project(arrays, None, proj))
        # AND / OR of comparisons over nullable inputs: comparisons are never null, so neither is the result
        proj = [(col(0) < col(1)) & (col(2) > lit(0)), (col(0) > lit(0.5)) | (col(1) > lit(0.5)), col(0)]
        assert_nullable_equal(gpu_fp(ctx, arrays, None, proj), O.filter_project(arrays, None, proj))
    finally:
        O.set_extensions(filter_all_primitives=False)


def test_nulls_aggregates(ctx):
    rng = np.random.default_rng(43)
    n = 120_000
    k = rng.integers(0, 500, n, dtype=np.int32)
    v, w = rng.random(n), rng.random(n)
    vk, vv, vw = rng.random(n) > 0.1, rng.random(n) > 0.4, rng.random(n) > 0.5
    arrays = [nullable(k, vk), nullable(v, vv), nullable(w, vw)]
    aggs = [AggregateFunction("sum", col(1)), AggregateFunction("min", col(1)), AggregateFunction("max", col(1)),
            AggregateFunction("count", col(1)), AggregateFunction("count", col(2))]
    got = gpu_agg(ctx, arrays, [col(0)], aggs)
    exp = O.aggregate(arrays, [col(0)], aggs)
    check_groupby(got, exp, 1, set(), {1})
    # arithmetic over nullable columns as an aggregate argument (null reads as 0, aggregate.rs:561-601): small input,
    # the reference re-evaluates the argument per row
    m = 3000
    small = [nullable(k[:m], vk[:m]), nullable(v[:m], vv[:m]), nullable(w[:m], vw[:m])]
    aggs2 = [AggregateFunction("sum", col(1) + col(2)), AggregateFunction("count", col(1) + col(2))]
    check_groupby(gpu_agg(ctx, small, [col(0)], aggs2), O.aggregate(small, [col(0)], aggs2), 1, set(), {1})
    # no GROUP BY: array_ops min/max/sum skip nulls
    aggs3 = [AggregateFunction("min", col(1)), AggregateFunction("max", col(1)), AggregateFunction("sum", col(1)), AggregateFunction("count", col(1))]
    g, e = gpu_agg(ctx, arrays, [], aggs3, nbatches=3), O.aggregate(arrays, [], aggs3, batch_size=40_000)
    assert g[0][0] == e[0][0] and g[1][0] == e[1][0] and g[3][0] == e[3][0] == int(vv.sum())
    assert abs(g[2][0] - e[2][0]) <= SUM_RTOL * abs(e[2][0])
    # all-null column: MIN/MAX/SUM are null, COUNT is 0
    allnull = [nullable(v[:1000], np.zeros(1000, dtype=bool))]
    g = gpu_agg(ctx, allnull, [], [AggregateFunction("sum", col(0)), AggregateFunction("min", col(0)), AggregateFunction("count", col(0))])
    assert not unpack(g[0])[1][0] and not unpack(g[1])[1][0]
    assert unpack(g[2])[0][0] == 0 and unpack(g[2])[1][0]


def test_fuzz_random_expression_trees(ctx):
    """120 random queries (predicate + 1-3 projections, depth <= 3) over f64 / i64 / i32 / f32 columns:
    the GPU result must equal the oracle's bit for bit — the same rows, in the same order."""
    import fuzz_exprs as F
    rng = np.random.default_rng(20260923)
    n = 20_011
    data = [rng.random(n) * 4 - 2, rng.random(n) * 4 - 2, rng.integers(-6, 7, n, dtype=np.int64), rng.integers(-6, 7, n, dtype=np.int64),
            rng.integers(-100, 100, n, dtype=np.int32), (rng.random(n) * 4 - 2).astype(np.float32), (rng.random(n) * 4 - 2).astype(np.float32)]
    schema = [A.DTYPE_OF_NP[a.dtype] for a in data]
    b = ctx.upload(data)
    O.set_extensions(filter_all_primitives=True)
    ran = 0
    try:
        for q in range(120):
            pred, proj = F.gen_query(rng, schema)
            try:
                exp = O.filter_project(data, pred, proj)
            except O.OracleError as e:
                # e.g. a literal-only projection is fine for the oracle but needs a column on the GPU path
                raise AssertionError("oracle rejected a generated query: %s / %r %r" % (e, pred, proj))
            if not any(F.references_column(e) for e in proj + ([pred] if pred is not None else [])):
                continue
            r = ctx.filter_project(b, pred, proj)
            got = r.columns()
            r.free()
            assert len(got) == len(exp), (pred, proj)
            for g, e in zip(got, exp):
                assert g.dtype == e.dtype and g.shape == e.shape and np.array_equal(g.view(np.uint8), e.view(np.uint8)), (q, pred, proj)
            ran += 1
    finally:
        O.set_extensions(filter_all_primitives=False)
        b.free()
    assert ran >= 100
