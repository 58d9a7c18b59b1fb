"""Every GROUP BY and reduce kernel instantiation against the exact reference of tests/groupby_ref.py.

Each case runs with DFGPU_TRACE set, reads the names of the kernels the library launched, and asserts that the
instantiation it is named for ran, so a change in the dispatch cannot silently move a case onto another kernel.
Inputs carry the value edges where kernels go wrong: NaN, ±0.0, ±inf, subnormals, the integer extremes, UInt64 values with
the top bit set, and the keys that pack to the table's empty marker."""

import numpy as np
import pytest

import groupby_ref as R
from kernel_trace import traced_set as traced
from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import engine
from datafusion_archive_b200.expr import AggregateFunction, col, lit

pytestmark = pytest.mark.gpu

F64, I64, U64 = np.float64, np.int64, np.uint64
FUNC_OF_BIT = {1: R.MIN, 2: R.MAX, 4: R.SUM, 8: R.COUNT}
MT = {np.dtype(F64): 1, np.dtype(np.float32): 2, np.dtype(I64): 3, np.dtype(U64): 4}  # expr_vm.cuh MT_*


@pytest.fixture(scope="module")
def ctx():
    c = engine.GpuContext(0)
    yield c
    c.close()


def run_agg(ctx, batches, keys, aggs, expected=0, pred=None):
    """GROUP BY over the given batches (lists of columns); returns (result columns, kernels launched)."""
    def go():
        bs = [ctx.upload(b) for b in batches]
        try:
            r = ctx.aggregate(bs, keys, aggs, expected, pred=pred)
            try:
                return r.columns()
            finally:
                r.free()
        finally:
            for b in bs:
                b.free()
    return traced(go)


def assert_launched(names, *want):
    for w in want:
        assert w in names, (w, sorted(names))


def key_pool(rng, dt, ngroups):
    """ngroups distinct keys of dtype dt, the empty-marker key (-1 / all ones) and the extremes among them."""
    info = np.iinfo(dt)
    special = np.array(sorted({info.min, info.max, 0, np.array(-1).astype(dt).item()}), dtype=dt)
    if ngroups <= len(special):
        return special[:ngroups]
    lo, hi = max(info.min, -(2 ** 62)), min(info.max, 2 ** 62)
    rest = np.unique(rng.integers(lo, hi, 2 * ngroups, dtype=dt))
    rest = rest[~np.isin(rest, special)]
    rng.shuffle(rest)
    return np.concatenate([special, rest[:ngroups - len(special)]])


def keys_from(rng, pool, n):
    """n keys drawing every pool entry at least once."""
    k = pool[rng.integers(0, len(pool), n)]
    k[rng.choice(n, len(pool), replace=False)] = pool
    return k


def values(rng, dt, n, for_sum):
    return R.sprinkle(rng, R.random_values(rng, dt, n), R.edges(dt, for_sum))


def agg_exprs(spec):
    """[(func, column index)] -> AggregateFunction list."""
    return [AggregateFunction(f, col(c)) for f, c in spec]


def reference(key_cols, cols, spec):
    return R.aggregate(key_cols, [(f, cols[c]) for f, c in spec])


def concat(batches):
    return [np.concatenate([b[i] for b in batches]) for i in range(len(batches[0]))]


# ---- k_hash_agg_lean<M, MT>: all 15 aggregate masks x 3 argument machine types ------------------------------
@pytest.mark.parametrize("mask", range(1, 16))
@pytest.mark.parametrize("adt", [F64, I64, U64], ids=["f64", "i64", "u64"])
def test_lean_kernel(ctx, mask, adt):
    rng = np.random.default_rng(1000 * mask + MT[np.dtype(adt)])
    n = 200_001  # odd: the last thread holds one row
    kdt = U64 if (adt == U64 or mask % 2) else I64  # both key types; -1 / 2^64 - 1 is the empty-marker key
    k = keys_from(rng, key_pool(rng, kdt, 5000), n)
    v = values(rng, adt, n, for_sum=bool(mask & 4))
    funcs = [FUNC_OF_BIT[b] for b in (1, 2, 4, 8) if mask & b]
    funcs = [funcs[i] for i in rng.permutation(len(funcs))]  # the MIN / MAX words come from the layout, not the order
    spec = [(f, 1) for f in funcs]
    got, names = run_agg(ctx, [[k, v]], [col(0)], agg_exprs(spec))
    assert_launched(names, "k_hash_agg_lean<%d,%d>" % (mask, MT[np.dtype(adt)]))
    R.assert_matches(got, reference([k], [k, v], spec), "lean %d %s" % (mask, np.dtype(adt)))


# ---- k_hash_agg_plain<2|4, FRONT> and the front-table boundaries ---------------------------------------------
def plain_columns(rng, n, pool, four):
    k = keys_from(rng, pool, n)
    if not four:
        return [k, values(rng, np.float32, n, for_sum=False)], [(R.MIN, 1), (R.MAX, 1), (R.COUNT, 1)]
    cols = [k, values(rng, np.float32, n, for_sum=False), values(rng, np.int32, n, for_sum=True), values(rng, np.uint32, n, for_sum=False)]
    return cols, [(R.MAX, 3), (R.SUM, 2), (R.MIN, 1), (R.MIN, 2), (R.COUNT, 3), (R.MAX, 1), (R.MIN, 3), (R.MAX, 2)]


@pytest.mark.parametrize("four", [False, True], ids=["2col", "4col"])
def test_plain_kernel(ctx, four):
    rng = np.random.default_rng(7 + four)
    n = 300_001
    cols, spec = plain_columns(rng, n, key_pool(rng, np.int32, 20_000), four)
    got, names = run_agg(ctx, [cols], [col(0)], agg_exprs(spec))
    assert_launched(names, "k_hash_agg_plain<%d,0>" % (4 if four else 2))
    R.assert_matches(got, reference([cols[0]], cols, spec), "plain")


@pytest.mark.parametrize("ngroups", [1, 64, 65, 66, 1024, 1025, 1026])
@pytest.mark.parametrize("four", [False, True], ids=["2col", "4col"])
def test_plain_front_table(ctx, ngroups, four):
    # a first batch of >= 1 Mi rows with <= 1024 groups sends the next batch through the shared-memory front table
    # (one table per warp up to 64 groups, one per CTA beyond).  The empty-marker key (in every pool of more than
    # one key) lives in its own slot, outside both tables, so it is not counted against either limit
    rng = np.random.default_rng(ngroups * 2 + four)
    pool = key_pool(rng, np.int32, ngroups)
    b1, spec = plain_columns(rng, 1_100_000, pool, four)
    b2, _ = plain_columns(rng, 400_001, pool, four)
    got, names = run_agg(ctx, [b1, b2], [col(0)], agg_exprs(spec))
    nc = 4 if four else 2
    assert_launched(names, "k_hash_agg_plain<%d,0>" % nc)
    front = "k_hash_agg_plain<%d,1>" % nc
    counted = ngroups - int(np.any(pool == -1))
    assert (front in names) == (counted <= 1024), sorted(names)
    allc = concat([b1, b2])
    R.assert_matches(got, reference([allc[0]], allc, spec), "front %d" % ngroups)


# ---- k_hash_agg_plain with a fused WHERE chain, and the interpreter fallback -----------------------------------
OPS = ["eq", "ne", "lt", "le", "gt", "ge"]


def cmp_expr(e, op, rhs):
    return {"eq": lambda: e.eq(rhs), "ne": lambda: e.not_eq(rhs), "lt": lambda: e < rhs, "le": lambda: e <= rhs,
            "gt": lambda: e > rhs, "ge": lambda: e >= rhs}[op]()


def cmp_np(x, op, y):
    return {"eq": np.equal, "ne": np.not_equal, "lt": np.less, "le": np.less_equal, "gt": np.greater, "ge": np.greater_equal}[op](x, y)


PRED_DTYPES = [(np.float64, A.FLOAT64), (np.float32, A.FLOAT32), (np.int32, A.INT32), (np.int64, A.INT64),
               (np.uint32, A.UINT32), (np.uint64, A.UINT64)]


def pred_data(rng, dt, n):
    dt = np.dtype(dt)
    if np.issubdtype(dt, np.floating):
        x = rng.integers(-8, 8, n).astype(dt) * dt.type(0.5)  # repeats: EQ / LE / GE have something to find
        return R.sprinkle(rng, x, R.edges(dt))
    return R.sprinkle(rng, rng.integers(-8, 8, n).astype(dt), R.edges(dt))


def literal_for(dt, code):
    dt = np.dtype(dt)
    if np.issubdtype(dt, np.floating):
        return -1.5, lit(-1.5, code)
    if np.issubdtype(dt, np.signedinteger):
        return -3, lit(-3, code)  # a negative literal against sign-extended column values
    return 3, lit(3, code)


@pytest.mark.parametrize("dt,code", PRED_DTYPES, ids=[np.dtype(d).name for d, _ in PRED_DTYPES])
def test_plain_fused_where_single_comparisons(ctx, dt, code):
    rng = np.random.default_rng(int(np.dtype(dt).num))
    n = 100_001
    k = keys_from(rng, key_pool(rng, np.int64, 300), n)
    v = values(rng, np.float64, n, for_sum=True)
    a, b = pred_data(rng, dt, n), pred_data(rng, dt, n)
    spec = [(R.MIN, 1), (R.MAX, 1), (R.SUM, 1), (R.COUNT, 1)]
    litv, litx = literal_for(dt, code)
    for op in OPS:
        for rhs_col in (False, True):
            pred = cmp_expr(col(2), op, col(3) if rhs_col else litx)
            m = cmp_np(a, op, b if rhs_col else np.dtype(dt).type(litv))
            got, names = run_agg(ctx, [[k, v, a, b]], [col(0)], agg_exprs(spec), pred=pred)
            assert_launched(names, "k_hash_agg_plain<4,0>")
            assert not any(x.startswith("k_hash_agg<") for x in names), sorted(names)
            R.assert_matches(got, reference([k[m]], [k[m], v[m]], spec), "%s %s col=%s" % (np.dtype(dt), op, rhs_col))


def test_plain_fused_where_chains(ctx):
    # 2 - 4 comparisons joined left to right by AND / OR: the plain kernel; 5 terms: the interpreter, same answer
    rng = np.random.default_rng(99)
    n = 200_001
    k = keys_from(rng, key_pool(rng, np.int32, 500), n)
    v = values(rng, np.float64, n, for_sum=True)
    a = pred_data(rng, np.int32, n)
    b = pred_data(rng, np.float64, n)
    spec = [(R.SUM, 1), (R.MIN, 1), (R.COUNT, 1), (R.MAX, 1)]
    for nterms in [2, 3, 4, 5, 2, 3, 4, 5]:
        expr, mask = None, None
        for t in range(nterms):
            op = OPS[rng.integers(0, 6)]
            if rng.random() < 0.5:
                e, m = cmp_expr(col(2), op, lit(int(rng.integers(-4, 4)), A.INT32)), None
                m = cmp_np(a, op, np.int32(e.right.value))
            else:
                c = float(rng.integers(-6, 6)) * 0.5
                e, m = cmp_expr(col(3), op, lit(c)), cmp_np(b, op, c)
            if expr is None:
                expr, mask = e, m
            elif rng.random() < 0.5:
                expr, mask = expr & e, mask & m
            else:
                expr, mask = expr | e, mask | m
        got, names = run_agg(ctx, [[k, v, a, b]], [col(0)], agg_exprs(spec), pred=expr)
        if nterms <= 4:
            assert_launched(names, "k_hash_agg_plain<4,0>")
        else:
            assert_launched(names, "k_hash_agg<2,0,0>")
        R.assert_matches(got, reference([k[mask]], [k[mask], v[mask]], spec), "chain %r" % expr)


# ---- k_hash_agg<DEPTH, FRONT, false>: the interpreter at every stack-depth bucket, global and front table -------
def depth_key(depth, c=0):
    """An integer expression equal to col(c) whose register stack depth is `depth` (1, 2, 4 or 8):
    col(c) + ((k - k) + ((k - k) + ...)), right-nested, keeps depth - 1 partial results on the stack."""
    if depth == 1:
        return col(c) + lit(0)
    e = col(c) - col(c)
    for _ in range(depth - 2):
        e = (col(c) - col(c)) + e
    return col(c) + e


@pytest.mark.parametrize("ngroups", [40, 700], ids=["per_warp", "per_cta"])
@pytest.mark.parametrize("depth", [1, 2, 4, 8])
def test_interpreter_depths_and_front(ctx, depth, ngroups):
    # <= 64 groups after the first batch: one front table per warp; up to 1024: one per CTA
    rng = np.random.default_rng(depth * 1000 + ngroups)
    pool = key_pool(rng, np.int64, ngroups)
    mk = lambda n: [keys_from(rng, pool, n), values(rng, F64, n, for_sum=False), values(rng, I64, n, for_sum=True)]  # noqa: E731
    b1, b2 = mk(1_100_001), mk(300_000)
    spec = [(R.MIN, 1), (R.MAX, 1), (R.SUM, 2), (R.COUNT, 1), (R.MIN, 2), (R.MAX, 2)]
    got, names = run_agg(ctx, [b1, b2], [depth_key(depth)], agg_exprs(spec))
    assert_launched(names, "k_hash_agg<%d,0,0>" % depth, "k_hash_agg<%d,1,0>" % depth)
    allc = concat([b1, b2])
    R.assert_matches(got, reference([allc[0]], allc, spec), "depth %d" % depth)
    # an expression argument (the identity col * 1.0) with a plain key: the interpreter with the global table
    spec2 = [(R.MIN, 1), (R.MAX, 1), (R.COUNT, 1)]
    got, names = run_agg(ctx, [b2], [col(0)], [AggregateFunction(f, col(1) * lit(1.0)) for f, _ in spec2])
    assert_launched(names, "k_hash_agg<1,0,0>")
    R.assert_matches(got, reference([b2[0]], b2, spec2), "expression argument")


# ---- nulls: k_hash_agg<8, false, true> and k_hash_agg_wide<8, true> ---------------------------------------------
def test_nullable_narrow_keys(ctx):
    rng = np.random.default_rng(41)
    n = 300_001
    k = keys_from(rng, key_pool(rng, np.int32, 3000), n)
    v, s, i = values(rng, F64, n, False), values(rng, F64, n, True), values(rng, I64, n, True)
    vk, vv, vs, vi = (rng.random(n) > p for p in (0.1, 0.3, 0.5, 0.2))
    arrays = [R.arrow_nullable(k, vk), R.arrow_nullable(v, vv), R.arrow_nullable(s, vs), R.arrow_nullable(i, vi)]
    spec = [(R.MIN, 1), (R.MAX, 1), (R.SUM, 2), (R.COUNT, 1), (R.COUNT, 2), (R.SUM, 3), (R.MIN, 3), (R.MAX, 3), ]
    got, names = run_agg(ctx, [arrays], [col(0)], agg_exprs(spec))
    assert_launched(names, "k_hash_agg<8,0,1>")
    cols = [(k, vk), (v, vv), (s, vs), (i, vi)]
    R.assert_matches(got, reference([k], cols, spec), "nullable")


def test_nullable_wide_keys(ctx):
    rng = np.random.default_rng(42)
    n = 300_001
    pool1 = key_pool(rng, np.int64, 60)
    k1, k2 = keys_from(rng, pool1, n), keys_from(rng, key_pool(rng, np.int64, 50), n)
    v, s = values(rng, F64, n, False), values(rng, U64, n, True)
    vk1, vv, vs = rng.random(n) > 0.1, rng.random(n) > 0.3, rng.random(n) > 0.4
    arrays = [R.arrow_nullable(k1, vk1), k2, R.arrow_nullable(v, vv), R.arrow_nullable(s, vs)]
    spec = [(R.MIN, 2), (R.MAX, 2), (R.SUM, 3), (R.COUNT, 2), (R.MIN, 3), (R.MAX, 3), (R.COUNT, 3)]
    got, names = run_agg(ctx, [arrays], [col(0), col(1)], agg_exprs(spec))
    assert_launched(names, "k_hash_agg_wide<8,1>")
    R.assert_matches(got, reference([k1, k2], [(k1, vk1), k2, (v, vv), (s, vs)], spec), "wide nullable")
    # the same without nulls: k_hash_agg_wide<8, false>
    got, names = run_agg(ctx, [[k1, k2, v, s]], [col(0), col(1)], agg_exprs(spec))
    assert_launched(names, "k_hash_agg_wide<8,0>")
    R.assert_matches(got, reference([k1, k2], [k1, k2, v, s], spec), "wide")


# ---- growth and replay: k_compact + k_merge, k_wide_move ---------------------------------------------------------
def distinct_keys(rng, dt, n):
    k = np.unique(rng.integers(np.iinfo(dt).min, np.iinfo(dt).max, int(n * 1.01) + 16, dtype=dt, endpoint=True))
    rng.shuffle(k)
    k = k[:n]
    k[:2] = [np.array(-1).astype(dt), np.iinfo(dt).min]
    return k


@pytest.mark.parametrize("hint", [0, 1_500_000], ids=["hybrid", "line"])
def test_growth_and_replay(ctx, hint):
    # more distinct keys than the initial table admits: the scan overflows, the table grows (k_compact + k_merge)
    # and the refused rows are replayed through the interpreter
    rng = np.random.default_rng(51 + hint)
    n = 2_400_001
    k = distinct_keys(rng, np.int64, 2_300_000)
    k = np.concatenate([k, k[rng.integers(0, len(k), n - len(k))]])
    v = values(rng, I64, n, for_sum=True)
    spec = [(R.MIN, 1), (R.MAX, 1), (R.COUNT, 1)]
    got, names = run_agg(ctx, [[k, v]], [col(0)], agg_exprs(spec), expected=hint)
    assert_launched(names, "k_compact", "k_merge", "k_hash_agg<1,0,0>",
                    "k_hash_agg_lean<11,3>" if hint == 0 else "k_hash_agg_plain<2,0>")
    R.assert_matches(got, reference([k], [k, v], spec), "growth")


def test_front_launch_overflow_replay(ctx):
    # the first batch shows <= 64 groups, the second brings ~2.5 M new keys: the front launch overflows the global
    # table, which grows, and the refused rows are replayed
    rng = np.random.default_rng(52)
    pool = key_pool(rng, np.int64, 40)
    b1 = [keys_from(rng, pool, 1_100_000), values(rng, I64, 1_100_000, True), values(rng, F64, 1_100_000, False)]
    k2 = distinct_keys(rng, np.int64, 2_500_000)
    b2 = [k2, values(rng, I64, len(k2), True), values(rng, F64, len(k2), False)]
    spec = [(R.MIN, 1), (R.MAX, 1), (R.SUM, 1), (R.MAX, 2), (R.MIN, 2), (R.COUNT, 2)]
    got, names = run_agg(ctx, [b1, b2], [col(0)], agg_exprs(spec))
    assert_launched(names, "k_hash_agg_plain<4,1>", "k_compact", "k_merge", "k_hash_agg<1,0,0>")
    allc = concat([b1, b2])
    R.assert_matches(got, reference([allc[0]], allc, spec), "front overflow")


def test_wide_key_growth(ctx):
    rng = np.random.default_rng(53)
    n = 2_200_000
    a = distinct_keys(rng, np.int64, n)
    b = rng.integers(-3, 3, n, dtype=np.int64)
    v = values(rng, F64, n, for_sum=False)
    spec = [(R.MIN, 2), (R.MAX, 2), (R.COUNT, 2)]
    got, names = run_agg(ctx, [[a, b, v]], [col(0), col(1)], agg_exprs(spec))
    assert_launched(names, "k_wide_move", "k_hash_agg_wide<8,0>")
    R.assert_matches(got, reference([a, b], [a, b, v], spec), "wide growth")


# ---- narrow composite keys packed into one 64-bit word -----------------------------------------------------------
@pytest.mark.parametrize("dts", [(np.int32, np.int32), (np.int16, np.int16, np.int32), (np.uint8, np.int8, np.uint16, np.int32)],
                         ids=["i32_i32", "i16_i16_i32", "u8_i8_u16_i32"])
def test_narrow_composite_keys(ctx, dts):
    rng = np.random.default_rng(len(dts))
    n = 300_001
    keys = [rng.integers(max(np.iinfo(dt).min, -40), min(np.iinfo(dt).max, 40), n, endpoint=True).astype(dt) for dt in dts]
    for kc in keys:
        kc[::97] = np.array(-1).astype(kc.dtype)  # every part all ones: the packed key is the empty marker
        kc[5::101] = np.iinfo(kc.dtype).min
        kc[7::103] = np.iinfo(kc.dtype).max
    v = values(rng, I64, n, for_sum=True)
    spec = [(R.MIN, 0), (R.MAX, 0), (R.SUM, 0), (R.COUNT, 0)]
    nk = len(dts)
    got, names = run_agg(ctx, [keys + [v]], [col(i) for i in range(nk)], [AggregateFunction(f, col(nk)) for f, _ in spec])
    assert_launched(names, "k_hash_agg_plain<4,0>" if nk == 2 else "k_hash_agg<1,0,0>")
    R.assert_matches(got, R.aggregate(keys, [(f, v) for f, _ in spec]), str(dts))


# ---- no GROUP BY: k_reduce_f64, k_reduce<DEPTH, false>, k_reduce<8, true> ------------------------------------------
REDUCE_SPEC = [(R.MIN, 0), (R.MAX, 0), (R.SUM, 0), (R.COUNT, 0)]


def reduce_inputs(rng, dt, n):
    """Columns of n rows: edge values, -0.0 before / after +0.0, and a NaN first (skipped: DESIGN §7)."""
    dt = np.dtype(dt)
    out = []
    if np.issubdtype(dt, np.floating):
        if n <= 3:
            z = np.array([-0.0, 0.0, -0.0], dtype=dt)[:n]
            out += [z.copy(), z[::-1].copy()]
        else:
            # one zero of the other sign, late in the column: it meets the rest only in the combine across CTAs
            neg, pos = np.full(n, -0.0, dtype=dt), np.full(n, 0.0, dtype=dt)
            neg[n - 5], pos[n - 7] = 0.0, -0.0
            out += [neg, pos]
        out.append(np.full(n, -0.0, dtype=dt))
        nanfirst = np.full(n, 2.5, dtype=dt)
        nanfirst[0] = np.nan
        out.append(nanfirst)
    out.append(values(rng, dt, n, for_sum=True) if n > 3 else R.edges(dt, True)[rng.integers(0, len(R.edges(dt, True)), n)])
    return out


@pytest.mark.parametrize("n", [1, 2, 3, 1_000_001])
@pytest.mark.parametrize("dt", [F64, np.float32, I64, U64, np.int32], ids=["f64", "f32", "i64", "u64", "i32"])
def test_reduce(ctx, n, dt):
    rng = np.random.default_rng(n + MT.get(np.dtype(dt), 9))
    want = "k_reduce_f64" if dt == F64 else "k_reduce<1,0>"
    for x in reduce_inputs(rng, dt, n):
        got, names = run_agg(ctx, [[x]], [], agg_exprs(REDUCE_SPEC))
        assert_launched(names, want)
        R.assert_matches(got, R.aggregate([], [(f, x) for f, _ in REDUCE_SPEC]), "reduce %s %d" % (np.dtype(dt), n))


def test_reduce_expressions_predicates_and_nulls(ctx):
    rng = np.random.default_rng(61)
    n = 700_001
    x = values(rng, F64, n, for_sum=True)
    w = pred_data(rng, np.int64, n)
    spec = [AggregateFunction(f, col(0)) for f in (R.MIN, R.MAX, R.SUM, R.COUNT)]
    # fused WHERE over a plain Float64 column: k_reduce<1, false>
    got, names = run_agg(ctx, [[x, w]], [], spec, pred=col(1) >= lit(-2))
    assert_launched(names, "k_reduce<1,0>")
    m = w >= -2
    R.assert_matches(got, R.aggregate([], [(f, x[m]) for f in (R.MIN, R.MAX, R.SUM, R.COUNT)]), "reduce where")
    # expression arguments that keep the values: x * 1.0 (not x + 0.0, which turns -0.0 into +0.0), and integer
    # identities of each stack-depth bucket over the Int64 column
    got, names = run_agg(ctx, [[x, w]], [], [AggregateFunction(f, col(0) * lit(1.0)) for f in (R.MIN, R.MAX, R.SUM, R.COUNT)])
    assert_launched(names, "k_reduce<1,0>")
    R.assert_matches(got, R.aggregate([], [(f, x) for f in (R.MIN, R.MAX, R.SUM, R.COUNT)]), "reduce expression")
    for d in (2, 4, 8):
        got, names = run_agg(ctx, [[x, w]], [], [AggregateFunction(f, depth_key(d, 1)) for f in (R.MIN, R.MAX, R.SUM)])
        assert_launched(names, "k_reduce<%d,0>" % d)
        R.assert_matches(got, R.aggregate([], [(f, w) for f in (R.MIN, R.MAX, R.SUM)]), "reduce depth %d" % d)
    # nulls: k_reduce<8, true> skips null values
    vx = rng.random(n) > 0.3
    got, names = run_agg(ctx, [[R.arrow_nullable(x, vx)]], [], spec[:4])
    assert_launched(names, "k_reduce<8,1>")
    R.assert_matches(got, R.aggregate([], [(f, (x, vx)) for f in (R.MIN, R.MAX, R.SUM, R.COUNT)]), "reduce nulls")
