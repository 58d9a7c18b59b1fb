"""The reference evaluator of tests/expr_ref.py and the full-language generator of tests/fuzz_exprs.py, without a GPU:
the evaluator against the CPU oracle on the oracle's subset of the language (every null profile, with and without a
WHERE), its numpy shortcuts against the exact arithmetic and CAST references, the worked examples of DESIGN §7, and the
generator's programs (they type-check, every node kind and operator occurs, a stated share reaches stack depth 6, and
some CASEs keep a division by zero in a branch not taken)."""
import numpy as np
import pyarrow as pa
import pytest

import arith_ref
import cast_ref
import expr_ref as R
import fuzz_exprs as F
from groupby_ref import arrow_nullable
import oracle_lib as O
from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import engine
from datafusion_archive_b200.expr import BinaryExpr, Case, Cast, ScalarFunction, Utf8Function, case, col, fn, lit, utf8_fn


def unpack(c):
    if isinstance(c, tuple):
        return np.asarray(c[0]), np.asarray(c[1], dtype=bool)
    return np.asarray(c), np.ones(len(c), dtype=bool)


def assert_same_column(got, exp, what):
    """got: (values, valid) of the engine or oracle; exp: an expr_ref.Value over the kept rows.  Validity equal, valid
    values bit for bit (NaNs as a class)."""
    gv, gm = got
    assert np.array_equal(gm, exp.valid), (what, "validity", np.flatnonzero(gm != exp.valid)[:8])
    ev = np.asarray(exp.values)
    if ev.dtype == np.bool_ or gv.dtype == np.bool_:
        assert np.array_equal(gv[gm].astype(bool), ev[gm].astype(bool)), (what, "values")
        return
    bad = cast_ref.same(gv[gm], ev[gm].astype(gv.dtype))
    assert not len(bad), (what, "values", bad[:8], gv[gm][bad[:8]], ev[gm][bad[:8]])


def rows_of(v, keep):
    return R.Value(v.values[keep], v.valid[keep], v.err[keep])


@pytest.mark.parametrize("profile", F.PROFILES)
def test_reference_matches_the_oracle_on_its_subset(profile):
    """gen_fp_query's queries (the oracle's subset: + - * /, comparisons, And / Or, the oracle's CASTs) over gen_table's
    nullable columns with garbage under their nulls: the reference gives the oracle's rows, values and validity bit for
    bit, and raises exactly where the oracle does."""
    rng = np.random.default_rng(list(F.PROFILES).index(profile) + 100)
    t = F.gen_table(rng, 2_000, profiles=profile, surviving_zero=True)
    T = R.Table(t.arrays)
    compared = raised = 0
    for q in range(80):
        pred, proj = F.gen_fp_query(rng, t, with_pred=q % 3 != 0)
        bad, keep = R.raises(T, pred, proj)
        try:
            exp = O.rows(t.arrays, pred, proj)
        except O.OracleError as e:
            assert "DivideByZero" in e.msg and bad, (q, pred, proj, e.msg)
            raised += 1
            continue
        assert not bad, (q, pred, proj)
        for i, e in enumerate(proj):
            assert_same_column(unpack(exp[i]), rows_of(R.evaluate(e, T, pred is None), keep), (profile, q, i, pred, e))
        compared += 1
    assert compared >= 60, (compared, raised)


def test_float_shortcuts_match_the_exact_references():
    """expr_ref's numpy float arithmetic and float-to-float CAST equal arith_ref / cast_ref over their edge operands."""
    rng = np.random.default_rng(7)
    for dt in (np.float32, np.float64):
        a, b = arith_ref.operands(rng, dt, 6_000)
        for op in arith_ref.OPS:
            gv, gbad = R.arith(op, a, b)
            ev, ebad = arith_ref.arith(op, a, b)
            assert np.array_equal(gbad, ebad), (dt, op)
            assert not len(cast_ref.same(gv, ev)), (dt, op)
    for src, dst in ((np.float64, np.float32), (np.float32, np.float64)):
        x = cast_ref.fill(rng, src, dst, 4_000)
        assert not len(cast_ref.same(R.cast(x, dst), cast_ref.cast(x, dst))), (src, dst)


# ---- DESIGN §7, worked by hand ---------------------------------------------------------------------------------------
def table():
    x = np.array([10, 7, -9, 4, 0], dtype=np.int64)
    y = pa.array(np.array([2, 0, 3, 0, 5], dtype=np.int64), mask=np.array([0, 0, 0, 1, 0], bool))  # row 3: null over 0
    f = np.array([-0.0, 0.0, 2.5, -3.0, np.nan])
    s = pa.array([b"abc", None, b"", b"\xc3\xa9t\xc3\xa9", b"a\0b"], type=pa.binary())
    return [x, y, f, s]


def test_guarded_division_never_raises_and_a_where_reads_every_row():
    t = table()
    e = case([(col(1).not_eq(lit(0)), col(0) / col(1))], lit(0))
    v = R.evaluate(e, t)
    assert not v.err.any()
    # row 3: `null <> 0` is true (a comparison orders the null), and `x / null` is null
    assert v.values.tolist() == [5, 0, -3, 0, 0] and v.valid.tolist() == [True, True, True, False, True]
    assert not R.evaluate(e, t, read_bitmaps=False).err.any()
    # WHERE y <> 0 AND x / y > 1: the WHERE reads every row, so the zero divisor of row 1 raises
    pred = col(1).not_eq(lit(0)) & (col(0) / col(1) > lit(1))
    assert R.raises(t, pred, [col(0)])[0]
    # a projection's zero divisor raises only in rows the WHERE keeps
    bad, keep = R.raises(t, col(0) > lit(5), [col(0) / col(1)])
    assert bad and keep.tolist() == [True, True, False, False, False]
    assert not R.raises(t, col(0) > lit(8), [col(0) / col(1)])[0]
    # under a WHERE the 0 stored under row 3's null is divided like any other value
    assert R.raises(t, col(0).eq(lit(4)), [col(0) / col(1)])[0]


def test_case_conditions_and_validity():
    t = table()
    # a null condition is not taken (comparisons never give a null: this condition is a CASE-made one)
    cond = case([(col(0) > lit(5), col(0) > lit(0))])
    assert R.evaluate(cond, t).valid.tolist() == [True, True, False, False, False]
    v = R.evaluate(case([(cond, lit(1))], lit(2)), t)
    assert v.values.tolist() == [1, 1, 2, 2, 2] and v.valid.all()
    # without ELSE a row where no WHEN is taken is null with value 0; a select takes the chosen branch's validity
    v = R.evaluate(case([(col(0) > lit(5), col(1))]), t)
    assert v.valid.tolist() == [True, True, False, False, False] and v.values.tolist() == [2, 0, 0, 0, 0]
    v = R.evaluate(case([(col(0) < lit(5), col(1))], lit(9)), t)
    assert v.valid.tolist() == [True, True, True, False, True] and v.values.tolist() == [9, 9, 3, 0, 5]
    # under a WHERE the input bitmap is dropped: row 3 reads its stored 0
    v = R.evaluate(case([(col(0) < lit(5), col(1))], lit(9)), t, read_bitmaps=False)
    assert v.valid.all() and v.values.tolist() == [9, 9, 3, 0, 5]
    # a CASE that selects a null passes the value stored under it through; only a CASE-made null is 0
    stored = arrow_nullable(np.array([7, 8], np.int64), np.array([False, True]))
    v = R.evaluate(case([(col(0).eq(col(0)), col(0))], lit(1)), [stored])  # null = null is true
    assert v.valid.tolist() == [False, True] and v.values.tolist() == [7, 8]
    # DivideByZero only from the conditions up to the first true one and the value chosen
    e = case([(col(0) > lit(5), lit(1)), (col(0) / col(1) > lit(0), lit(2))], lit(100) / col(1))
    assert R.evaluate(e, t).err.tolist() == [False, False, False, False, False]
    e = case([(col(0) > lit(8), lit(1)), (col(0) / col(1) > lit(0), lit(2))], lit(3))
    assert R.evaluate(e, t).err.tolist() == [False, True, False, False, False]


def test_functions_and_utf8():
    t = table()
    assert R.evaluate(fn("signum", col(2)), t).values[:2].tolist() == [-1.0, 1.0]  # signum(-0.0) = -1
    v = R.evaluate(fn("round", lit(-0.4)), [np.zeros(1)]).values
    assert np.signbit(v[0]) and v[0] == 0
    like = R.evaluate(col(3).like(lit(b"%")), t)
    assert like.values.tolist() == [True, False, True, True, True] and like.valid.all()  # LIKE on a null is false
    assert R.evaluate(col(3).not_like(lit(b"%")), t).values.tolist() == [False] * 5
    assert R.evaluate(col(3).like(lit(b"_t_")), t).values.tolist() == [False, False, False, True, False]  # é is one character
    # substr with start <= 0: the characters at [start, start + count) clipped to [1, n]
    sub = R.evaluate(utf8_fn("substr", col(3), lit(0, A.INT64), lit(2, A.INT64)), t)
    assert sub.values.tolist() == [b"a", b"", b"", b"\xc3\xa9", b"a"] and sub.valid.tolist() == [True, False, True, True, True]
    assert R.evaluate(utf8_fn("substr", col(3), lit(-1, A.INT64), lit(2, A.INT64)), t).values.tolist() == [b""] * 5
    n = R.evaluate(utf8_fn("length", col(3)), t)
    assert n.values.tolist() == [3, 0, 0, 3, 3] and n.valid.tolist() == [True, False, True, True, True]
    assert R.evaluate(utf8_fn("length", col(3)), t, read_bitmaps=False).valid.all()
    # null ordering: a numeric `<` is true when the left side is null; Utf8 orders a null below every string
    lt = R.evaluate(col(1) < lit(-1000), t)
    assert lt.values.tolist() == [False, False, False, True, False] and lt.valid.all()
    assert R.evaluate(lit(-1000) < col(1), t).values.tolist() == [True, True, True, False, True]
    assert R.evaluate(col(3) < lit(b""), t).values.tolist() == [False, True, False, False, False]
    assert R.evaluate(col(3).eq(col(3)), t).values.all()
    assert R.evaluate(lit(b"a") <= col(3), t).values.tolist() == [True, False, False, True, True]


# ---- the generator ---------------------------------------------------------------------------------------------------
def kinds(e, schema, out):
    """Every (kind, detail) in e: operators, function names, CAST pairs, CASE shapes."""
    if isinstance(e, BinaryExpr):
        out.add(("op", e.op))
        kinds(e.left, schema, out)
        kinds(e.right, schema, out)
    elif isinstance(e, Cast):
        out.add(("cast_to", e.dtype))
        out.add(("cast_from", e.expr.get_type(schema)))
        kinds(e.expr, schema, out)
    elif isinstance(e, ScalarFunction):
        out.add(("fn", R.FN_NAME[e.code]))
        for a in e.args:
            kinds(a, schema, out)
    elif isinstance(e, Utf8Function):
        out.add(("utf8_fn", e.code))
        kinds(e.args[0], schema, out)
    elif isinstance(e, Case):
        out.add(("case", (len(e.whens), e.else_ is not None)))
        for c, v in e.whens:
            kinds(c, schema, out)
            kinds(v, schema, out)
        if e.else_ is not None:
            kinds(e.else_, schema, out)


def lazy_division(e, T, rb):
    """Whether some CASE in e holds a division whose zero divisor sits only in rows where its branch is not taken."""
    if isinstance(e, Case):
        for _, v in e.whens:
            if isinstance(v, BinaryExpr) and v.op == A.OP_DIV:
                inner = R.evaluate(v, T, rb).err
                if inner.any() and not (R.evaluate(e, T, rb).err & inner).all():
                    return True
        return any(lazy_division(x, T, rb) for w in e.whens for x in w) or (e.else_ is not None and lazy_division(e.else_, T, rb))
    if isinstance(e, BinaryExpr):
        return lazy_division(e.left, T, rb) or lazy_division(e.right, T, rb)
    if isinstance(e, (Cast,)):
        return lazy_division(e.expr, T, rb)
    if isinstance(e, ScalarFunction):
        return any(lazy_division(a, T, rb) for a in e.args)
    return False


def test_full_generator():
    rng = np.random.default_rng(2026)
    n = 1_500
    t = F.gen_table(rng, n)
    F.add_strings(rng, t, n)
    kc = F.add_keys(rng, t, [A.INT32, A.INT64], n)
    T = R.Table(t.arrays)
    seen, found, deep, lazy, raising, total = set(), set(), 0, 0, 0, 0
    queries = [F.gen_fp_query(rng, t, with_pred=q % 2 == 0, full=True, seen=seen) for q in range(160)]
    for q in range(40):
        pred, keys, aggs = F.gen_agg_query(rng, t, kc[:1 + q % 2], q % 2 == 0, False, True, full=True, seen=seen)
        queries.append((pred, keys + [a.arg for a in aggs]))
    for pred, exprs in queries:
        progs = exprs + ([pred] if pred is not None else [])
        for e in progs:
            engine.check_program(t.dtype, e)  # raises as the operators would
            kinds(e, t.dtype, found)
        total += 1
        deep += max(R.stack_depth(e, t.dtype) for e in progs) >= 6
        lazy += any(lazy_division(e, T, pred is None) for e in exprs)
        raising += R.raises(T, pred, exprs)[0]
    assert seen == set(F.FULL_KINDS) | {"bool_case", "nested_case", "deep"}, seen
    ops = {d for k, d in found if k == "op"}
    assert ops == set(R.CMP) | set(R.MATH) | {A.OP_AND, A.OP_OR, A.OP_LIKE, A.OP_NOT_LIKE}, ops
    assert {d for k, d in found if k == "fn"} == set(F.EXACT_FNS) | set(F.TRANSCENDENTAL)
    assert {d for k, d in found if k == "utf8_fn"} == {A.UTF8FN_UPPER, A.UTF8FN_LOWER, A.UTF8FN_TRIM, A.UTF8FN_LTRIM, A.UTF8FN_RTRIM,
                                                       A.UTF8FN_SUBSTR, A.UTF8FN_SUBSTR_FROM, A.UTF8FN_LENGTH, A.UTF8FN_OCTET_LENGTH}
    assert {d for k, d in found if k == "cast_to"} >= set(F.NUMERIC) and {d for k, d in found if k == "cast_from"} >= set(F.NUMERIC)
    shapes = {d for k, d in found if k == "case"}
    assert shapes >= {(w, e) for w in (1, 2, 3, 4) for e in (False, True)}, shapes
    # at least a quarter of the queries reach stack depth 6 (the spilled entries of the extended interpreter)
    assert deep >= total // 4, (deep, total)
    assert lazy >= 5 and 3 <= raising <= total // 3, (lazy, raising, total)


def test_generator_default_is_the_oracle_subset():
    """Without full=True the generator makes only what the oracle implements, as before."""
    rng = np.random.default_rng(3)
    t = F.gen_table(rng, 500)
    found = set()
    for q in range(100):
        pred, proj = F.gen_fp_query(rng, t, with_pred=q % 2 == 0)
        for e in proj + ([pred] if pred is not None else []):
            kinds(e, t.dtype, found)
    assert not {k for k, _ in found} & {"fn", "utf8_fn", "case"}
    assert {d for k, d in found if k == "cast_to"} <= {A.INT16, A.INT32, A.FLOAT64}
