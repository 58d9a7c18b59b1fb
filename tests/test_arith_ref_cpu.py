"""The exact arithmetic reference of tests/arith_ref.py, checked on its own (no GPU): against numpy where numpy's
arithmetic is exact, against a table of hand-worked results, and against the oracle's filter_project."""
import math
from fractions import Fraction

import numpy as np
import pytest

import arith_ref as AR
import oracle_lib as O
from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200.expr import col, lit

I8, I16, I32, I64 = np.int8, np.int16, np.int32, np.int64
U8, U16, U32, U64 = np.uint8, np.uint16, np.uint32, np.uint64
F32, F64 = np.float32, np.float64
NAME = {np.dtype(d): np.dtype(d).name for d in AR.NUMERIC}
NP_OP = {"+": np.add, "-": np.subtract, "*": np.multiply, "/": np.divide}
CODE = {np.dtype(d): c for d, c in zip(AR.NUMERIC, [A.INT8, A.INT16, A.INT32, A.INT64, A.UINT8, A.UINT16, A.UINT32, A.UINT64, A.FLOAT32, A.FLOAT64])}


@pytest.mark.parametrize("dt", AR.NUMERIC, ids=NAME.get)
def test_agrees_with_numpy(dt):
    # numpy's integer + - * wrap like the reference, and its IEEE + - * / are correctly rounded; numpy's integer
    # division floors, so only the quotients of operands with one sign are compared with it
    rng = np.random.default_rng(np.dtype(dt).num)
    a, b = AR.operands(rng, dt, 30_000)
    for op in AR.OPS:
        got, dbz = AR.arith(op, a, b)
        assert np.array_equal(dbz, (b == 0) & (op == "/")), op
        with np.errstate(all="ignore"):
            if AR.is_float(dt):
                fin = np.isfinite(a) & np.isfinite(b) & ~dbz
                exp = NP_OP[op](a, b)
                bad = AR.same(got[fin], exp[fin])
            elif op == "/":
                ok = ~dbz & ((a >= 0) == (b > 0))
                ok &= ~((a == np.iinfo(dt).min) & (b == -1)) if AR.is_signed(dt) else ok
                bad = AR.same(got[ok], a[ok] // b[ok])
            else:
                bad = AR.same(got, NP_OP[op](a, b))
        assert not len(bad), (op, bad[:5])


def test_float_specials_agree_with_numpy():
    # every IEEE special but a zero divisor: numpy's results, NaN compared as a class
    for dt in AR.FLOATS:
        e = AR.edges(dt)
        a, b = np.repeat(e, len(e)), np.tile(e, len(e))
        for op in AR.OPS:
            got, dbz = AR.arith(op, a, b)
            with np.errstate(all="ignore"):
                exp = NP_OP[op](a, b)
            assert not len(AR.same(got[~dbz], exp[~dbz])), (dt, op)


# (op, dtype, a, b, exact result)
KNOWN = [
    ("/", I8, -128, -1, -128), ("/", I16, -32768, -1, -32768), ("/", I32, -(2 ** 31), -1, -(2 ** 31)), ("/", I64, -(2 ** 63), -1, -(2 ** 63)),
    ("/", I32, -7, 2, -3), ("/", I32, 7, -2, -3), ("/", I32, -7, -2, 3), ("/", I64, -1, 2, 0), ("/", U64, 2 ** 64 - 1, 2, 2 ** 63 - 1),
    ("/", U8, 255, 2, 127), ("/", U32, 2 ** 31, 3, 715827882), ("/", I8, -128, 1, -128), ("/", I8, 127, -1, -127),
    ("*", U64, 2 ** 64 - 1, 2 ** 64 - 1, 1), ("*", I64, 2 ** 32 + 1, 2 ** 32 - 1, -1), ("*", I8, 16, 16, 0), ("*", I8, -128, -1, -128),
    ("*", U16, 257, 255, 65535), ("*", U32, 65537, 65537, 131073), ("*", I16, 182, 182, 33124 - 65536),
    ("+", I8, 100, 100, -56), ("+", I8, 127, 1, -128), ("+", U8, 255, 1, 0), ("-", U16, 0, 1, 65535), ("-", I32, -(2 ** 31), 1, 2 ** 31 - 1),
    ("-", U64, 0, 1, 2 ** 64 - 1), ("+", U64, 2 ** 63, 2 ** 63, 0), ("-", I64, -(2 ** 63) + 1, 2, 2 ** 63 - 1),
    # ties to even: 1 + 2^-53 and (1 + 2^-52) + 2^-53 are halfway between two doubles
    ("+", F64, 1.0, 2.0 ** -53, 1.0), ("+", F64, 1.0 + 2.0 ** -52, 2.0 ** -53, 1.0 + 2.0 ** -51), ("-", F64, 1.0, 2.0 ** -54, 1.0), ("-", F64, 1.0, 3 * 2.0 ** -54, 1.0 - 2.0 ** -52),
    ("+", F32, 1.0, 2.0 ** -24, 1.0), ("+", F32, 1.0 + 2.0 ** -23, 2.0 ** -24, 1.0 + 2.0 ** -22),
    ("*", F64, 1.0 + 2.0 ** -52, 1.5, 1.5 + 2.0 ** -51), ("*", F32, 1.0 + 2.0 ** -23, 1.5, 1.5 + 2.0 ** -22),
    # subnormal products and their ties: half the smallest subnormal rounds to 0, 1.5 of it to 2
    ("*", F64, 5e-324, 0.5, 0.0), ("*", F64, 3 * 5e-324, 0.5, 2 * 5e-324), ("*", F64, -5e-324, 0.5, -0.0),
    ("*", F64, 2.2250738585072014e-308, 0.5, 1.1125369292536007e-308), ("*", F32, 1.401298464324817e-45, 0.5, 0.0),
    ("*", F32, 3 * 1.401298464324817e-45, 0.5, 2 * 1.401298464324817e-45), ("*", F32, 1.1754943508222875e-38, 0.25, 2.938735877055719e-39),
    ("-", F32, 1.1754943508222875e-38, 1.401298464324817e-45, 1.1754942106924411e-38), ("/", F64, 5e-324, 2.0, 0.0),
    ("/", F64, 3 * 5e-324, 2.0, 2 * 5e-324),
    # overflow: MAX + half an ulp is a tie with 2^1024, which is odd-to-even -> inf; just below it stays MAX
    ("+", F64, 1.7976931348623157e308, 2.0 ** 970, math.inf), ("+", F64, 1.7976931348623157e308, 2.0 ** 970 * (1 - 2.0 ** -53), 1.7976931348623157e308),
    ("+", F32, 3.4028234663852886e38, 2.0 ** 103, math.inf), ("*", F32, 3.4028234663852886e38, 2.0, math.inf), ("*", F64, -1.7976931348623157e308, 2.0, -math.inf),
    ("/", F32, 1.0, 3.0, 0.3333333432674408), ("/", F64, 1.0, 3.0, 0.3333333333333333), ("/", F32, 2.0, 3.0, 0.6666666865348816),
    # signed zeros and the other specials
    ("+", F64, -0.0, 0.0, 0.0), ("+", F64, -0.0, -0.0, -0.0), ("-", F64, 0.0, 0.0, 0.0), ("-", F64, -0.0, 0.0, -0.0), ("-", F32, 1.0, 1.0, 0.0),
    ("*", F64, 0.0, -1.0, -0.0), ("*", F32, -0.0, -0.0, 0.0), ("/", F64, -0.0, 3.0, -0.0), ("/", F64, 1.0, -math.inf, -0.0),
    ("-", F64, math.inf, math.inf, math.nan), ("+", F32, -math.inf, math.inf, math.nan), ("*", F64, 0.0, math.inf, math.nan),
    ("/", F64, math.inf, -math.inf, math.nan), ("/", F64, -math.inf, 2.0, -math.inf), ("+", F64, math.nan, 1.0, math.nan),
]


@pytest.mark.parametrize("op,dt,a,b,want", KNOWN, ids=["%s_%s_%r_%r" % (k[1].__name__, {"+": "add", "-": "sub", "*": "mul", "/": "div"}[k[0]], k[2], k[3]) for k in KNOWN])
def test_known_results(op, dt, a, b, want):
    got = AR.scalar(op, a, b, dt)
    if isinstance(want, float) and math.isnan(want):
        assert math.isnan(got)
        return
    assert got == want and (math.copysign(1, got) == math.copysign(1, want) if isinstance(want, float) else True), (got, want)
    # the array form agrees with the scalar form
    v, dbz = AR.arith(op, np.array([a], dtype=dt), np.array([b], dtype=dt))
    assert not dbz[0] and not len(AR.same(v, np.array([want], dtype=dt)))


def test_zero_divisors():
    for dt in AR.NUMERIC:
        zeros = [0.0, -0.0] if AR.is_float(dt) else [0]
        for z in zeros:
            with pytest.raises(AR.DivideByZero):
                AR.scalar("/", 1, z, dt)
            with pytest.raises(AR.DivideByZero):
                AR.scalar("/", 0, z, dt)
        for op in "+-*":
            AR.scalar(op, 1, 0, dt)  # only division raises
    v, dbz = AR.arith("/", np.array([1.0, 2.0, 3.0]), np.array([0.0, -0.0, 2.0]))
    assert dbz.tolist() == [True, True, False] and v[2] == 1.5


def test_edge_pairs_are_what_they_say():
    for dt in AR.FLOATS:
        p = np.finfo(dt).nmant + 1
        ties = 0
        for a, b in AR._ulp_pairs(dt):
            for op in "+*":
                if math.isinf(a) or math.isinf(b) or math.isnan(a) or math.isnan(b):
                    continue
                x = Fraction(a) + Fraction(b) if op == "+" else Fraction(a) * Fraction(b)
                r = AR.scalar(op, a, b, dt)
                if x == 0 or abs(r) >= float(np.finfo(dt).max) or Fraction(r) == x:
                    continue
                other = float(np.nextafter(dt(r), dt(-np.inf) if Fraction(r) > x else dt(np.inf)))
                if math.isinf(other):
                    continue
                lo, hi = sorted([Fraction(r), Fraction(other)])
                if x - lo == hi - x:  # a tie: the even significand won
                    ties += 1
                    assert int(np.array(r, dtype=dt).view(AR._UINT[np.dtype(dt).itemsize])) % 2 == 0, (a, b, op)
        assert ties >= 8, (dt, ties, p)
        # an exact overflow tie and a sum just below it
        mx = float(np.finfo(dt).max)
        assert AR.scalar("+", mx, 2.0 ** (np.finfo(dt).maxexp - 1 - p), dt) == math.inf
        assert AR.scalar("+", mx, float(np.nextafter(dt(2.0 ** (np.finfo(dt).maxexp - 1 - p)), dt(0))), dt) == mx


@pytest.mark.parametrize("dt", AR.NUMERIC, ids=NAME.get)
def test_operands_cover_the_edges(dt):
    rng = np.random.default_rng(1)
    a, b = AR.operands(rng, dt, 20_000)
    u = AR._UINT[np.dtype(dt).itemsize]
    pairs = set(zip(a.view(u).tolist(), b.view(u).tolist()))
    e = AR.edges(dt).view(u).tolist()
    assert all((x, y) in pairs for x in e for y in e)
    if not AR.is_float(dt):
        lo, hi = AR.int_bounds(dt)
        assert {lo, hi, 0, 1, hi - 1, lo + 1} <= set(AR.edges(dt).tolist())
        if AR.is_signed(dt):
            assert -1 in set(AR.edges(dt).tolist())


@pytest.mark.parametrize("dt", AR.NUMERIC, ids=NAME.get)
def test_oracle_agrees(dt):
    # the oracle's filter_project (no WHERE, so every dtype is projected) over the generator's rows, all four operators;
    # the oracle refuses a zero divisor in any row, so division runs with the zero divisors replaced by 1
    rng = np.random.default_rng(7 + np.dtype(dt).num)
    a, b = AR.operands(rng, dt, 40_000)
    b1 = np.where(b == 0, dt(1), b).astype(dt)
    x, y = AR.operands(rng, dt, 3)
    lv = x[0].item() if AR.is_float(dt) else int(x[0])
    for op in AR.OPS:
        bb = b1 if op == "/" else b
        lhs = lambda e, r: {"+": e + r, "-": e - r, "*": e * r, "/": e / r}[op]  # noqa: E731
        lit1 = lit(lv if lv != 0 or op != "/" else 1, CODE[np.dtype(dt)])
        exprs = [lhs(col(0), col(1)), lhs(col(0), lit1), lhs(lit(int(y[0]) if not AR.is_float(dt) else y[0].item(), CODE[np.dtype(dt)]), col(1))]
        got = O.filter_project([a, bb], None, exprs)
        ref = [AR.value(op, a, bb), AR.value(op, a, np.dtype(dt).type(lit1.value)), AR.value(op, np.dtype(dt).type(y[0]), bb)]
        for g, e, what in zip(got, ref, ("a op b", "a op lit", "lit op b")):
            bad = AR.same(g, e)
            assert not len(bad), (op, what, bad[:5], g[bad[:5]], e[bad[:5]])
