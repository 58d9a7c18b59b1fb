"""The exact Rust `as` reference of tests/cast_ref.py, checked on its own (no GPU): against a table of known Rust
results, against numpy where numpy's conversion is exact, and against the oracle's cast_column (-> Int16 / Int32)."""
import math
from fractions import Fraction

import numpy as np
import pytest

import cast_ref as CR

I8, I16, I32, I64 = np.int8, np.int16, np.int32, np.int64
U8, U16, U32, U64 = np.uint8, np.uint16, np.uint32, np.uint64
F32, F64 = np.float32, np.float64
NAN, INF = math.nan, math.inf

# (value, source, target, Rust `value as target`)
KNOWN = [
    (300, I64, U8, 44), (-1, I8, U64, 2 ** 64 - 1), (-1, I64, U32, 2 ** 32 - 1), (200, U8, I8, -56), (2 ** 63, U64, I64, -(2 ** 63)),
    (2 ** 64 - 1, U64, I64, -1), (-129, I16, I8, 127), (65536 + 7, I32, U16, 7), (-(2 ** 31), I32, U64, 2 ** 64 - 2 ** 31),
    (NAN, F64, I32, 0), (NAN, F32, U64, 0), (NAN, F64, I64, 0), (INF, F64, I8, 127), (-INF, F64, I8, -128), (INF, F32, U64, 2 ** 64 - 1),
    (-INF, F64, U16, 0), (1e300, F64, U64, 2 ** 64 - 1), (-1e300, F64, I64, -(2 ** 63)), (-0.9, F64, U8, 0), (-0.0, F64, U32, 0),
    (-0.7, F32, U64, 0), (-0.7, F64, I8, 0), (255.9, F64, U8, 255), (256.0, F64, U8, 255), (-128.9, F64, I8, -128), (-129.0, F64, I8, -128),
    (127.9, F64, I8, 127), (2147483647.5, F64, I32, 2147483647), (-2147483648.5, F64, I32, -2147483648), (2147483648.0, F64, I32, 2147483647),
    (9.223372036854775e18, F64, I64, 9223372036854774784), (9223372036854775808.0, F64, I64, 2 ** 63 - 1),
    (18446744073709549568.0, F64, U64, 18446744073709549568), (18446744073709551616.0, F64, U64, 2 ** 64 - 1), (-1.0, F64, U64, 0),
    (-1.0, F64, I64, -1), (4294967295.9, F64, U32, 4294967295), (-2.5, F64, I16, -2), (2.5, F32, I16, 2),
    (16777217, I32, F32, 16777216.0), (16777219, I32, F32, 16777220.0), (2 ** 64 - 1, U64, F32, 1.8446744073709552e19),
    (2 ** 64 - 1, U64, F64, 1.8446744073709552e19), (2 ** 63 + 1, U64, F64, 9.223372036854775808e18), (2 ** 53 + 1, I64, F64, 9007199254740992.0),
    (2 ** 53 + 3, I64, F64, 9007199254740996.0), (-(2 ** 63), I64, F32, -9.223372036854775808e18),
    ((1 << 60) + (1 << 36) + 1, I64, F32, 1.1529216420458004e18), ((1 << 63) + (1 << 39) + 1, U64, F32, 9.223373136366404e18),
    # Float32 max + half an ulp is a tie between an odd significand and 2^128: it rounds to inf; just below, to the max
    (1e300, F64, F32, INF), (-1e300, F64, F32, -INF), (3.4028235677973366e38, F64, F32, INF),
    (3.4028235677973362e38, F64, F32, 3.4028234663852886e38), (-3.4028235677973362e38, F64, F32, -3.4028234663852886e38), (1e-46, F64, F32, 0.0), (-1e-46, F64, F32, -0.0),
    (1e-45, F64, F32, 1.401298464324817e-45), (1.0000000596046448, F64, F32, 1.0), (1.0000000596046450, F64, F32, 1.0000001192092896),
    (0.1, F64, F32, 0.10000000149011612), (0.1, F32, F64, 0.10000000149011612), (NAN, F64, F32, NAN), (-0.0, F64, F32, -0.0),
]


@pytest.mark.parametrize("v,src,dst,want", KNOWN, ids=["%r_%s_as_%s" % (k[0], np.dtype(k[1]).name, np.dtype(k[2]).name) for k in KNOWN])
def test_known_rust_results(v, src, dst, want):
    if CR.is_float(src):
        v = float(np.dtype(src).type(v))
    got = CR.cast_scalar(v, src, dst)
    if isinstance(want, float) and math.isnan(want):
        assert math.isnan(got)
        return
    assert got == want and type(got) is type(want), (got, want)
    if isinstance(want, float) and want == 0:
        assert math.copysign(1, got) == math.copysign(1, want)
    # the array form agrees with the scalar form
    arr = np.array([v], dtype=src)
    assert not len(CR.same(CR.cast(arr, dst), np.array([want], dtype=dst)))


def test_double_rounding_integers_round_once():
    # the correctly rounded Float32 of each differs from rounding through Float64 first, which leaves an exact tie
    for i in CR.DOUBLE_ROUNDING:
        direct = CR.cast_scalar(i, I64 if i < 2 ** 63 else U64, F32)
        via = float(np.float32(float(i)))
        assert direct != via and abs(int(direct) - i) < abs(int(via) - i), (i, direct, via)


@pytest.mark.parametrize("dst", CR.FLOATS, ids=["f32", "f64"])
def test_int_to_float_is_correctly_rounded(dst):
    # nearest by exhaustive comparison with both neighbours, ties to the even significand
    rng = np.random.default_rng(3)
    xs = [int(x) for x in rng.integers(-(2 ** 63), 2 ** 63 - 1, 2000, dtype=np.int64)] + [2 ** 64 - 1 - k for k in range(50)]
    t = np.dtype(dst).type
    for x in xs:
        f = CR.cast_scalar(x, U64 if x >= 2 ** 63 else I64, dst)
        lo, hi = float(np.nextafter(t(f), t(-np.inf))), float(np.nextafter(t(f), t(np.inf)))
        d = abs(Fraction(f) - x)
        assert d <= abs(Fraction(lo) - x) and (math.isinf(hi) or d <= abs(Fraction(hi) - x)), x
        if d == abs(Fraction(lo) - x) or (not math.isinf(hi) and d == abs(Fraction(hi) - x)):
            assert int(np.array(f, dtype=dst).view(CR._UINT[np.dtype(dst).itemsize])) % 2 == 0, x


@pytest.mark.parametrize("src", CR.INTS, ids=lambda d: np.dtype(d).name)
def test_int_to_int_agrees_with_numpy(src):
    rng = np.random.default_rng(np.dtype(src).num)
    for dst in CR.INTS:
        x = CR.fill(rng, src, dst, 20_000)
        assert not len(CR.same(CR.cast(x, dst), x.astype(dst))), (src, dst)


def test_f32_to_f64_agrees_with_numpy():
    rng = np.random.default_rng(5)
    x = CR.fill(rng, F32, F64, 20_000)
    bits = rng.integers(0, 2 ** 32, 5000, dtype=np.uint64).astype(np.uint32).view(F32)  # every class of Float32, NaNs included
    x = np.concatenate([x, bits])
    with np.errstate(invalid="ignore"):
        assert not len(CR.same(CR.cast(x, F64), x.astype(F64)))


def test_f64_to_f32_agrees_with_numpy_on_normal_values():
    # numpy's double -> float is the C conversion, correctly rounded under the default rounding mode
    rng = np.random.default_rng(6)
    x = np.concatenate([CR.fill(rng, F64, F32, 20_000), rng.standard_normal(5000) * 10.0 ** rng.integers(-40, 40, 5000)])
    with np.errstate(over="ignore"):
        assert not len(CR.same(CR.cast(x, F32), x.astype(F32)))


@pytest.mark.parametrize("src", CR.NUMERIC, ids=lambda d: np.dtype(d).name)
@pytest.mark.parametrize("dst", CR.NUMERIC, ids=lambda d: np.dtype(d).name)
def test_edges_cover_the_bounds(src, dst):
    e = CR.edges(src, dst)
    assert e.dtype == np.dtype(src) and len(e) >= 8
    vals = set(e.tolist()) if not CR.is_float(src) else None
    if CR.is_float(dst):
        if CR.is_float(src):
            assert np.isnan(e).any() and np.isinf(e).any() and (e == 0).sum() == 2
        return
    lo, hi = CR.int_bounds(dst)
    if not CR.is_float(src):
        slo, shi = CR.int_bounds(src)
        for b in (lo - 1, lo, hi, hi + 1):
            if slo <= b <= shi:
                assert b in vals, (b, src, dst)
    else:
        assert np.isnan(e).any() and np.isinf(e).any() and np.signbit(e[e == 0]).any()
        assert (e == np.dtype(src).type(float(hi) + 1)).any() or float(np.dtype(src).type(hi)) != hi


@pytest.mark.parametrize("src", CR.NUMERIC, ids=lambda d: np.dtype(d).name)
def test_agrees_with_oracle_cast_column(src):
    # the reference implements CAST(column) to Int16 and Int32 only; over every edge value of the pair
    import oracle_lib as O
    from datafusion_archive_b200.expr import col
    rng = np.random.default_rng(11)
    for dst in (I16, I32):
        x = np.concatenate([CR.edges(src, dst), CR.fill(rng, src, dst, 3000)])
        got = O.filter_project([x], None, [col(0).cast(CR.CODE[np.dtype(dst)])])[0]
        bad = CR.same(got, CR.cast(x, dst))
        assert not len(bad), (src, dst, x[bad[:5]], got[bad[:5]])


def test_planner_coercion_helper_matches_the_planner():
    # cast_ref.coerce predicts, for every pair of column types, whether the planner plans `a + b` and which operands
    # it casts; the planner's own plan text is the check
    from datafusion_archive_b200 import host
    host.build()
    c = host.Catalog()
    names = {np.dtype(d): "c_" + np.dtype(d).name for d in CR.NUMERIC}
    c.add_table("t", [(names[np.dtype(d)], CR.CODE[np.dtype(d)]) for d in CR.NUMERIC])
    idx = {np.dtype(d): i for i, d in enumerate(CR.NUMERIC)}
    for a in CR.NUMERIC:
        for b in CR.NUMERIC:
            st = host.supertype(CR.CODE[np.dtype(a)], CR.CODE[np.dtype(b)])
            sql = "SELECT %s + %s FROM t" % (names[np.dtype(a)], names[np.dtype(b)])
            one = np.zeros(1, dtype=a), np.zeros(1, dtype=b)
            if st is None:
                with pytest.raises(host.ExecutionError) as e:
                    c.plan(sql)
                assert "No common supertype" in e.value.msg
                continue
            want = CR.coerce(one[0], one[1], CR.DTYPE[st])
            if want is None:
                with pytest.raises(host.ExecutionError) as e:
                    c.plan(sql)
                assert "Cannot automatically convert" in e.value.msg, (a, b, e.value.msg)
                continue
            side = lambda d: "#%d" % idx[np.dtype(d)] if np.dtype(d) == CR.DTYPE[st] else "CAST(#%d AS %s)" % (  # noqa: E731
                idx[np.dtype(d)], {v: k for k, v in _DEBUG.items()}[st])
            assert c.plan(sql).splitlines()[0] == "Projection: %s Plus %s" % (side(a), side(b)), (a, b)


_DEBUG = {"Int8": CR.CODE[np.dtype(I8)], "Int16": CR.CODE[np.dtype(I16)], "Int32": CR.CODE[np.dtype(I32)], "Int64": CR.CODE[np.dtype(I64)],
          "UInt8": CR.CODE[np.dtype(U8)], "UInt16": CR.CODE[np.dtype(U16)], "UInt32": CR.CODE[np.dtype(U32)],
          "UInt64": CR.CODE[np.dtype(U64)], "Float32": CR.CODE[np.dtype(F32)], "Float64": CR.CODE[np.dtype(F64)]}
