"""Exact reference of Rust `as` between the ten numeric dtypes, and of the SQL planner's implicit coercions.

Computed over Python ints and `fractions.Fraction`, never through a numpy conversion whose rounding path is
unspecified:
* float -> int: NaN -> 0; otherwise truncate toward zero and saturate to [MIN, MAX] of the target, so ±inf give the
  extremes and -0.0 / -0.7 give 0 for every target, unsigned ones included;
* int -> int: wrap modulo 2^width and reinterpret in the target's signedness;
* int -> float and Float64 -> Float32: one correctly rounded step from the exact value, round-half-to-even, with
  overflow to ±inf and subnormal results (never through a double for Float32);
* Float32 -> Float64 is exact; NaN stays NaN (compare NaNs as a class, not by payload).
"""
import math
from fractions import Fraction

import numpy as np

from datafusion_archive_b200 import _abi as A

INTS = [np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64]
FLOATS = [np.float32, np.float64]
NUMERIC = INTS + FLOATS
CODE = {np.dtype(np.int8): A.INT8, np.dtype(np.int16): A.INT16, np.dtype(np.int32): A.INT32, np.dtype(np.int64): A.INT64,
        np.dtype(np.uint8): A.UINT8, np.dtype(np.uint16): A.UINT16, np.dtype(np.uint32): A.UINT32, np.dtype(np.uint64): A.UINT64,
        np.dtype(np.float32): A.FLOAT32, np.dtype(np.float64): A.FLOAT64}
DTYPE = {v: k for k, v in CODE.items()}
# (significand bits, minimum normal exponent, maximum exponent) of the IEEE binary formats
_FMT = {np.dtype(np.float32): (24, -126, 127), np.dtype(np.float64): (53, -1022, 1023)}
_UINT = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}


def is_float(dt):
    return np.dtype(dt).kind == "f"


def is_signed(dt):
    return np.dtype(dt).kind == "i"


def int_bounds(dt):
    info = np.iinfo(dt)
    return int(info.min), int(info.max)


def round_float(x, dt):
    """The value of dtype dt (Float32 / Float64) nearest to the exact rational x, ties to even; ±inf past the largest
    finite value, subnormals below the smallest normal.  A zero keeps the sign of x (-0.0 for a negative x that rounds
    to zero).  Returned as a Python float, which holds every Float32 value exactly."""
    p, emin, emax = _FMT[np.dtype(dt)]
    x = Fraction(x)
    if x == 0:
        return 0.0
    neg, a = x < 0, abs(x)
    e = a.numerator.bit_length() - a.denominator.bit_length()  # 2^e <= a < 2^(e+2)
    if Fraction(2) ** e > a:
        e -= 1
    if Fraction(2) ** (e + 1) <= a:
        e += 1
    e = max(e, emin)  # below the normal range the quantum stays 2^(emin - p + 1)
    q = Fraction(2) ** (e - p + 1)
    m = a / q
    n = m.numerator // m.denominator
    r = m - n
    if r > Fraction(1, 2) or (r == Fraction(1, 2) and n % 2 == 1):
        n += 1
    v = n * q
    if v >= Fraction(2) ** (emax + 1):
        return -math.inf if neg else math.inf
    f = float(v)  # exact: v has at most p significant bits and lies in the Float64 range
    return -f if neg else f


def cast_scalar(v, src, dst):
    """Rust `v as dst` for one value v of dtype src (a Python int / float, or a numpy scalar).  Returns a Python int
    for an integer target and a Python float (the exact value of the target dtype) for a float target."""
    src, dst = np.dtype(src), np.dtype(dst)
    if is_float(src):
        x = float(v)
        if is_float(dst):
            if math.isnan(x) or math.isinf(x) or x == 0 or src == dst or dst == np.dtype(np.float64):
                return x  # Float32 -> Float64 is exact
            return round_float(Fraction(x), dst)
        if math.isnan(x):
            return 0
        lo, hi = int_bounds(dst)
        if math.isinf(x):
            return hi if x > 0 else lo
        return min(hi, max(lo, math.trunc(x)))
    i = int(v)
    if is_float(dst):
        return round_float(i, dst)
    bits = 8 * dst.itemsize
    w = i % (1 << bits)
    return w - (1 << bits) if is_signed(dst) and w >= 1 << (bits - 1) else w


def cast(values, dst):
    """Rust `as` over a numpy array, exactly: the reference is computed once per distinct bit pattern."""
    values = np.asarray(values)
    src, dst = values.dtype, np.dtype(dst)
    if len(values) == 0:
        return np.zeros(0, dtype=dst)
    bits = values.view(_UINT[src.itemsize])
    u, inv = np.unique(bits, return_inverse=True)
    keys = u.view(src)
    out = np.array([cast_scalar(k, src, dst) for k in keys.tolist()], dtype=object)
    res = np.array(out.tolist(), dtype=dst) if is_float(dst) else np.array([int(x) for x in out], dtype=dst)
    return res[inv.reshape(-1)]


def same(got, exp):
    """Bit-for-bit equality, with NaNs compared as a class.  Returns the indices that differ."""
    got, exp = np.asarray(got), np.asarray(exp)
    assert got.dtype == exp.dtype and got.shape == exp.shape, (got.dtype, exp.dtype, got.shape, exp.shape)
    if is_float(got.dtype):
        gn, en = np.isnan(got), np.isnan(exp)
        diff = (gn != en) | (~en & (got.view(_UINT[got.dtype.itemsize]) != exp.view(_UINT[exp.dtype.itemsize])))
    else:
        diff = got != exp
    return np.flatnonzero(diff)


# ---- edge values --------------------------------------------------------------------------------------------------
def _representable(x, src):
    """x (a Python int / float) as a value of src, or None when src cannot hold it exactly."""
    src = np.dtype(src)
    if is_float(src):
        if isinstance(x, float):
            if math.isnan(x) or math.isinf(x):
                return x
            return x if round_float(Fraction(x), src) == x else None
        f = round_float(x, src)
        return f if not math.isinf(f) and Fraction(f) == x else None
    if isinstance(x, float):
        if math.isnan(x) or math.isinf(x) or x != math.trunc(x):
            return None
        x = int(x)
    lo, hi = int_bounds(src)
    return x if lo <= x <= hi else None


def _neighbours(f, dt):
    """f and its nearest values of float dtype dt on either side."""
    t = np.dtype(dt).type
    return [float(np.nextafter(t(f), t(-np.inf))), float(t(f)), float(np.nextafter(t(f), t(np.inf)))]


# integers whose correctly rounded Float32 differs from rounding through Float64 first
# (just above a Float32 tie; Float64 drops the +1 and leaves an exact tie, which then rounds to even)
DOUBLE_ROUNDING = [s * ((1 << k) + (1 << (k - 24)) + 1) for k in (55, 60, 62) for s in (1, -1)] + [(1 << 63) + (1 << 39) + 1]


def edges(src, dst):
    """Values of dtype src where `CAST(x AS dst)` goes wrong: the target's MIN - 1, MIN, MAX and MAX + 1; ±0.5 and
    ±1 ulp around the float images of those bounds; NaN, ±inf, ±0.0, subnormals, 2^53 ± 1, integers that Float32
    would double-round through Float64, the largest Float32 and Float64 values just beyond it; the source's own
    extremes.  Only values src can represent are kept; returned sorted by bit pattern, without duplicates."""
    src, dst = np.dtype(src), np.dtype(dst)
    xs = []
    if is_float(dst):
        lo, hi = None, None
    else:
        lo, hi = int_bounds(dst)
        xs += [lo - 1, lo, lo + 1, hi - 1, hi, hi + 1]
        for b in (lo, hi, lo - 1, hi + 1):
            xs += [b - 0.5, b + 0.5, b - 0.9, b + 0.9]
            for fdt in FLOATS:
                xs += _neighbours(float(b), fdt)
    xs += [0, 1, -1, 2, -2, 127, 128, 255, 256, -128, -129, 200, 300, 65535, 65536, 2 ** 31, 2 ** 32, 2 ** 63, 2 ** 64,
           (1 << 53) - 1, 1 << 53, (1 << 53) + 1, 16777217, -16777217, (1 << 64) - 1, (1 << 63) - 1, -(1 << 63)]
    xs += DOUBLE_ROUNDING
    xs += [math.nan, -math.nan, math.inf, -math.inf, 0.0, -0.0, 0.5, -0.5, 0.7, -0.7, 0.9, -0.9, 1.5, -1.5, 2.5, -2.5,
           5e-324, -5e-324, 2.2250738585072014e-308, 1e-40, -1e-40, 1.1754944e-38, 1e-45, 1e-300, -1e-300,
           1e300, -1e300, 1.7976931348623157e308, -1.7976931348623157e308, 255.9, -128.9, 2147483647.5, -2147483648.5,
           9007199254740993.0, 1.8446744073709552e19, 9.223372036854775e18]
    f32max = float(np.finfo(np.float32).max)
    xs += _neighbours(f32max, np.float64) + [-f32max, float(np.nextafter(-f32max, -np.inf)), f32max * (1 + 2.0 ** -25),
                                             f32max * (1 + 2.0 ** -24), 1.401298464324817e-45 * 0.5, 1.401298464324817e-45 * 1.5]
    if is_float(src):
        xs += [float(np.finfo(src).max), -float(np.finfo(src).max), float(np.finfo(src).tiny), float(np.finfo(src).smallest_subnormal)]
    else:
        slo, shi = int_bounds(src)
        xs += [slo, slo + 1, shi - 1, shi, shi // 2, shi // 2 + 1]
    vals = []
    for x in xs:
        r = _representable(x, src)
        if r is not None:
            vals.append(r)
    arr = np.array(vals, dtype=src) if is_float(src) else np.array(vals, dtype=object).astype(src)
    u = np.unique(arr.view(_UINT[src.itemsize]))
    return u.view(src)


def fill(rng, src, dst, n, pool=4096):
    """n values of dtype src: every edge of (src, dst) at least once (of every target when dst is None), the rest
    drawn from a pool of random values of every magnitude the source holds."""
    src = np.dtype(src)
    e = edges(src, dst) if dst is not None else np.unique(np.concatenate([edges(src, d) for d in NUMERIC]).view(_UINT[src.itemsize])).view(src)
    if is_float(src):
        mag = 10.0 ** rng.uniform(-3, 20 if src == np.float64 else 12, pool)
        p = (rng.choice([-1.0, 1.0], pool) * mag).astype(src)
    else:
        lo, hi = int_bounds(src)
        p = rng.integers(lo, hi, pool, dtype=src, endpoint=True)
        p[: pool // 2] = rng.integers(max(lo, -300), min(hi, 300), pool // 2, endpoint=True).astype(src)
    pool_vals = np.concatenate([e, p])
    out = pool_vals[rng.integers(0, len(pool_vals), n)]
    out[rng.choice(n, len(e), replace=False)] = e
    return out


# ---- the SQL planner's coercions ----------------------------------------------------------------------------------
def can_coerce_from(to, frm):
    """The planner's can_coerce_from: which implicit CAST(frm AS to) it inserts (sqlplanner's cast_to)."""
    to, frm = np.dtype(to), np.dtype(frm)
    if to == frm:
        return True
    if to.kind in "iu":
        return frm.kind == to.kind and frm.itemsize <= to.itemsize
    if to == np.float32:
        return frm.kind in "iu"
    return frm.kind in "iuf"


def coerce(a, b, supertype):
    """What the planner computes for `a op b` with operands a, b (arrays) under `supertype` (a dtype, from
    host.supertype): both operands cast to it, or None when the planner refuses to convert one of them
    ("Cannot automatically convert")."""
    st = np.dtype(supertype)
    if not (can_coerce_from(st, a.dtype) and can_coerce_from(st, b.dtype)):
        return None
    return (a if a.dtype == st else cast(a, st)), (b if b.dtype == st else cast(b, st))


def wrap_int(x, dt):
    """Integer arithmetic result x (numpy object or int array) wrapped to dtype dt, like Rust's release build."""
    bits = 8 * np.dtype(dt).itemsize
    w = np.array([int(v) % (1 << bits) for v in x], dtype=object)
    if is_signed(dt):
        w = np.array([v - (1 << bits) if v >= 1 << (bits - 1) else v for v in w], dtype=object)
    return w.astype(dt)
