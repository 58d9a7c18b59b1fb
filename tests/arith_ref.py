"""Exact reference of the binary arithmetic `a + b`, `a - b`, `a * b`, `a / b` over the ten numeric dtypes.

Computed over Python ints and `fractions.Fraction`, with cast_ref's correctly rounded Fraction -> Float32 / Float64
step, never through numpy's arithmetic:
* integers: the exact result wrapped to the operand width (Rust's release build).  `/` truncates toward zero, and
  `MIN / -1` wraps to MIN.  Unsigned operands are never read as signed.
* floats: the exact rational `a op b` rounded once to the operand type, to nearest with ties to even.  Subnormal
  results stay subnormal; overflow gives ±inf.  The IEEE specials are spelled out: the sign of a zero result,
  `inf - inf`, `0 * inf`, `inf / inf` and `0 / 0` (NaN), NaN operands.
* a zero divisor, of any type and including -0.0, is DivideByZero.
NaN results compare as a class (cast_ref.same): the GPU's canonical NaN is not x86's.
"""
import math
from fractions import Fraction

import numpy as np

from cast_ref import FLOATS, INTS, NUMERIC, _UINT, cast_scalar, int_bounds, is_float, is_signed, round_float, same, wrap_int  # noqa: F401

OPS = ("+", "-", "*", "/")


class DivideByZero(ArithmeticError):
    pass


def int_op(op, a, b, dt):
    """a op b for Python ints a, b of integer dtype dt, wrapped to dt."""
    if op == "+":
        r = a + b
    elif op == "-":
        r = a - b
    elif op == "*":
        r = a * b
    else:
        if b == 0:
            raise DivideByZero
        q = abs(a) // abs(b)  # truncation toward zero; MIN / -1 = -MIN, which wraps to MIN
        r = q if (a < 0) == (b < 0) else -q
    return cast_scalar(r, np.int64, dt)  # Rust `as` from a wider integer: wraps to dt


def _neg(x):
    return -x if x == x else x


def float_op(op, a, b, dt):
    """a op b for Python floats a, b holding values of float dtype dt; the result as a Python float (exact value of
    dt).  NaN results are some NaN."""
    if op == "/" and b == 0:
        raise DivideByZero
    if math.isnan(a) or math.isnan(b):
        return math.nan
    if op == "-":
        return float_op("+", a, _neg(b), dt)
    if op == "+":
        if math.isinf(a) or math.isinf(b):
            if math.isinf(a) and math.isinf(b) and a != b:
                return math.nan
            return a if math.isinf(a) else b
        if a == 0 and b == 0:  # -0 + -0 = -0; every other sum of zeros is +0
            return -0.0 if math.copysign(1, a) < 0 and math.copysign(1, b) < 0 else 0.0
        r = Fraction(a) + Fraction(b)
        return 0.0 if r == 0 else round_float(r, dt)  # an exact zero sum of nonzero operands is +0 (to nearest)
    neg = (math.copysign(1, a) < 0) != (math.copysign(1, b) < 0)
    if op == "*":
        if math.isinf(a) or math.isinf(b):
            if a == 0 or b == 0:
                return math.nan
            return -math.inf if neg else math.inf
        if a == 0 or b == 0:
            return -0.0 if neg else 0.0
        return round_float(Fraction(a) * Fraction(b), dt)
    # division, b != 0
    if math.isinf(a):
        return math.nan if math.isinf(b) else (-math.inf if neg else math.inf)
    if math.isinf(b) or a == 0:
        return -0.0 if neg else 0.0
    return round_float(Fraction(a) / Fraction(b), dt)


def scalar(op, a, b, dt):
    """a op b for one pair of values of dtype dt (Python or numpy scalars): a Python int or float; raises
    DivideByZero."""
    if is_float(dt):
        return float_op(op, float(a), float(b), dt)
    return int_op(op, int(a), int(b), dt)


def _pairs(a, b):
    """Row indices of the distinct (a, b) bit-pattern pairs, and the pair index of every row."""
    u = _UINT[a.dtype.itemsize]
    ux, ix = np.unique(a.view(u), return_inverse=True)
    uy, iy = np.unique(b.view(u), return_inverse=True)
    m = len(ux) * len(uy)
    if m <= 1 << 25:  # few distinct operands (every generator here): a dense table of the pairs, no sort of the rows
        code = ix.reshape(-1).astype(np.int64) * len(uy) + iy.reshape(-1)
        row = np.full(m, -1, dtype=np.int64)
        row[code] = np.arange(len(a))  # some row of each pair that occurs
        present = row >= 0
        return row[present], (np.cumsum(present) - 1)[code]
    x, y = a.view(u), b.view(u)
    order = np.lexsort((y, x))
    sx, sy = x[order], y[order]
    new = np.ones(len(a), dtype=bool)
    new[1:] = (sx[1:] != sx[:-1]) | (sy[1:] != sy[:-1])
    inv = np.empty(len(a), dtype=np.int64)
    inv[order] = np.cumsum(new) - 1
    return order[new], inv


def arith(op, a, b):
    """Exact `a op b` over numpy arrays (or scalars broadcast to the other operand) of one dtype.  Returns (values,
    divide_by_zero): the row's result, and a mask of the rows whose divisor is zero (their value is 0).  The
    reference is computed once per distinct operand pair."""
    a, b = np.asarray(a), np.asarray(b)
    dt = a.dtype if a.ndim else b.dtype
    a, b = np.broadcast_arrays(a.astype(dt), b.astype(dt))
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    n = len(a)
    if n == 0:
        return np.zeros(0, dtype=dt), np.zeros(0, dtype=bool)
    first, inv = _pairs(a, b)
    vals, bad = [], np.zeros(len(first), dtype=bool)
    for i, (x, y) in enumerate(zip(a[first].tolist(), b[first].tolist())):
        try:
            vals.append(scalar(op, x, y, dt))
        except DivideByZero:
            vals.append(0)
            bad[i] = True
    if is_float(dt):
        res = np.array(vals, dtype=np.float64).astype(dt)  # exact: every value is one of dt
    else:
        res = np.array(vals, dtype=object).astype(dt)
    return res[inv], bad[inv]


def value(op, a, b):
    """arith() when no divisor is zero (asserted)."""
    v, bad = arith(op, a, b)
    assert not bad.any(), "zero divisor in %d rows" % bad.sum()
    return v


# ---- edge values ----------------------------------------------------------------------------------------------------
def _ulp_pairs(dt):
    """Float pairs (a, b) where + - * / round at their hardest: exact ties (to even, both directions), sums that land
    exactly on the overflow threshold or just below it, results in the subnormal range and subnormal ties."""
    f = np.finfo(dt)
    p = f.nmant + 1
    t = np.dtype(dt).type
    one_up = 1.0 + 2.0 ** (1 - p)          # 1 + ulp(1): odd significand
    half = 2.0 ** -p                       # half an ulp of 1
    mx, tiny, sub = float(f.max), float(f.tiny), float(f.smallest_subnormal)
    half_ulp_max = 2.0 ** (f.maxexp - 1 - p)  # half an ulp of MAX
    pairs = [
        (1.0, half), (one_up, half), (-1.0, -half), (-one_up, -half), (1.0, -half / 2), (2.0, -half),  # + ties
        (one_up, 1.5), (1.5, one_up), (3.0, one_up), (-3.0, one_up),  # * ties
        (mx, half_ulp_max), (mx, float(np.nextafter(t(half_ulp_max), t(0)))), (-mx, -half_ulp_max), (mx, mx), (mx, -mx),
        (mx, 2.0), (mx, 0.5), (mx, 1.0 + 2.0 ** (1 - p)),  # overflow on the threshold and just below
        (tiny, -sub), (3 * sub, -2 * sub), (tiny, 0.5), (sub, 0.5), (3 * sub, 0.5), (-3 * sub, 0.5), (sub, -0.5),  # subnormal
        (tiny, -tiny), (sub, 2.0), (3 * sub, 2.0), (tiny * 1.5, 0.25), (1.0, 3.0), (2.0, 3.0), (tiny, 3.0), (mx, tiny),
        (0.0, -0.0), (-0.0, -0.0), (-0.0, 0.0), (0.0, -1.0), (-1.0, 0.0), (math.inf, -math.inf), (math.inf, math.inf),
        (0.0, math.inf), (-0.0, math.inf), (math.inf, 2.0), (2.0, -math.inf), (math.nan, 1.0), (1.0, math.nan),
    ]
    return [(float(t(x)), float(t(y))) for x, y in pairs]


def edges(dt):
    """The edge values of dtype dt, sorted by bit pattern, without duplicates.
    Integers: 0, ±1, ±2, ±7, MIN, MIN+1, MAX, MAX-1, 2^(w/2) and its neighbours (multiply overflow), 2^(w-1) and its
    neighbours (the unsigned sign bit).  Floats: ±0, ±inf, NaN, the smallest and largest subnormal, the smallest
    normal, MAX, 1 and its neighbours, and a few ordinary values."""
    dt = np.dtype(dt)
    if is_float(dt):
        f = np.finfo(dt)
        t = dt.type
        xs = [0.0, 1.0, 2.0, 0.5, 3.0, 0.1, 7.0, 1.5, 100.0, math.inf, math.nan, float(f.smallest_subnormal),
              float(np.nextafter(t(f.tiny), t(0))), float(f.tiny), float(f.max), float(np.nextafter(t(1), t(2))),
              float(np.nextafter(t(1), t(0))), float(np.nextafter(t(f.max), t(0)))]
        xs += [-x for x in xs]
        arr = np.array(xs, dtype=dt)
    else:
        lo, hi = int_bounds(dt)
        w = 8 * dt.itemsize
        h = 1 << (w // 2)
        xs = [0, 1, -1, 2, -2, 7, -7, lo, lo + 1, hi, hi - 1, h - 1, h, h + 1, -h - 1, -h, -h + 1, 1 << (w - 1),
              (1 << (w - 1)) - 1, (1 << (w - 1)) + 1, 3, 100, -100]
        arr = np.array([x for x in xs if lo <= x <= hi], dtype=object).astype(dt)
    u = np.unique(arr.view(_UINT[dt.itemsize]))
    return u.view(dt)


def pool(rng, dt, k):
    """k random values of dtype dt, of every magnitude the dtype holds (small integers half the time)."""
    dt = np.dtype(dt)
    if is_float(dt):
        top = 300 if dt == np.float64 else 36
        mag = 10.0 ** rng.uniform(-top, top, k)
        return (rng.choice([-1.0, 1.0], k) * mag).astype(dt)
    lo, hi = int_bounds(dt)
    p = rng.integers(lo, hi, k, dtype=dt, endpoint=True)
    p[: k // 2] = rng.integers(max(lo, -300), min(hi, 300), k // 2, endpoint=True).astype(dt)
    return p


def operands(rng, dt, n, k=64):
    """Two columns (a, b) of n rows of dtype dt.  Every pair of the edges and k random values occurs at least once
    (when n allows), and so does every pair of _ulp_pairs for floats; the other rows repeat random such pairs.  A small
    set of distinct pairs keeps the exact reference cheap at any n."""
    dt = np.dtype(dt)
    v = np.concatenate([edges(dt), pool(rng, dt, k)])
    ia, ib = np.meshgrid(np.arange(len(v)), np.arange(len(v)), indexing="ij")
    pa, pb = v[ia.ravel()], v[ib.ravel()]
    if is_float(dt):
        sp = np.array(_ulp_pairs(dt), dtype=dt)
        pa, pb = np.concatenate([pa, sp[:, 0], sp[:, 1]]), np.concatenate([pb, sp[:, 1], sp[:, 0]])
    m = len(pa)
    idx = rng.integers(0, m, n)
    if n >= m:
        idx[rng.choice(n, m, replace=False)] = np.arange(m)
    return pa[idx], pb[idx]
