"""Exact CPU reference of the GROUP BY / reduce operator (numpy only), for checking every kernel instantiation and every
aggregate function the operator accepts: MIN, MAX, SUM, COUNT, AVG and COUNT(DISTINCT).

The semantics are those DESIGN §7 states for the GPU path:
* keys are grouped by value and keep their own dtype; the bytes under a null key slot are the key;
* MIN / MAX are exact under the total order of non-NaN values with -0.0 < +0.0; NaN is skipped, and a group
  whose values are all NaN yields some NaN (only `isnan` is checked, not the payload bits);
* integer SUM is exact and wraps at the width of its output dtype, which is the argument dtype;
* COUNT counts the valid values, as uint64;
* float SUM: NaN if a NaN or both infinities are present, else the infinity present, else within
  gamma(n) * sum|v| of the exact sum, gamma(n) = n u / (1 - n u): a bound that holds for any summation order.  The
  bound is 0 (the sum is exact) when every value is a multiple of a power of two q >= the dtype's smallest normal and
  sum|v| < 2^p q (p = 53, or 24 for Float32): then every partial sum in any order is exactly representable and no
  partial sum is subnormal, so Float32's flush to zero cannot apply;
* AVG: Float64, the mean of the valid values, each first rounded to f64 (integers beyond 2^53 round to nearest).  Null
  when the group has no valid value.  NaN if a NaN or both infinities are present, else the infinity present, else
  within the f64 SUM bound above divided by the count, plus the rounding of that one division; when the sum is exact,
  it is exactly the f64 quotient sum / count;
* COUNT(DISTINCT): the number of distinct valid values, as uint64; +0.0 and -0.0 are one value, and all NaNs are one
  value;
* GROUP BY reads MIN / MAX / SUM arguments ignoring the validity bitmap (arrow 0.12 `value(row)`), while COUNT, AVG and
  COUNT(DISTINCT) skip null values, so a group whose values are all null counts 0 and its AVG is null;
* without GROUP BY every aggregate skips null values and the result is one row, also over zero rows: COUNT and
  COUNT(DISTINCT) are 0 there, and MIN / MAX / SUM / AVG are null when no value is valid;
* WHERE: `where` is the per-row pass mask, and only the rows it passes are aggregated.  The keys and arguments of those
  rows are read as over FilterRelation's output, which has no bitmaps: the value under a null slot of a column is an
  ordinary valid value there, and only an expression such as a CASE without ELSE can still be null.  The caller passes
  keys and arguments evaluated that way.  With the rules above, a COUNT under a WHERE that passes nothing is 0
  without GROUP BY, and the other aggregates are null.
"""
import numpy as np

MIN, MAX, SUM, COUNT, AVG, COUNT_DISTINCT = "min", "max", "sum", "count", "avg", "count_distinct"
_P = {np.dtype(np.float64): 53, np.dtype(np.float32): 24}  # significand bits; the unit roundoff u is 2^-p


def func_of(agg):
    """The reference's name for an expr.AggregateFunction."""
    return COUNT_DISTINCT if agg.distinct else agg.name


def _vm(x):
    """(values, valid) of a column given as an array or as a (values, valid-or-None) pair."""
    if isinstance(x, tuple):
        v, m = x
        return np.asarray(v), (None if m is None else np.asarray(m, dtype=bool))
    return np.asarray(x), None


class Expected:
    """Sorted distinct keys and, per aggregate, what the result column must hold."""

    def __init__(self, keys, aggs):
        self.keys = keys   # list of arrays, one per key column, sorted by key tuple
        self.aggs = aggs   # list of dicts, see aggregate


def _segments(keys, n):
    """Row order that sorts by the key tuple, segment starts of equal keys, and the keys of each segment."""
    order = np.lexsort([k for k in reversed(keys)])
    sk = [k[order] for k in keys]
    change = np.zeros(n, dtype=bool)
    if n:
        change[0] = True
    for k in sk:
        change[1:] |= k[1:] != k[:-1]
    starts = np.flatnonzero(change)
    return order, starts, [k[starts] for k in sk]


def _reduce(ufunc, x, seg, nseg, empty):
    """ufunc over the elements of each segment (seg: the sorted segment id of each element); `empty` for a segment
    without element."""
    out = np.full(nseg, empty, dtype=x.dtype)
    if len(x):
        present, starts = np.unique(seg, return_index=True)
        out[present] = ufunc.reduceat(x, starts)
    return out


def _min_max(func, v, seg, nseg):
    dt = v.dtype
    if not np.issubdtype(dt, np.floating):
        ufunc, empty = (np.minimum, np.iinfo(dt).max) if func == MIN else (np.maximum, np.iinfo(dt).min)
        return {"values": _reduce(ufunc, v, seg, nseg, empty), "isnan": np.zeros(nseg, dtype=bool)}
    nan = np.isnan(v)
    fill = np.inf if func == MIN else -np.inf
    w = np.where(nan, dt.type(fill), v)
    ufunc = np.minimum if func == MIN else np.maximum
    r = _reduce(ufunc, w, seg, nseg, fill).astype(dt)
    all_nan = np.bincount(seg, weights=~nan, minlength=nseg) == 0
    # the total order puts -0.0 below +0.0: a zero extremum is -0.0 for MIN when the group holds a -0.0,
    # and +0.0 for MAX when it holds a +0.0
    want_sign = func == MIN
    has = np.bincount(seg, weights=(w == 0) & (np.signbit(w) == want_sign), minlength=nseg) > 0
    zero = r == 0
    r[zero & has] = dt.type(-0.0 if want_sign else 0.0)
    r[zero & ~has] = dt.type(0.0 if want_sign else -0.0)
    return {"values": r, "isnan": all_nan}


def _lowest_bit(x):
    """The value of the lowest set significand bit of each nonzero finite x, a power of two."""
    m, e = np.frexp(x.astype(np.float64))  # x = m 2^e, 0.5 <= |m| < 1, and m 2^53 is an integer
    sig = np.abs(np.ldexp(m, 53)).astype(np.uint64)
    return np.ldexp((sig & (~sig + np.uint64(1))).astype(np.float64), e - 53)


def _float_sum(v, seg, nseg):
    dt = v.dtype
    u = 2.0 ** -_P[dt]
    flags = lambda m: np.bincount(seg, weights=m, minlength=nseg) > 0  # noqa: E731
    nan, pinf, ninf = flags(np.isnan(v)), flags(v == np.inf), flags(v == -np.inf)
    fin = np.where(np.isfinite(v), v, dt.type(0))
    exact = _reduce(np.add, fin.astype(np.longdouble), seg, nseg, 0)
    absum = _reduce(np.add, np.abs(fin).astype(np.longdouble), seg, nseg, 0)
    counts = np.bincount(seg, minlength=nseg)
    nu = counts.astype(np.float64) * u
    gamma = nu / (1.0 - nu)
    # the long-double reference sum has an error bound of its own (64-bit significand), well below gamma
    bound = (gamma + counts * 2.0 ** -63) * absum.astype(np.float64)
    q = _reduce(np.minimum, np.where(fin != 0, _lowest_bit(fin), np.inf), seg, nseg, np.inf)
    bound[(absum < np.ldexp(q, _P[dt]).astype(np.longdouble)) & (q >= np.finfo(dt).tiny)] = 0.0
    special = np.where(nan | (pinf & ninf), 1, np.where(pinf, 2, np.where(ninf, 3, 0)))
    return {"exact": exact, "bound": bound, "special": special}


def _avg(x, seg, nseg, nvalid):
    """AVG of the f64 values x: the SUM rule above, divided by the count."""
    s = _float_sum(x, seg, nseg)
    c = np.maximum(nvalid, 1).astype(np.float64)
    exact, bound = s["exact"], s["bound"]
    s["exact"] = np.where(bound == 0, (exact.astype(np.float64) / c).astype(np.longdouble), exact / c)
    s["bound"] = np.where(bound == 0, 0.0, (bound + 2.0 ** -53 * (np.abs(exact).astype(np.float64) + bound)) / c)
    return s


def _count_distinct(v, seg, nseg):
    if v.dtype.kind == "f":
        w = v.astype(np.float64) + 0.0  # -0.0 + 0.0 is +0.0
        v = w.view(np.uint64).copy()
        v[np.isnan(w)] = 0x7FF8000000000000
    order = np.lexsort((v, seg))
    s, x = seg[order], v[order]
    first = np.ones(len(order), dtype=bool)
    first[1:] = (s[1:] != s[:-1]) | (x[1:] != x[:-1])
    return np.bincount(s[first], minlength=nseg).astype(np.uint64)


def aggregate(keys, aggs, where=None):
    """keys: list of key columns, none without GROUP BY; aggs: list of (func, column) with func one of MIN / MAX / SUM /
    COUNT / AVG / COUNT_DISTINCT; where: the per-row pass mask of a WHERE, or None.  A column is an array or a (values,
    valid) pair.  Returns an Expected, keys sorted by tuple (numpy order of each dtype)."""
    kv = [_vm(k)[0] for k in keys]
    n = len(_vm(aggs[0][1])[0]) if aggs else len(kv[0])
    take = np.ones(n, dtype=bool) if where is None else np.asarray(where, dtype=bool)
    kv = [k[take] for k in kv]
    n = int(take.sum())
    grouped = len(keys) > 0
    order, starts, ukeys = _segments(kv, n) if grouped else (np.arange(n), np.zeros(1, dtype=np.int64), [])
    nseg = len(starts)
    seg = np.repeat(np.arange(nseg), np.diff(np.append(starts, n)))
    out = []
    for func, c in aggs:
        v, valid = _vm(c)
        v = v[take][order]
        valid = np.ones(n, dtype=bool) if valid is None else valid[take][order]
        nvalid = np.bincount(seg[valid], minlength=nseg).astype(np.uint64)
        d = {"func": func, "null": np.zeros(nseg, dtype=bool)}
        if func == COUNT:
            d.update(values=nvalid, dtype=np.dtype(np.uint64))
        elif func == COUNT_DISTINCT:
            d.update(values=_count_distinct(v[valid], seg[valid], nseg), dtype=np.dtype(np.uint64))
        elif func == AVG:
            d.update(_avg(v[valid].astype(np.float64), seg[valid], nseg, nvalid), dtype=np.dtype(np.float64), null=nvalid == 0)
        else:
            sel, sseg = (v, seg) if grouped else (v[valid], seg[valid])
            if not grouped:
                d["null"] = nvalid == 0
            if func in (MIN, MAX):
                d.update(_min_max(func, sel, sseg, nseg), dtype=v.dtype)
            elif np.issubdtype(v.dtype, np.floating):
                d.update(_float_sum(sel, sseg, nseg), dtype=v.dtype)
            else:
                wide = sel.astype(np.int64).view(np.uint64) if np.issubdtype(v.dtype, np.signedinteger) else sel.astype(np.uint64)
                d.update(values=_reduce(np.add, wide, sseg, nseg, 0).astype(v.dtype), dtype=v.dtype)  # wraps at the output width
        out.append(d)
    return Expected(ukeys, out)


def _unpack(c, n):
    if isinstance(c, tuple):
        return np.asarray(c[0]), np.asarray(c[1], dtype=bool)
    return (np.asarray(c) if not isinstance(c, list) else c), np.ones(n, dtype=bool)


def assert_matches(got, exp, ctx=""):
    """`got`: result columns (keys first, then aggregates; a nullable column as (values, valid)), any row order."""
    nk = len(exp.keys)
    assert len(got) == nk + len(exp.aggs), ctx
    n = len(_unpack(got[0], 0)[0])
    cols = [_unpack(c, n) for c in got]
    if nk:
        for (v, m), e in zip(cols[:nk], exp.keys):
            assert m.all(), ctx
            assert v.dtype == e.dtype, (ctx, v.dtype, e.dtype)
        order = np.lexsort([cols[k][0] for k in reversed(range(nk))])
        assert n == len(exp.keys[0]), (ctx, "groups", n, len(exp.keys[0]))
        for k in range(nk):
            g = cols[k][0][order]
            bad = np.flatnonzero(g != exp.keys[k])
            assert not len(bad), (ctx, "key", k, bad[:5], g[bad[:5]], exp.keys[k][bad[:5]])
    else:
        order = np.arange(n)
        assert n == 1, ctx
    for i, e in enumerate(exp.aggs):
        v, m = cols[nk + i]
        v, m = v[order], m[order]
        where = "%s agg %d (%s)" % (ctx, i, e["func"])
        assert v.dtype == e["dtype"], (where, v.dtype, e["dtype"])
        assert np.array_equal(~m, e["null"]), (where, "nulls")
        ok = m
        if "special" in e:
            sp = e["special"][ok]
            g = v[ok].astype(np.float64)
            assert np.array_equal(np.isnan(g), sp == 1), (where, "NaN")
            assert np.array_equal(g == np.inf, sp == 2) and np.array_equal(g == -np.inf, sp == 3), (where, "inf")
            fin = sp == 0
            err = np.abs(g[fin].astype(np.longdouble) - e["exact"][ok][fin]).astype(np.float64)
            bad = np.flatnonzero(err > e["bound"][ok][fin])
            assert not len(bad), (where, "sum error", bad[:5], g[fin][bad[:5]], e["exact"][ok][fin][bad[:5]], e["bound"][ok][fin][bad[:5]])
        else:
            gv, ev = v[ok], e["values"][ok]
            if "isnan" in e:
                nanm = e["isnan"][ok]
                if np.issubdtype(gv.dtype, np.floating):
                    assert np.isnan(gv[nanm]).all(), (where, "all-NaN group")
                    assert not np.isnan(gv[~nanm]).any(), (where, "unexpected NaN")
                gv, ev = gv[~nanm], ev[~nanm]
            bad = np.flatnonzero(gv.view(_uint_of(gv.dtype)) != ev.view(_uint_of(ev.dtype)))
            assert not len(bad), (where, "bits", bad[:5], gv[bad[:5]], ev[bad[:5]])


def _uint_of(dt):
    return {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[np.dtype(dt).itemsize]


def arrow_nullable(values, valid):
    """pyarrow array over our own buffers, so the bytes under null slots are known (for the engine and oracle)."""
    import pyarrow as pa
    values = np.ascontiguousarray(values)
    bits = np.packbits(np.asarray(valid, dtype=bool), bitorder="little")
    return pa.Array.from_buffers(pa.from_numpy_dtype(values.dtype), len(values), [pa.py_buffer(bits.tobytes()), pa.py_buffer(values.tobytes())])


# ---- edge values ------------------------------------------------------------------------------------------
def _f(dt, xs):
    return np.array(xs, dtype=dt)


def edges(dt, for_sum=False):
    """Values where kernels go wrong, for an argument dtype.  for_sum: only values whose sums cannot overflow in
    any order, and no Float32 subnormal (Float32 SUM flushes subnormals to zero, DESIGN §7).  The SUM bound
    scales with the group's sum of |v|, so in the few groups that draw ±1e300 (±1e30 for Float32) a lost or
    doubled ordinary row is below the bound; every other group still resolves a single row."""
    dt = np.dtype(dt)
    if dt == np.float64:
        xs = [0.0, -0.0, 1.0, -1.0, 2.5e-308, -2.2250738585072014e-308, 5e-324, -5e-324, np.inf, -np.inf, np.nan,
              -np.nan, 1e300 if for_sum else 1.7976931348623157e308, -1e300 if for_sum else -1.7976931348623157e308]
        return _f(dt, xs)
    if dt == np.float32:
        xs = [0.0, -0.0, 1.0, -1.0, np.inf, -np.inf, np.nan, -np.nan, 1.1754944e-38, -1.1754944e-38,
              1e30 if for_sum else 3.4028235e38, -1e30 if for_sum else -3.4028235e38]
        if not for_sum:
            xs += [1e-45, -1e-45, 1e-40]
        return _f(dt, xs)
    info = np.iinfo(dt)
    xs = {info.min, info.max, 0, 1, info.max - 1, info.min + 1}
    if info.min < 0:
        xs |= {-1, info.min // 2}
    else:
        xs |= {info.max // 2 + 1}  # the top bit set: >= 2^63 for UInt64
    return _f(dt, sorted(xs))


def random_values(rng, dt, n):
    """Bulk values of dtype dt: both signs, a few thousand distinct values (repeats exercise the MIN / MAX skip)."""
    dt = np.dtype(dt)
    if np.issubdtype(dt, np.floating):
        return ((rng.random(n) - 0.5) * 2000.0).astype(dt)
    info = np.iinfo(dt)
    lo, hi = max(info.min, -(10 ** 6)), min(info.max, 10 ** 6)
    return rng.integers(lo, hi, n, dtype=dt, endpoint=True)


def sprinkle(rng, v, e, frac=0.01):
    """v with every value of e written to random rows (about frac of the rows in all)."""
    v = v.copy()
    m = max(len(e), int(len(v) * frac))
    rows = rng.choice(len(v), size=min(m, len(v)), replace=False)
    v[rows] = e[np.arange(len(rows)) % len(e)]
    return v
