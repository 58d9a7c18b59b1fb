"""Exact CPU reference of the GROUP BY / reduce operator (numpy only), for checking every kernel instantiation.

The semantics are those DESIGN §7 states for the GPU path:
* keys are grouped by value and keep their own dtype; the bytes under a null key slot are the key;
* MIN / MAX are exact under the total order of non-NaN values with -0.0 < +0.0; NaN is skipped, and a group
  whose values are all NaN yields some NaN (only `isnan` is checked, not the payload bits);
* integer SUM is exact and wraps at the width of its output dtype, which is the argument dtype;
* COUNT counts the valid values, as uint64;
* float SUM: NaN if a NaN or both infinities are present, else the infinity present, else within
  gamma(n) * sum|v| of the exact sum, gamma(n) = n u / (1 - n u): a bound that holds for any summation order;
* GROUP BY reads MIN / MAX / SUM arguments ignoring the validity bitmap (arrow 0.12 `value(row)`), while a
  reduction without GROUP BY skips null values and is null when no value is valid.
"""
import numpy as np

MIN, MAX, SUM, COUNT = "min", "max", "sum", "count"
_U = {np.dtype(np.float64): 2.0 ** -53, np.dtype(np.float32): 2.0 ** -24}


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
        self.aggs = aggs   # list of dicts, see _agg


def _segments(keys, n):
    """Row order that sorts by the key tuple, segment starts of equal keys, and the keys of each segment."""
    if not keys:
        return np.arange(n), (np.zeros(1, dtype=np.int64) if n else np.zeros(0, dtype=np.int64)), []
    order = np.lexsort([k for k in reversed(keys)])
    sk = [k[order] for k in keys]
    change = np.zeros(n, dtype=bool)
    if n:
        change[0] = True
    for k in sk:
        change[1:] |= k[1:] != k[:-1]
    starts = np.flatnonzero(change)
    return order, starts, [k[starts] for k in sk]


def _reduceat(ufunc, x, starts, empty):
    """ufunc.reduceat over segments, where an empty segment (possible only without GROUP BY) yields `empty`."""
    if len(x) == 0:
        return np.full(len(starts), empty, dtype=x.dtype)
    return ufunc.reduceat(x, starts)


def _min_max(func, v, starts, counts):
    dt = v.dtype
    if not np.issubdtype(dt, np.floating):
        ufunc, empty = (np.minimum, np.iinfo(dt).max) if func == MIN else (np.maximum, np.iinfo(dt).min)
        return {"values": _reduceat(ufunc, v, starts, empty), "isnan": np.zeros(len(starts), dtype=bool)}
    nan = np.isnan(v)
    fill = np.inf if func == MIN else -np.inf
    w = np.where(nan, dt.type(fill), v)
    ufunc = np.minimum if func == MIN else np.maximum
    r = _reduceat(ufunc, w, starts, fill).astype(dt)
    seg = np.repeat(np.arange(len(starts)), counts)
    all_nan = np.bincount(seg, weights=~nan, minlength=len(starts)) == 0
    # the total order puts -0.0 below +0.0: a zero extremum is -0.0 for MIN when the group holds a -0.0,
    # and +0.0 for MAX when it holds a +0.0
    want_sign = func == MIN
    has = np.bincount(seg, weights=(w == 0) & (np.signbit(w) == want_sign), minlength=len(starts)) > 0
    zero = r == 0
    r[zero & has] = dt.type(-0.0 if want_sign else 0.0)
    r[zero & ~has] = dt.type(0.0 if want_sign else -0.0)
    return {"values": r, "isnan": all_nan}


def _float_sum(v, starts, counts):
    dt = v.dtype
    u = _U[dt]
    nseg = len(starts)
    seg = np.repeat(np.arange(nseg), counts)
    flags = lambda m: np.bincount(seg, weights=m, minlength=nseg) > 0  # noqa: E731
    nan, pinf, ninf = flags(np.isnan(v)), flags(v == np.inf), flags(v == -np.inf)
    fin = np.where(np.isfinite(v), v, dt.type(0)).astype(np.longdouble)
    exact = _reduceat(np.add, fin, starts, 0).astype(np.longdouble) if nseg else np.zeros(0, dtype=np.longdouble)
    absum = _reduceat(np.add, np.abs(fin), starts, 0).astype(np.float64) if nseg else np.zeros(0)
    nu = counts.astype(np.float64) * u
    gamma = nu / (1.0 - nu)
    # the long-double reference sum has an error bound of its own (64-bit significand), well below gamma
    bound = (gamma + counts * 2.0 ** -63) * absum
    special = np.where(nan | (pinf & ninf), 1, np.where(pinf, 2, np.where(ninf, 3, 0)))
    return {"exact": exact, "bound": bound, "special": special}


def aggregate(keys, aggs):
    """keys: list of key columns; aggs: list of (func, column) with func in MIN / MAX / SUM / COUNT.  A column is
    an array or a (values, valid) pair.  Returns an Expected, keys sorted by tuple (numpy order of each dtype)."""
    kv = [_vm(k)[0] for k in keys]
    n = len(_vm(aggs[0][1])[0]) if aggs else len(kv[0])
    order, starts, ukeys = _segments(kv, n)
    grouped = len(keys) > 0
    out = []
    for func, c in aggs:
        v, valid = _vm(c)
        v = v[order]
        valid = np.ones(n, dtype=bool) if valid is None else valid[order]
        if grouped:
            counts = np.diff(np.append(starts, n))
            nvalid = np.add.reduceat(valid.astype(np.uint64), starts) if n else np.zeros(0, dtype=np.uint64)
            sel, sstarts, scounts = v, starts, counts
        else:
            # no GROUP BY: null values are skipped, and an aggregate over no valid value is null
            sel = v[valid]
            nvalid = np.array([valid.sum()], dtype=np.uint64)
            sstarts, scounts = np.zeros(1, dtype=np.int64), np.array([len(sel)])
        d = {"func": func, "null": (nvalid == 0) if not grouped and func != COUNT else np.zeros(len(starts), dtype=bool)}
        if func == COUNT:
            d.update(values=nvalid.astype(np.uint64), dtype=np.dtype(np.uint64))
        elif func in (MIN, MAX):
            d.update(_min_max(func, sel, sstarts, scounts), dtype=v.dtype)
        elif np.issubdtype(v.dtype, np.floating):
            d.update(_float_sum(sel, sstarts, scounts), dtype=v.dtype)
        else:
            wide = sel.astype(np.int64).view(np.uint64) if np.issubdtype(v.dtype, np.signedinteger) else sel.astype(np.uint64)
            s = _reduceat(np.add, wide, sstarts, 0)
            d.update(values=s.astype(v.dtype), dtype=v.dtype)  # wraps at the output width
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
