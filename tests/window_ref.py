"""Exact CPU reference of dfgpu_window and of window functions under SQL (numpy only).

* Order: sort_ref.order over the partition keys (ascending) and then the ORDER BY keys, the row number last, so rows that
  tie keep their input order.
* Partitions and peers: a partition starts where a partition key's encoding (sort_ref.encode) or null bit differs from
  the previous sorted row; a peer group also starts where an ORDER BY key's does.
* Frames: with ORDER BY a row's frame is its partition's sorted rows through its last peer, without ORDER BY the whole
  partition.
* ROW_NUMBER, RANK and DENSE_RANK count positions, first peers and peer groups within the partition, from 1 (UInt64).
* The aggregates skip null values and follow groupby_ref's value rules: integer SUM wraps at its width, MIN / MAX order
  -0.0 below +0.0 and skip NaN (some NaN when every value is NaN), COUNT is UInt64, float SUM and AVG are exact when
  groupby_ref proves the sum exact in any order and within its gamma bound otherwise.  A frame without a valid value is
  null, except for COUNT, which is 0.
"""
import numpy as np

from datafusion_archive_b200 import _abi as A

import groupby_ref as G
import sort_ref

ROW_NUMBER, RANK, DENSE_RANK = "row_number", "rank", "dense_rank"
MIN, MAX, SUM, COUNT, AVG = G.MIN, G.MAX, G.SUM, G.COUNT, G.AVG
FUNC_CODE = {ROW_NUMBER: A.WIN_ROW_NUMBER, RANK: A.WIN_RANK, DENSE_RANK: A.WIN_DENSE_RANK, MIN: A.AGG_MIN, MAX: A.AGG_MAX, SUM: A.AGG_SUM,
             COUNT: A.AGG_COUNT, AVG: A.AGG_AVG}


def _key_words(dtype, vals, valid, idx):
    e = sort_ref.encode(dtype, vals, valid)[idx]
    v = np.ones(len(idx), dtype=bool) if valid is None else np.asarray(valid, dtype=bool)[idx]
    return e, v


def structure(n, part, order):
    """(perm, pid, gid, pstart, gstart) in sorted order.  part: [(dtype, values, valid)]; order: [(dtype, values, valid,
    desc)]."""
    perm = sort_ref.order(n, [(d, v, m, False) for d, v, m in part] + list(order))
    pstart = np.zeros(n, dtype=bool)
    if n:
        pstart[0] = True
    gstart = pstart.copy()
    for i, k in enumerate(list(part) + list(order)):
        e, v = _key_words(k[0], k[1], k[2], perm)
        diff = np.zeros(n, dtype=bool)
        diff[1:] = (e[1:] != e[:-1]) | (v[1:] != v[:-1])
        if i < len(part):
            pstart |= diff
        gstart |= diff
    return perm, np.cumsum(pstart) - 1, np.cumsum(gstart) - 1, pstart, gstart


def _decode(dtype, e):
    w = np.dtype(A.NP_OF[dtype]).itemsize
    u = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[w]
    sign = np.uint64(1 << (8 * w - 1))
    mask = np.uint64((1 << (8 * w)) - 1)
    if dtype in (A.FLOAT32, A.FLOAT64):
        raw = np.where((e & sign) != 0, e ^ sign, ~e & mask)
    elif dtype in (A.INT8, A.INT16, A.INT32, A.INT64):
        raw = e ^ sign
    else:
        raw = e
    return raw.astype(u).view(A.NP_OF[dtype])


def window(n, part, order, fns):
    """Expected output of each function of `fns`, [(func, (dtype, values, valid) or None)], in input row order: a dict
    with "values", "null" and "dtype", and for float SUM / AVG "exact", "bound" and "special" as groupby_ref has them,
    for float MIN / MAX "isnan"."""
    perm, pid, gid, pstart, gstart = structure(n, part, order)
    pfirst = np.flatnonzero(pstart)
    gfirst = np.flatnonzero(gstart)
    glast = np.append(gfirst[1:] - 1, n - 1).astype(np.int64) if n else np.zeros(0, np.int64)
    frame_end = glast[gid] if n else np.zeros(0, np.int64)  # sorted position of each sorted row's frame end
    pos = np.arange(n)
    bounds = list(zip(pfirst, np.append(pfirst[1:], n)))
    out = []
    for func, arg in fns:
        d = {"func": func, "null": np.zeros(n, dtype=bool)}
        if func in (ROW_NUMBER, RANK, DENSE_RANK):
            if func == ROW_NUMBER:
                s = pos - pfirst[pid] + 1
            elif func == RANK:
                s = gfirst[gid] - pfirst[pid] + 1
            else:
                s = gid - gid[pfirst[pid]] + 1
            d.update(values=_scatter(perm, np.asarray(s, dtype=np.uint64)), dtype=np.dtype(np.uint64))
            out.append(d)
            continue
        dtype, vals, valid = arg
        v = np.asarray(vals)[perm]
        ok = np.ones(n, dtype=bool) if valid is None else np.asarray(valid, dtype=bool)[perm]
        cnt = np.zeros(n, dtype=np.int64)
        for a, b in bounds:
            cnt[a:b] = np.cumsum(ok[a:b])
        c = cnt[frame_end]
        if func != COUNT:
            d["null"] = _scatter(perm, c == 0)
        if func == COUNT:
            d.update(values=_scatter(perm, c.astype(np.uint64)), dtype=np.dtype(np.uint64))
        elif func in (MIN, MAX):
            e = sort_ref.encode(dtype, v)
            isf = dtype in (A.FLOAT32, A.FLOAT64)
            nan = np.isnan(v) if isf else np.zeros(n, dtype=bool)
            acc = np.zeros(n, dtype=np.uint64)
            if func == MIN:
                e = np.where(ok, e, np.uint64(2 ** 64 - 1))
                for a, b in bounds:
                    acc[a:b] = np.minimum.accumulate(e[a:b])
            else:
                e = np.where(ok & ~nan, e, np.uint64(0))
                for a, b in bounds:
                    acc[a:b] = np.maximum.accumulate(e[a:b])
            nn = np.zeros(n, dtype=np.int64)  # valid non-NaN values so far
            for a, b in bounds:
                nn[a:b] = np.cumsum(ok[a:b] & ~nan[a:b])
            r = acc[frame_end]
            allnan = (nn[frame_end] == 0) & (c > 0) if isf else np.zeros(n, dtype=bool)
            r = np.where(allnan | (c == 0), np.uint64(0), r)
            d.update(values=_scatter(perm, _decode(dtype, r)), dtype=np.dtype(A.NP_OF[dtype]))
            if isf:
                d["isnan"] = _scatter(perm, allnan)
        elif func == SUM and dtype not in (A.FLOAT32, A.FLOAT64):
            t = A.NP_OF[dtype]
            wide = v.astype(np.int64).view(np.uint64) if np.issubdtype(t, np.signedinteger) else v.astype(np.uint64)
            wide = np.where(ok, wide, np.uint64(0))
            acc = np.zeros(n, dtype=np.uint64)
            for a, b in bounds:
                acc[a:b] = np.cumsum(wide[a:b], dtype=np.uint64)
            d.update(values=_scatter(perm, acc[frame_end].astype(t)), dtype=np.dtype(t))
        else:
            x = v.astype(np.float64) if func == AVG else v
            d.update(_float_prefix(x, ok, bounds, frame_end, c, func == AVG))
            d["dtype"] = np.dtype(np.float64) if func == AVG else np.dtype(A.NP_OF[dtype])
            for k in ("exact", "bound", "special"):
                d[k] = _scatter(perm, d[k])
        out.append(d)
    return out


def _scatter(perm, s):
    o = np.empty_like(s)
    o[perm] = s
    return o


def _float_prefix(x, ok, bounds, frame_end, c, avg):
    """groupby_ref's SUM (or AVG) rule for each sorted row's frame, from per-partition prefix sums."""
    n = len(x)
    dt = x.dtype
    u = 2.0 ** -G._P[dt]
    fin = np.where(ok & np.isfinite(x), x, dt.type(0))
    lb = np.where(fin != 0, G._lowest_bit(fin) if n else fin, np.inf)
    exact = np.zeros(n, dtype=np.longdouble)
    absum = np.zeros(n, dtype=np.longdouble)
    q = np.zeros(n)
    fl = {k: np.zeros(n, dtype=bool) for k in ("nan", "pinf", "ninf")}
    for a, b in bounds:
        exact[a:b] = np.cumsum(fin[a:b].astype(np.longdouble))
        absum[a:b] = np.cumsum(np.abs(fin[a:b]).astype(np.longdouble))
        q[a:b] = np.minimum.accumulate(lb[a:b])
        fl["nan"][a:b] = np.logical_or.accumulate(ok[a:b] & np.isnan(x[a:b]))
        fl["pinf"][a:b] = np.logical_or.accumulate(ok[a:b] & (x[a:b] == np.inf))
        fl["ninf"][a:b] = np.logical_or.accumulate(ok[a:b] & (x[a:b] == -np.inf))
    exact, absum, q = exact[frame_end], absum[frame_end], q[frame_end]
    nan, pinf, ninf = (fl[k][frame_end] for k in ("nan", "pinf", "ninf"))
    nu = c.astype(np.float64) * u
    bound = (nu / (1.0 - nu) + c * 2.0 ** -63) * absum.astype(np.float64)
    bound[(absum < np.ldexp(q, G._P[dt]).astype(np.longdouble)) & (q >= np.finfo(dt).tiny)] = 0.0
    special = np.where(nan | (pinf & ninf), 1, np.where(pinf, 2, np.where(ninf, 3, 0)))
    if avg:
        cc = np.maximum(c, 1).astype(np.float64)
        exact, bound = (np.where(bound == 0, (exact.astype(np.float64) / cc).astype(np.longdouble), exact / cc),
                        np.where(bound == 0, 0.0, (bound + 2.0 ** -53 * (np.abs(exact).astype(np.float64) + bound)) / cc))
    return {"exact": exact, "bound": bound, "special": special}


def assert_matches(got, exp, ctx=""):
    """`got`: the result columns in input row order, a nullable column as (values, valid)."""
    assert len(got) == len(exp), ctx
    for i, e in enumerate(exp):
        where = "%s fn %d (%s)" % (ctx, i, e["func"])
        v, m = G._unpack(got[i], len(e["null"]))
        assert len(v) == len(e["null"]), (where, "rows", len(v), len(e["null"]))
        assert v.dtype == e["dtype"], (where, v.dtype, e["dtype"])
        bad = np.flatnonzero(~m != e["null"])
        assert not len(bad), (where, "nulls", bad[:5])
        if "special" in e:
            sp = e["special"][m]
            g = v[m].astype(np.float64)
            assert np.array_equal(np.isnan(g), sp == 1), (where, "NaN")
            assert np.array_equal(g == np.inf, sp == 2) and np.array_equal(g == -np.inf, sp == 3), (where, "inf")
            fin = sp == 0
            err = np.abs(g[fin].astype(np.longdouble) - e["exact"][m][fin]).astype(np.float64)
            bad = np.flatnonzero(err > e["bound"][m][fin])
            assert not len(bad), (where, "sum error", bad[:5], g[fin][bad[:5]], e["exact"][m][fin][bad[:5]], e["bound"][m][fin][bad[:5]])
            continue
        gv, ev = v[m], e["values"][m]
        if "isnan" in e:
            nanm = e["isnan"][m]
            assert np.isnan(gv[nanm]).all(), (where, "all-NaN frame")
            gv, ev = gv[~nanm], ev[~nanm]
        bad = np.flatnonzero(gv.view(G._uint_of(gv.dtype)) != ev.view(G._uint_of(ev.dtype)))
        assert not len(bad), (where, "bits", bad[:5], gv[bad[:5]], ev[bad[:5]])


def window_loop(n, part, order, fns):
    """The same as window(), by a per-row Python loop over explicit frames (small inputs only): for the self-check."""
    perm, pid, gid, _, _ = structure(n, part, order)
    where = np.empty(n, dtype=np.int64)
    where[perm] = np.arange(n)
    out = []
    for func, arg in fns:
        vals, nulls = [], []
        for r in range(n):
            i = where[r]
            same_p = [j for j in range(n) if pid[j] == pid[i]]
            if func == ROW_NUMBER:
                vals.append(i - same_p[0] + 1)
            elif func == RANK:
                vals.append(min(j for j in same_p if gid[j] == gid[i]) - same_p[0] + 1)
            elif func == DENSE_RANK:
                vals.append(gid[i] - gid[same_p[0]] + 1)
            else:
                dtype, v, valid = arg
                frame = [perm[j] for j in same_p if gid[j] <= gid[i]]
                xs = [v[k] for k in frame if valid is None or valid[k]]
                if func == COUNT:
                    vals.append(len(xs))
                    continue
                nulls.append(not xs)
                vals.append(xs)
        out.append((vals, nulls))
    return out
