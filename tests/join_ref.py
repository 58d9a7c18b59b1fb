"""Exact CPU reference of the joins (numpy and pyarrow only): the pairs of an inner equi-join and the passing probe rows
of a semi, anti or null-aware anti join, per the semantics of include/dfgpu.h.

A key is a list of parts, each a numpy array or a pyarrow array (which may hold nulls), integer or Utf8.  Two keys are
equal when every part is equal: integers by value, Utf8 byte for byte.  A key with a null part never matches.
* inner: every (probe row, build row) pair with equal keys; the pairs' order is unspecified, so callers compare them as a
  sorted multiset;
* semi: the probe rows with a match; anti: the probe rows without one, a row with a null part included;
* null-aware anti (NOT IN): every probe row when the build side is empty; otherwise none when some build key has a null
  part, and else the rows with no null part and no match.
Semi and anti results are probe row numbers in probe order."""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc

from datafusion_archive_b200 import _abi as A


def _is_arrow(a):
    return isinstance(a, (pa.Array, pa.ChunkedArray))


def _valid(a):
    return np.asarray(a.is_valid()) if _is_arrow(a) else np.ones(len(a), dtype=bool)


def _int_words(a):
    """(sign, 64-bit word) columns of an integer part: equal exactly when the values are equal, whatever the dtypes."""
    v = a.fill_null(0).to_numpy(zero_copy_only=False) if _is_arrow(a) else np.asarray(a)
    v = np.asarray(v)
    if v.dtype.kind == "i":
        w = v.astype(np.int64)
        return (w < 0).astype(np.int64), w.view(np.uint64)
    return np.zeros(len(v), np.int64), v.astype(np.uint64)


def _part_codes(p, b):
    """Columns identifying each value of one key part across both sides (probe rows first), and the valid masks."""
    p, b = (pa.array(x) if isinstance(x, list) or (not _is_arrow(x) and np.asarray(x).dtype.kind in "OUS") else x for x in (p, b))
    pv, bv = _valid(p), _valid(b)
    types = [x.type for x in (p, b) if _is_arrow(x) and (pa.types.is_string(x.type) or pa.types.is_large_string(x.type))]
    if types:
        both = pa.chunked_array([pa.array(x).cast(types[0]) if not _is_arrow(x) or x.type != types[0] else x for x in (p, b)], type=types[0])
        enc = pc.dictionary_encode(both.combine_chunks())
        return [np.asarray(enc.indices.fill_null(0).to_numpy(zero_copy_only=False), dtype=np.int64)], pv, bv
    ps, pw = _int_words(p)
    bs, bw = _int_words(b)
    return [np.concatenate([ps, bs]), np.concatenate([pw, bw])], pv, bv


def _key_ids(pkeys, bkeys):
    """(probe key ids, probe valid, build key ids, build valid): equal keys have equal ids."""
    n_p, n_b = len(pkeys[0]), len(bkeys[0])
    pv, bv = np.ones(n_p, bool), np.ones(n_b, bool)
    cols = []
    for pk, bk in zip(pkeys, bkeys):
        c, pvalid, bvalid = _part_codes(pk, bk)
        cols += c
        pv &= pvalid
        bv &= bvalid
    if n_p + n_b == 0:
        return np.zeros(0, np.int64), pv, np.zeros(0, np.int64), bv
    _, ids = np.unique(np.rec.fromarrays(cols), return_inverse=True)
    ids = ids.reshape(-1)
    return ids[:n_p], pv, ids[n_p:], bv


def inner(pkeys, bkeys):
    """(probe rows, build rows) of every matching pair."""
    n_p, n_b = len(pkeys[0]), len(bkeys[0])
    if n_p == 0 or n_b == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    pid, pv, bid, bv = _key_ids(pkeys, bkeys)
    brows = np.nonzero(bv)[0]
    order = np.argsort(bid[brows], kind="stable")
    sorted_ids, sorted_rows = bid[brows][order], brows[order]
    lo = np.searchsorted(sorted_ids, pid, "left")
    hi = np.searchsorted(sorted_ids, pid, "right")
    cnt = np.where(pv, hi - lo, 0)
    total = int(cnt.sum())
    prow = np.repeat(np.arange(n_p), cnt)
    first = np.repeat(lo, cnt) + (np.arange(total) - np.repeat(np.cumsum(cnt) - cnt, cnt))
    return prow, sorted_rows[first]


def passing(kind, pkeys, bkeys):
    """The probe rows a semi (A.JOIN_SEMI), anti (A.JOIN_ANTI) or null-aware anti (A.JOIN_ANTI_NULL_AWARE) join passes, in probe order."""
    n_p, n_b = len(pkeys[0]), len(bkeys[0])
    if n_p == 0:
        return np.zeros(0, np.int64)
    pid, pv, bid, bv = _key_ids(pkeys, bkeys)
    hit = pv & np.isin(pid, bid[bv])
    if kind == A.JOIN_SEMI:
        ok = hit
    elif kind == A.JOIN_ANTI:
        ok = ~hit
    elif kind == A.JOIN_ANTI_NULL_AWARE:
        ok = np.ones(n_p, bool) if n_b == 0 else (pv & ~hit if bv.all() else np.zeros(n_p, bool))
    else:
        raise ValueError(kind)
    return np.flatnonzero(ok).astype(np.int64)


def same_pairs(got, exp):
    """got and exp, (probe rows, build rows), hold the same pairs."""
    g = np.lexsort((got[1], got[0]))
    e = np.lexsort((exp[1], exp[0]))
    assert len(got[0]) == len(exp[0]), (len(got[0]), len(exp[0]))
    assert np.array_equal(np.asarray(got[0])[g], np.asarray(exp[0])[e])
    assert np.array_equal(np.asarray(got[1])[g], np.asarray(exp[1])[e])
