"""The reference order of dfgpu_sort: np.lexsort over each key's order-preserving encoding, with the row number as the last
key so that ties keep the input order.  A key is (dtype, values, valid or None, desc); Utf8 values are bytes (or str)."""
import numpy as np

from datafusion_archive_b200 import _abi as A

_WIDTH = {A.INT8: 1, A.UINT8: 1, A.INT16: 2, A.UINT16: 2, A.INT32: 4, A.UINT32: 4, A.FLOAT32: 4, A.INT64: 8, A.UINT64: 8, A.FLOAT64: 8}
_UINT = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}


def encode(dtype, vals, valid=None):
    """Each row's order-preserving unsigned word (nulls 0): integers by value, floats with -0.0 below +0.0 and every NaN
    after +inf, Utf8 as the dense rank of its bytes (a proper prefix first; a null as '')."""
    n = len(vals)
    if dtype == A.UTF8:
        b = [(v.encode("utf-8", "surrogatepass") if isinstance(v, str) else bytes(v)) for v in vals]
        if valid is not None:
            b = [x if ok else b"" for x, ok in zip(b, valid)]
        rank = {s: i for i, s in enumerate(sorted(set(b)))}
        e = np.array([rank[x] for x in b], dtype=np.uint64)
    else:
        w = _WIDTH[dtype]
        u = _UINT[w]
        sign = np.uint64(1 << (8 * w - 1))
        raw = np.asarray(vals, dtype=A.NP_OF[dtype]).view(u).astype(np.uint64)
        if dtype in (A.FLOAT32, A.FLOAT64):
            mask = np.uint64((1 << (8 * w)) - 1)
            f = np.asarray(vals, dtype=A.NP_OF[dtype])
            neg = (raw & sign) != 0
            e = np.where(neg, ~raw & mask, raw ^ sign)
            e = np.where(np.isnan(f), mask, e)
        elif dtype in (A.INT8, A.INT16, A.INT32, A.INT64):
            e = raw ^ sign
        else:
            e = raw
    if valid is not None:
        e = np.where(np.asarray(valid, dtype=bool), e, np.uint64(0))
    return e.astype(np.uint64) if n else np.zeros(0, np.uint64)


def order(n, keys, keep=None):
    """The kept row numbers (keep: bool per row, or None) in dfgpu_sort's order."""
    rows = np.arange(n) if keep is None else np.flatnonzero(np.asarray(keep, dtype=bool))
    cols = [rows]
    for dtype, vals, valid, desc in reversed(keys):
        e = encode(dtype, vals, valid)[rows]
        # a descending key: the encoding complemented, i.e. its order reversed (as uint64, ~e reverses any width)
        cols.append(~e if desc else e)
        if valid is not None:
            v = np.asarray(valid, dtype=bool)[rows].astype(np.uint8)
            cols.append(1 - v if desc else v)
    return rows[np.lexsort(cols)] if len(rows) else rows
