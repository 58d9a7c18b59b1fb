"""ctypes wrapper around oracle/libdf_oracle.so — TEST INFRASTRUCTURE ONLY (the CPU restatement of
the reference's operators).  Imported by tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs; never by the product package."""
import ctypes as C
import os
import subprocess

import numpy as np

from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200.expr import col

_ROOT = A.repo_root()
_LIB = None


def build(force=False):
    so = os.path.join(_ROOT, "oracle", "libdf_oracle.so")
    src = os.path.join(_ROOT, "oracle", "df_oracle.cpp")
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", os.path.join(_ROOT, "oracle"), "-s"])
    return so


def lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(build())
        L.oracle_last_error.restype = C.c_char_p
        PI = C.POINTER(A.Insn)
        L.oracle_filter_project.argtypes = [C.POINTER(A.Col), C.c_int, C.c_int64, PI, C.c_int, C.POINTER(PI),
                                            C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_void_p)]
        L.oracle_aggregate.argtypes = [C.POINTER(A.Col), C.c_int, C.c_int64, C.POINTER(PI), C.POINTER(C.c_int), C.c_int,
                                       C.POINTER(A.Agg), C.c_int, C.POINTER(C.c_void_p)]
        L.oracle_result_shape.argtypes = [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int)]
        L.oracle_result_col_dtype.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int32)]
        L.oracle_result_col_bytes.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int64)]
        L.oracle_result_col_nulls.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int64)]
        L.oracle_result_copy_col.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        L.oracle_result_free.argtypes = [C.c_void_p]
        L.oracle_set_extensions.argtypes = [C.c_int, C.c_int]
        _LIB = L
    return _LIB


class OracleError(Exception):
    def __init__(self, code, msg):
        super().__init__("oracle error %d: %s" % (code, msg))
        self.code, self.msg = code, msg


def _check(rc):
    if rc != 0:
        raise OracleError(rc, lib().oracle_last_error().decode())


def fetch_result(L, prefix, handle):
    """Generic result reader shared with the product wrapper (same accessor shapes).
    Returns list of columns: numpy arrays (primitive, with .mask via tuple) or list[str]."""
    nrows, ncols = C.c_int64(), C.c_int()
    getattr(L, prefix + "_result_shape")(handle, C.byref(nrows), C.byref(ncols))
    cols = []
    for i in range(ncols.value):
        dt = C.c_int32()
        getattr(L, prefix + "_result_col_dtype")(handle, i, C.byref(dt))
        nulls = C.c_int64()
        getattr(L, prefix + "_result_col_nulls")(handle, i, C.byref(nulls))
        n = nrows.value
        validity = np.zeros((n + 7) // 8, dtype=np.uint8) if nulls.value else None
        vptr = validity.ctypes.data if validity is not None else None
        if dt.value == A.UTF8:
            nb = C.c_int64()
            getattr(L, prefix + "_result_col_bytes")(handle, i, C.byref(nb))
            data = np.zeros(max(1, nb.value), dtype=np.uint8)
            offs = np.zeros(n + 1, dtype=np.int32)
            rc = getattr(L, prefix + "_result_copy_col")(handle, i, data.ctypes.data, vptr, offs.ctypes.data)
            assert rc == 0
            raw = data.tobytes()
            vals = [raw[offs[k]:offs[k + 1]].decode() for k in range(n)]
        elif dt.value == A.BOOL:
            vals = np.zeros(max(1, n), dtype=np.uint8)
            rc = getattr(L, prefix + "_result_copy_col")(handle, i, vals.ctypes.data, vptr, None)
            assert rc == 0
            vals = vals[:n].astype(bool)
        else:
            vals = np.zeros(max(1, n), dtype=A.NP_OF[dt.value])
            rc = getattr(L, prefix + "_result_copy_col")(handle, i, vals.ctypes.data, vptr, None)
            assert rc == 0
            vals = vals[:n]
        if validity is not None:
            mask = np.unpackbits(validity, bitorder="little")[:n].astype(bool)
            cols.append((vals, mask))
        else:
            cols.append(vals)
    return cols


def set_extensions(filter_all_primitives=False, count=True):
    lib().oracle_set_extensions(int(filter_all_primitives), int(count))


def filter_project(arrays, pred=None, proj=(), batch_size=0, schema=None):
    """arrays: list of numpy / pyarrow arrays.  pred: Expr or None.  proj: list of Expr."""
    L = lib()
    keep = []
    cols = A.make_cols(arrays, keep)
    schema = schema or [c.dtype for c in cols[:len(arrays)]]
    pprog = pred.program(schema) if pred is not None else []
    parr = (A.Insn * max(1, len(pprog)))(*pprog)
    ptrs, lens, n = A.make_programs([e.program(schema) for e in proj], keep)
    out = C.c_void_p()
    _check(L.oracle_filter_project(cols, len(arrays), batch_size, parr, len(pprog), ptrs, lens, n, C.byref(out)))
    try:
        return fetch_result(L, "oracle", out)
    finally:
        L.oracle_result_free(out)


def aggregate(arrays, keys=(), aggs=(), batch_size=0, schema=None):
    """keys: list of Expr; aggs: list of expr.AggregateFunction."""
    L = lib()
    keep = []
    cols = A.make_cols(arrays, keep)
    schema = schema or [c.dtype for c in cols[:len(arrays)]]
    kptrs, klens, nk = A.make_programs([k.program(schema) for k in keys], keep)
    aggarr = A.make_aggs([a.lower(schema) for a in aggs], keep)
    out = C.c_void_p()
    _check(L.oracle_aggregate(cols, len(arrays), batch_size, kptrs, klens, nk, aggarr, len(aggs), C.byref(out)))
    try:
        return fetch_result(L, "oracle", out)
    finally:
        L.oracle_result_free(out)


def rows(arrays, pred, exprs):
    """FilterRelation + ProjectRelation: the value of each expression on each row that passes `pred`.  Filter gathers
    every fixed-width column, which the reference's filter() does for Float64 / Utf8 only (filter.rs:82-108)."""
    set_extensions(filter_all_primitives=True)
    try:
        return filter_project(arrays, pred, exprs)
    finally:
        set_extensions(filter_all_primitives=False)


def filtered_aggregate(arrays, pred, keys, aggs):
    """The reference's wiring of a WHERE under an aggregate: FilterRelation (gathers every column, dropping the bitmaps)
    feeding AggregateRelation (context.rs:126-139, 162-192)."""
    if pred is None:
        return aggregate(arrays, keys, aggs)
    return aggregate(rows(arrays, pred, [col(i) for i in range(len(arrays))]), keys, aggs)
