"""ctypes binding of libdfhost.so — the C++ mirror of the reference's ExecutionContext / Relation /
SQL planner API (csrc/host/).  `ExecutionContext.sql()` returns a pull-based Relation whose
`next()` yields host record batches, like the reference (src/execution/context.rs:44)."""
import ctypes as C
import os
import subprocess

import numpy as np

from . import _abi as A

_LIB = None


class ExecutionError(Exception):
    def __init__(self, code, msg):
        super().__init__("ExecutionError(code=%d): %s" % (code, msg))
        self.code, self.msg = code, msg


def lib_path():
    return os.path.join(os.path.dirname(os.path.abspath(__file__)), "libdfhost.so")


def build(force=False):
    here = os.path.dirname(os.path.abspath(__file__))
    hostdir = os.path.join(here, "csrc", "host")
    so = lib_path()
    srcs = [os.path.join(hostdir, f) for f in os.listdir(hostdir) if f.endswith((".cpp", ".h"))]
    dep = os.path.join(here, "libdfgpu.so")
    stale = not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs + [dep])
    if force or stale:
        subprocess.check_call(["make", "-C", hostdir, "-s", "-j4"])
    return so


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(lib_path()):
            raise RuntimeError("libdfhost.so is not built (run __graft_entry__.build())")
        L = C.CDLL(lib_path())
        vp, cp = C.c_void_p, C.c_char_p
        L.dfhost_last_error.restype = cp
        L.dfhost_free_string.argtypes = [vp]
        L.dfhost_catalog_new.argtypes = [C.POINTER(vp)]
        L.dfhost_catalog_free.argtypes = [vp]
        L.dfhost_catalog_add_table.argtypes = [vp, cp, C.c_int, C.POINTER(cp), C.POINTER(C.c_int32)]
        L.dfhost_catalog_add_function.argtypes = [vp, cp, C.c_int, C.POINTER(C.c_int32), C.c_int32]
        L.dfhost_catalog_add_builtin_functions.argtypes = [vp]
        L.dfhost_plan_sql.argtypes = [vp, cp, C.POINTER(vp)]
        L.dfhost_supertype.argtypes = [C.c_int32, C.c_int32, C.POINTER(C.c_int32)]
        L.dfhost_debug_f64.argtypes = [C.c_double, C.POINTER(vp)]
        L.dfhost_csv_open.argtypes = [cp, C.c_int, C.POINTER(cp), C.POINTER(C.c_int32), C.c_int64, C.POINTER(vp)]
        L.dfhost_datasource_next.argtypes = [vp, C.POINTER(vp)]
        L.dfhost_datasource_free.argtypes = [vp]
        L.dfhost_context_new.argtypes = [C.c_int, C.POINTER(vp)]
        L.dfhost_context_free.argtypes = [vp]
        L.dfhost_context_set_verbose.argtypes = [vp, C.c_int]
        L.dfhost_context_set_partition.argtypes = [vp, C.c_int, C.c_int, C.c_char_p]
        L.dfhost_register_csv.argtypes = [vp, cp, cp, C.c_int, C.POINTER(cp), C.POINTER(C.c_int32), C.c_int64]
        L.dfhost_register_memory.argtypes = [vp, cp, C.c_int, C.POINTER(cp), C.POINTER(A.Col), C.c_int64]
        L.dfhost_sql.argtypes = [vp, cp, C.POINTER(vp)]
        L.dfhost_plan_debug.argtypes = [vp, cp, C.POINTER(vp)]
        L.dfhost_relation_free.argtypes = [vp]
        L.dfhost_relation_schema.argtypes = [vp, C.POINTER(C.c_int)]
        L.dfhost_relation_field.argtypes = [vp, C.c_int, C.POINTER(vp), C.POINTER(C.c_int32)]
        L.dfhost_relation_next.argtypes = [vp, C.POINTER(vp)]
        L.dfhost_batch_free.argtypes = [vp]
        L.dfhost_batch_shape.argtypes = [vp, C.POINTER(C.c_int64), C.POINTER(C.c_int)]
        L.dfhost_batch_col.argtypes = [vp, C.c_int, C.POINTER(A.Col), C.POINTER(C.c_int64)]
        _LIB = L
    return _LIB


def _check(rc):
    if rc != 0:
        raise ExecutionError(rc, lib().dfhost_last_error().decode())


def _take_string(p):
    s = C.cast(p, C.c_char_p).value.decode()
    lib().dfhost_free_string(p)
    return s


def _names_dtypes(fields):
    names = (C.c_char_p * len(fields))(*[n.encode() for n, _ in fields])
    dts = (C.c_int32 * len(fields))(*[d for _, d in fields])
    return names, dts


class Catalog:
    """SchemaProvider for planner-only use (mirrors MockSchemaProvider, src/sqlplanner.rs:761-789)."""

    def __init__(self):
        self.h = C.c_void_p()
        _check(lib().dfhost_catalog_new(C.byref(self.h)))

    def add_table(self, name, fields):
        names, dts = _names_dtypes(fields)
        _check(lib().dfhost_catalog_add_table(self.h, name.encode(), len(fields), names, dts))

    def add_function(self, name, arg_dtypes, return_dtype):
        args = (C.c_int32 * len(arg_dtypes))(*arg_dtypes)
        _check(lib().dfhost_catalog_add_function(self.h, name.encode(), len(arg_dtypes), args, return_dtype))

    def add_builtin_functions(self):
        """The built-in scalar functions ExecutionContext plans and runs (sqrt, abs, power, ...)."""
        _check(lib().dfhost_catalog_add_builtin_functions(self.h))

    def plan(self, sql):
        """`format!("{:?}", plan)` of the logical plan for `sql`."""
        out = C.c_void_p()
        _check(lib().dfhost_plan_sql(self.h, sql.encode(), C.byref(out)))
        return _take_string(out)

    def __del__(self):
        try:
            lib().dfhost_catalog_free(self.h)
        except Exception:
            pass


def supertype(l, r):
    out = C.c_int32()
    lib().dfhost_supertype(l, r, C.byref(out))
    return out.value or None


def debug_f64(x):
    out = C.c_void_p()
    _check(lib().dfhost_debug_f64(float(x), C.byref(out)))
    return _take_string(out)


def _col_to_py(col, nulls):
    n = col.len
    if col.dtype == A.UTF8:
        offs = np.ctypeslib.as_array(C.cast(col.offsets, C.POINTER(C.c_int32)), shape=(col.offset + n + 1,))[col.offset:]
        raw = C.string_at(col.values, int(offs[-1])) if n else b""
        vals = [raw[offs[k]:offs[k + 1]].decode() for k in range(n)]
    elif col.dtype == A.BOOL:  # bit-packed, LSB first
        bits = np.frombuffer(C.string_at(col.values, (col.offset + n + 7) // 8), dtype=np.uint8) if n else np.zeros(0, np.uint8)
        vals = np.unpackbits(bits, bitorder="little")[col.offset:col.offset + n].astype(bool)
    else:
        dt = np.dtype(A.NP_OF[col.dtype])
        buf = C.string_at(col.values + col.offset * dt.itemsize, n * dt.itemsize) if n else b""
        vals = np.frombuffer(buf, dtype=dt).copy()
    if nulls:
        bits = np.frombuffer(C.string_at(col.validity, (col.offset + n + 7) // 8), dtype=np.uint8)
        mask = np.unpackbits(bits, bitorder="little")[col.offset:col.offset + n].astype(bool)
        return (vals, mask)
    return vals


def _batch_to_py(b):
    try:
        nrows, ncols = C.c_int64(), C.c_int()
        lib().dfhost_batch_shape(b, C.byref(nrows), C.byref(ncols))
        cols = []
        for i in range(ncols.value):
            col, nulls = A.Col(), C.c_int64()
            _check(lib().dfhost_batch_col(b, i, C.byref(col), C.byref(nulls)))
            cols.append(_col_to_py(col, nulls.value))
        return cols
    finally:
        lib().dfhost_batch_free(b)


class CsvDataSource:
    """CsvDataSource::new(filename, schema, batch_size) (src/execution/datasource.rs:39-43); CPU only."""

    def __init__(self, filename, fields, batch_size=1024):
        names, dts = _names_dtypes(fields)
        self.h = C.c_void_p()
        _check(lib().dfhost_csv_open(filename.encode(), len(fields), names, dts, batch_size, C.byref(self.h)))

    def next(self):
        b = C.c_void_p()
        _check(lib().dfhost_datasource_next(self.h, C.byref(b)))
        return _batch_to_py(b) if b else None

    def __del__(self):
        try:
            lib().dfhost_datasource_free(self.h)
        except Exception:
            pass


class Relation:
    def __init__(self, handle, keepalive):
        self.h, self._keep = handle, keepalive

    def schema(self):
        n = C.c_int()
        lib().dfhost_relation_schema(self.h, C.byref(n))
        out = []
        for i in range(n.value):
            name, dt = C.c_void_p(), C.c_int32()
            _check(lib().dfhost_relation_field(self.h, i, C.byref(name), C.byref(dt)))
            out.append((_take_string(name), dt.value))
        return out

    def next(self):
        """Relation::next(): list of columns (numpy arrays / list[str]) or None when exhausted."""
        b = C.c_void_p()
        _check(lib().dfhost_relation_next(self.h, C.byref(b)))
        if not b:
            return None
        return _batch_to_py(b)

    def collect(self):
        out = []
        while True:
            b = self.next()
            if b is None:
                return out
            out.append(b)

    def __del__(self):
        try:
            lib().dfhost_relation_free(self.h)
        except Exception:
            pass


class ExecutionContext:
    """ExecutionContext::new / register_datasource / sql (src/execution/context.rs:33-102)."""

    def __init__(self, device=0):
        self.h = C.c_void_p()
        self._keep = []
        _check(lib().dfhost_context_new(device, C.byref(self.h)))

    def register_csv(self, table, filename, fields, batch_size=1024):
        """CsvDataSource::new(filename, schema, batch_size) + register_datasource."""
        names, dts = _names_dtypes(fields)
        _check(lib().dfhost_register_csv(self.h, table.encode(), filename.encode(), len(fields), names, dts, batch_size))

    def register_memory(self, table, named_arrays, batch_size=0):
        """In-memory DataSource over numpy / pyarrow buffers (borrowed: kept alive by this context)."""
        arrays = [a for _, a in named_arrays]
        cols = A.make_cols(arrays, self._keep)
        names = (C.c_char_p * len(arrays))(*[n.encode() for n, _ in named_arrays])
        self._keep.append(cols)
        _check(lib().dfhost_register_memory(self.h, table.encode(), len(arrays), names, cols, batch_size))

    def set_partition(self, rank, world, unique_id):
        """One process per GPU: join the NCCL communicator (unique_id from engine.comm_unique_id() on rank 0)
        and work on this rank's row range of every table; aggregates return the global result on every rank."""
        _check(lib().dfhost_context_set_partition(self.h, rank, world, unique_id))

    def sql(self, sql):
        out = C.c_void_p()
        _check(lib().dfhost_sql(self.h, sql.encode(), C.byref(out)))
        return Relation(out, self)

    def plan(self, sql):
        out = C.c_void_p()
        _check(lib().dfhost_plan_debug(self.h, sql.encode(), C.byref(out)))
        return _take_string(out)

    def close(self):
        if self.h:
            lib().dfhost_context_free(self.h)
            self.h = None
