"""ctypes binding of libdfgpu.so (the sm_90a engine behind include/dfgpu.h).

This is the harness-side view of the C ABI: tests and bench.py drive the kernels through it with
host (numpy / pyarrow) buffers, exactly as the Rust shim of INTEGRATION.md would.  There is no CPU
fallback: if the shared library is missing or no H100 is present, calls raise.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from . import _abi as A

_LIB = None


class DfGpuError(Exception):
    def __init__(self, code, msg):
        super().__init__("dfgpu error %d: %s" % (code, msg))
        self.code, self.msg = code, msg


def lib_path():
    # DFGPU_LIB: A/B-test another build of the same ABI (profiling experiments only)
    return os.environ.get("DFGPU_LIB") or os.path.join(os.path.dirname(os.path.abspath(__file__)), "libdfgpu.so")


def build(force=False):
    """Compile csrc/*.cu for sm_90a into libdfgpu.so (nvcc cross-compiles without a GPU)."""
    here = os.path.dirname(os.path.abspath(__file__))
    csrc = os.path.join(here, "csrc")
    so = lib_path()
    srcs = [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cu", ".cuh"))]
    srcs.append(os.path.join(A.repo_root(), "include", "dfgpu.h"))
    stale = not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs)
    if force or stale:
        subprocess.check_call(["make", "-C", csrc, "-s", "-j4"])
    return so


def lib():
    global _LIB
    if _LIB is not None:
        return _LIB
    so = lib_path()
    if not os.path.exists(so):
        raise RuntimeError("libdfgpu.so is not built (run __graft_entry__.build()); there is no CPU fallback")
    L = C.CDLL(so)
    PI = C.POINTER(A.Insn)
    vp = C.c_void_p
    L.dfgpu_last_error.restype = C.c_char_p
    L.dfgpu_init.argtypes = [C.c_int, C.POINTER(vp)]
    L.dfgpu_shutdown.argtypes = [vp]
    L.dfgpu_device_count.argtypes = [C.POINTER(C.c_int)]
    L.dfgpu_sync.argtypes = [vp]
    L.dfgpu_host_alloc.argtypes = [C.c_size_t, C.POINTER(vp)]
    L.dfgpu_host_free.argtypes = [vp]
    L.dfgpu_timer_start.argtypes = [vp]
    L.dfgpu_timer_stop.argtypes = [vp, C.POINTER(C.c_float)]
    L.dfgpu_flush_l2.argtypes = [vp]
    L.dfgpu_kernel_launches.argtypes = [vp, C.POINTER(C.c_int64)]
    L.dfgpu_profile_enable.argtypes = [vp, C.c_int]
    L.dfgpu_profile_get.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(C.c_int64)]
    L.dfgpu_batch_upload.argtypes = [vp, C.POINTER(A.Col), C.c_int, C.POINTER(vp)]
    L.dfgpu_batch_rows.argtypes = [vp, C.POINTER(C.c_int64)]
    L.dfgpu_batch_free.argtypes = [vp]
    L.dfgpu_filter_project.argtypes = [vp, vp, PI, C.c_int, C.POINTER(PI), C.POINTER(C.c_int), C.c_int, C.POINTER(vp)]
    L.dfgpu_filter_project_host.argtypes = [vp, C.POINTER(A.Col), C.c_int, PI, C.c_int, C.POINTER(PI), C.POINTER(C.c_int), C.c_int, C.c_int64, C.POINTER(vp)]
    L.dfgpu_result_col_host_ptr.argtypes = [vp, C.c_int, C.POINTER(vp)]
    L.dfgpu_result_on_host.argtypes = [vp, C.POINTER(C.c_int)]
    L.dfgpu_aggregate_create.argtypes = [vp, C.POINTER(PI), C.POINTER(C.c_int), C.c_int, C.POINTER(A.Agg), C.c_int, C.c_int64, C.POINTER(vp)]
    L.dfgpu_aggregate_set_predicate.argtypes = [vp, PI, C.c_int]
    L.dfgpu_aggregate_update.argtypes = [vp, vp]
    L.dfgpu_aggregate_update_host.argtypes = [vp, C.POINTER(A.Col), C.c_int, C.c_int64]
    L.dfgpu_aggregate_finish.argtypes = [vp, C.POINTER(vp)]
    L.dfgpu_aggregate_free.argtypes = [vp]
    L.dfgpu_result_shape.argtypes = [vp, C.POINTER(C.c_int64), C.POINTER(C.c_int)]
    L.dfgpu_result_col_dtype.argtypes = [vp, C.c_int, C.POINTER(C.c_int32)]
    L.dfgpu_result_col_bytes.argtypes = [vp, C.c_int, C.POINTER(C.c_int64)]
    L.dfgpu_result_col_nulls.argtypes = [vp, C.c_int, C.POINTER(C.c_int64)]
    L.dfgpu_result_copy_col.argtypes = [vp, C.c_int, vp, vp, vp]
    L.dfgpu_result_col_device_ptr.argtypes = [vp, C.c_int, C.POINTER(vp)]
    L.dfgpu_result_free.argtypes = [vp]
    L.dfgpu_comm_unique_id.argtypes = [C.c_char_p]
    L.dfgpu_comm_init.argtypes = [vp, C.c_int, C.c_int, C.c_char_p]
    L.dfgpu_comm_destroy.argtypes = [vp]
    PC = C.POINTER(C.c_int)
    L.dfgpu_join_build.argtypes = [vp, vp, C.POINTER(PI), PC, C.c_int, PC, C.c_int, C.POINTER(vp)]
    L.dfgpu_join_probe.argtypes = [vp, vp, C.POINTER(PI), PC, C.c_int, PC, C.c_int, PC, C.c_int, C.POINTER(vp)]
    L.dfgpu_join_semi.argtypes = [vp, vp, C.POINTER(PI), PC, C.c_int, C.c_int, PC, C.c_int, C.POINTER(vp)]
    L.dfgpu_join_free.argtypes = [vp]
    L.dfgpu_sort.argtypes = [vp, vp, PI, C.c_int, C.POINTER(PI), PC, C.POINTER(C.c_int32), C.c_int, C.c_int64, C.POINTER(vp)]
    L.dfgpu_result_as_batch.argtypes = [vp, C.POINTER(vp)]
    L.dfgpu_window.argtypes = [vp, vp, C.POINTER(PI), PC, C.c_int, C.POINTER(PI), PC, C.POINTER(C.c_int32), C.c_int, C.POINTER(A.Agg), C.c_int,
                               C.POINTER(vp)]
    if L.dfgpu_abi_version() != A.ABI_VERSION:
        raise RuntimeError("libdfgpu.so ABI version mismatch")
    _LIB = L
    return L


def check(rc):
    if rc != 0:
        raise DfGpuError(rc, lib().dfgpu_last_error().decode())


class PinnedBuffer:
    """cudaMallocHost-backed numpy array (Arrow buffers allocated this way upload as one DMA)."""

    def __init__(self, shape, dtype):
        self.dtype = np.dtype(dtype)
        n = int(np.prod(shape))
        self.ptr = C.c_void_p()
        check(lib().dfgpu_host_alloc(max(8, n * self.dtype.itemsize), C.byref(self.ptr)))
        buf = (C.c_uint8 * (n * self.dtype.itemsize)).from_address(self.ptr.value)
        self.array = np.frombuffer(buf, dtype=self.dtype, count=n).reshape(shape)

    def free(self):
        if self.ptr:
            self.array = None
            lib().dfgpu_host_free(self.ptr)
            self.ptr = None


class Result:
    """An operator's output.  `shape_on_first_use`: the operator may have returned before its kernel finished
    (dfgpu_filter_project), so the shape is read, waiting for the kernel, when nrows / ncols is first asked for;
    other results read it here, so that it stays available after free()."""

    def __init__(self, ctx, handle, shape_on_first_use=False):
        self.ctx, self.h = ctx, handle
        self._shape = None
        if not shape_on_first_use:
            self._read_shape()

    def _read_shape(self):
        if self._shape is None:
            if not self.h:
                raise RuntimeError("the result was freed before its shape was read")
            nrows, ncols = C.c_int64(), C.c_int()
            check(lib().dfgpu_result_shape(self.h, C.byref(nrows), C.byref(ncols)))
            self._shape = (nrows.value, ncols.value)
        return self._shape

    @property
    def nrows(self):
        return self._read_shape()[0]

    @property
    def ncols(self):
        return self._read_shape()[1]

    def dtype(self, i):
        dt = C.c_int32()
        check(lib().dfgpu_result_col_dtype(self.h, i, C.byref(dt)))
        return dt.value

    @property
    def on_host(self):
        """True when the columns live in pinned host memory (chunk-pipelined filter_project_host)."""
        f = C.c_int()
        check(lib().dfgpu_result_on_host(self.h, C.byref(f)))
        return bool(f.value)

    def host_view(self, i):
        """Zero-copy numpy view of column i of a host-resident result (filter_project_host)."""
        p = C.c_void_p()
        check(lib().dfgpu_result_col_host_ptr(self.h, i, C.byref(p)))
        dt = np.dtype(A.NP_OF[self.dtype(i)])
        buf = (C.c_uint8 * (self.nrows * dt.itemsize)).from_address(p.value) if self.nrows else (C.c_uint8 * 0)()
        return np.frombuffer(buf, dtype=dt, count=self.nrows)

    def copy_into(self, i, dst):
        """Copy column i into a caller-allocated numpy buffer (first nrows elements)."""
        check(lib().dfgpu_result_copy_col(self.h, i, dst.ctypes.data, None, None))

    def columns(self):
        """All columns as numpy arrays; nullable columns come back as (values, valid_mask)."""
        from_fetch = _fetch_result(lib(), self.h)
        return from_fetch

    def free(self):
        if self.h:
            if self.ctx.h:  # after ctx.close() the device memory is gone with the context
                check(lib().dfgpu_result_free(self.h))
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def _fetch_result(L, handle):
    nrows, ncols = C.c_int64(), C.c_int()
    check(L.dfgpu_result_shape(handle, C.byref(nrows), C.byref(ncols)))
    n = nrows.value
    cols = []
    for i in range(ncols.value):
        dt, nulls = C.c_int32(), C.c_int64()
        check(L.dfgpu_result_col_dtype(handle, i, C.byref(dt)))
        check(L.dfgpu_result_col_nulls(handle, i, C.byref(nulls)))
        validity = np.zeros((n + 7) // 8, dtype=np.uint8) if nulls.value else None
        vptr = validity.ctypes.data if validity is not None else None
        if dt.value == A.UTF8:
            nb = C.c_int64()
            check(L.dfgpu_result_col_bytes(handle, i, C.byref(nb)))
            data = np.zeros(max(1, nb.value), dtype=np.uint8)
            offs = np.zeros(n + 1, dtype=np.int32)
            check(L.dfgpu_result_copy_col(handle, i, data.ctypes.data, vptr, offs.ctypes.data))
            raw = data.tobytes()
            vals = [raw[offs[k]:offs[k + 1]].decode() for k in range(n)]
        elif dt.value == A.BOOL:  # bit-packed, LSB first
            packed = np.zeros(max(1, (n + 7) // 8), dtype=np.uint8)
            check(L.dfgpu_result_copy_col(handle, i, packed.ctypes.data, vptr, None))
            vals = np.unpackbits(packed, bitorder="little")[:n].astype(bool)
        else:
            vals = np.zeros(max(1, n), dtype=A.NP_OF[dt.value])
            check(L.dfgpu_result_copy_col(handle, i, vals.ctypes.data, vptr, None))
            vals = vals[:n]
        if validity is not None:
            cols.append((vals, np.unpackbits(validity, bitorder="little")[:n].astype(bool)))
        else:
            cols.append(vals)
    return cols


def check_program(schema_dtypes, expr):
    """dfgpu_check_program: type-check `expr` against a schema (list of dtype codes) on the host, no GPU.
    Returns the result dtype; raises DfGpuError exactly as the operators would."""
    prog = expr.program(list(schema_dtypes))
    arr = (A.Insn * max(1, len(prog)))(*prog)
    dts = (C.c_int32 * max(1, len(schema_dtypes)))(*schema_dtypes)
    out = C.c_int32()
    L = lib()
    L.dfgpu_check_program.argtypes = [C.POINTER(C.c_int32), C.c_int, C.POINTER(A.Insn), C.c_int, C.POINTER(C.c_int32)]
    check(L.dfgpu_check_program(dts, len(schema_dtypes), arr, len(prog), C.byref(out)))
    return out.value


def utf8_like_host(s, pattern):
    """dfgpu_utf8_like_host: (match, pattern class) of `s LIKE pattern` (bytes or str) by the engine's own pattern
    compiler and matcher, on the host.  Classes: 0 exact, 1 prefix, 2 suffix, 3 contains, 4 general."""
    s = s.encode("utf-8") if isinstance(s, str) else bytes(s)
    pattern = pattern.encode("utf-8") if isinstance(pattern, str) else bytes(pattern)
    m, cls = C.c_int32(), C.c_int32()
    L = lib()
    L.dfgpu_utf8_like_host.argtypes = [C.c_char_p, C.c_int64, C.c_char_p, C.c_int64, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    check(L.dfgpu_utf8_like_host(s, len(s), pattern, len(pattern), C.byref(m), C.byref(cls)))
    return bool(m.value), cls.value


def utf8_fn_host(s, expr):
    """dfgpu_utf8_fn_host: the value of `expr`, a Utf8 function nest over column 0, for the one string `s` (bytes or str),
    by the engine's own per-row code on the host: bytes for a Utf8 result, int for an Int64 one."""
    s = s.encode("utf-8") if isinstance(s, str) else bytes(s)
    prog = expr.program([A.UTF8])
    arr = (A.Insn * len(prog))(*prog)
    out = C.create_string_buffer(max(1, len(s)))
    out_len, out_int, out_dtype = C.c_int64(), C.c_int64(), C.c_int32()
    L = lib()
    L.dfgpu_utf8_fn_host.argtypes = [C.c_char_p, C.c_int64, C.POINTER(A.Insn), C.c_int, C.c_char_p, C.POINTER(C.c_int64),
                                     C.POINTER(C.c_int64), C.POINTER(C.c_int32)]
    check(L.dfgpu_utf8_fn_host(s, len(s), arr, len(prog), out, C.byref(out_len), C.byref(out_int), C.byref(out_dtype)))
    return out.raw[:out_len.value] if out_dtype.value == A.UTF8 else out_int.value


class Batch:
    def __init__(self, ctx, handle, schema):
        self.ctx, self.h, self.schema = ctx, handle, schema
        n = C.c_int64()
        lib().dfgpu_batch_rows(self.h, C.byref(n))
        self.nrows = n.value

    def free(self):
        if self.h:
            if self.ctx.h:
                check(lib().dfgpu_batch_free(self.h))
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class GpuContext:
    """One dfgpu_ctx = one H100 + stream + memory pool."""

    def __init__(self, device=0):
        self.h = C.c_void_p()
        check(lib().dfgpu_init(device, C.byref(self.h)))
        self.device = device

    # -- data movement ------------------------------------------------------------------------
    def upload(self, arrays):
        keep = []
        cols = A.make_cols(arrays, keep)
        out = C.c_void_p()
        check(lib().dfgpu_batch_upload(self.h, cols, len(arrays), C.byref(out)))
        return Batch(self, out, [cols[i].dtype for i in range(len(arrays))])

    # -- FilterRelation + ProjectRelation -------------------------------------------------------
    def filter_project(self, batch, pred=None, proj=()):
        schema = batch.schema
        pprog = pred.program(schema) if pred is not None else []
        parr = (A.Insn * max(1, len(pprog)))(*pprog)
        keep = []
        ptrs, lens, n = A.make_programs([e.program(schema) for e in proj], keep)
        out = C.c_void_p()
        check(lib().dfgpu_filter_project(self.h, batch.h, parr, len(pprog), ptrs, lens, n, C.byref(out)))
        return Result(self, out, shape_on_first_use=True)

    def filter_project_host(self, arrays, pred=None, proj=(), chunk_rows=0):
        """Host buffers in, host (pinned) buffers out; upload / kernel / download pipelined by chunk."""
        keep = []
        cols = A.make_cols(arrays, keep)
        schema = [cols[i].dtype for i in range(len(arrays))]
        pprog = pred.program(schema) if pred is not None else []
        parr = (A.Insn * max(1, len(pprog)))(*pprog)
        ptrs, lens, n = A.make_programs([e.program(schema) for e in proj], keep)
        out = C.c_void_p()
        check(lib().dfgpu_filter_project_host(self.h, cols, len(arrays), parr, len(pprog), ptrs, lens, n, chunk_rows, C.byref(out)))
        return Result(self, out)

    # -- AggregateRelation ------------------------------------------------------------------------
    def aggregate(self, batches, keys=(), aggs=(), expected_groups=0, pred=None):
        """AggregateRelation over `batches`; `pred` = the WHERE clause of a Selection under it, fused into the scan."""
        if isinstance(batches, Batch):
            batches = [batches]
        schema = batches[0].schema
        keep = []
        kptrs, klens, nk = A.make_programs([k.program(schema) for k in keys], keep)
        aggarr = A.make_aggs([a.lower(schema) for a in aggs], keep)
        st = C.c_void_p()
        check(lib().dfgpu_aggregate_create(self.h, kptrs, klens, nk, aggarr, len(aggs), expected_groups, C.byref(st)))
        try:
            if pred is not None:
                pprog = pred.program(schema)
                parr = (A.Insn * max(1, len(pprog)))(*pprog)
                check(lib().dfgpu_aggregate_set_predicate(st, parr, len(pprog)))
            for b in batches:
                check(lib().dfgpu_aggregate_update(st, b.h))
            out = C.c_void_p()
            check(lib().dfgpu_aggregate_finish(st, C.byref(out)))
            return Result(self, out)
        finally:
            lib().dfgpu_aggregate_free(st)

    def aggregate_host(self, arrays, keys=(), aggs=(), expected_groups=0, pred=None, chunk_rows=0):
        """AggregateRelation over one big HOST batch: chunked H2D overlapped with the scan inside the library."""
        keep = []
        cols = A.make_cols(arrays, keep)
        schema = [cols[i].dtype for i in range(len(arrays))]
        kptrs, klens, nk = A.make_programs([k.program(schema) for k in keys], keep)
        aggarr = A.make_aggs([a.lower(schema) for a in aggs], keep)
        st = C.c_void_p()
        check(lib().dfgpu_aggregate_create(self.h, kptrs, klens, nk, aggarr, len(aggs), expected_groups, C.byref(st)))
        try:
            if pred is not None:
                pprog = pred.program(schema)
                parr = (A.Insn * max(1, len(pprog)))(*pprog)
                check(lib().dfgpu_aggregate_set_predicate(st, parr, len(pprog)))
            check(lib().dfgpu_aggregate_update_host(st, cols, len(arrays), chunk_rows))
            out = C.c_void_p()
            check(lib().dfgpu_aggregate_finish(st, C.byref(out)))
            return Result(self, out)
        finally:
            lib().dfgpu_aggregate_free(st)

    # -- inner equi-join ---------------------------------------------------------------------------
    def join_build(self, batch, keys, keep_cols=None):
        """dfgpu_join_build: the hash table over `batch` (the right input) on the integer or Utf8 key
        expressions `keys`.  `keep_cols` (default: every column) are the columns later probes may return; the batch may
        be freed after."""
        keep = []
        kptrs, klens, nk = A.make_programs([k.program(batch.schema) for k in keys], keep)
        cols = list(range(len(batch.schema))) if keep_cols is None else list(keep_cols)
        carr = (C.c_int * max(1, len(cols)))(*cols)
        out = C.c_void_p()
        check(lib().dfgpu_join_build(self.h, batch.h, kptrs, klens, nk, carr, len(cols), C.byref(out)))
        return Join(self, out, keep_cols=cols)

    # -- ORDER BY / LIMIT / HAVING ------------------------------------------------------------------
    def sort(self, batch, keys=(), desc=None, keep=None, limit=-1):
        """dfgpu_sort: every column of `batch` (a Batch, or a device Result viewed in place), the rows where `keep` is true,
        stably ordered by the expressions `keys` (`desc[i]` true: descending), the first `limit` of them (< 0: all)."""
        view = None
        if isinstance(batch, Result):
            h = C.c_void_p()
            check(lib().dfgpu_result_as_batch(batch.h, C.byref(h)))
            view = Batch(self, h, [batch.dtype(i) for i in range(batch.ncols)])
            batch = view
        try:
            keep_alive = []
            kptrs, klens, nk = A.make_programs([k.program(batch.schema) for k in keys], keep_alive)
            kprog = keep.program(batch.schema) if keep is not None else []
            karr = (A.Insn * max(1, len(kprog)))(*kprog)
            d = list(desc) if desc is not None else [False] * nk
            darr = (C.c_int32 * max(1, nk))(*[int(bool(x)) for x in d])
            out = C.c_void_p()
            check(lib().dfgpu_sort(self.h, batch.h, karr, len(kprog), kptrs, klens, darr, nk, limit, C.byref(out)))
            return Result(self, out)
        finally:
            if view is not None:
                view.free()

    # -- window functions ----------------------------------------------------------------------------
    def window(self, batch, fns, partition=(), order=(), desc=None):
        """dfgpu_window: one column per function of `fns`, each (func, arg expression or None, out_dtype or 0) with func
        one of A.WIN_ROW_NUMBER / WIN_RANK / WIN_DENSE_RANK (arg None) or A.AGG_MIN / MAX / SUM / COUNT / AVG, over the
        rows of `batch` partitioned by the expressions `partition` and ordered by `order` (`desc[i]` true: descending),
        in the batch's row order."""
        keep = []
        pptrs, plens, npart = A.make_programs([k.program(batch.schema) for k in partition], keep)
        optrs, olens, nord = A.make_programs([k.program(batch.schema) for k in order], keep)
        d = list(desc) if desc is not None else [False] * nord
        darr = (C.c_int32 * max(1, nord))(*[int(bool(x)) for x in d])
        farr = A.make_aggs([(f, a.program(batch.schema) if a is not None else [], dt) for f, a, dt in fns], keep)
        out = C.c_void_p()
        check(lib().dfgpu_window(self.h, batch.h, pptrs, plens, npart, optrs, olens, darr, nord, farr, len(fns), C.byref(out)))
        return Result(self, out)

    # -- utilities ------------------------------------------------------------------------------
    def sync(self):
        check(lib().dfgpu_sync(self.h))

    def flush_l2(self):
        check(lib().dfgpu_flush_l2(self.h))

    def timer_start(self):
        check(lib().dfgpu_timer_start(self.h))

    def timer_stop(self):
        ms = C.c_float()
        check(lib().dfgpu_timer_stop(self.h, C.byref(ms)))
        return ms.value

    def kernel_launches(self):
        n = C.c_int64()
        check(lib().dfgpu_kernel_launches(self.h, C.byref(n)))
        return n.value

    def profile_enable(self, on=True):
        check(lib().dfgpu_profile_enable(self.h, int(on)))

    def profile_get(self):
        ms, n = C.c_double(), C.c_int64()
        check(lib().dfgpu_profile_get(self.h, C.byref(ms), C.byref(n)))
        return ms.value, n.value

    def comm_init(self, rank, world, unique_id):
        check(lib().dfgpu_comm_init(self.h, rank, world, unique_id))

    def close(self):
        if self.h:
            check(lib().dfgpu_shutdown(self.h))
            self.h = None


class Join:
    """A built join (dfgpu_join): probe it with any number of batches of the left input."""

    def __init__(self, ctx, handle, keep_cols):
        self.ctx, self.h, self.keep_cols = ctx, handle, keep_cols

    def probe(self, batch, keys, probe_cols=None, build_cols=None):
        """dfgpu_join_probe: one row per matching (probe row, build row) pair, the `probe_cols` of `batch` (default:
        all) followed by the `build_cols` of the build batch (default: every kept column)."""
        keep = []
        kptrs, klens, nk = A.make_programs([k.program(batch.schema) for k in keys], keep)
        pc = list(range(len(batch.schema))) if probe_cols is None else list(probe_cols)
        bc = list(self.keep_cols) if build_cols is None else list(build_cols)
        parr = (C.c_int * max(1, len(pc)))(*pc)
        barr = (C.c_int * max(1, len(bc)))(*bc)
        out = C.c_void_p()
        check(lib().dfgpu_join_probe(self.h, batch.h, kptrs, klens, nk, parr, len(pc), barr, len(bc), C.byref(out)))
        return Result(self.ctx, out)

    def semi(self, batch, keys, kind=A.JOIN_SEMI, probe_cols=None):
        """dfgpu_join_semi: the `probe_cols` of `batch` (default: all) of the probe rows that pass, in probe order.
        `kind` is A.JOIN_SEMI, A.JOIN_ANTI or A.JOIN_ANTI_NULL_AWARE (include/dfgpu.h has the rules)."""
        keep = []
        kptrs, klens, nk = A.make_programs([k.program(batch.schema) for k in keys], keep)
        pc = list(range(len(batch.schema))) if probe_cols is None else list(probe_cols)
        parr = (C.c_int * max(1, len(pc)))(*pc)
        out = C.c_void_p()
        check(lib().dfgpu_join_semi(self.h, batch.h, kptrs, klens, nk, kind, parr, len(pc), C.byref(out)))
        return Result(self.ctx, out)

    def free(self):
        if self.h:
            if self.ctx.h:
                check(lib().dfgpu_join_free(self.h))
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def comm_unique_id():
    buf = C.create_string_buffer(128)
    check(lib().dfgpu_comm_unique_id(buf))
    return buf.raw


def device_count():
    n = C.c_int()
    check(lib().dfgpu_device_count(C.byref(n)))
    return n.value
