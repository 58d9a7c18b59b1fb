"""ctypes mirror of include/dfgpu.h (the C ABI of the sm_90a engine).

Only plain-old-data definitions live here so that the test-only CPU checker under
tests/ can share them.  Nothing in this module touches a GPU.
"""
import ctypes as C
import os

import numpy as np

ABI_VERSION = 2

# error codes
OK, ERR_GENERAL, ERR_EXECUTION, ERR_NOT_IMPLEMENTED, ERR_INVALID_COLUMN, ERR_INTERNAL, ERR_ARROW, ERR_CUDA, ERR_OOM = range(9)

# dtypes (arrow::datatypes::DataType)
BOOL, INT8, INT16, INT32, INT64, UINT8, UINT16, UINT32, UINT64, FLOAT32, FLOAT64, UTF8 = range(1, 13)

DTYPE_NAMES = {
    BOOL: "Boolean", INT8: "Int8", INT16: "Int16", INT32: "Int32", INT64: "Int64", UINT8: "UInt8",
    UINT16: "UInt16", UINT32: "UInt32", UINT64: "UInt64", FLOAT32: "Float32", FLOAT64: "Float64", UTF8: "Utf8",
}
NP_OF = {
    INT8: np.int8, INT16: np.int16, INT32: np.int32, INT64: np.int64, UINT8: np.uint8, UINT16: np.uint16,
    UINT32: np.uint32, UINT64: np.uint64, FLOAT32: np.float32, FLOAT64: np.float64,
}
DTYPE_OF_NP = {np.dtype(v): k for k, v in NP_OF.items()}

# expression opcodes
OP_COL, OP_LIT, OP_CAST, OP_LIT_UTF8 = 1, 2, 3, 4
OP_ADD, OP_SUB, OP_MUL, OP_DIV = 10, 11, 12, 13
OP_EQ, OP_NE, OP_LT, OP_LE, OP_GT, OP_GE = 20, 21, 22, 23, 24, 25
OP_LIKE, OP_NOT_LIKE = 26, 27
UTF8_LITERAL_MAX = 4096  # longest Utf8 literal or LIKE pattern, in bytes
OP_AND, OP_OR = 30, 31
OP_FN = 40

# built-in scalar functions (DFGPU_OP_FN: `col` = code); all Float64 -> Float64
FN_SQRT, FN_ABS, FN_FLOOR, FN_CEIL, FN_TRUNC, FN_ROUND, FN_SIGNUM = 1, 2, 3, 4, 5, 6, 7
FN_EXP, FN_LN, FN_LOG2, FN_LOG10 = 8, 9, 10, 11
FN_SIN, FN_COS, FN_TAN, FN_ASIN, FN_ACOS, FN_ATAN = 12, 13, 14, 15, 16, 17
FN_POWER, FN_ATAN2 = 18, 19
FN_CODES = {
    "sqrt": FN_SQRT, "abs": FN_ABS, "floor": FN_FLOOR, "ceil": FN_CEIL, "trunc": FN_TRUNC, "round": FN_ROUND,
    "signum": FN_SIGNUM, "exp": FN_EXP, "ln": FN_LN, "log2": FN_LOG2, "log10": FN_LOG10, "sin": FN_SIN, "cos": FN_COS,
    "tan": FN_TAN, "asin": FN_ASIN, "acos": FN_ACOS, "atan": FN_ATAN, "power": FN_POWER, "atan2": FN_ATAN2,
}
FN_ARITY = {code: (2 if code in (FN_POWER, FN_ATAN2) else 1) for code in FN_CODES.values()}

# Utf8 functions (DFGPU_OP_UTF8_FN: `col` = code, `dtype` = result type); the Utf8 operand first, then Int64 literals
OP_UTF8_FN = 41
# CASE WHEN c1 THEN v1 .. [ELSE e] END (DFGPU_OP_CASE): operands c1 v1 .. cn vn [e] first, `col` = their number, `dtype` =
# the result type
OP_CASE = 42
UTF8FN_UPPER, UTF8FN_LOWER, UTF8FN_TRIM, UTF8FN_LTRIM, UTF8FN_RTRIM = 1, 2, 3, 4, 5
UTF8FN_SUBSTR_FROM, UTF8FN_SUBSTR, UTF8FN_LENGTH, UTF8FN_OCTET_LENGTH = 6, 7, 8, 9
UTF8_FN_CODES = {
    "upper": UTF8FN_UPPER, "lower": UTF8FN_LOWER, "trim": UTF8FN_TRIM, "ltrim": UTF8FN_LTRIM, "rtrim": UTF8FN_RTRIM,
    "substr": UTF8FN_SUBSTR, "length": UTF8FN_LENGTH, "char_length": UTF8FN_LENGTH, "octet_length": UTF8FN_OCTET_LENGTH,
}

AGG_MIN, AGG_MAX, AGG_SUM, AGG_COUNT, AGG_COUNT_DISTINCT, AGG_AVG = 1, 2, 3, 4, 5, 6
# dfgpu_window's rank functions (the aggregates above are its other functions)
WIN_ROW_NUMBER, WIN_RANK, WIN_DENSE_RANK = 16, 17, 18

# dfgpu_join_semi kinds
JOIN_SEMI, JOIN_ANTI, JOIN_ANTI_NULL_AWARE = 1, 2, 3


class Col(C.Structure):
    _fields_ = [
        ("dtype", C.c_int32), ("_pad", C.c_int32), ("len", C.c_int64), ("offset", C.c_int64),
        ("values", C.c_void_p), ("validity", C.c_void_p), ("offsets", C.c_void_p), ("values_bytes", C.c_int64),
    ]


class _Lit(C.Union):
    _fields_ = [("f64", C.c_double), ("i64", C.c_int64), ("u64", C.c_uint64), ("f32", C.c_float), ("str", C.c_void_p)]


class Insn(C.Structure):
    _fields_ = [("op", C.c_int32), ("col", C.c_int32), ("dtype", C.c_int32), ("_pad", C.c_int32), ("lit", _Lit)]


class Agg(C.Structure):
    _fields_ = [
        ("func", C.c_int32), ("arg_len", C.c_int32), ("arg", C.POINTER(Insn)), ("out_dtype", C.c_int32), ("_pad", C.c_int32),
    ]


def repo_root():
    return os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def make_col(arr, keepalive):
    """Borrowed dfgpu_col view of a numpy array, a pyarrow primitive/string array, or a list of str."""
    c = Col()
    try:
        import pyarrow as pa
    except ImportError:  # pragma: no cover
        pa = None
    if pa is not None and isinstance(arr, (pa.Array, pa.ChunkedArray)):
        if isinstance(arr, pa.ChunkedArray):
            arr = arr.combine_chunks()
        bufs = arr.buffers()
        keepalive.append(arr)
        c.len = len(arr)
        c.offset = arr.offset
        if arr.null_count and bufs[0] is not None:
            c.validity = bufs[0].address
        if pa.types.is_string(arr.type) or pa.types.is_binary(arr.type):
            c.dtype = UTF8
            c.offsets = bufs[1].address
            c.values = bufs[2].address if bufs[2] is not None else None
            c.values_bytes = bufs[2].size if bufs[2] is not None else 0
        elif pa.types.is_boolean(arr.type):  # BooleanArray: bit-packed values, LSB first
            c.dtype = BOOL
            c.values = bufs[1].address
        else:
            c.dtype = DTYPE_OF_NP[np.dtype(arr.type.to_pandas_dtype())]
            c.values = bufs[1].address
        return c
    if isinstance(arr, (list, tuple)) and (len(arr) == 0 or isinstance(arr[0], str)):
        import pyarrow as pa2
        return make_col(pa2.array(list(arr), type=pa2.string()), keepalive)
    a = np.ascontiguousarray(arr)
    if a.dtype == np.bool_:  # numpy bools -> arrow BooleanArray layout
        bits = np.packbits(a, bitorder="little")
        keepalive.append(bits)
        c.dtype, c.len, c.offset, c.values = BOOL, a.shape[0], 0, bits.ctypes.data
        return c
    keepalive.append(a)
    c.dtype = DTYPE_OF_NP[a.dtype]
    c.len = a.shape[0]
    c.offset = 0
    c.values = a.ctypes.data
    return c


def make_cols(arrays, keepalive):
    cols = (Col * max(1, len(arrays)))()
    for i, a in enumerate(arrays):
        cols[i] = make_col(a, keepalive)
    return cols


def make_programs(progs, keepalive):
    """list[list[Insn-tuple]] -> (const dfgpu_insn* const*, const int*, n)"""
    n = len(progs)
    arrs = []
    for p in progs:
        arr = (Insn * max(1, len(p)))(*p)
        arrs.append(arr)
    ptrs = (C.POINTER(Insn) * max(1, n))(*[C.cast(a, C.POINTER(Insn)) for a in arrs])
    lens = (C.c_int * max(1, n))(*[len(p) for p in progs])
    keepalive.extend(arrs)
    keepalive.append(ptrs)
    keepalive.append(lens)
    return ptrs, lens, n


def make_aggs(aggs, keepalive):
    """list[(func, program, out_dtype)] -> dfgpu_agg[]"""
    out = (Agg * max(1, len(aggs)))()
    for i, (func, prog, out_dtype) in enumerate(aggs):
        arr = (Insn * max(1, len(prog)))(*prog)
        keepalive.append(arr)
        out[i].func = func
        out[i].arg = C.cast(arr, C.POINTER(Insn))
        out[i].arg_len = len(prog)
        out[i].out_dtype = out_dtype
    return out
