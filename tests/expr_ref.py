"""Exact reference evaluator of the whole expression language (datafusion_archive_b200/expr.py), per row, over numpy.

`evaluate(expr, table, read_bitmaps)` returns `Value(values, valid, err)`: each row's value, whether it is valid, and
its pending DivideByZero bit.  It is assembled from the per-feature references rather than restating them:
arithmetic from arith_ref (wrap-around, truncating `/`, `MIN / -1 = MIN`, one IEEE rounding per float operation), CAST
from cast_ref (Rust `as`), the Utf8 functions from utf8_fn_ref.  The rules below are those of DESIGN §7 and
include/dfgpu.h, each written once:

* Nulls.  A null operand gives a null result, and a computed null (arithmetic, And / Or, CAST, a function) has value 0.
  A plain column keeps its stored value under a null, and so does a CASE that selects it; GROUP BY SUM / MIN / MAX
  and GROUP BY keys read that stored value.
* Comparisons never give a null.  Numeric ones order a null as arrow 0.12's `bool_op` over `Option` does: `=` is true
  when both sides are null, `<` / `<=` are true when the left side is null, `>` / `>=` when the right side is.  Utf8
  ones compare bytes (a proper prefix first), a null equals a null and sorts below every string (`cmp3`).  LIKE and
  NOT LIKE on a null are false.
* Utf8 predicates and functions always read the Utf8 column's own nulls, under a WHERE too: they are evaluated over
  the batch before the scan.  An Int64 function result (`length`, `octet_length`) is 0 under a null source row and
  shares its validity, which a WHERE drops like any input bitmap.
* CASE.  A false or null condition is not taken; the result is the first taken WHEN's value, else the ELSE value,
  else a null with value 0.  The result takes the chosen branch's validity.
* DivideByZero.  A zero divisor (of any type, -0.0 included) where both operands are valid sets the row's bit.  A row
  raises only from the conditions up to and including the first true one and from the value chosen.  Only rows that
  survive the WHERE raise, and a WHERE itself reads every row (`raises`).
* WHERE.  `read_bitmaps=False` is the rule under a WHERE or a fused WHERE: every input column reads as valid, so only a
  CASE-made null is a null.
* Scalar functions take and return Float64.  The exact ones (`sqrt abs floor ceil trunc round signum`) follow the Rust
  f64 methods bit for bit; the others are computed in long double (values of dtype longdouble), to be compared within
  `test_scalar_fn_gpu.within_ulps`.
"""
import re
from collections import namedtuple

import numpy as np

import arith_ref
import cast_ref
import utf8_fn_ref
from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200.expr import BinaryExpr, Case, Cast, Column, Literal, ScalarFunction, Utf8Function

Value = namedtuple("Value", "values valid err")

CMP = (A.OP_EQ, A.OP_NE, A.OP_LT, A.OP_LE, A.OP_GT, A.OP_GE)
MATH = {A.OP_ADD: "+", A.OP_SUB: "-", A.OP_MUL: "*", A.OP_DIV: "/"}


# ---- Rust f64 methods (the exact scalar functions) ------------------------------------------------------------------
def rust_round(x):
    """f64::round: half away from zero.  x - trunc(x) is exact, so 0.49999999999999994 is not a half."""
    t = np.trunc(x)
    with np.errstate(invalid="ignore"):
        return np.where(np.abs(x - t) >= 0.5, t + np.copysign(1.0, x), t)


def rust_signum(x):
    return np.where(np.isnan(x), np.nan, np.copysign(1.0, x))


def rust_abs(x):
    return (x.view(np.uint64) & np.uint64(0x7FFFFFFFFFFFFFFF)).view(np.float64)


EXACT_REF = {"sqrt": np.sqrt, "abs": rust_abs, "floor": np.floor, "ceil": np.ceil, "trunc": np.trunc, "round": rust_round,
             "signum": rust_signum}
LONG = {"exp": np.exp, "ln": np.log, "log2": np.log2, "log10": np.log10, "sin": np.sin, "cos": np.cos, "tan": np.tan,
        "asin": np.arcsin, "acos": np.arccos, "atan": np.arctan}
LONG2 = {"power": np.power, "atan2": np.arctan2}
FN_NAME = {code: name for name, code in A.FN_CODES.items()}


# ---- Utf8 comparisons and LIKE --------------------------------------------------------------------------------------
def cmp3(a, b):
    if a is None or b is None:
        return (a is not None) - (b is not None)
    return (a > b) - (a < b)


def py_like(s, p):
    rx = b"".join(b"[\\x00-\\xff]*" if ch == 0x25 else b"[\\x00-\\xff][\\x80-\\xbf]*+" if ch == 0x5F else re.escape(bytes([ch]))
                  for ch in p)
    return re.fullmatch(rx, s, re.DOTALL) is not None


def like_ref(vals, p, neg=False):
    return np.array([v is not None and (py_like(v, p) != neg) for v in vals], bool)


_CMP3 = {A.OP_EQ: lambda c: c == 0, A.OP_NE: lambda c: c != 0, A.OP_LT: lambda c: c < 0, A.OP_LE: lambda c: c <= 0,
         A.OP_GT: lambda c: c > 0, A.OP_GE: lambda c: c >= 0}
_NP_CMP = {A.OP_EQ: np.equal, A.OP_NE: np.not_equal, A.OP_LT: np.less, A.OP_LE: np.less_equal, A.OP_GT: np.greater,
           A.OP_GE: np.greater_equal}


# ---- arithmetic and CAST at table sizes -----------------------------------------------------------------------------
def arith(op, a, b):
    """arith_ref.arith(op, a, b): (values, divide_by_zero).  Integers go to arith_ref as they are (their operands take
    few distinct values); float operands are rounded once by numpy's IEEE operation of the operand dtype, which
    test_expr_ref_cpu pins to arith_ref over its edge operands, since the exact rational path costs seconds per
    hundred thousand distinct pairs."""
    if a.dtype.kind != "f":
        return arith_ref.arith(op, a, b)
    bad = (b == 0) if op == "/" else np.zeros(len(a), bool)
    with np.errstate(all="ignore"):
        v = {"+": np.add, "-": np.subtract, "*": np.multiply, "/": np.divide}[op](a, b)
    return np.where(bad, a.dtype.type(0), v).astype(a.dtype), bad


def cast(values, dst):
    """cast_ref.cast (Rust `as`); between the float dtypes numpy's conversion, exact (Float32 -> Float64) or correctly
    rounded (Float64 -> Float32), which test_expr_ref_cpu pins to cast_ref."""
    dst = np.dtype(dst)
    if values.dtype.kind == "f" and dst.kind == "f":
        with np.errstate(over="ignore"):
            return values.astype(dst)
    return cast_ref.cast(values, dst)


# ---- the table ----------------------------------------------------------------------------------------------------
def column_data(a):
    """(dtype code, values, valid) of one input column: a numpy array, or a pyarrow array whose stored values under its
    nulls are read from its buffers.  Utf8 / binary values are an object array of bytes (b'' under a null)."""
    import pyarrow as pa
    if not isinstance(a, pa.Array):
        a = np.asarray(a)
        return (A.BOOL if a.dtype == np.bool_ else A.DTYPE_OF_NP[a.dtype]), a, np.ones(len(a), bool)
    n = len(a)
    valid = np.ones(n, bool) if a.null_count == 0 else np.asarray(a.is_valid().to_numpy(zero_copy_only=False), bool)
    if pa.types.is_binary(a.type) or pa.types.is_string(a.type) or pa.types.is_large_binary(a.type):
        vals = [b"" if v is None else (v.encode("utf-8") if isinstance(v, str) else bytes(v)) for v in a.to_pylist()]
        out = np.empty(n, dtype=object)
        out[:] = vals
        return A.UTF8, out, valid
    buf = a.buffers()[1]
    if pa.types.is_boolean(a.type):
        bits = np.unpackbits(np.frombuffer(buf, np.uint8), bitorder="little")[a.offset:a.offset + n].astype(bool)
        return A.BOOL, bits, valid
    npd = np.dtype(a.type.to_pandas_dtype())
    return A.DTYPE_OF_NP[npd], np.frombuffer(buf, npd)[a.offset:a.offset + n].copy(), valid


class Table:
    def __init__(self, arrays):
        self.cols = [column_data(a) for a in arrays]
        self.n = len(self.cols[0][1]) if self.cols else 0


# ---- the evaluator ------------------------------------------------------------------------------------------------
def evaluate(expr, table, read_bitmaps=True):
    """Value(values, valid, err) of `expr` on every row of `table` (a list of arrays, or a Table)."""
    t = table if isinstance(table, Table) else Table(table)
    return _ev(expr, t, read_bitmaps)


def raises(table, pred, exprs, read_bitmaps=None):
    """Whether filter/project (or an aggregate's fused WHERE) of `exprs` under `pred` raises DivideByZero, and the rows
    `pred` keeps (all rows without one).  The predicate reads the input bitmaps; the expressions read them only without
    a predicate (read_bitmaps=None)."""
    t = table if isinstance(table, Table) else Table(table)
    keep, err = np.ones(t.n, bool), np.zeros(t.n, bool)
    if pred is not None:
        p = _ev(pred, t, True)
        keep = p.values.astype(bool) & p.valid
        err = p.err.copy()
    rb = pred is None if read_bitmaps is None else read_bitmaps
    for e in exprs:
        err |= _ev(e, t, rb).err & keep
    return bool(err.any()), keep


def _zeros_like(v):
    if v.dtype == object:
        out = np.empty(len(v), dtype=object)
        out[:] = b""
        return out
    return np.zeros_like(v)


def _ev(e, t, rb):
    n = t.n
    none = np.zeros(n, bool)
    if isinstance(e, Column):
        dt, v, valid = t.cols[e.index]
        return Value(v, valid if (rb or dt == A.UTF8) else np.ones(n, bool), none)
    if isinstance(e, Literal):
        if e.dtype == A.UTF8:
            v = np.empty(n, dtype=object)
            v[:] = e.value.encode("utf-8") if isinstance(e.value, str) else bytes(e.value)
        elif e.dtype == A.BOOL:
            v = np.full(n, bool(e.value))
        else:
            v = np.full(n, e.value, dtype=A.NP_OF[e.dtype])
        return Value(v, np.ones(n, bool), none)
    if isinstance(e, Cast):
        x = _ev(e.expr, t, rb)
        v = cast(x.values, A.NP_OF[e.dtype])
        return Value(np.where(x.valid, v, v.dtype.type(0)), x.valid, x.err)
    if isinstance(e, Case):
        return _case(e, t, rb)
    if isinstance(e, ScalarFunction):
        return _scalar_fn(e, t, rb)
    if isinstance(e, Utf8Function):
        return _utf8_fn(e, t, rb)
    assert isinstance(e, BinaryExpr), e
    a, b = _ev(e.left, t, rb), _ev(e.right, t, rb)
    op = e.op
    err = a.err | b.err
    if op in (A.OP_LIKE, A.OP_NOT_LIKE):
        pat = b.values[0] if n else b""
        m = like_ref([x if ok else None for x, ok in zip(a.values, a.valid)], pat, op == A.OP_NOT_LIKE)
        return Value(m, np.ones(n, bool), err)
    if a.values.dtype == object:  # Utf8 comparison
        f = _CMP3[op]
        v = np.array([f(cmp3(x if va else None, y if vb else None)) for x, va, y, vb in zip(a.values, a.valid, b.values, b.valid)], bool)
        return Value(v.reshape(n), np.ones(n, bool), err)
    both = a.valid & b.valid
    if op in CMP:
        with np.errstate(invalid="ignore"):
            v = _NP_CMP[op](a.values, b.values)
        ln, rn = ~a.valid, ~b.valid
        nv = {A.OP_EQ: ln & rn, A.OP_NE: ~(ln & rn), A.OP_LT: ln, A.OP_LE: ln, A.OP_GT: rn, A.OP_GE: rn}[op]
        return Value(np.where(both, v, nv), np.ones(n, bool), err)
    if op in (A.OP_AND, A.OP_OR):
        v = (a.values & b.values) if op == A.OP_AND else (a.values | b.values)
        return Value(v & both, both, err)
    v, bad = arith(MATH[op], a.values, b.values)
    return Value(np.where(both, v, v.dtype.type(0)), both, err | (bad & both))


def _case(e, t, rb):
    n = t.n
    if e.else_ is not None:
        acc = _ev(e.else_, t, rb)
        v, valid, err = acc.values, acc.valid, acc.err
    else:
        v0 = _ev(e.whens[-1][1], t, rb).values
        v, valid, err = _zeros_like(v0), np.zeros(n, bool), np.zeros(n, bool)
    for c, x in reversed(e.whens):  # the fold backward from the ELSE, as the compiler lowers it
        cv, xv = _ev(c, t, rb), _ev(x, t, rb)
        taken = cv.values.astype(bool) & cv.valid
        v = np.where(taken, xv.values, v)
        valid = np.where(taken, xv.valid, valid)
        err = cv.err | np.where(taken, xv.err, err)
    return Value(v, valid, err)


def _scalar_fn(e, t, rb):
    args = [_ev(a, t, rb) for a in e.args]
    valid = np.logical_and.reduce([a.valid for a in args])
    err = np.logical_or.reduce([a.err for a in args])
    name = FN_NAME[e.code]
    with np.errstate(all="ignore"):
        if name in EXACT_REF:
            v = EXACT_REF[name](np.asarray(args[0].values, np.float64))
            zero = 0.0
        else:
            L = [np.asarray(a.values, np.float64).astype(np.longdouble) for a in args]
            v = (LONG[name] if name in LONG else LONG2[name])(*L)
            zero = np.longdouble(0)
    return Value(np.where(valid, v, zero), valid, err)


def _utf8_fn(e, t, rb):
    inner = _ev(e.args[0], t, True)
    extra = [int(a.value) for a in e.args[1:]]
    name = {A.UTF8FN_SUBSTR_FROM: "substr"}.get(e.code) or next(k for k, c in A.UTF8_FN_CODES.items() if c == e.code)
    n = t.n
    if e.dtype == A.INT64:
        v = np.array([utf8_fn_ref.apply(name, s, *extra) if ok else 0 for s, ok in zip(inner.values, inner.valid)], np.int64).reshape(n)
        return Value(v, inner.valid if rb else np.ones(n, bool), inner.err)
    out = np.empty(n, dtype=object)
    out[:] = [utf8_fn_ref.apply(name, s, *extra) if ok else b"" for s, ok in zip(inner.values, inner.valid)]
    return Value(out, inner.valid, inner.err)


def is_approx(expr):
    """Whether `expr` is a transcendental function, whose value is compared within the ulp bound."""
    return isinstance(expr, ScalarFunction) and FN_NAME[expr.code] not in EXACT_REF


def _synthetic(e, schema):
    """Whether the compiler turns `e` into a column or literal node: a column, a literal, a Utf8 function nest (a view)
    or a Utf8 predicate (a Boolean synthetic column)."""
    if isinstance(e, (Column, Literal, Utf8Function)):
        return True
    return isinstance(e, BinaryExpr) and (e.op in (A.OP_LIKE, A.OP_NOT_LIKE) or e.left.get_type(schema) == A.UTF8)


def stack_depth(e, schema):
    """The register-stack depth the expression compiler gives `e` over a table of dtypes `schema`: a column or literal
    right operand is folded into its instruction, any other right operand keeps the left one live beneath it (a
    right-nested operand keeps one more entry live); a CASE is a fold backward from its ELSE, so a condition is
    evaluated over the fold and a value over the fold and its condition."""
    if _synthetic(e, schema):
        return 1
    if isinstance(e, Cast):
        return stack_depth(e.expr, schema)
    if isinstance(e, ScalarFunction) and len(e.args) == 1:
        return stack_depth(e.args[0], schema)
    if isinstance(e, (BinaryExpr, ScalarFunction)):
        left, right = (e.left, e.right) if isinstance(e, BinaryExpr) else e.args
        if _synthetic(right, schema):
            return stack_depth(left, schema)
        return max(stack_depth(left, schema), 1 + stack_depth(right, schema))
    assert isinstance(e, Case), e
    items = [x for w in e.whens for x in w]
    if e.else_ is not None:
        d, pairs = stack_depth(e.else_, schema), items
    else:
        d, pairs = max(stack_depth(items[-2], schema), 1 + stack_depth(items[-1], schema)), items[:-2]
    for k in range(0, len(pairs), 2):  # over the fold: 1 live entry under a condition, 2 under a value
        d = max(d, 1 + stack_depth(pairs[k], schema), 2 + stack_depth(pairs[k + 1], schema))
    return d
