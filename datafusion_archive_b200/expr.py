"""Python mirror of the reference's expression IR (src/logicalplan.rs:67-167), used by the test and
bench harness to build the postfix expression programs the C ABI takes (include/dfgpu.h).

The production host layer is the C++ mirror under csrc/host/ (the reference is compiled code);
this module only exists so tests read like the reference's own tests, which build `Expr` by hand
(src/execution/aggregate.rs:971-988).
"""
import ctypes as C
import struct

from . import _abi as A

_CMP = {A.OP_EQ, A.OP_NE, A.OP_LT, A.OP_LE, A.OP_GT, A.OP_GE}
_BOOLOP = {A.OP_AND, A.OP_OR, A.OP_LIKE, A.OP_NOT_LIKE}
_OPNAME = {
    A.OP_ADD: "Plus", A.OP_SUB: "Minus", A.OP_MUL: "Multiply", A.OP_DIV: "Divide", A.OP_EQ: "Eq", A.OP_NE: "NotEq",
    A.OP_LT: "Lt", A.OP_LE: "LtEq", A.OP_GT: "Gt", A.OP_GE: "GtEq", A.OP_AND: "And", A.OP_OR: "Or",
    A.OP_LIKE: "Like", A.OP_NOT_LIKE: "NotLike",
}


class Expr:
    def _bin(self, op, other):
        return BinaryExpr(self, op, _wrap(other))

    def __add__(self, o): return self._bin(A.OP_ADD, o)
    def __sub__(self, o): return self._bin(A.OP_SUB, o)
    def __mul__(self, o): return self._bin(A.OP_MUL, o)
    def __truediv__(self, o): return self._bin(A.OP_DIV, o)
    def __lt__(self, o): return self._bin(A.OP_LT, o)
    def __le__(self, o): return self._bin(A.OP_LE, o)
    def __gt__(self, o): return self._bin(A.OP_GT, o)
    def __ge__(self, o): return self._bin(A.OP_GE, o)
    def eq(self, o): return self._bin(A.OP_EQ, o)
    def not_eq(self, o): return self._bin(A.OP_NE, o)
    def __and__(self, o): return self._bin(A.OP_AND, o)
    def __or__(self, o): return self._bin(A.OP_OR, o)
    def like(self, pattern): return self._bin(A.OP_LIKE, pattern)
    def not_like(self, pattern): return self._bin(A.OP_NOT_LIKE, pattern)

    def cast(self, dtype):
        return Cast(self, dtype)

    def program(self, schema_dtypes):
        out = []
        self._emit(schema_dtypes, out)
        return out


class Column(Expr):
    def __init__(self, index):
        self.index = index

    def get_type(self, schema):
        return schema[self.index] if 0 <= self.index < len(schema) else 0

    def _emit(self, schema, out):
        i = A.Insn()
        # an out-of-range index is passed through: the engine reports InvalidColumn
        i.op, i.col, i.dtype = A.OP_COL, self.index, (schema[self.index] if 0 <= self.index < len(schema) else 0)
        out.append(i)

    def __repr__(self):
        return "#%d" % self.index


class Literal(Expr):
    """Expr::Literal(ScalarValue); default typing follows the planner: Python int -> Int64,
    float -> Float64, str -> Utf8 (src/sqlplanner.rs:214-218).  A Utf8 literal (str or bytes) is emitted as
    DFGPU_OP_LIT_UTF8 pointing at an encoded copy that every emitted instruction keeps alive."""

    def __init__(self, value, dtype=None):
        if dtype is None:
            dtype = A.UTF8 if isinstance(value, (str, bytes)) else A.FLOAT64 if isinstance(value, float) else A.INT64
        self.value, self.dtype = value, dtype
        if dtype == A.UTF8:
            raw = value.encode("utf-8") if isinstance(value, str) else bytes(value)
            self._bytes = C.create_string_buffer(raw, max(1, len(raw)))
            self._len = len(raw)

    def get_type(self, schema):
        return self.dtype

    def _emit(self, schema, out):
        i = A.Insn()
        i.op, i.dtype = A.OP_LIT, self.dtype
        if self.dtype == A.UTF8:
            i.op, i.col = A.OP_LIT_UTF8, self._len
            i.lit.str = C.addressof(self._bytes)
            i._keep = self._bytes  # the program borrows the bytes: they live as long as the instruction
        elif self.dtype == A.FLOAT64:
            i.lit.f64 = float(self.value)
        elif self.dtype == A.FLOAT32:
            i.lit.u64 = 0
            i.lit.f32 = float(self.value)
        elif self.dtype in (A.UINT8, A.UINT16, A.UINT32, A.UINT64):
            i.lit.u64 = int(self.value)
        else:
            i.lit.i64 = int(self.value)
        out.append(i)

    def __repr__(self):
        return "%s(%r)" % (A.DTYPE_NAMES[self.dtype], self.value)


class Cast(Expr):
    def __init__(self, expr, dtype):
        self.expr, self.dtype = expr, dtype

    def get_type(self, schema):
        return self.dtype

    def _emit(self, schema, out):
        self.expr._emit(schema, out)
        i = A.Insn()
        i.op, i.dtype, i.col = A.OP_CAST, self.dtype, self.expr.get_type(schema)
        out.append(i)

    def __repr__(self):
        return "CAST(%r AS %s)" % (self.expr, A.DTYPE_NAMES[self.dtype])


class BinaryExpr(Expr):
    def __init__(self, left, op, right):
        self.left, self.op, self.right = left, op, right

    def get_type(self, schema):
        if self.op in _CMP or self.op in _BOOLOP:
            return A.BOOL
        return self.left.get_type(schema)  # op_type = left type (expression.rs:408)

    def _emit(self, schema, out):
        self.left._emit(schema, out)
        self.right._emit(schema, out)
        i = A.Insn()
        i.op = self.op
        i.dtype = self.left.get_type(schema)  # operand type (advisory: the engine re-infers and checks)
        out.append(i)

    def __repr__(self):
        return "%r %s %r" % (self.left, _OPNAME[self.op], self.right)


class ScalarFunction(Expr):
    """Expr::ScalarFunction{name,args,return_type} (src/logicalplan.rs:156-160) for a built-in function: Float64
    arguments, Float64 result.  Like the C ABI, it casts nothing; cast integer arguments with `.cast(A.FLOAT64)`."""

    def __init__(self, name, *args):
        self.name, self.args = name, [_wrap(a) for a in args]
        self.code = A.FN_CODES[name.lower()]

    def get_type(self, schema):
        return A.FLOAT64

    def _emit(self, schema, out):
        for a in self.args:
            a._emit(schema, out)
        i = A.Insn()
        i.op, i.col, i.dtype = A.OP_FN, self.code, A.FLOAT64
        out.append(i)

    def __repr__(self):
        return "%s(%s)" % (self.name, ", ".join(repr(a) for a in self.args))


class Utf8Function(Expr):
    """Expr::ScalarFunction of a Utf8 function (DFGPU_OP_UTF8_FN): upper, lower, trim, ltrim, rtrim, substr(s, start
    [, count]), length / char_length, octet_length.  The first argument is the Utf8 operand, the others Int64 literals;
    length and octet_length return Int64, the others Utf8."""

    def __init__(self, name, *args):
        self.name, self.args = name, [_wrap(a) for a in args]
        self.code = A.UTF8_FN_CODES[name.lower()]
        if self.code == A.UTF8FN_SUBSTR and len(self.args) == 2:
            self.code = A.UTF8FN_SUBSTR_FROM
        self.dtype = A.INT64 if self.code in (A.UTF8FN_LENGTH, A.UTF8FN_OCTET_LENGTH) else A.UTF8

    def get_type(self, schema):
        return self.dtype

    def _emit(self, schema, out):
        for a in self.args:
            a._emit(schema, out)
        i = A.Insn()
        i.op, i.col, i.dtype = A.OP_UTF8_FN, self.code, self.dtype
        out.append(i)

    def __repr__(self):
        return "%s(%s)" % (self.name, ", ".join(repr(a) for a in self.args))


class Case(Expr):
    """CASE WHEN c1 THEN v1 [WHEN ..] [ELSE e] END (DFGPU_OP_CASE): `whens` is a list of (condition, value) pairs,
    `else_` the ELSE value or None.  Like the C ABI, it casts nothing: every value has the result type."""

    def __init__(self, whens, else_=None):
        self.whens = [(c, _wrap(v)) for c, v in whens]
        self.else_ = None if else_ is None else _wrap(else_)

    def get_type(self, schema):
        return self.whens[0][1].get_type(schema)

    def _emit(self, schema, out):
        for c, v in self.whens:
            c._emit(schema, out)
            v._emit(schema, out)
        if self.else_ is not None:
            self.else_._emit(schema, out)
        i = A.Insn()
        i.op, i.col, i.dtype = A.OP_CASE, 2 * len(self.whens) + (self.else_ is not None), self.get_type(schema)
        out.append(i)

    def __repr__(self):
        s = "CASE" + "".join(" WHEN %r THEN %r" % w for w in self.whens)
        return s + (" ELSE %r" % self.else_ if self.else_ is not None else "") + " END"


class AggregateFunction:
    """Expr::AggregateFunction{name,args,return_type} (src/logicalplan.rs:162-166)."""

    _F = {"min": A.AGG_MIN, "max": A.AGG_MAX, "sum": A.AGG_SUM, "count": A.AGG_COUNT, "avg": A.AGG_AVG}

    def __init__(self, name, arg, return_type=None, distinct=False):
        """distinct=True: COUNT(DISTINCT arg), the number of distinct non-null values (count only)."""
        if distinct and name.lower() != "count":
            raise ValueError("DISTINCT is only supported in COUNT(DISTINCT expr)")
        self.name, self.arg, self.return_type, self.distinct = name, _wrap(arg), return_type, distinct

    def lower(self, schema):
        func = A.AGG_COUNT_DISTINCT if self.distinct else self._F[self.name.lower()]
        rt = self.return_type
        if rt is None:
            if func in (A.AGG_COUNT, A.AGG_COUNT_DISTINCT):
                rt = A.UINT64
            elif func == A.AGG_AVG:
                rt = A.FLOAT64
            else:
                rt = self.arg.get_type(schema)
        return (func, self.arg.program(schema), rt)


def _wrap(x):
    return x if isinstance(x, Expr) else Literal(x)


def col(i):
    return Column(i)


def lit(v, dtype=None):
    return Literal(v, dtype)


def case(whens, else_=None):
    return Case(whens, else_)


def fn(name, *args):
    return ScalarFunction(name, *args)


def utf8_fn(name, *args):
    return Utf8Function(name, *args)


def f64_bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]
