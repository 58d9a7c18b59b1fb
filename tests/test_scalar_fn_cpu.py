"""Built-in scalar functions (sqrt, abs, power, ...) without a GPU: the C ABI's type check of DFGPU_OP_FN, the plan text of
the SQL front-end over the built-in catalogue, the Python lowering, and the function codes of the header against the
Python and Rust mirrors."""
import os
import re

import pytest

from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import engine, host
from datafusion_archive_b200.expr import ScalarFunction, col, fn, lit

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UNARY = ["sqrt", "abs", "floor", "ceil", "trunc", "round", "signum", "exp", "ln", "log2", "log10", "sin", "cos", "tan",
         "asin", "acos", "atan"]
BINARY = ["power", "atan2"]


class Raw:
    """A postfix program given instruction by instruction: (op, col, dtype) triples."""

    def __init__(self, *insns):
        self.insns = insns

    def program(self, schema):
        out = []
        for op, c, dt in self.insns:
            i = A.Insn()
            i.op, i.col, i.dtype = op, c, dt
            out.append(i)
        return out


def check_err(schema, e):
    with pytest.raises(engine.DfGpuError) as ei:
        engine.check_program(schema, e)
    return ei.value


@pytest.mark.parametrize("name", UNARY)
def test_unary_result_type(name):
    assert engine.check_program([A.FLOAT64], fn(name, col(0))) == A.FLOAT64
    assert engine.check_program([A.INT32], fn(name, col(0).cast(A.FLOAT64))) == A.FLOAT64
    assert engine.check_program([A.FLOAT64], fn(name, fn("abs", col(0))) > 1.0) == A.BOOL


@pytest.mark.parametrize("name", BINARY)
def test_binary_result_type(name):
    schema = [A.FLOAT64, A.FLOAT64]
    for e in [fn(name, col(0), col(1)), fn(name, col(0), 2.0), fn(name, col(0), col(0) + col(1)), fn(name, 2.0, col(1)),
              fn(name, lit(2).cast(A.FLOAT64), col(0))]:
        assert engine.check_program(schema, e) == A.FLOAT64


@pytest.mark.parametrize("dt", [A.INT64, A.INT32, A.UINT8, A.FLOAT32, A.BOOL])
def test_non_float64_argument_is_an_execution_error(dt):
    err = check_err([dt, A.FLOAT64], fn("sqrt", col(0)))
    assert err.code == A.ERR_EXECUTION and "'sqrt'" in err.msg and "Float64" in err.msg
    err = check_err([dt, A.FLOAT64], fn("power", col(1), col(0)))
    assert err.code == A.ERR_EXECUTION and "'power'" in err.msg
    err = check_err([dt, A.FLOAT64], fn("atan2", col(0), col(1)))
    assert err.code == A.ERR_EXECUTION and "'atan2'" in err.msg
    err = check_err([A.FLOAT64], fn("power", col(0), lit(2)))  # an Int64 literal is not cast by the ABI either
    assert err.code == A.ERR_EXECUTION


def test_too_few_arguments_name_the_function_and_its_arity():
    err = check_err([A.FLOAT64], Raw((A.OP_FN, A.FN_SQRT, A.FLOAT64)))
    assert err.code == A.ERR_EXECUTION and "'sqrt' takes 1 argument" in err.msg
    err = check_err([A.FLOAT64], Raw((A.OP_COL, 0, A.FLOAT64), (A.OP_FN, A.FN_POWER, A.FLOAT64)))
    assert err.code == A.ERR_EXECUTION and "'power' takes 2 arguments" in err.msg
    # one argument too many leaves two values on the stack: a malformed program
    err = check_err([A.FLOAT64], Raw((A.OP_COL, 0, A.FLOAT64), (A.OP_COL, 0, A.FLOAT64), (A.OP_FN, A.FN_SQRT, A.FLOAT64)))
    assert err.code == A.ERR_GENERAL


@pytest.mark.parametrize("code", [0, -1, 20, 40, 1000])
def test_unknown_function_code_is_an_error(code):
    err = check_err([A.FLOAT64], Raw((A.OP_COL, 0, A.FLOAT64), (A.OP_FN, code, A.FLOAT64)))
    assert err.code == A.ERR_EXECUTION and "unknown scalar function code" in err.msg


def test_cast_of_a_function_stays_unsupported():
    err = check_err([A.FLOAT64], fn("sqrt", col(0)).cast(A.INT64))
    assert err.code == A.ERR_GENERAL and err.msg == "CAST not implemented for expression"


def test_python_lowering():
    prog = fn("Power", col(1), col(0) + 1.0).program([A.INT64, A.FLOAT64])
    assert [(i.op, i.col) for i in prog] == [(A.OP_COL, 1), (A.OP_COL, 0), (A.OP_LIT, 0), (A.OP_ADD, 0), (A.OP_FN, A.FN_POWER)]
    assert prog[-1].dtype == A.FLOAT64
    assert repr(ScalarFunction("sqrt", col(3).cast(A.FLOAT64))) == "sqrt(CAST(#3 AS Float64))"
    with pytest.raises(KeyError):
        fn("foo", col(0))


@pytest.fixture(scope="module")
def cat():
    host.build()
    c = host.Catalog()
    c.add_table("person", [("id", A.UINT32), ("first_name", A.UTF8), ("last_name", A.UTF8), ("age", A.INT32), ("state", A.UTF8), ("salary", A.FLOAT64)])
    c.add_builtin_functions()
    return c


@pytest.mark.parametrize("sql,expected", [
    ("SELECT sqrt(age), power(salary, 2) FROM person",
     "Projection: sqrt(CAST(#3 AS Float64)), power(#5, CAST(Int64(2) AS Float64))\n  TableScan: person projection=None"),
    ("SELECT SQRT(age), Power(salary, 2.5) FROM person",
     "Projection: SQRT(CAST(#3 AS Float64)), Power(#5, Float64(2.5))\n  TableScan: person projection=None"),
    ("SELECT id FROM person WHERE atan2(salary, age) > 1",
     "Projection: #0\n  Selection: atan2(#5, CAST(#3 AS Float64)) Gt CAST(Int64(1) AS Float64)\n    TableScan: person projection=None"),
    ("SELECT state, SUM(ln(salary)), COUNT(round(age)) FROM person GROUP BY state",
     "Aggregate: groupBy=[[#4]], aggr=[[SUM(ln(#5)), COUNT(round(CAST(#3 AS Float64)))]]\n  TableScan: person projection=None"),
    ("SELECT abs(sin(salary) - cos(age)) FROM person",
     "Projection: abs(sin(#5) Minus cos(CAST(#3 AS Float64)))\n  TableScan: person projection=None"),
])
def test_plan_text(cat, sql, expected):
    assert cat.plan(sql) == expected


def test_every_builtin_is_in_the_catalogue(cat):
    for name in UNARY:
        assert cat.plan("SELECT %s(salary) FROM person" % name.upper()).startswith("Projection: %s(#5)" % name.upper())
    for name in BINARY:
        assert cat.plan("SELECT %s(salary, salary) FROM person" % name).startswith("Projection: %s(#5, #5)" % name)


def test_unknown_and_extra_arguments(cat):
    with pytest.raises(host.ExecutionError) as ei:
        cat.plan("SELECT foo(age) FROM person")
    assert ei.value.code == A.ERR_GENERAL and "Invalid function 'foo'" in str(ei.value)
    with pytest.raises(host.ExecutionError) as ei:
        cat.plan("SELECT sqrt(age, 2) FROM person")
    assert ei.value.code == A.ERR_INTERNAL


def test_a_catalogue_without_builtins_is_unchanged():
    c = host.Catalog()
    c.add_table("t", [("a", A.FLOAT64)])
    with pytest.raises(host.ExecutionError) as ei:
        c.plan("SELECT sqrt(a) FROM t")
    assert "Invalid function 'sqrt'" in str(ei.value)


def test_function_codes_match_the_header_and_mirrors():
    with open(os.path.join(ROOT, "include", "dfgpu.h")) as f:
        header = f.read()
    with open(os.path.join(ROOT, "shim", "src", "execution", "gpu", "ffi.rs")) as f:
        ffi = f.read()
    codes = {m.group(1): int(m.group(2)) for m in re.finditer(r"DFGPU_FN_(\w+)\s*=\s*(\d+)", header)}
    assert len(codes) == len(UNARY) + len(BINARY)
    assert int(re.search(r"DFGPU_OP_FN\s*=\s*(\d+)", header).group(1)) == A.OP_FN == 40
    assert re.search(r"pub const OP_FN: i32 = 40;", ffi)
    assert re.search(r"#define DFGPU_ABI_VERSION 2\b", header) and A.ABI_VERSION == 2
    for name, code in codes.items():
        assert getattr(A, "FN_" + name) == code, name
        assert re.search(r"pub const FN_%s: i32 = %d;" % (name, code), ffi), name
        assert A.FN_CODES[name.lower()] == code
    assert sorted(A.FN_CODES) == sorted(UNARY + BINARY)
