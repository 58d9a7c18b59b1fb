"""Utf8 functions without a GPU: the C ABI's typing of DFGPU_OP_UTF8_FN and its refusals, the plan text of the SQL
front-end, the constants of the header against the Python and Rust mirrors, and dfgpu_utf8_fn_host (the kernels' own
per-row code) fuzzed against the Python reference of utf8_fn_ref over random byte strings."""
import os
import re

import pytest

from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import engine, host
from datafusion_archive_b200.expr import col, lit, utf8_fn
from utf8_fn_ref import EDGE_COUNTS, EDGE_STARTS, NESTS, build, ev, random_strings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def check_err(schema, e):
    with pytest.raises(engine.DfGpuError) as ei:
        engine.check_program(schema, e)
    return ei.value


def test_result_types():
    for name in ["upper", "lower", "trim", "ltrim", "rtrim"]:
        assert engine.check_program([A.UTF8], utf8_fn(name, col(0))) == A.UTF8
    assert engine.check_program([A.UTF8], utf8_fn("substr", col(0), 2)) == A.UTF8
    assert engine.check_program([A.UTF8], utf8_fn("substr", col(0), 2, 3)) == A.UTF8
    for name in ["length", "char_length", "octet_length"]:
        assert engine.check_program([A.UTF8], utf8_fn(name, col(0))) == A.INT64
        assert engine.check_program([A.UTF8], utf8_fn(name, col(0)) > 3) == A.BOOL
        assert engine.check_program([A.UTF8], utf8_fn(name, col(0)) + 1) == A.INT64
        assert engine.check_program([A.UTF8], utf8_fn(name, col(0)).cast(A.FLOAT64)) == A.FLOAT64
    schema = [A.UTF8, A.UTF8, A.INT64]
    for e in [utf8_fn("lower", col(0)).like(lit("ab%")), utf8_fn("upper", col(0)).eq(lit("X")), lit("X") < utf8_fn("trim", col(1)),
              utf8_fn("upper", col(0)).eq(utf8_fn("upper", col(1))), (utf8_fn("length", col(0)) > col(2)) & utf8_fn("trim", col(1)).not_like(lit("%a"))]:
        assert engine.check_program(schema, e) == A.BOOL
    assert engine.check_program([A.UTF8], build(("upper", ("trim", ("substr", "s", 2))))) == A.UTF8


def test_refusals():
    err = check_err([A.INT32], utf8_fn("upper", col(0)))
    assert err.code == A.ERR_EXECUTION and err.msg == "function 'upper' takes a Utf8 argument, not Int32"
    err = check_err([A.UTF8], utf8_fn("upper", lit("x")))
    assert err.code == A.ERR_NOT_IMPLEMENTED
    err = check_err([A.UTF8], utf8_fn("substr", col(0), 1, -1))
    assert err.code == A.ERR_EXECUTION and err.msg == "negative substring length not allowed"
    for e in [utf8_fn("substr", col(0), col(1)), utf8_fn("substr", col(0), 1.5), utf8_fn("substr", col(0), lit(1, A.INT32)),
              utf8_fn("substr", col(0), 1, col(1))]:
        assert check_err([A.UTF8, A.INT64], e).code == A.ERR_NOT_IMPLEMENTED
    err = check_err([A.UTF8], utf8_fn("upper", utf8_fn("length", col(0))))
    assert err.code == A.ERR_EXECUTION and "not Int64" in err.msg
    # a Utf8 result is not a number; comparing it with one is "comparison_ops", as for a Utf8 column
    assert check_err([A.UTF8], utf8_fn("upper", col(0)) > 3).msg == "comparison_ops"
    assert check_err([A.UTF8], utf8_fn("upper", col(0)).cast(A.INT64)).code == A.ERR_NOT_IMPLEMENTED
    assert check_err([A.UTF8], utf8_fn("upper", col(0)) + utf8_fn("lower", col(0))).msg == "math_ops"


def raw(*insns):
    class Raw:
        def program(self, schema):
            out = []
            for op, c, dt in insns:
                i = A.Insn()
                i.op, i.col, i.dtype = op, c, dt
                out.append(i)
            return out
    return Raw()


def test_malformed_programs():
    err = check_err([A.UTF8], raw((A.OP_UTF8_FN, A.UTF8FN_UPPER, A.UTF8)))
    assert err.code == A.ERR_EXECUTION and "'upper' takes 1 argument" in err.msg
    err = check_err([A.UTF8], raw((A.OP_COL, 0, A.UTF8), (A.OP_UTF8_FN, A.UTF8FN_SUBSTR, A.UTF8)))
    assert err.code == A.ERR_EXECUTION and "'substr' takes 3 arguments" in err.msg
    err = check_err([A.UTF8], raw((A.OP_COL, 0, A.UTF8), (A.OP_UTF8_FN, A.UTF8FN_LENGTH, A.UTF8)))  # wrong result type
    assert err.code == A.ERR_GENERAL
    for code in [0, -1, 10, 41]:
        err = check_err([A.UTF8], raw((A.OP_COL, 0, A.UTF8), (A.OP_UTF8_FN, code, A.UTF8)))
        assert err.code == A.ERR_EXECUTION and "unknown Utf8 function code" in err.msg
    # DFGPU_OP_FN codes stay the math functions only
    err = check_err([A.UTF8], raw((A.OP_COL, 0, A.UTF8), (A.OP_FN, 20, A.FLOAT64)))
    assert "unknown scalar function code" in err.msg


def test_python_lowering():
    prog = utf8_fn("SUBSTR", col(1), 2).program([A.INT64, A.UTF8])
    assert [(i.op, i.col) for i in prog] == [(A.OP_COL, 1), (A.OP_LIT, 0), (A.OP_UTF8_FN, A.UTF8FN_SUBSTR_FROM)]
    assert prog[-1].dtype == A.UTF8
    prog = utf8_fn("length", utf8_fn("substr", col(0), 1, 2)).program([A.UTF8])
    assert [i.col for i in prog][-2:] == [A.UTF8FN_SUBSTR, A.UTF8FN_LENGTH] and prog[-1].dtype == A.INT64
    assert repr(utf8_fn("upper", utf8_fn("trim", col(0)))) == "upper(trim(#0))"
    assert "upper" not in A.FN_CODES
    with pytest.raises(KeyError):
        utf8_fn("foo", col(0))


def test_constants_match_the_header_and_mirrors():
    header = open(os.path.join(ROOT, "include", "dfgpu.h")).read()
    ffi = open(os.path.join(ROOT, "shim", "src", "execution", "gpu", "ffi.rs")).read()
    assert int(re.search(r"DFGPU_OP_UTF8_FN\s*=\s*(\d+)", header).group(1)) == A.OP_UTF8_FN == 41
    assert re.search(r"pub const OP_UTF8_FN: i32 = 41;", ffi)
    codes = {m.group(1): int(m.group(2)) for m in re.finditer(r"DFGPU_UTF8FN_(\w+)\s*=\s*(\d+)", header)}
    assert len(codes) == 9
    for name, code in codes.items():
        assert getattr(A, "UTF8FN_" + name) == code, name
        assert re.search(r"pub const UTF8FN_%s: i32 = %d;" % (name, code), ffi), name
    assert set(A.UTF8_FN_CODES.values()) == set(codes.values()) - {A.UTF8FN_SUBSTR_FROM}


@pytest.fixture(scope="module")
def cat():
    host.build()
    c = host.Catalog()
    c.add_table("person", [("id", A.UINT32), ("first_name", A.UTF8), ("last_name", A.UTF8), ("age", A.INT32), ("state", A.UTF8), ("salary", A.FLOAT64)])
    c.add_builtin_functions()
    return c


@pytest.mark.parametrize("sql,expected", [
    ("SELECT upper(first_name), lower(state), trim(last_name), ltrim(state), rtrim(state) FROM person",
     "Projection: upper(#1), lower(#4), trim(#2), ltrim(#4), rtrim(#4)\n  TableScan: person projection=None"),
    ("SELECT substr(first_name, 2), substr(first_name, 1, 3), LENGTH(state), char_length(state), octet_length(state) FROM person",
     "Projection: substr(#1, Int64(2)), substr(#1, Int64(1), Int64(3)), LENGTH(#4), char_length(#4), octet_length(#4)\n  TableScan: person projection=None"),
    ("SELECT upper(trim(substr(first_name, 2))), length(lower(state)) FROM person",
     "Projection: upper(trim(substr(#1, Int64(2)))), length(lower(#4))\n  TableScan: person projection=None"),
    ("SELECT id FROM person WHERE lower(first_name) LIKE 'a%'",
     "Projection: #0\n  Selection: lower(#1) Like Utf8(\"a%\")\n    TableScan: person projection=None"),
    ("SELECT id FROM person WHERE length(state) > 1 AND age > 3",
     "Projection: #0\n  Selection: length(#4) Gt Int64(1) And CAST(#3 AS Int64) Gt Int64(3)\n    TableScan: person projection=None"),
    ("SELECT length(state), SUM(length(first_name)) FROM person GROUP BY length(state)",
     "Aggregate: groupBy=[[length(#4)]], aggr=[[SUM(length(#1))]]\n  TableScan: person projection=None"),
])
def test_plan_text(cat, sql, expected):
    assert cat.plan(sql) == expected


def test_sql_refusals(cat):
    with pytest.raises(host.ExecutionError) as ei:
        cat.plan("SELECT substr(first_name, 1, 2, 3) FROM person")
    assert ei.value.code == A.ERR_INTERNAL
    with pytest.raises(host.ExecutionError):
        cat.plan("SELECT upper(age) FROM person")  # the planner's CAST of Int32 to Utf8
    for sql in ["SELECT TRIM(BOTH ' ' FROM state) FROM person", "SELECT SUBSTRING(state FROM 1 FOR 2) FROM person"]:
        with pytest.raises(host.ExecutionError):
            cat.plan(sql)


def test_host_function_matches_the_reference():
    vals = [v for v in random_strings(400, 21) if v is not None] + [b"", b" ", b"  a  ", b"\x80", b"\x80\x80a", b"a\x80", b"\xf0\x9f\x98\x80" * 3]
    nests = list(NESTS)
    for s in EDGE_STARTS:
        nests.append(("substr", "s", s))
        for c in EDGE_COUNTS:
            nests.append(("substr", "s", s, c))
    for n in (2, 3, 4):  # start at n, n + 1 of a 3-character string
        nests.append(("substr", "s", n, 1))
    for nest in nests:
        e = build(nest)
        for v in vals:
            assert engine.utf8_fn_host(v, e) == ev(nest, v), (nest, v)


def test_host_function_refuses_other_programs():
    with pytest.raises(engine.DfGpuError):
        engine.utf8_fn_host(b"abc", col(0))
    with pytest.raises(engine.DfGpuError):
        engine.utf8_fn_host(b"abc", utf8_fn("length", col(0)) > 1)
