"""CASE WHEN .. THEN .. ELSE .. END without a GPU: plan text of both forms with their supertype CASTs, nesting, CASE at
every site of a query, column collection through CASE operands, every parser, planner and dfgpu_check_program error, and
the Python lowering to DFGPU_OP_CASE."""
import os
import re

import pytest

from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import engine, host
from datafusion_archive_b200.expr import Case, case, col, lit

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCAN = "TableScan: person projection=None"


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


@pytest.fixture(scope="module")
def cat():
    host.build()
    c = host.Catalog()
    c.add_table("person", [("id", A.UINT32), ("first_name", A.UTF8), ("last_name", A.UTF8), ("age", A.INT32), ("state", A.UTF8), ("salary", A.FLOAT64)])
    c.add_table("orders", [("id", A.INT64), ("person_id", A.INT64), ("qty", A.INT64), ("price", A.FLOAT64)])
    c.add_builtin_functions()
    return c


@pytest.mark.parametrize("sql,expected", [
    ("SELECT CASE WHEN age > 30 THEN salary ELSE 0 END FROM person",
     "Projection: CASE WHEN CAST(#3 AS Int64) Gt Int64(30) THEN #5 ELSE CAST(Int64(0) AS Float64) END\n  " + SCAN),
    ("SELECT CASE WHEN age > 30 THEN 1 WHEN age > 20 THEN 2.5 END FROM person",
     "Projection: CASE WHEN CAST(#3 AS Int64) Gt Int64(30) THEN CAST(Int64(1) AS Float64) WHEN CAST(#3 AS Int64) Gt Int64(20) "
     "THEN Float64(2.5) END\n  " + SCAN),
    # the simple form is the searched form with conditions x Eq a, coerced like any Eq
    ("SELECT CASE age WHEN 1 THEN age WHEN 2 THEN 7 ELSE 0 END FROM person",
     "Projection: CASE WHEN CAST(#3 AS Int64) Eq Int64(1) THEN CAST(#3 AS Int64) WHEN CAST(#3 AS Int64) Eq Int64(2) THEN Int64(7) "
     "ELSE Int64(0) END\n  " + SCAN),
    ("SELECT case state when 'CA' then 1 end FROM person",
     "Projection: CASE WHEN #4 Eq Utf8(\"CA\") THEN Int64(1) END\n  " + SCAN),
    # nesting: in a THEN, in a condition, under arithmetic and a function
    ("SELECT CASE WHEN age > 1 THEN CASE WHEN salary > 1 THEN 1 ELSE 2 END END + 1 FROM person",
     "Projection: CASE WHEN CAST(#3 AS Int64) Gt Int64(1) THEN CASE WHEN #5 Gt CAST(Int64(1) AS Float64) THEN Int64(1) ELSE Int64(2) "
     "END END Plus Int64(1)\n  " + SCAN),
    ("SELECT sqrt(CASE WHEN CASE WHEN age > 1 THEN salary END > 2 THEN salary ELSE 0.5 END) FROM person",
     "Projection: sqrt(CASE WHEN CASE WHEN CAST(#3 AS Int64) Gt Int64(1) THEN #5 END Gt CAST(Int64(2) AS Float64) THEN #5 "
     "ELSE Float64(0.5) END)\n  " + SCAN),
    # WHERE, GROUP BY and aggregate arguments
    ("SELECT id FROM person WHERE CASE WHEN age <> 0 THEN salary / age > 1 ELSE age > 5 END",
     "Projection: #0\n  Selection: CASE WHEN CAST(#3 AS Int64) NotEq Int64(0) THEN #5 Divide CAST(#3 AS Float64) Gt "
     "CAST(Int64(1) AS Float64) ELSE CAST(#3 AS Int64) Gt Int64(5) END\n    " + SCAN),
    ("SELECT COUNT(id) FROM person GROUP BY CASE WHEN age < 10 THEN 0 WHEN age < 100 THEN 1 ELSE 2 END",
     "Aggregate: groupBy=[[CASE WHEN CAST(#3 AS Int64) Lt Int64(10) THEN Int64(0) WHEN CAST(#3 AS Int64) Lt Int64(100) THEN Int64(1) "
     "ELSE Int64(2) END]], aggr=[[COUNT(#0)]]\n  " + SCAN),
    ("SELECT state, SUM(CASE WHEN age > 3 THEN salary ELSE 0 END), COUNT(CASE WHEN age > 10 THEN 1 END), "
     "COUNT(DISTINCT CASE WHEN age > 3 THEN age END) FROM person WHERE salary > 1 GROUP BY state",
     "Aggregate: groupBy=[[#4]], aggr=[[SUM(CASE WHEN CAST(#3 AS Int64) Gt Int64(3) THEN #5 ELSE CAST(Int64(0) AS Float64) END), "
     "COUNT(CASE WHEN CAST(#3 AS Int64) Gt Int64(10) THEN Int64(1) END), COUNT(DISTINCT CASE WHEN CAST(#3 AS Int64) Gt Int64(3) "
     "THEN #3 END)]]\n  Selection: #5 Gt CAST(Int64(1) AS Float64)\n    " + SCAN),
    # a coercion of a CASE casts its values, not the CASE: the engine casts columns and literals only
    ("SELECT CASE WHEN age > 1 THEN age END + 1 FROM person",
     "Projection: CASE WHEN CAST(#3 AS Int64) Gt Int64(1) THEN CAST(#3 AS Int64) END Plus Int64(1)\n  " + SCAN),
    ("SELECT sqrt(CASE WHEN age > 1 THEN age ELSE 2 END) FROM person",
     "Projection: sqrt(CASE WHEN CAST(#3 AS Int64) Gt Int64(1) THEN CAST(#3 AS Float64) ELSE "
     "CAST(Int64(2) AS Float64) END)\n  " + SCAN),
    ("SELECT CASE WHEN first_name LIKE 'A%' THEN 1 ELSE 0 END FROM person",
     "Projection: CASE WHEN #1 Like Utf8(\"A%\") THEN Int64(1) ELSE Int64(0) END\n  " + SCAN),
])
def test_plan_text(cat, sql, expected):
    assert cat.plan(sql) == expected


def test_join_keys_and_subquery_keys_see_case_operands(cat):
    # a CASE over one side's columns is a key: the planner collects the columns of every operand
    plan = cat.plan("SELECT p.id FROM person p JOIN orders o ON CASE WHEN p.age > 0 THEN p.age ELSE 0 END = o.person_id")
    assert "Join: on=[CASE WHEN CAST(#3 AS Int64) Gt Int64(0) THEN CAST(#3 AS Int64) ELSE Int64(0) END Eq #7]" in plan
    plan = cat.plan("SELECT p.id FROM person p JOIN orders o ON p.age = o.person_id AND CASE WHEN o.qty > 1 THEN p.age ELSE 0 END > 2")
    assert plan.startswith("Projection: #0\n  Selection: CASE WHEN #8 Gt Int64(1) THEN CAST(#3 AS Int64) ELSE Int64(0) END Gt Int64(2)")
    plan = cat.plan("SELECT id FROM person WHERE CASE WHEN age > 1 THEN age ELSE 0 END IN (SELECT person_id FROM orders)")
    assert "SemiJoin: on=[CASE WHEN CAST(#3 AS Int64) Gt Int64(1) THEN CAST(#3 AS Int64) ELSE Int64(0) END Eq #6]" in plan
    plan = cat.plan("SELECT id FROM person p WHERE EXISTS (SELECT id FROM orders o WHERE o.person_id = CASE WHEN p.age > 1 THEN p.age END)")
    assert "SemiJoin: on=[CASE WHEN CAST(#3 AS Int64) Gt Int64(1) THEN CAST(#3 AS Int64) END Eq #6]" in plan


@pytest.mark.parametrize("sql,code,msg", [
    ("SELECT CASE END FROM person", A.ERR_GENERAL, 'ParserError("Expected WHEN after CASE, found: END")'),
    ("SELECT CASE age ELSE 1 END FROM person", A.ERR_GENERAL, 'ParserError("Expected WHEN after CASE, found: ELSE")'),
    ("SELECT CASE WHEN age > 1 THEN 1 FROM person", A.ERR_GENERAL, 'ParserError("Expected END, found: FROM")'),
    ("SELECT CASE WHEN age > 1 THEN 1 ELSE 2 FROM person", A.ERR_GENERAL, 'ParserError("Expected END, found: FROM")'),
    ("SELECT CASE WHEN age > 1 1 END FROM person", A.ERR_GENERAL, 'ParserError("Expected THEN, found: 1")'),
    ("SELECT end FROM person", A.ERR_GENERAL, 'ParserError("Expected an expression, found: end")'),
    ("SELECT id FROM person AS when", A.ERR_GENERAL, "ParserError"),
    ("SELECT CASE WHEN age > 1 THEN 'a' ELSE 1 END FROM person", A.ERR_GENERAL,
     "No common supertype found for CASE with input types Utf8 and Int64"),
    ("SELECT CASE WHEN age > 1 THEN salary WHEN age > 2 THEN 1 ELSE first_name END FROM person", A.ERR_GENERAL,
     "No common supertype found for CASE with input types Float64 and Utf8"),
    ("SELECT CASE age WHEN 'x' THEN 1 END FROM person", A.ERR_GENERAL,
     "No common supertype found for binary operator Eq with input types Int32 and Utf8"),
])
def test_parser_and_planner_errors(cat, sql, code, msg):
    with pytest.raises(host.ExecutionError) as ei:
        cat.plan(sql)
    assert ei.value.code == code and msg in str(ei.value)


def test_case_over_an_aggregate_is_not_an_aggregate(cat):
    # planned as a projection, like sqrt(SUM(x)); executing it is refused when the aggregate is lowered
    assert cat.plan("SELECT CASE WHEN SUM(age) > 0 THEN 1 ELSE 0 END FROM person").startswith("Projection: CASE WHEN CAST(SUM(#3)")


# ---- dfgpu_check_program ------------------------------------------------------------------------------------------
S = [A.INT64, A.FLOAT64, A.BOOL, A.UTF8, A.INT32, A.UINT8, A.FLOAT32]


@pytest.mark.parametrize("dt", [A.INT8, A.INT16, A.INT32, A.INT64, A.UINT8, A.UINT16, A.UINT32, A.UINT64, A.FLOAT32, A.FLOAT64])
def test_result_type_is_the_branches_type(dt):
    schema = [A.FLOAT64, dt]
    assert engine.check_program(schema, case([(col(0) > 0.5, col(1))], lit(1, dt))) == dt
    assert engine.check_program(schema, case([(col(0) > 0.5, col(1)), (col(0) < 0.1, col(1) + col(1))])) == dt
    assert engine.check_program(schema, case([(col(0) > 0.5, col(1))]).eq(col(1))) == A.BOOL


def test_boolean_results_and_conditions():
    assert engine.check_program(S, case([(col(2), col(2))], col(1) > 1.0)) == A.BOOL
    assert engine.check_program(S, case([(col(3).like("a%"), col(0))], 0)) == A.INT64
    assert engine.check_program(S, case([(col(3).eq(lit("x")), col(1))])) == A.FLOAT64
    assert engine.check_program(S, case([(case([(col(2), col(1) > 1.0)]), col(0))])) == A.INT64


def test_cast_of_a_case_stays_unsupported_at_the_abi():
    # the planner never emits one (it casts the values); through the ABI it is refused like any CAST of an expression
    e = check_err(S, case([(col(2), col(4))]).cast(A.INT64))
    assert e.code == A.ERR_GENERAL and e.msg == "CAST not implemented for expression"


def test_type_errors():
    e = check_err(S, case([(col(0), col(1))]))
    assert e.code == A.ERR_EXECUTION and e.msg == "CASE WHEN condition did not evaluate to boolean"
    e = check_err(S, case([(col(2), col(1)), (col(1), col(1))]))
    assert e.code == A.ERR_EXECUTION and e.msg == "CASE WHEN condition did not evaluate to boolean"
    e = check_err(S, case([(col(2), col(0))], col(1)))
    assert e.code == A.ERR_EXECUTION and e.msg == "CASE branch types differ: Int64 and Float64"
    e = check_err(S, case([(col(2), col(4)), (col(2), col(5))]))
    assert e.code == A.ERR_EXECUTION and e.msg == "CASE branch types differ: Int32 and UInt8"
    e = check_err(S, case([(col(2), col(3))]))
    assert e.code == A.ERR_NOT_IMPLEMENTED and e.msg == "CASE with a Utf8 result"
    e = check_err(S, case([(col(2), col(0))], lit("x")))
    assert e.code == A.ERR_NOT_IMPLEMENTED and e.msg == "CASE with a Utf8 result"


@pytest.mark.parametrize("insns", [
    [(A.OP_COL, 2, A.BOOL), (A.OP_CASE, 1, A.BOOL)],                          # fewer than 2 operands
    [(A.OP_COL, 2, A.BOOL), (A.OP_COL, 0, A.INT64), (A.OP_CASE, 3, A.INT64)],  # more operands than on the stack
    [(A.OP_COL, 2, A.BOOL), (A.OP_COL, 0, A.INT64), (A.OP_CASE, 2, A.FLOAT64)],  # dtype is not the result type
    [(A.OP_COL, 0, A.INT64), (A.OP_COL, 2, A.BOOL), (A.OP_COL, 0, A.INT64), (A.OP_CASE, 2, A.INT64)],  # two values left
])
def test_malformed_programs(insns):
    e = check_err(S, Raw(*insns))
    assert e.code == A.ERR_GENERAL and e.msg == "malformed expression program"


def test_instruction_limit():
    # each WHEN is 4 instructions (column, compare with the literal folded in, value, select): 1 + 4 * 24 = 97 is over the
    # 96 of one operator
    e = case([(col(1) > float(i), col(1)) for i in range(24)], 0.0)
    err = check_err(S, e)
    assert err.code == A.ERR_NOT_IMPLEMENTED and "exceed 96 instructions" in err.msg
    assert engine.check_program(S, case([(col(1) > float(i), col(1)) for i in range(23)], 0.0)) == A.FLOAT64


# ---- Python lowering and the header -------------------------------------------------------------------------------
def test_python_lowering():
    e = case([(col(0) > 1, col(1)), (col(2), 2.0)], 0.5)
    prog = e.program(S)
    assert [(i.op, i.col) for i in prog] == [(A.OP_COL, 0), (A.OP_LIT, 0), (A.OP_GT, 0), (A.OP_COL, 1), (A.OP_COL, 2),
                                             (A.OP_LIT, 0), (A.OP_LIT, 0), (A.OP_CASE, 5)]
    assert prog[-1].dtype == A.FLOAT64
    assert [(i.op, i.col) for i in case([(col(2), col(0))]).program(S)][-1] == (A.OP_CASE, 2)
    assert repr(Case([(col(0) > 1, col(1))], 0.5)) == "CASE WHEN #0 Gt Int64(1) THEN #1 ELSE Float64(0.5) END"
    assert repr(case([(col(2), col(0))])) == "CASE WHEN #2 THEN #0 END"


def test_opcode_matches_the_header():
    with open(os.path.join(ROOT, "include", "dfgpu.h")) as f:
        header = f.read()
    assert int(re.search(r"DFGPU_OP_CASE\s*=\s*(\d+)", header).group(1)) == A.OP_CASE == 42
