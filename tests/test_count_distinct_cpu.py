"""COUNT(DISTINCT expr) in the SQL front-end and the C ABI, without a GPU: plan text, parser and planner errors, and
the function code."""
import os
import re

import pytest

from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import host
from datafusion_archive_b200.expr import AggregateFunction, col


@pytest.fixture(scope="module")
def cat():
    host.build()
    c = host.Catalog()
    c.add_table("person", [("id", A.UINT32), ("first_name", A.UTF8), ("last_name", A.UTF8), ("age", A.INT32), ("state", A.UTF8), ("salary", A.FLOAT64)])
    return c


@pytest.mark.parametrize("sql,expected", [
    ("SELECT state, COUNT(DISTINCT age) FROM person GROUP BY state",
     "Aggregate: groupBy=[[#4]], aggr=[[COUNT(DISTINCT #3)]]\n  TableScan: person projection=None"),
    ("SELECT COUNT(DISTINCT salary) FROM person", "Aggregate: groupBy=[[]], aggr=[[COUNT(DISTINCT #5)]]\n  TableScan: person projection=None"),
    ("SELECT count(distinct age + age), SUM(salary) FROM person",
     "Aggregate: groupBy=[[]], aggr=[[count(DISTINCT #3 Plus #3), SUM(#5)]]\n  TableScan: person projection=None"),
    ("SELECT id, SUM(salary), COUNT(DISTINCT age), COUNT(age) FROM person WHERE salary > 1.0 GROUP BY id",
     "Aggregate: groupBy=[[#0]], aggr=[[SUM(#5), COUNT(DISTINCT #3), COUNT(#3)]]\n  Selection: #5 Gt Float64(1.0)\n"
     "    TableScan: person projection=None"),
])
def test_plan_text(cat, sql, expected):
    assert cat.plan(sql) == expected


@pytest.mark.parametrize("sql,code,msg", [
    ("SELECT SUM(DISTINCT age) FROM person", A.ERR_GENERAL, "DISTINCT is only supported in COUNT(DISTINCT expr)"),
    ("SELECT MIN(DISTINCT age) FROM person", A.ERR_GENERAL, "DISTINCT is only supported in COUNT(DISTINCT expr)"),
    ("SELECT COUNT(DISTINCT *) FROM person", A.ERR_GENERAL, "COUNT(DISTINCT *) is not supported"),
    ("SELECT COUNT(DISTINCT age, salary) FROM person", A.ERR_GENERAL, "COUNT(DISTINCT) takes exactly one argument"),
    ("SELECT DISTINCT age FROM person", A.ERR_GENERAL, "Unexpected token after end of statement"),
])
def test_errors(cat, sql, code, msg):
    with pytest.raises(host.ExecutionError) as e:
        cat.plan(sql)
    assert e.value.code == code and msg in e.value.msg


def test_abi_constant_matches_header():
    with open(os.path.join(A.repo_root(), "include", "dfgpu.h")) as f:
        m = re.search(r"DFGPU_AGG_COUNT_DISTINCT\s*=\s*(\d+)", f.read())
    assert m and int(m.group(1)) == A.AGG_COUNT_DISTINCT == 5
    assert A.ABI_VERSION == 2


def test_python_ir():
    func, prog, rt = AggregateFunction("count", col(1), distinct=True).lower([A.INT64, A.FLOAT32])
    assert func == A.AGG_COUNT_DISTINCT and rt == A.UINT64 and len(prog) == 1
    assert AggregateFunction("count", col(1)).lower([A.INT64, A.FLOAT32])[0] == A.AGG_COUNT
    with pytest.raises(ValueError):
        AggregateFunction("sum", col(0), distinct=True)
