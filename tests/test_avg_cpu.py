"""AVG(expr) in the SQL front-end, the C ABI and the Python harness, without a GPU: plan text, the function code and
the lowering."""
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
    ("SELECT AVG(age) FROM person", "Aggregate: groupBy=[[]], aggr=[[AVG(#3)]]\n  TableScan: person projection=None"),
    ("SELECT state, AVG(age) FROM person GROUP BY state",
     "Aggregate: groupBy=[[#4]], aggr=[[AVG(#3)]]\n  TableScan: person projection=None"),
    ("SELECT id, SUM(salary), avg(salary), COUNT(salary) FROM person WHERE age > 30 GROUP BY id",
     "Aggregate: groupBy=[[#0]], aggr=[[SUM(#5), avg(#5), COUNT(#5)]]\n  Selection: CAST(#3 AS Int64) Gt Int64(30)\n"
     "    TableScan: person projection=None"),
])
def test_plan_text(cat, sql, expected):
    assert cat.plan(sql) == expected


def test_avg_distinct_is_a_parse_error(cat):
    with pytest.raises(host.ExecutionError) as e:
        cat.plan("SELECT AVG(DISTINCT age) FROM person")
    assert e.value.code == A.ERR_GENERAL and "DISTINCT is only supported in COUNT(DISTINCT expr)" in e.value.msg


def test_abi_constant_matches_header():
    with open(os.path.join(A.repo_root(), "include", "dfgpu.h")) as f:
        text = f.read()
    m = re.search(r"DFGPU_AGG_AVG\s*=\s*(\d+)", text)
    assert m and int(m.group(1)) == A.AGG_AVG == 6
    assert int(re.search(r"#define DFGPU_ABI_VERSION (\d+)", text).group(1)) == A.ABI_VERSION == 2


def test_python_ir():
    for dt in (A.INT8, A.INT32, A.UINT64, A.FLOAT32, A.FLOAT64):
        func, prog, rt = AggregateFunction("avg", col(1)).lower([A.INT64, dt])
        assert func == A.AGG_AVG == 6 and rt == A.FLOAT64 and len(prog) == 1
    assert AggregateFunction("AVG", col(0)).lower([A.INT16])[0] == A.AGG_AVG
    assert AggregateFunction("avg", col(0), return_type=A.FLOAT32).lower([A.INT16])[2] == A.FLOAT32  # passed through as given
