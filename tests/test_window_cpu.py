"""Window functions without a GPU: the plan text of each shape, every refusal with its code and message, plans of queries
without a window call, and a self-check of tests/window_ref.py against a per-row loop over explicit frames."""
import numpy as np
import pytest

from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import host

import window_ref as W

SCAN = "TableScan: person projection=None"


@pytest.fixture(scope="module")
def cat():
    host.build()
    c = host.Catalog()
    c.add_table("person", [("id", A.UINT32), ("first_name", A.UTF8), ("last_name", A.UTF8), ("age", A.INT32), ("state", A.UTF8), ("salary", A.FLOAT64)])
    c.add_table("orders", [("oid", A.UINT32), ("pid", A.UINT32), ("amount", A.FLOAT64)])
    c.add_builtin_functions()
    return c


@pytest.mark.parametrize("sql,expected", [
    ("SELECT id, RANK() OVER (PARTITION BY state ORDER BY salary DESC) FROM person",
     "Projection: #0, #6\n  Window: windowExpr=[[RANK() OVER (PARTITION BY #4 ORDER BY #5 DESC)]]\n    " + SCAN),
    ("SELECT row_number() OVER (), Dense_Rank() OVER (ORDER BY age, id DESC) FROM person",
     "Projection: #6, #7\n  Window: windowExpr=[[row_number() OVER (), Dense_Rank() OVER (ORDER BY #3 ASC, #0 DESC)]]\n    " + SCAN),
    ("SELECT SUM(age) OVER (PARTITION BY state ORDER BY id), MIN(salary) OVER (PARTITION BY state, age), "
     "max(salary) OVER (), COUNT(*) OVER (), avg(age) OVER (ORDER BY salary) FROM person",
     "Projection: #6, #7, #8, #9, #10\n  Window: windowExpr=[[SUM(#3) OVER (PARTITION BY #4 ORDER BY #0 ASC), MIN(#5) OVER (PARTITION BY #4, #3), "
     "max(#5) OVER (), COUNT(#0) OVER (), avg(#3) OVER (ORDER BY #5 ASC)]]\n    " + SCAN),
    # inside expressions; equal calls share one column
    ("SELECT salary - AVG(salary) OVER (PARTITION BY state), AVG(salary) OVER (PARTITION BY state) FROM person WHERE age > 20",
     "Projection: #5 Minus #6, #6\n  Window: windowExpr=[[AVG(#5) OVER (PARTITION BY #4)]]\n    Selection: CAST(#3 AS Int64) Gt Int64(20)\n      " + SCAN),
    ("SELECT CAST(RANK() OVER (ORDER BY age) AS BIGINT) * 10 FROM person",
     "Projection: CAST(#6 AS Int64) Multiply Int64(10)\n  Window: windowExpr=[[RANK() OVER (ORDER BY #3 ASC)]]\n    " + SCAN),
    # over a join and over a semi join
    ("SELECT SUM(amount) OVER (PARTITION BY state ORDER BY o.oid) FROM person p JOIN orders o ON p.id = o.pid",
     "Projection: #9\n  Window: windowExpr=[[SUM(#8) OVER (PARTITION BY #4 ORDER BY #6 ASC)]]\n    Join: on=[#0 Eq #7]\n      " + SCAN +
     "\n      TableScan: orders projection=None"),
    ("SELECT MIN(age) OVER () + 1 FROM person WHERE id IN (SELECT pid FROM orders)",
     "Projection: CAST(#6 AS Int64) Plus Int64(1)\n  Window: windowExpr=[[MIN(#3) OVER ()]]\n    SemiJoin: on=[#0 Eq #6]\n      " + SCAN +
     "\n      Projection: #1\n        TableScan: orders projection=None"),
    # a query-level ORDER BY plans as before, over the projection
    ("SELECT id, RANK() OVER (ORDER BY age) FROM person ORDER BY id",
     "Sort: #0 ASC\n  Projection: #0, #6\n    Window: windowExpr=[[RANK() OVER (ORDER BY #3 ASC)]]\n      " + SCAN),
])
def test_plans(cat, sql, expected):
    assert cat.plan(sql) == expected


@pytest.mark.parametrize("sql,expected", [
    ("SELECT id, age FROM person WHERE age > 3", "Projection: #0, #3\n  Selection: CAST(#3 AS Int64) Gt Int64(3)\n    " + SCAN),
    ("SELECT over FROM over_t", None),  # OVER is no reserved word
    ("SELECT state, MAX(age) FROM person GROUP BY state", "Aggregate: groupBy=[[#4]], aggr=[[MAX(#3)]]\n  " + SCAN),
])
def test_queries_without_windows_plan_unchanged(cat, sql, expected):
    if expected is None:
        c = host.Catalog()
        c.add_table("over_t", [("over", A.INT64), ("partition", A.INT64)])
        assert c.plan(sql) == "Projection: #0\n  TableScan: over_t projection=None"
        assert c.plan("SELECT partition FROM over_t WHERE over > 1") == \
            "Projection: #1\n  Selection: #0 Gt Int64(1)\n    TableScan: over_t projection=None"
        return
    assert cat.plan(sql) == expected


@pytest.mark.parametrize("sql,code,msg", [
    ("SELECT id FROM person WHERE RANK() OVER () > 1", A.ERR_GENERAL, "window functions are not allowed in WHERE"),
    ("SELECT id FROM person p JOIN orders o ON p.id = o.pid AND RANK() OVER () = 1", A.ERR_GENERAL, "window functions are not allowed in ON"),
    ("SELECT state, COUNT(age) FROM person GROUP BY state, RANK() OVER ()", A.ERR_GENERAL, "window functions are not allowed in GROUP BY"),
    ("SELECT state, COUNT(age) FROM person GROUP BY state HAVING RANK() OVER () > 1", A.ERR_GENERAL, "window functions are not allowed in HAVING"),
    ("SELECT SUM(RANK() OVER ()) FROM person", A.ERR_GENERAL, "window functions are not allowed in an aggregate argument"),
    ("SELECT id FROM person WHERE id IN (SELECT RANK() OVER () FROM orders)", A.ERR_GENERAL,
     "window functions are not allowed in an IN / EXISTS subquery"),
    ("SELECT id FROM person WHERE EXISTS (SELECT oid FROM orders WHERE orders.pid = person.id AND RANK() OVER () > 1)", A.ERR_GENERAL,
     "window functions are not allowed in an IN / EXISTS subquery"),
    ("SELECT SUM(RANK() OVER ()) OVER () FROM person", A.ERR_GENERAL, "window functions cannot be nested"),
    ("SELECT RANK() OVER (PARTITION BY SUM(age) OVER ()) FROM person", A.ERR_GENERAL, "window functions cannot be nested"),
    ("SELECT state, COUNT(age), RANK() OVER () FROM person GROUP BY state", A.ERR_NOT_IMPLEMENTED,
     "window functions are not supported in an aggregate query"),
    ("SELECT COUNT(age), RANK() OVER () FROM person", A.ERR_NOT_IMPLEMENTED, "window functions are not supported in an aggregate query"),
    ("SELECT RANK() OVER (ORDER BY age ROWS BETWEEN 1 PRECEDING AND CURRENT ROW) FROM person", A.ERR_NOT_IMPLEMENTED,
     "window frame clauses are not supported"),
    ("SELECT SUM(age) OVER (ORDER BY age RANGE UNBOUNDED PRECEDING) FROM person", A.ERR_NOT_IMPLEMENTED, "window frame clauses are not supported"),
    ("SELECT COUNT(DISTINCT age) OVER () FROM person", A.ERR_NOT_IMPLEMENTED, "COUNT(DISTINCT x) OVER (..) is not supported"),
    ("SELECT RANK() OVER w FROM person", A.ERR_GENERAL, 'ParserError("named windows are not supported: write OVER (..)")'),
    ("SELECT LAG(age) OVER () FROM person", A.ERR_GENERAL, "Invalid function 'LAG'"),
    ("SELECT NTILE(4) OVER (ORDER BY age) FROM person", A.ERR_GENERAL, "Invalid function 'NTILE'"),
    ("SELECT FIRST_VALUE(age) OVER () FROM person", A.ERR_GENERAL, "Invalid function 'FIRST_VALUE'"),
    ("SELECT RANK() OVER (PARTITION BY age > 3) FROM person", A.ERR_NOT_IMPLEMENTED, "PARTITION BY a Boolean key is not supported"),
    ("SELECT RANK() OVER (ORDER BY age > 3) FROM person", A.ERR_NOT_IMPLEMENTED, "ORDER BY a Boolean key is not supported"),
    ("SELECT RANK(age) OVER () FROM person", A.ERR_GENERAL, "RANK() takes no arguments"),
])
def test_refusals(cat, sql, code, msg):
    with pytest.raises(host.ExecutionError) as e:
        cat.plan(sql)
    assert (e.value.code, e.value.msg) == (code, msg)


def test_window_clause_does_not_parse(cat):
    with pytest.raises(host.ExecutionError) as e:
        cat.plan("SELECT RANK() OVER () FROM person WINDOW w AS ()")
    assert e.value.code == A.ERR_GENERAL and e.value.msg.startswith("ParserError")


def test_reference_against_per_row_loop():
    rng = np.random.default_rng(1)
    for t in range(60):
        n = int(rng.integers(0, 40))
        k = rng.integers(0, 3, n)
        kv = rng.random(n) < 0.8
        o = rng.integers(0, 4, n).astype(np.float64)
        o[rng.random(n) < 0.1] = np.nan
        o[rng.random(n) < 0.1] = -0.0
        v = rng.integers(-5, 5, n).astype(np.int8) * 40
        vv = rng.random(n) < 0.7
        f = rng.integers(-8, 8, n) / 4.0
        part = [(A.INT64, k, kv)] if t % 3 else []
        order = [(A.FLOAT64, o, None, bool(t % 2))] if t % 4 else []
        arg, farg = (A.INT8, v, vv), (A.FLOAT64, f, vv)
        fns = [(W.ROW_NUMBER, None), (W.RANK, None), (W.DENSE_RANK, None), (W.COUNT, arg), (W.SUM, arg), (W.MIN, arg), (W.MAX, arg),
               (W.SUM, farg), (W.AVG, farg)]
        exp = W.window(n, part, order, fns)
        loop = W.window_loop(n, part, order, fns)
        for e, (vals, nulls), (fn, a) in zip(exp, loop, fns):
            if fn in (W.ROW_NUMBER, W.RANK, W.DENSE_RANK, W.COUNT):
                assert list(e["values"]) == vals, (t, fn)
                continue
            assert list(e["null"]) == nulls, (t, fn)
            for r in range(n):
                if nulls[r]:
                    continue
                xs = vals[r]
                if fn == W.SUM and a is arg:
                    want = np.array([sum(int(x) for x in xs)]).astype(np.int64).astype(np.int8)[0]
                elif fn == W.MIN:
                    want = min(xs)
                elif fn == W.MAX:
                    want = max(xs)
                else:  # multiples of 1/4: every sum is exact
                    want = sum(xs) / (len(xs) if fn == W.AVG else 1)
                    assert e["bound"][r] == 0 and float(e["exact"][r]) == want, (t, fn, r)
                    continue
                assert e["values"][r] == want, (t, fn, r)
