"""HAVING, ORDER BY and LIMIT over aggregate queries without a GPU: the plan text of each shape, every new planner error,
the refusals that stay, and a self-check of the reference order the GPU tests compare against."""
import functools
import math
import random
import struct

import pytest

from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import host

import sort_ref as R

SCAN = "TableScan: person projection=None"


@pytest.fixture(scope="module")
def cat():
    host.build()
    c = host.Catalog()
    c.add_table("person", [("id", A.UINT32), ("first_name", A.UTF8), ("last_name", A.UTF8), ("age", A.INT32), ("state", A.UTF8), ("salary", A.FLOAT64)])
    c.add_builtin_functions()
    return c


@pytest.mark.parametrize("sql,expected", [
    # ORDER BY only
    ("SELECT state, MIN(age), MAX(age) FROM person GROUP BY state ORDER BY state",
     "Sort: #0 ASC\n  Aggregate: groupBy=[[#4]], aggr=[[MIN(#3), MAX(#3)]]\n    " + SCAN),
    ("SELECT state, MIN(age), MAX(age) FROM person GROUP BY state ORDER BY MAX(age) DESC, state",
     "Sort: #2 DESC, #0 ASC\n  Aggregate: groupBy=[[#4]], aggr=[[MIN(#3), MAX(#3)]]\n    " + SCAN),
    # LIMIT only
    ("SELECT state, MIN(age), MAX(age) FROM person GROUP BY state LIMIT 3",
     "Limit: 3\n  Aggregate: groupBy=[[#4]], aggr=[[MIN(#3), MAX(#3)]]\n    " + SCAN),
    # HAVING only, over a SELECT-list aggregate
    ("SELECT state, MIN(age), MAX(age) FROM person GROUP BY state HAVING MAX(age) > 30",
     "Selection: CAST(#2 AS Int64) Gt Int64(30)\n  Aggregate: groupBy=[[#4]], aggr=[[MIN(#3), MAX(#3)]]\n    " + SCAN),
    # all three
    ("SELECT state, MIN(age), MAX(age) FROM person GROUP BY state HAVING MIN(age) < 20 ORDER BY MAX(age) DESC LIMIT 5",
     "Limit: 5\n  Sort: #2 DESC\n    Selection: CAST(#1 AS Int64) Lt Int64(20)\n      Aggregate: groupBy=[[#4]], aggr=[[MIN(#3), MAX(#3)]]\n        " + SCAN),
    # hidden aggregates: appended to aggr and dropped by the top Projection
    # (COUNT is UInt64, which the coercion lattice does not widen to Int64: the literal needs a CAST, as in WHERE)
    ("SELECT state, MIN(age) FROM person GROUP BY state HAVING CAST(COUNT(id) AS BIGINT) > 10 ORDER BY SUM(salary) DESC",
     "Projection: #0, #1\n  Sort: #3 DESC\n    Selection: CAST(#2 AS Int64) Gt Int64(10)\n"
     "      Aggregate: groupBy=[[#4]], aggr=[[MIN(#3), COUNT(#0), SUM(#5)]]\n        " + SCAN),
    # an ORDER BY aggregate equal to a SELECT-list one is not added again
    ("SELECT state, COUNT(id) FROM person GROUP BY state HAVING CAST(COUNT(id) AS BIGINT) > 1 ORDER BY COUNT(id)",
     "Sort: #1 ASC\n  Selection: CAST(#1 AS Int64) Gt Int64(1)\n    Aggregate: groupBy=[[#4]], aggr=[[COUNT(#0)]]\n      " + SCAN),
    # ordinals name SELECT-list items, in SELECT order (the aggregate's output puts the keys first)
    ("SELECT MIN(age), state FROM person GROUP BY state ORDER BY 2 DESC, 1",
     "Sort: #0 DESC, #1 ASC\n  Aggregate: groupBy=[[#4]], aggr=[[MIN(#3)]]\n    " + SCAN),
    # expression keys: arithmetic over aggregates, a function of a key
    ("SELECT state, SUM(salary), COUNT(salary) FROM person GROUP BY state ORDER BY SUM(salary) / COUNT(salary)",
     "Sort: #1 Divide CAST(#2 AS Float64) ASC\n  Aggregate: groupBy=[[#4]], aggr=[[SUM(#5), COUNT(#5)]]\n    " + SCAN),
    ("SELECT state, COUNT(id) FROM person GROUP BY state ORDER BY lower(state) DESC",
     "Sort: lower(#0) DESC\n  Aggregate: groupBy=[[#4]], aggr=[[COUNT(#0)]]\n    " + SCAN),
    # a GROUP BY expression matched as a whole
    ("SELECT age + 1, COUNT(id) FROM person GROUP BY age + 1 ORDER BY age + 1 DESC",
     "Sort: #0 DESC\n  Aggregate: groupBy=[[CAST(#3 AS Int64) Plus Int64(1)]], aggr=[[COUNT(#0)]]\n    " + SCAN),
    # no GROUP BY
    ("SELECT COUNT(id) FROM person HAVING CAST(COUNT(id) AS BIGINT) > 100",
     "Selection: CAST(#0 AS Int64) Gt Int64(100)\n  Aggregate: groupBy=[[]], aggr=[[COUNT(#0)]]\n    " + SCAN),
])
def test_plan_text(cat, sql, expected):
    assert cat.plan(sql) == expected


def test_plan_text_without_the_clauses_is_unchanged(cat):
    assert cat.plan("SELECT state, MIN(age), MAX(age) FROM person GROUP BY state") == "Aggregate: groupBy=[[#4]], aggr=[[MIN(#3), MAX(#3)]]\n  " + SCAN
    assert cat.plan("SELECT id FROM person ORDER BY id DESC LIMIT 10") == "Limit: 10\n  Sort: #0 DESC\n    Projection: #0\n      " + SCAN


@pytest.mark.parametrize("sql,code,msg", [
    ("SELECT state, COUNT(id) FROM person GROUP BY state ORDER BY age", A.ERR_GENERAL,
     "Column 'age' must appear in the GROUP BY clause or be used in an aggregate function"),
    ("SELECT state, COUNT(id) FROM person GROUP BY state HAVING salary > 1", A.ERR_GENERAL,
     "Column 'salary' must appear in the GROUP BY clause or be used in an aggregate function"),
    ("SELECT state, COUNT(id) FROM person GROUP BY state ORDER BY 3", A.ERR_GENERAL, "ORDER BY position 3 is not in select list"),
    ("SELECT state, COUNT(id) FROM person GROUP BY state ORDER BY 0", A.ERR_GENERAL, "ORDER BY position 0 is not in select list"),
    ("SELECT state, COUNT(id) FROM person GROUP BY state ORDER BY MIN(age) > 1", A.ERR_NOT_IMPLEMENTED, "ORDER BY a Boolean expression is not supported"),
    ("SELECT state, COUNT(id) FROM person GROUP BY state HAVING COUNT(id)", A.ERR_GENERAL, "HAVING expression did not evaluate to boolean"),
    ("SELECT state, COUNT(id) FROM person GROUP BY state LIMIT x", A.ERR_GENERAL, "LIMIT parameter is not a number"),
])
def test_planner_errors(cat, sql, code, msg):
    with pytest.raises(host.ExecutionError) as ei:
        cat.plan(sql)
    assert ei.value.code == code and msg in ei.value.msg


@pytest.mark.parametrize("sql,msg", [
    # no aggregate in the SELECT list: HAVING is still refused
    ("SELECT id FROM person GROUP BY id HAVING id > 1", "HAVING is not implemented yet"),
    # inside a subquery the clauses are still refused
    ("SELECT id FROM person WHERE id IN (SELECT id FROM person ORDER BY id)", "GROUP BY, HAVING, ORDER BY and LIMIT are not supported in an IN subquery"),
    ("SELECT id FROM person WHERE id IN (SELECT id FROM person LIMIT 1)", "GROUP BY, HAVING, ORDER BY and LIMIT are not supported in an IN subquery"),
])
def test_refusals_stay(cat, sql, msg):
    with pytest.raises(host.ExecutionError) as ei:
        cat.plan(sql)
    assert msg in ei.value.msg


def test_nulls_first_last_is_still_a_parse_error(cat):
    with pytest.raises(host.ExecutionError) as ei:
        cat.plan("SELECT state, COUNT(id) FROM person GROUP BY state ORDER BY state NULLS FIRST")
    assert "ParserError" in ei.value.msg


# ---- the reference order ---------------------------------------------------------------------------------------------
def _cmp_value(dtype, a, b):
    """The engine's order of two non-null values, from the definitions (not from the encoding)."""
    if dtype == A.UTF8:
        return (a > b) - (a < b)
    if dtype in (A.FLOAT32, A.FLOAT64):
        na, nb = math.isnan(a), math.isnan(b)
        if na or nb:
            return (na > nb) - (na < nb)
        if a == b == 0.0:
            sa, sb = math.copysign(1, a) < 0, math.copysign(1, b) < 0
            return (sb > sa) - (sb < sa)
    return (a > b) - (a < b)


def _cmp_rows(keys, i, j):
    for dtype, vals, valid, desc in keys:
        vi = valid is None or valid[i]
        vj = valid is None or valid[j]
        if not vi or not vj:
            c = (vi > vj) - (vi < vj)  # null below every value
        else:
            c = _cmp_value(dtype, vals[i], vals[j])
        if desc:
            c = -c
        if c:
            return c
    return (i > j) - (i < j)


@pytest.mark.parametrize("seed", range(6))
def test_reference_order_matches_sorted(seed):
    rng = random.Random(seed)
    n = 300
    f64 = [rng.choice([0.0, -0.0, 1.5, -1.5, math.inf, -math.inf, math.nan, struct.unpack("<d", struct.pack("<Q", 0xfff8000000000001))[0], 5e-324])
           for _ in range(n)]
    ints = [rng.randrange(-3, 3) for _ in range(n)]
    strs = [rng.choice(["", "a", "a\0", "ab", "b", "\x80", "aaaaaaaaa", "aaaaaaaab"]) for _ in range(n)]
    u64 = [rng.choice([0, 1, 2 ** 64 - 1, 2 ** 63]) for _ in range(n)]
    valid = [rng.random() > 0.2 for _ in range(n)]
    keys = [(A.FLOAT64, f64, None, rng.random() < 0.5), (A.INT32, ints, valid, rng.random() < 0.5),
            (A.UTF8, [s.encode("utf-8", "surrogatepass") for s in strs], None, rng.random() < 0.5), (A.UINT64, u64, None, rng.random() < 0.5)]
    rng.shuffle(keys)
    want = sorted(range(n), key=functools.cmp_to_key(lambda i, j: _cmp_rows(keys, i, j)))
    got = R.order(n, keys)
    assert list(got) == want
