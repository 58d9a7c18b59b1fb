"""IN / NOT IN / EXISTS / NOT EXISTS subqueries in the SQL front end (CPU only, mock catalog): the plan text of each
form as a semi or anti join, scoping, and every refusal."""
import pytest

from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import host


@pytest.fixture(scope="module")
def cat():
    host.build()
    c = host.Catalog()
    c.add_table("person", [("id", A.UINT32), ("first_name", A.UTF8), ("age", A.INT32), ("city", A.INT32)])
    c.add_table("city", [("id", A.INT32), ("name", A.UTF8), ("pop", A.INT64)])
    c.add_table("orders", [("oid", A.INT64), ("pid", A.UINT32), ("amount", A.FLOAT64), ("qty", A.INT32)])
    return c


S = {t: "TableScan: %s projection=None" % t for t in ("person", "city", "orders")}


def test_in(cat):
    assert cat.plan("SELECT first_name FROM person WHERE city IN (SELECT id FROM city WHERE pop > 1000)") == (
        "Projection: #1\n  SemiJoin: on=[#3 Eq #4]\n    %s\n    Projection: #0\n      Selection: #2 Gt Int64(1000)\n        %s"
        % (S["person"], S["city"]))


def test_not_in_with_coercion_casts(cat):
    # Int32 city against Int64 pop: the cast goes on the outer side; UInt32 id against Int64 oid on the subquery side
    assert cat.plan("SELECT first_name FROM person WHERE city NOT IN (SELECT pop FROM city)") == (
        "Projection: #1\n  AntiJoin (null-aware): on=[CAST(#3 AS Int64) Eq #4]\n    %s\n    Projection: #2\n      %s" % (S["person"], S["city"]))
    assert cat.plan("SELECT oid FROM orders WHERE oid IN (SELECT age FROM person)") == (
        "Projection: #0\n  SemiJoin: on=[#0 Eq #4]\n    %s\n    Projection: CAST(#2 AS Int64)\n      %s" % (S["orders"], S["person"]))


def test_exists_with_two_keys_and_select_star(cat):
    plan = ("Projection: #1\n  SemiJoin: on=[#0 Eq #4, #2 Eq #5]\n    %s\n    Projection: #1, #3\n      Selection: #2 Gt Float64(2.5)\n"
            "        %s" % (S["person"], S["orders"]))
    assert cat.plan("SELECT first_name FROM person p WHERE EXISTS (SELECT * FROM orders WHERE pid = p.id AND p.age = qty AND amount > 2.5)") == plan
    assert cat.plan("SELECT first_name FROM person p WHERE EXISTS (SELECT 1 FROM orders WHERE pid = p.id AND p.age = qty AND amount > 2.5)") == plan
    assert cat.plan("SELECT first_name FROM person WHERE NOT EXISTS (SELECT oid FROM orders WHERE orders.pid = person.id)") == (
        "Projection: #1\n  AntiJoin: on=[#0 Eq #4]\n    %s\n    Projection: #1\n      %s" % (S["person"], S["orders"]))


def test_correlated_in(cat):
    assert cat.plan("SELECT first_name FROM person p WHERE city IN (SELECT id FROM city WHERE pop = p.age)") == (
        "Projection: #1\n  SemiJoin: on=[#3 Eq #4, CAST(#2 AS Int64) Eq #5]\n    %s\n    Projection: #0, #2\n      %s" % (S["person"], S["city"]))


def test_two_subqueries_and_other_terms(cat):
    assert cat.plan("SELECT first_name FROM person WHERE age > 3 AND city IN (SELECT id FROM city) AND id NOT IN (SELECT pid FROM orders) "
                    "AND age < 90") == (
        "Projection: #1\n  Selection: CAST(#2 AS Int64) Gt Int64(3) And CAST(#2 AS Int64) Lt Int64(90)\n"
        "    AntiJoin (null-aware): on=[#0 Eq #4]\n      SemiJoin: on=[#3 Eq #4]\n        %s\n        Projection: #0\n          %s\n"
        "      Projection: #1\n        %s" % (S["person"], S["city"], S["orders"]))


def test_under_group_by_with_the_fused_selection(cat):
    assert cat.plan("SELECT city, COUNT(id), SUM(age) FROM person WHERE age > 1 AND city IN (SELECT id FROM city) GROUP BY city") == (
        "Aggregate: groupBy=[[#3]], aggr=[[COUNT(#0), SUM(#2)]]\n  Selection: CAST(#2 AS Int64) Gt Int64(1)\n    SemiJoin: on=[#3 Eq #4]\n"
        "      %s\n      Projection: #0\n        %s" % (S["person"], S["city"]))


def test_under_a_join_with_its_residual(cat):
    assert cat.plan("SELECT oid FROM orders JOIN person ON pid = person.id AND qty > age WHERE city IN (SELECT id FROM city)") == (
        "Projection: #0\n  Selection: #3 Gt #6\n    SemiJoin: on=[#7 Eq #8]\n      Join: on=[#1 Eq #4]\n        %s\n        %s\n"
        "      Projection: #0\n        %s" % (S["orders"], S["person"], S["city"]))


def test_nested_subquery(cat):
    assert cat.plan("SELECT first_name FROM person WHERE id IN (SELECT pid FROM orders WHERE qty IN (SELECT id FROM city WHERE pop > 5))") == (
        "Projection: #1\n  SemiJoin: on=[#0 Eq #4]\n    %s\n    Projection: #1\n      SemiJoin: on=[#3 Eq #4]\n        %s\n"
        "        Projection: #0\n          Selection: #2 Gt Int64(5)\n            %s" % (S["person"], S["orders"], S["city"]))


def test_scoping(cat):
    # `id` and `name`-less `pop` resolve in the subquery (city.id shadows person.id); `p.id` reaches the outer query
    assert cat.plan("SELECT first_name FROM person p WHERE EXISTS (SELECT 1 FROM city WHERE id = p.city AND pop > 7)") == (
        "Projection: #1\n  SemiJoin: on=[#3 Eq #4]\n    %s\n    Projection: #0\n      Selection: #2 Gt Int64(7)\n        %s" % (S["person"], S["city"]))
    assert cat.plan("SELECT first_name FROM person WHERE EXISTS (SELECT 1 FROM city WHERE CAST(id AS BIGINT) = CAST(person.id AS BIGINT))") == (
        "Projection: #1\n  SemiJoin: on=[CAST(#0 AS Int64) Eq #4]\n    %s\n    Projection: CAST(#0 AS Int64)\n      %s" % (S["person"], S["city"]))
    # a subquery over the outer query's own table
    assert cat.plan("SELECT first_name FROM person WHERE id IN (SELECT id FROM person WHERE age > 3)") == (
        "Projection: #1\n  SemiJoin: on=[#0 Eq #4]\n    %s\n    Projection: #0\n      Selection: CAST(#2 AS Int64) Gt Int64(3)\n        %s"
        % (S["person"], S["person"]))


@pytest.mark.parametrize("sql,code,msg", [
    ("SELECT age FROM person WHERE EXISTS (SELECT 1 FROM city WHERE pop > 3)", A.ERR_NOT_IMPLEMENTED,
     "EXISTS subquery without a correlated equality is not supported"),
    ("SELECT age FROM person p WHERE city IN (SELECT id FROM city WHERE pop > p.age)", A.ERR_NOT_IMPLEMENTED,
     "a correlated subquery term must be an equality between an inner and an outer expression"),
    ("SELECT age FROM person p WHERE city IN (SELECT id FROM city WHERE p.age > 3)", A.ERR_NOT_IMPLEMENTED,
     "a subquery WHERE term over outer columns only is not supported"),
    ("SELECT age FROM person p WHERE city NOT IN (SELECT id FROM city WHERE pop = p.age)", A.ERR_NOT_IMPLEMENTED,
     "correlated NOT IN subqueries are not supported"),
    ("SELECT age FROM person p WHERE city IN (SELECT id FROM city WHERE id IN (SELECT qty FROM orders WHERE oid = p.age))",
     A.ERR_NOT_IMPLEMENTED, "correlation that skips a level"),
    ("SELECT age FROM person WHERE city IN (SELECT MAX(id) FROM city)", A.ERR_NOT_IMPLEMENTED, "aggregates are not supported in an IN subquery"),
    ("SELECT age FROM person p WHERE EXISTS (SELECT COUNT(id) FROM city WHERE id = p.city)", A.ERR_NOT_IMPLEMENTED,
     "aggregates are not supported in an EXISTS subquery"),
    ("SELECT age FROM person WHERE city IN (SELECT id FROM city GROUP BY id)", A.ERR_NOT_IMPLEMENTED, "GROUP BY, HAVING, ORDER BY and LIMIT"),
    ("SELECT age FROM person WHERE city IN (SELECT id FROM city ORDER BY id)", A.ERR_NOT_IMPLEMENTED, "GROUP BY, HAVING, ORDER BY and LIMIT"),
    ("SELECT age FROM person WHERE city IN (SELECT id FROM city LIMIT 3)", A.ERR_NOT_IMPLEMENTED, "GROUP BY, HAVING, ORDER BY and LIMIT"),
    ("SELECT age FROM person WHERE city IN (SELECT id, pop FROM city)", A.ERR_GENERAL, "IN subquery must return exactly one column"),
    ("SELECT age FROM person WHERE age > 1 OR city IN (SELECT id FROM city)", A.ERR_NOT_IMPLEMENTED,
     "IN / EXISTS subqueries are supported only as AND terms of WHERE"),
    ("SELECT city IN (SELECT id FROM city) FROM person", A.ERR_NOT_IMPLEMENTED, "supported only as AND terms of WHERE"),
    ("SELECT age FROM person JOIN city ON person.city = city.id AND pop IN (SELECT oid FROM orders)", A.ERR_NOT_IMPLEMENTED,
     "supported only as AND terms of WHERE"),
    ("SELECT COUNT(age) FROM person GROUP BY city IN (SELECT id FROM city)", A.ERR_NOT_IMPLEMENTED, "supported only as AND terms of WHERE"),
    ("SELECT SUM(age) FROM person p WHERE NOT (EXISTS (SELECT 1 FROM city WHERE id = p.city))", A.ERR_GENERAL, "Invalid function 'NOT'"),
    ("SELECT age FROM person WHERE city IN (1, 2)", A.ERR_NOT_IMPLEMENTED, "IN over a list of values is not supported"),
    ("SELECT age FROM person WHERE city IN city", A.ERR_GENERAL, "ParserError"),
    ("SELECT age FROM person WHERE city NOT BETWEEN 1 AND 2", A.ERR_GENERAL, "ParserError"),
    ("SELECT age FROM person WHERE EXISTS(1)", A.ERR_GENERAL, "Invalid function 'EXISTS'"),
    ("SELECT age FROM person WHERE first_name IN (SELECT pop FROM city)", A.ERR_GENERAL, "No common supertype found for binary operator Eq"),
])
def test_refusals(cat, sql, code, msg):
    with pytest.raises(host.ExecutionError) as e:
        cat.plan(sql)
    assert e.value.code == code and msg in e.value.msg, e.value.msg
