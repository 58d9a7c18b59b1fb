"""JOIN in the SQL front end (CPU only, mock catalog): plan text of inner joins, qualified names and aliases, and every
refusal."""
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


SCANS = {t: "TableScan: %s projection=None" % t for t in ("person", "city", "orders")}


def test_two_table_join(cat):
    assert cat.plan("SELECT first_name, name FROM person JOIN city ON city = city.id") == (
        "Projection: #1, #5\n  Join: on=[#3 Eq #4]\n    %s\n    %s" % (SCANS["person"], SCANS["city"]))
    # INNER JOIN is the same plan; the key is oriented left / right whichever side it is written on
    assert cat.plan("SELECT first_name FROM person INNER JOIN city ON city.id = person.city") == (
        "Projection: #1\n  Join: on=[#3 Eq #4]\n    %s\n    %s" % (SCANS["person"], SCANS["city"]))


def test_qualified_names_and_aliases(cat):
    assert cat.plan("SELECT person.id, city.id FROM person JOIN city ON person.city = city.id") == (
        "Projection: #0, #4\n  Join: on=[#3 Eq #4]\n    %s\n    %s" % (SCANS["person"], SCANS["city"]))
    assert cat.plan("SELECT p.id, c.name FROM person AS p JOIN city c ON p.city = c.id") == (
        "Projection: #0, #5\n  Join: on=[#3 Eq #4]\n    %s\n    %s" % (SCANS["person"], SCANS["city"]))
    # qualified names in a single-table query; the plan text is unchanged
    assert cat.plan("SELECT person.age FROM person WHERE person.age > 3") == cat.plan("SELECT age FROM person WHERE age > 3")
    assert cat.plan("SELECT p.age FROM person p") == "Projection: #2\n  %s" % SCANS["person"]


def test_self_join_through_aliases(cat):
    assert cat.plan("SELECT a.id, b.id FROM person a JOIN person b ON a.age = b.age") == (
        "Projection: #0, #4\n  Join: on=[#2 Eq #6]\n    %s\n    %s" % (SCANS["person"], SCANS["person"]))


def test_two_keys_and_coercion_cast(cat):
    # UInt32 person.id against UInt32 orders.pid: no cast; Int32 qty against Int64 city.pop: CAST on the narrower side
    assert cat.plan("SELECT oid FROM orders JOIN person ON pid = person.id AND qty = age") == (
        "Projection: #0\n  Join: on=[#1 Eq #4, #3 Eq #6]\n    %s\n    %s" % (SCANS["orders"], SCANS["person"]))
    assert cat.plan("SELECT name FROM person JOIN city ON person.city = city.pop") == (
        "Projection: #5\n  Join: on=[CAST(#3 AS Int64) Eq #6]\n    %s\n    %s" % (SCANS["person"], SCANS["city"]))


def test_residual_terms_and_where_in_one_selection(cat):
    assert cat.plan("SELECT first_name FROM person JOIN city ON person.city = city.id AND pop > 1000 AND age < pop "
                    "WHERE person.age > 5") == (
        "Projection: #1\n  Selection: #6 Gt Int64(1000) And CAST(#2 AS Int64) Lt #6 And CAST(#2 AS Int64) Gt Int64(5)\n"
        "    Join: on=[#3 Eq #4]\n      %s\n      %s" % (SCANS["person"], SCANS["city"]))


def test_join_under_group_by(cat):
    assert cat.plan("SELECT name, SUM(age), COUNT(DISTINCT person.id) FROM person JOIN city ON person.city = city.id GROUP BY name") == (
        "Aggregate: groupBy=[[#5]], aggr=[[SUM(#2), COUNT(DISTINCT #0)]]\n  Join: on=[#3 Eq #4]\n    %s\n    %s"
        % (SCANS["person"], SCANS["city"]))


def test_three_table_chain(cat):
    assert cat.plan("SELECT oid, name FROM orders JOIN person ON pid = person.id JOIN city ON person.city = city.id WHERE amount > 1.5") == (
        "Projection: #0, #9\n  Selection: #2 Gt Float64(1.5)\n    Join: on=[#7 Eq #8]\n      Join: on=[#1 Eq #4]\n"
        "        %s\n        %s\n      %s" % (SCANS["orders"], SCANS["person"], SCANS["city"]))


@pytest.mark.parametrize("sql,code,msg", [
    ("SELECT id FROM person JOIN city ON person.city = city.id", A.ERR_GENERAL, "Ambiguous reference to column 'id'"),
    ("SELECT x.id FROM person JOIN city ON person.city = city.id", A.ERR_EXECUTION, "Invalid identifier 'x.id'"),
    ("SELECT person.nope FROM person", A.ERR_EXECUTION, "Invalid identifier 'person.nope'"),
    ("SELECT age FROM person JOIN person ON age = age", A.ERR_GENERAL, "appears more than once in FROM: give each occurrence an alias"),
    ("SELECT age FROM person JOIN city ON pop + 1", A.ERR_GENERAL, "JOIN ON expression did not evaluate to boolean"),
    ("SELECT age FROM person JOIN city ON age > pop", A.ERR_NOT_IMPLEMENTED, "JOIN needs at least one equality between the two inputs"),
    ("SELECT age FROM person JOIN city ON age = 3", A.ERR_NOT_IMPLEMENTED, "JOIN needs at least one equality between the two inputs"),
    ("SELECT age FROM person LEFT JOIN city ON person.city = city.id", A.ERR_NOT_IMPLEMENTED, "LEFT JOIN"),
    ("SELECT age FROM person RIGHT JOIN city ON person.city = city.id", A.ERR_NOT_IMPLEMENTED, "RIGHT JOIN"),
    ("SELECT age FROM person FULL OUTER JOIN city ON person.city = city.id", A.ERR_NOT_IMPLEMENTED, "FULL JOIN"),
    ("SELECT age FROM person LEFT OUTER JOIN city ON person.city = city.id", A.ERR_NOT_IMPLEMENTED, "LEFT JOIN"),
    ("SELECT age FROM person CROSS JOIN city", A.ERR_NOT_IMPLEMENTED, "CROSS JOIN"),
    ("SELECT age FROM person NATURAL JOIN city", A.ERR_NOT_IMPLEMENTED, "NATURAL JOIN"),
    ("SELECT age FROM person JOIN city USING (id)", A.ERR_GENERAL, "ParserError"),
    ("SELECT age FROM person, city", A.ERR_GENERAL, "ParserError"),
    ("SELECT age FROM person JOIN city", A.ERR_GENERAL, "ParserError"),
])
def test_join_errors(cat, sql, code, msg):
    with pytest.raises(host.ExecutionError) as e:
        cat.plan(sql)
    assert e.value.code == code and msg in e.value.msg, e.value.msg
