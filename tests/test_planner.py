"""The reference's planner tests replayed against the C++ host mirror (CPU only): every plan-text
test of src/sqlplanner.rs:547-686 verbatim, plus the coercion lattice and Rust Debug formatting."""
import pytest

from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import host


@pytest.fixture(scope="module")
def mock():
    host.build()
    c = host.Catalog()
    # MockSchemaProvider (src/sqlplanner.rs:761-789)
    c.add_table("person", [("id", A.UINT32), ("first_name", A.UTF8), ("last_name", A.UTF8), ("age", A.INT32), ("state", A.UTF8), ("salary", A.FLOAT64)])
    c.add_function("sqrt", [A.FLOAT64], A.FLOAT64)
    return c


CASES = [
    # (sql, expected plan text) — src/sqlplanner.rs:547-686
    ("SELECT 1", "Projection: Int64(1)\n  EmptyRelation"),
    ("SELECT sqrt(9)", "Projection: sqrt(CAST(Int64(9) AS Float64))\n  EmptyRelation"),
    ("SELECT id, first_name, last_name FROM person WHERE state = 'CO'",
     "Projection: #0, #1, #2\n  Selection: #4 Eq Utf8(\"CO\")\n    TableScan: person projection=None"),
    ("SELECT id, first_name, last_name FROM person WHERE state = 'CO' AND age >= 21 AND age <= 65",
     "Projection: #0, #1, #2\n  Selection: #4 Eq Utf8(\"CO\") And CAST(#3 AS Int64) GtEq Int64(21) And CAST(#3 AS Int64) LtEq Int64(65)\n    TableScan: person projection=None"),
    ("SELECT age, first_name, last_name FROM person WHERE age = 21 AND age != 21 AND age > 21 AND age >= 21 AND age < 65 AND age <= 65",
     "Projection: #3, #1, #2\n  Selection: CAST(#3 AS Int64) Eq Int64(21) And CAST(#3 AS Int64) NotEq Int64(21) And CAST(#3 AS Int64) Gt Int64(21) "
     "And CAST(#3 AS Int64) GtEq Int64(21) And CAST(#3 AS Int64) Lt Int64(65) And CAST(#3 AS Int64) LtEq Int64(65)\n    TableScan: person projection=None"),
    ("SELECT MIN(age) FROM person", "Aggregate: groupBy=[[]], aggr=[[MIN(#3)]]\n  TableScan: person projection=None"),
    ("SELECT SUM(age) from person", "Aggregate: groupBy=[[]], aggr=[[SUM(#3)]]\n  TableScan: person projection=None"),
    ("SELECT state, MIN(age), MAX(age) FROM person GROUP BY state",
     "Aggregate: groupBy=[[#4]], aggr=[[MIN(#3), MAX(#3)]]\n  TableScan: person projection=None"),
    ("SELECT COUNT(1) FROM person", "Aggregate: groupBy=[[]], aggr=[[COUNT(#0)]]\n  TableScan: person projection=None"),
    ("SELECT sqrt(age) FROM person", "Projection: sqrt(CAST(#3 AS Float64))\n  TableScan: person projection=None"),
    ("SELECT id FROM person ORDER BY id", "Sort: #0 ASC\n  Projection: #0\n    TableScan: person projection=None"),
    ("SELECT id FROM person ORDER BY id DESC", "Sort: #0 DESC\n  Projection: #0\n    TableScan: person projection=None"),
    ("SELECT id FROM person ORDER BY id DESC LIMIT 10", "Limit: 10\n  Sort: #0 DESC\n    Projection: #0\n      TableScan: person projection=None"),
    ("SELECT id FROM person LIMIT 10", "Limit: 10\n  Projection: #0\n    TableScan: person projection=None"),
]


@pytest.mark.parametrize("sql,expected", CASES, ids=[c[0][:40] for c in CASES])
def test_reference_plan_text(mock, sql, expected):
    assert mock.plan(sql) == expected


def test_more_planner_rules(mock):
    # COUNT(*) -> COUNT(#0) (sqlplanner.rs:330-335)
    assert mock.plan("SELECT COUNT(*) FROM person") == "Aggregate: groupBy=[[]], aggr=[[COUNT(#0)]]\n  TableScan: person projection=None"
    # Double literal vs Float64 column: no cast; Long literal vs Float64 column: literal is cast (sqlplanner.rs:286-291)
    assert mock.plan("SELECT salary FROM person WHERE salary > 51.0 AND salary < 53") == (
        "Projection: #5\n  Selection: #5 Gt Float64(51.0) And #5 Lt CAST(Int64(53) AS Float64)\n    TableScan: person projection=None")
    # aggregate output = group exprs then aggregates, regardless of SELECT order (sqlplanner.rs:83-118)
    assert mock.plan("SELECT SUM(salary), state FROM person GROUP BY state") == (
        "Aggregate: groupBy=[[#4]], aggr=[[SUM(#5)]]\n  TableScan: person projection=None")
    assert mock.plan("SELECT CAST(salary AS int) FROM person") == "Projection: CAST(#5 AS Int32)\n  TableScan: person projection=None"
    assert mock.plan("SELECT salary + age, salary * 2 FROM person WHERE age < 30") == (
        "Projection: #5 Plus CAST(#3 AS Float64), #5 Multiply CAST(Int64(2) AS Float64)\n"
        "  Selection: CAST(#3 AS Int64) Lt Int64(30)\n    TableScan: person projection=None")
    # the i64 extremes are literals as written; INT64_MIN is `-9223372036854775807 - 1`
    assert mock.plan("SELECT age FROM person WHERE age < 9223372036854775807 AND age > -9223372036854775807 - 1") == (
        "Projection: #3\n  Selection: CAST(#3 AS Int64) Lt Int64(9223372036854775807) And "
        "CAST(#3 AS Int64) Gt Int64(-9223372036854775807) Minus Int64(1)\n    TableScan: person projection=None")


def test_planner_errors(mock):
    for sql, msg in [
        ("SELECT id FROM nope", "no schema found for table nope"),
        ("SELECT nope FROM person", "Invalid identifier 'nope' for schema"),
        ("SELECT foo(id) FROM person", "Invalid function 'foo'"),
        ("SELECT id FROM person WHERE first_name > 5", "No common supertype found for binary operator Gt with input types Utf8 and Int64"),
        ("SELECT id FROM person GROUP BY id HAVING id > 1", "HAVING is not implemented yet"),
        ("SELECT * FROM person", "SQL wildcard operator is not supported in projection"),
        ("SELECT id FROM person LIMIT x", "LIMIT parameter is not a number"),
        ("SELECT id FROM", "ParserError"),
        # get_supertype(Int32, UInt32) = Int32 but can_coerce_from(Int32, UInt32) is false: the reference's
        # own lattice inconsistency (logicalplan.rs:474 vs :565-568), reproduced
        ("SELECT id FROM person WHERE age < id", "Cannot automatically convert UInt32 to Int32"),
        # integer literals whose digits do not fit i64 are refused, not saturated (the prefix `-` is not part of
        # the literal, so INT64_MIN itself is refused too)
        ("SELECT id FROM person WHERE id > 9223372036854775808", "9223372036854775808"),
        ("SELECT id FROM person WHERE id > -9223372036854775808", "9223372036854775808"),
        ("SELECT id + 99999999999999999999999 FROM person", "99999999999999999999999"),
    ]:
        with pytest.raises(host.ExecutionError) as e:
            mock.plan(sql)
        assert msg in e.value.msg, e.value.msg


def test_supertype_lattice():
    # spot checks of every region of src/logicalplan.rs:456-553
    S = host.supertype
    assert S(A.UINT8, A.INT8) == A.INT8 and S(A.INT8, A.UINT8) == A.INT8
    assert S(A.UINT16, A.INT8) is None and S(A.INT8, A.UINT16) is None
    assert S(A.UINT32, A.INT64) == A.INT64 and S(A.UINT64, A.INT64) == A.INT64 and S(A.UINT64, A.INT32) is None
    assert S(A.INT16, A.INT64) == A.INT64 and S(A.UINT8, A.UINT32) == A.UINT32
    assert S(A.INT64, A.FLOAT32) == A.FLOAT32 and S(A.FLOAT64, A.UINT8) == A.FLOAT64
    assert S(A.FLOAT32, A.FLOAT64) == A.FLOAT64 and S(A.FLOAT32, A.FLOAT32) == A.FLOAT32
    assert S(A.UTF8, A.UTF8) == A.UTF8 and S(A.BOOL, A.BOOL) == A.BOOL
    assert S(A.UTF8, A.INT64) is None and S(A.BOOL, A.INT8) is None


def test_rust_debug_f64(golden):
    # the golden strings of tests/sql.rs are `{:?}` renderings; the formatter must reproduce them
    for s in ["50.494344999999996", "51.105844000000005", "-3.17909", "0.10231", "1.0", "13.2", "3.3000000000000003"]:
        assert host.debug_f64(float(s)) == s
    assert host.debug_f64(1e16) == "1e16" and host.debug_f64(1e15) == "1000000000000000.0"
    assert host.debug_f64(1.5e-7) == "1.5e-7" and host.debug_f64(0.00001) == "0.00001"
    assert host.debug_f64(-0.0) == "-0.0"


def test_hostile_sql_ends_in_parser_errors_not_crashes(mock):
    # the parser, planner and plan printer recurse over the tree: depth and size are bounded
    for sql in ["SELECT " + "(" * 100_000 + "age" + ")" * 100_000 + " FROM person",
                "SELECT " + " + ".join(["age"] * 100_000) + " FROM person",
                "SELECT " + "CAST(" * 50_000 + "age" + " AS int)" * 50_000 + " FROM person",
                "SELECT " + "sqrt(" * 50_000 + "age" + ")" * 50_000 + " FROM person"]:
        with pytest.raises(host.ExecutionError) as e:
            mock.plan(sql)
        assert "ParserError" in str(e.value)
    assert mock.plan("SELECT " + "(" * 300 + "age" + ")" * 300 + " FROM person").startswith("Projection: #3")
    assert mock.plan("SELECT " + " + ".join(["age"] * 3000) + " FROM person").count("Plus") == 2999
    # random token soup: every input is either planned or rejected with an error
    import random
    rnd = random.Random(7)
    toks = ["SELECT", "FROM", "WHERE", "GROUP", "BY", "ORDER", "LIMIT", "AND", "OR", "NOT", "AS", "CAST", "(", ")", ",", "*", "+", "-", "/", "%",
            "=", "<", ">", "<=", ">=", "<>", "!=", "id", "age", "salary", "state", "person", "nobody", "COUNT", "MIN", "sqrt", "1", "2.5", "'x'",
            "'", "NULL", "IS", "int", "double", ";", "DESC", "1e400", "99999999999999999999", ".", "--", "\\"]
    planned = 0
    for _ in range(3000):
        sql = ("SELECT " if rnd.random() < 0.6 else "") + " ".join(rnd.choice(toks) for _ in range(rnd.randint(1, 12)))
        if rnd.random() < 0.5:
            sql += " FROM person"
        try:
            mock.plan(sql)
            planned += 1
        except host.ExecutionError:
            pass
    assert planned > 0
