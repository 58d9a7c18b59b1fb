#!/usr/bin/env python
"""Generate tests/golden/reference_vectors.json from a checkout of the reference
(usage: make_fixtures.py <reference checkout>; the tests only read what it writes).

Inputs are the reference's own test fixtures (test/data/*.csv) and the golden strings / values its
tests assert (tests/sql.rs, src/execution/aggregate.rs).  The expected strings are extracted from
the reference's test sources by regex at generation time, not retyped.
"""
import csv
import json
import os
import re
import sys

REF = sys.argv[1]
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_vectors.json")


def read_csv(path, has_header):
    with open(path, newline="") as f:
        rows = list(csv.reader(f))
    # CsvDataSource::new passes has_headers = true unconditionally (src/execution/datasource.rs:41),
    # so line 1 is always swallowed — even for uk_cities.csv, which has no header (SURVEY App.A #5).
    return rows[1:] if has_header else rows


def rust_string_literal(src, after):
    """First Rust string literal following `after` in src, unescaped."""
    i = src.index(after)
    m = re.compile(r'"((?:[^"\\]|\\.)*)"', re.S).search(src, i + len(after))
    s = m.group(1)
    s = re.sub(r"\\\n\s*", "", s)  # line continuation
    return s.replace('\\"', '"').replace("\\t", "\t").replace("\\n", "\n").replace("\\\\", "\\")


def main():
    sql_rs = open(os.path.join(REF, "tests/sql.rs")).read()
    agg_rs = open(os.path.join(REF, "src/execution/aggregate.rs")).read()
    cities = read_csv(os.path.join(REF, "test/data/uk_cities.csv"), True)
    agg1 = read_csv(os.path.join(REF, "test/data/aggregate_test_1.csv"), True)
    agg2 = read_csv(os.path.join(REF, "test/data/aggregate_test_2.csv"), True)
    out = {
        "_generated_by": "tests/golden/make_fixtures.py from andygrove/datafusion-archive",
        "uk_cities": {  # schema tests/sql.rs:79-87
            "city": [r[0] for r in cities], "lat": [float(r[1]) for r in cities], "lng": [float(r[2]) for r in cities],
        },
        "aggregate_test_1": {"a": [int(r[0]) for r in agg1], "b": [float(r[1]) for r in agg1]},  # tests/sql.rs:42-45
        "aggregate_test_2": {"a": [r[0] for r in agg2], "b": [float(r[1]) for r in agg2]},        # tests/sql.rs:57-60
        "csv_query_with_predicate": {  # tests/sql.rs:30-37
            "sql": rust_string_literal(sql_rs, "fn csv_query_with_predicate"),
            "expected": rust_string_literal(sql_rs, "let expected= "),
        },
        "csv_query_group_by_int_min_max": {  # tests/sql.rs:40-52
            "sql": rust_string_literal(sql_rs[sql_rs.index("fn csv_query_group_by_int_min_max"):], "let sql = "),
            "expected": rust_string_literal(sql_rs[sql_rs.index("fn csv_query_group_by_int_min_max"):], "let expected = "),
        },
        "csv_query_group_by_string_min_max": {  # tests/sql.rs:55-67
            "sql": rust_string_literal(sql_rs[sql_rs.index("fn csv_query_group_by_string_min_max"):], "let sql = "),
            "expected": rust_string_literal(sql_rs[sql_rs.index("fn csv_query_group_by_string_min_max"):], "let expected = "),
        },
        "csv_query_cast": {  # tests/sql.rs:70-77
            "sql": rust_string_literal(sql_rs[sql_rs.index("fn csv_query_cast"):], "let sql = "),
            "expected": rust_string_literal(sql_rs[sql_rs.index("fn csv_query_cast"):], "let expected= "),
        },
        # src/execution/aggregate.rs:996,1030
        "min_lat": float(re.search(r"assert_eq!\(([0-9.]+), min_lat.value\(0\)\)", agg_rs).group(1)),
        "max_lat": float(re.search(r"assert_eq!\(([0-9.]+), max_lat.value\(0\)\)", agg_rs).group(1)),
        # src/execution/aggregate.rs:1113-1126: (a, min, max, sum) per output row
        "test_min_max_sum_group_by": [
            [float(x) for x in re.findall(r"assert_eq!\(([0-9.]+), (?:a|min|max|sum).value\(%d\)\)" % row, agg_rs)]
            for row in range(3)
        ],
    }
    with open(OUT, "w") as f:
        json.dump(out, f, indent=1)
    print("wrote", OUT)
    # byte-for-byte copies of the three CSV data files the hot-path tests open (test DATA, not source),
    # so CsvDataSource can be exercised without the reference checkout
    import shutil
    data = os.path.join(os.path.dirname(OUT), "data")
    os.makedirs(data, exist_ok=True)
    for name in ["uk_cities.csv", "aggregate_test_1.csv", "aggregate_test_2.csv", "people.csv"]:
        shutil.copyfile(os.path.join(REF, "test/data", name), os.path.join(data, name))
    print("copied CSV fixtures to", data)


if __name__ == "__main__":
    main()
