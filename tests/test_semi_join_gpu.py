"""Semi and anti joins on the GPU (dfgpu_join_semi, and [NOT] IN / [NOT] EXISTS subqueries through ctx.sql()), compared
exactly with tests/join_ref.py, the reference of include/dfgpu.h's table: the passing probe rows, in probe order."""
import os

import numpy as np
import pyarrow as pa
import pytest

from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import engine, host
from datafusion_archive_b200.expr import col, lit
from join_ref import passing

pytestmark = pytest.mark.gpu

INTS = [np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64]
KINDS = {"semi": A.JOIN_SEMI, "anti": A.JOIN_ANTI, "anti_null_aware": A.JOIN_ANTI_NULL_AWARE}


@pytest.fixture(scope="module")
def ctx():
    c = engine.GpuContext(0)
    yield c
    c.close()


def gpu_pass(ctx, kind, probe_arrays, pkeys, build_arrays, bkeys):
    """the passing probe rows' numbers (a row-number column is appended to the probe side)"""
    n = len(probe_arrays[0])
    pb = ctx.upload(list(probe_arrays) + [np.arange(n, dtype=np.int64)])
    bb = ctx.upload(list(build_arrays))
    j = ctx.join_build(bb, bkeys, keep_cols=[])
    bb.free()
    r = j.semi(pb, pkeys, kind, probe_cols=[len(probe_arrays)])
    got = r.columns()[0]
    r.free(); j.free(); pb.free()
    return np.asarray(got, dtype=np.int64)


def check(ctx, kind, probe, pkeys, build, bkeys, pref=None, bref=None):
    exp = passing(kind, pref if pref is not None else probe, bref if bref is not None else build)
    got = gpu_pass(ctx, kind, probe, pkeys, build, bkeys)
    assert np.array_equal(got, exp), (len(got), len(exp))


def nullable(vals, valid, dtype):
    return pa.array(np.asarray(vals, dtype=dtype), mask=~np.asarray(valid, bool))


# ---- the C ABI --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", list(KINDS.values()), ids=list(KINDS))
@pytest.mark.parametrize("dt", INTS, ids=lambda d: np.dtype(d).name)
def test_every_integer_key_dtype(ctx, dt, kind):
    rng = np.random.default_rng(1)
    info = np.iinfo(dt)
    lo = -3 if info.min < 0 else 0
    special = [0, info.max, info.min, -1 if info.min < 0 else info.max - 1, 1]
    pk = np.concatenate([np.array(special, dtype=dt), rng.integers(lo, 9, 3000).astype(dt)])
    bk = np.concatenate([np.array(special[:3] * 2, dtype=dt), rng.integers(lo, 6, 500).astype(dt)])  # duplicates
    pcol = nullable(pk, rng.random(len(pk)) > 0.1, dt)
    for bcol in (nullable(bk, rng.random(len(bk)) > 0.1, dt), bk):  # nulls in the build side, and none
        check(ctx, kind, [pcol], [col(0)], [bcol], [col(0)])


@pytest.mark.parametrize("kind", list(KINDS.values()), ids=list(KINDS))
def test_empty_build_and_empty_probe(ctx, kind):
    pk = nullable([1, 2, 3, 0], [True, True, False, True], np.int64)
    empty = np.zeros(0, np.int64)
    check(ctx, kind, [pk], [col(0)], [empty], [col(0)])  # anti and null-aware anti: every row, the null one included
    check(ctx, kind, [empty], [col(0)], [np.array([1, 2], np.int64)], [col(0)])


def test_null_aware_null_in_build(ctx):
    # one null build key: NOT IN is never true, with the probe columns' types and no kernel launched
    pb = ctx.upload([np.array([1, 2, 3], np.int64), pa.array(["a", None, "c"]), np.array([True, False, True])])
    bb = ctx.upload([nullable([7, 8], [True, False], np.int64)])
    j = ctx.join_build(bb, [col(0)], keep_cols=[])
    before = ctx.kernel_launches()
    r = j.semi(pb, [col(0)], A.JOIN_ANTI_NULL_AWARE)
    assert ctx.kernel_launches() == before
    assert r.nrows == 0 and [r.dtype(i) for i in range(3)] == [A.INT64, A.UTF8, A.BOOL]
    r.columns()
    r.free()
    # the plain anti join over the same build: 1, 2 and 3 pass
    r = j.semi(pb, [col(0)], A.JOIN_ANTI, probe_cols=[0])
    assert np.array_equal(r.columns()[0], [1, 2, 3])
    r.free(); j.free(); pb.free(); bb.free()


@pytest.mark.parametrize("kind", list(KINDS.values()), ids=list(KINDS))
def test_all_pass_and_none_pass(ctx, kind):
    n = 70_000  # many tiles of 2048 rows, the last one ragged
    pk = np.arange(n, dtype=np.int64)
    check(ctx, kind, [pk], [col(0)], [pk.copy()], [col(0)])
    check(ctx, kind, [pk], [col(0)], [pk + n], [col(0)])


def utf8_keys(rng, n, words, null_frac):
    return pa.array([words[i] for i in rng.integers(0, len(words), n)], mask=rng.random(n) < null_frac)


WORDS = ["w%d" % i * (1 + i % 5) for i in range(300)] + ["", "x" * 40, "é", "a ", "a"]


@pytest.mark.parametrize("bits", [None, "4", "1"], ids=["64-bit-tags", "4-bit-tags", "1-bit-tags"])
@pytest.mark.parametrize("kind", list(KINDS.values()), ids=list(KINDS))
def test_utf8_keys(ctx, kind, bits, monkeypatch):
    if bits:
        monkeypatch.setenv("DFGPU_JOIN_TAG_BITS", bits)
    rng = np.random.default_rng(2)
    ps = utf8_keys(rng, 6000, WORDS + ["p%d" % i for i in range(50)], 0.05)
    for bs in (utf8_keys(rng, 900, WORDS, 0.05), utf8_keys(rng, 900, WORDS, 0.0)):
        check(ctx, kind, [ps], [col(0)], [bs], [col(0)])


@pytest.mark.parametrize("bits", [None, "4"], ids=["64-bit-tags", "4-bit-tags"])
@pytest.mark.parametrize("kind", [A.JOIN_SEMI, A.JOIN_ANTI], ids=["semi", "anti"])
def test_utf8_int32_composite_key(ctx, kind, bits, monkeypatch):
    if bits:
        monkeypatch.setenv("DFGPU_JOIN_TAG_BITS", bits)
    rng = np.random.default_rng(3)
    ps, bs = utf8_keys(rng, 5000, WORDS[:40], 0.03), utf8_keys(rng, 700, WORDS[:40], 0.03)
    pi = nullable(rng.integers(0, 4, 5000), rng.random(5000) > 0.03, np.int32)
    bi = nullable(rng.integers(0, 4, 700), rng.random(700) > 0.03, np.int32)
    check(ctx, kind, [ps, pi], [col(0), col(1)], [bs, bi], [col(0), col(1)])


def test_payload_columns_keep_validity(ctx):
    rng = np.random.default_rng(4)
    n = 9000
    pk = rng.integers(0, 100, n).astype(np.int32)
    bk = rng.integers(0, 100, 60).astype(np.int32)
    f64 = nullable(rng.random(n), rng.random(n) > 0.2, np.float64)
    bools = pa.array(rng.random(n) > 0.5, mask=rng.random(n) < 0.2)
    strs = pa.array(["s%d" % (i % 13) * (i % 4) for i in range(n)], mask=rng.random(n) < 0.2)
    pb = ctx.upload([pk, f64, bools, strs])
    bb = ctx.upload([bk])
    j = ctx.join_build(bb, [col(0)], keep_cols=[])
    for kind in (A.JOIN_SEMI, A.JOIN_ANTI):
        r = j.semi(pb, [col(0)], kind, probe_cols=[3, 1, 2, 0])
        got = r.columns()
        r.free()
        sel = passing(kind, [pk], [bk])
        assert np.array_equal(got[3], pk[sel])
        for g, a in zip(got[:3], (strs, f64, bools)):
            vals, valid = g if isinstance(g, tuple) else (g, np.ones(len(sel), bool))
            exp = [a[int(i)].as_py() for i in sel]
            assert [v if ok else None for v, ok in zip(list(vals), valid.tolist())] == exp
    j.free(); pb.free(); bb.free()


def test_key_programs_and_refusals(ctx):
    # a CAST key and an arithmetic key, evaluated as projections
    pk = np.array([4294967295, 5, 2147483648, 7], dtype=np.uint32)
    bk = np.array([-1, 5, -2147483648, 8], dtype=np.int32)
    assert np.array_equal(gpu_pass(ctx, A.JOIN_SEMI, [pk], [col(0).cast(A.INT32)], [bk], [col(0)]), [0, 1, 2])
    assert np.array_equal(gpu_pass(ctx, A.JOIN_ANTI, [np.arange(6, dtype=np.int64)], [col(0) + lit(1)], [np.arange(4, dtype=np.int64)], [col(0)]),
                          [3, 4, 5])
    bb = ctx.upload([np.array([1, 2], np.int32), np.array([1, 2], np.int64), np.array([1.0, 2.0])])
    pb = ctx.upload([np.array([1, 2], np.int64), np.array([1, 2], np.int32)])
    j = ctx.join_build(bb, [col(0), col(0)], keep_cols=[])
    with pytest.raises(engine.DfGpuError) as e:
        j.semi(pb, [col(1), col(1)], A.JOIN_ANTI_NULL_AWARE)
    assert e.value.code == A.ERR_GENERAL and "exactly one key" in e.value.msg
    with pytest.raises(engine.DfGpuError) as e:
        j.semi(pb, [col(1), col(1)], 7)
    assert e.value.code == A.ERR_GENERAL and "unknown kind" in e.value.msg
    j.free()
    j = ctx.join_build(bb, [col(0)], keep_cols=[])
    with pytest.raises(engine.DfGpuError) as e:
        j.semi(pb, [col(0)], A.JOIN_SEMI)
    assert e.value.code == A.ERR_EXECUTION and "JOIN key types differ: Int64 and Int32" in e.value.msg
    j.free()
    with pytest.raises(engine.DfGpuError) as e:
        ctx.join_build(bb, [col(2)], keep_cols=[])
    assert e.value.code == A.ERR_NOT_IMPLEMENTED and "Float64" in e.value.msg
    bb.free(); pb.free()


def test_large_probe_in_order(ctx):
    rng = np.random.default_rng(5)
    n = 6_000_000
    pk = rng.integers(0, 4_000_000, n, dtype=np.int64)
    payload = rng.random(n)
    bk = rng.integers(0, 4_000_000, 1_000_000, dtype=np.int64)
    member = np.isin(pk, bk)
    pb, bb = ctx.upload([pk, payload]), ctx.upload([bk])
    j = ctx.join_build(bb, [col(0)], keep_cols=[])
    for kind, mask in ((A.JOIN_SEMI, member), (A.JOIN_ANTI, ~member), (A.JOIN_ANTI_NULL_AWARE, ~member)):
        r = j.semi(pb, [col(0)], kind)
        got = r.columns()
        r.free()
        assert np.array_equal(got[0], pk[mask]) and np.array_equal(got[1], payload[mask])
    j.free(); pb.free(); bb.free()


# ---- through ctx.sql() ------------------------------------------------------------------------------------------------
def rows(batches):
    out = []
    for b in batches:
        cols = [c if isinstance(c, list) else np.asarray(c).tolist() for c in b]
        out.extend(zip(*cols))
    return sorted(out, key=repr)


N_PEOPLE = 40_000


@pytest.fixture(scope="module")
def data():
    rng = np.random.default_rng(11)
    n = N_PEOPLE
    dept_valid = rng.random(n) > 0.05
    people = {"id": np.arange(n, dtype=np.int64), "dept": nullable(rng.integers(0, 60, n), dept_valid, np.int32),
              "grp": rng.integers(0, 80, n).astype(np.int32), "salary": (rng.integers(-800, 8000, n) / 8).astype(np.float64),
              "name": ["n%d" % (i % 37) for i in range(n)]}
    dept_id = list(range(50)) + list(range(10)) + [None]  # 0..9 twice, 50..59 absent, one null
    dept = {"dept_id": pa.array(dept_id, type=pa.int32()), "region": np.array([(d or 3) % 7 for d in dept_id], np.int64),
            "dname": ["d%d" % (d if d is not None else -1) for d in dept_id]}
    return people, dept


def py_tables(data):
    people, dept = data
    p = [dict(zip(people, r)) for r in zip(*[v.to_pylist() if isinstance(v, pa.Array) else list(np.asarray(v).tolist()) if not isinstance(v, list) else v
                                           for v in people.values()])]
    d = [dict(zip(dept, r)) for r in zip(*[v.to_pylist() if isinstance(v, pa.Array) else list(np.asarray(v).tolist()) if not isinstance(v, list) else v
                                          for v in dept.values()])]
    return p, d


def run_sql(data, sql, batch_size):
    hctx = host.ExecutionContext(0)
    try:
        people, dept = data
        hctx.register_memory("people", list(people.items()), batch_size=batch_size)
        hctx.register_memory("dept", list(dept.items()), batch_size=batch_size // 1000 if batch_size else 0)
        return rows(hctx.sql(sql).collect())
    finally:
        hctx.close()


def not_in(x, ys):
    ys = list(ys)
    if not ys:
        return True
    return x is not None and None not in ys and x not in ys


@pytest.mark.parametrize("batch_size", [0, 7000], ids=["one-batch", "multi-batch"])
def test_sql_forms(data, batch_size):
    p, d = py_tables(data)
    r4 = [r["dept_id"] for r in d if r["region"] == 4]
    r2 = [r["dept_id"] for r in d if r["region"] == 2]
    all_ids = [r["dept_id"] for r in d]
    assert None in all_ids
    cases = [
        ("SELECT id, name FROM people WHERE dept IN (SELECT dept_id FROM dept WHERE region = 4)",
         [(r["id"], r["name"]) for r in p if r["dept"] is not None and r["dept"] in r4]),
        ("SELECT id FROM people WHERE dept IN (SELECT dept_id FROM dept)", [(r["id"],) for r in p if r["dept"] is not None and r["dept"] in all_ids]),
        # NOT IN over a subquery holding a null: nothing; without one: the non-null keys outside the set
        ("SELECT id FROM people WHERE dept NOT IN (SELECT dept_id FROM dept)", [(r["id"],) for r in p if not_in(r["dept"], all_ids)]),
        ("SELECT id FROM people WHERE dept NOT IN (SELECT dept_id FROM dept WHERE region = 2)",
         [(r["id"],) for r in p if not_in(r["dept"], r2)]),
        ("SELECT id FROM people WHERE dept NOT IN (SELECT dept_id FROM dept WHERE region > 100)", [(r["id"],) for r in p]),
        ("SELECT id, salary FROM people p WHERE EXISTS (SELECT 1 FROM dept d WHERE d.dept_id = p.dept AND d.region < 3)",
         [(r["id"], r["salary"]) for r in p if any(x["dept_id"] == r["dept"] and r["dept"] is not None and x["region"] < 3 for x in d)]),
        ("SELECT id FROM people p WHERE NOT EXISTS (SELECT * FROM dept WHERE dept_id = p.dept AND region < 3)",
         [(r["id"],) for r in p if not any(x["dept_id"] == r["dept"] and r["dept"] is not None and x["region"] < 3 for x in d)]),
        ("SELECT id FROM people p WHERE NOT EXISTS (SELECT 1 FROM dept WHERE dept_id = p.dept)",
         [(r["id"],) for r in p if r["dept"] is None or r["dept"] not in all_ids]),
        # correlated IN: the IN pair and a correlated equality, two keys
        ("SELECT id FROM people p WHERE grp IN (SELECT dept_id FROM dept WHERE CAST(region AS INT) = p.dept)",
         [(r["id"],) for r in p if r["dept"] is not None and any(x["dept_id"] == r["grp"] and x["region"] == r["dept"] for x in d)]),
        ("SELECT id FROM people WHERE grp IN (SELECT dept_id FROM dept WHERE region < 5) AND salary > 100",
         [(r["id"],) for r in p if r["grp"] in [x["dept_id"] for x in d if x["region"] < 5] and r["salary"] > 100]),
        # a subquery over the outer query's own table
        ("SELECT id FROM people WHERE grp IN (SELECT grp FROM people WHERE salary > 990)",
         [(r["id"],) for r in p if r["grp"] in {x["grp"] for x in p if x["salary"] > 990}]),
    ]
    for sql, exp in cases:
        assert run_sql(data, sql, batch_size) == sorted(exp, key=repr), sql


@pytest.mark.parametrize("batch_size", [0, 7000], ids=["one-batch", "multi-batch"])
def test_sql_aggregate_over_semi_join(data, batch_size):
    p, d = py_tables(data)
    ids = {x["dept_id"] for x in d if x["region"] > 3}
    sel = [r for r in p if r["salary"] > 0 and r["dept"] is not None and r["dept"] in ids]
    groups = {}
    for r in sel:
        groups.setdefault(r["grp"], []).append(r)
    got = run_sql(data, "SELECT grp, COUNT(id), SUM(salary) FROM people WHERE salary > 0 AND dept IN (SELECT dept_id FROM dept WHERE region > 3) "
                        "GROUP BY grp", batch_size)
    assert got == sorted([(k, len(g), sum(r["salary"] for r in g)) for k, g in groups.items()], key=repr)
    got = run_sql(data, "SELECT COUNT(id), SUM(salary) FROM people WHERE dept NOT IN (SELECT dept_id FROM dept WHERE region > 3)", batch_size)
    rest = [r for r in p if not_in(r["dept"], [x["dept_id"] for x in d if x["region"] > 3])]
    assert got == [(len(rest), sum(r["salary"] for r in rest))]


def test_sql_self_join_reads_the_table_twice(data):
    p, d = py_tables(data)
    got = run_sql(data, "SELECT a.dname, b.dname FROM dept a JOIN dept b ON a.region = b.region WHERE a.dept_id < 5", 0)
    # a null orders below every value in this engine's comparisons, so the null dept_id passes `< 5`
    exp = [(a["dname"], b["dname"]) for a in d for b in d if a["region"] == b["region"] and (a["dept_id"] is None or a["dept_id"] < 5)]
    assert len(exp) > 0 and got == sorted(exp, key=repr)


def test_sql_csv(tmp_path, data):
    p, d = py_tables(data)
    path = os.path.join(tmp_path, "people.csv")
    with open(path, "w") as f:
        f.write("id,dept,salary\n")
        for r in p[:5000]:
            f.write("%d,%s,%r\n" % (r["id"], "" if r["dept"] is None else r["dept"], r["salary"]))
    fields = [("id", A.INT64), ("dept", A.INT32), ("salary", A.FLOAT64)]
    for sql, keep in [
        ("SELECT id FROM people WHERE dept IN (SELECT dept_id FROM dept WHERE region = 4)",
         lambda r: r["dept"] is not None and r["dept"] in [x["dept_id"] for x in d if x["region"] == 4]),
        ("SELECT id FROM people WHERE dept NOT IN (SELECT dept_id FROM dept)", lambda r: False),
        ("SELECT id FROM people WHERE dept NOT IN (SELECT dept_id FROM dept WHERE region = 2)",
         lambda r: not_in(r["dept"], [x["dept_id"] for x in d if x["region"] == 2])),
        ("SELECT id FROM people p WHERE NOT EXISTS (SELECT 1 FROM dept WHERE dept_id = p.dept)",
         lambda r: not any(x["dept_id"] == r["dept"] and r["dept"] is not None for x in d)),
        # the CSV table read twice in one query
        ("SELECT id FROM people WHERE id IN (SELECT dept FROM people WHERE salary > 500 AND dept > -1)",
         lambda r: r["id"] in {x["dept"] for x in p[:5000] if x["salary"] > 500 and x["dept"] is not None}),
    ]:
        hctx = host.ExecutionContext(0)
        try:
            hctx.register_csv("people", path, fields, batch_size=700)
            hctx.register_memory("dept", list(data[1].items()), batch_size=16)
            assert rows(hctx.sql(sql).collect()) == sorted([(r["id"],) for r in p[:5000] if keep(r)], key=repr), sql
        finally:
            hctx.close()


def test_sql_key_type_refusal(data):
    with pytest.raises(host.ExecutionError) as e:
        run_sql(data, "SELECT id FROM people WHERE salary IN (SELECT CAST(region AS DOUBLE) FROM dept)", 0)
    assert e.value.code == A.ERR_NOT_IMPLEMENTED and "Float64" in e.value.msg
