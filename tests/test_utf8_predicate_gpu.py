"""Utf8 comparisons and LIKE / NOT LIKE on the GPU, exact against a Python reference over bytes with the engine's null
rule (null equals null and orders below every string; a null satisfies neither LIKE nor NOT LIKE).  Every comparison
operator against a literal on either side and against a column, every LIKE pattern class, strings of 0 to 300 bytes with
shared prefixes, non-ASCII and emoji text, all-null, all-empty, zero-row and sliced inputs; in WHERE, ANDed / ORed with
numeric comparisons, as Boolean projections, in the aggregate's fused WHERE, after the caller freed its program, through
SQL and at 1e7 rows through the host paths.  Under DFGPU_TRACE the pre-pass kernel of each pattern class is asserted."""
import ctypes as C
import os

import numpy as np
import pyarrow as pa
import pytest

from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import engine, host
from datafusion_archive_b200.expr import AggregateFunction, col, lit
from expr_ref import cmp3, like_ref
from kernel_trace import traced_set as traced
from test_avg_gpu import rows

pytestmark = pytest.mark.gpu

DATA = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "data")
OPS = {"eq": lambda c: c == 0, "not_eq": lambda c: c != 0, "__lt__": lambda c: c < 0, "__le__": lambda c: c <= 0,
       "__gt__": lambda c: c > 0, "__ge__": lambda c: c >= 0}
MIRROR = {"eq": "eq", "not_eq": "not_eq", "__lt__": "__gt__", "__le__": "__ge__", "__gt__": "__lt__", "__ge__": "__le__"}


@pytest.fixture(scope="module")
def ctx():
    c = engine.GpuContext(0)
    yield c
    c.close()


def strings(n, seed, null_frac=0.1):
    rng = np.random.default_rng(seed)
    pieces = [b"abc", b"ab", b"Elgin, ", b"Scotland", b"the UK", b"\xc3\xa9", b"\xf0\x9f\x98\x80", b"x", b"_", b"%", b"\\",
              b"abcdefghijklmnopqrstuvwxyz", b"a" * 40]
    out = []
    for _ in range(n):
        if rng.random() < null_frac:
            out.append(None)
            continue
        k = int(rng.integers(0, 6)) if rng.random() < 0.9 else int(rng.integers(10, 25))
        out.append(b"".join(pieces[int(i)] for i in rng.integers(0, len(pieces), k))[:300])
    return out


def binary(vals):
    return pa.array(vals, type=pa.binary())


def project(ctx, arrays, exprs, pred=None):
    b = ctx.upload(arrays)
    try:
        r = ctx.filter_project(b, pred, exprs)
        try:
            return r.columns()
        finally:
            r.free()
    finally:
        b.free()


LITERALS = [b"", b"abc", b"ab", b"abcdefghijklmnopq", b"Elgin, Scotland", b"\xc3\xa9", b"a" * 40 + b"abc", b"\xff"]


def test_every_comparison_against_literals_and_columns(ctx):
    a, b = strings(3000, 1), strings(3000, 2)
    arrays = [binary(a), binary(b)]
    for op, f in OPS.items():
        for L in LITERALS:
            (got1, got2), k = traced(lambda: project(ctx, arrays, [getattr(col(0), op)(lit(L)), getattr(lit(L), op)(col(0))]))
            exp1 = np.array([f(cmp3(v, L)) for v in a])
            exp2 = np.array([f(cmp3(L, v)) for v in a])
            assert (got1 == exp1).all() and (got2 == exp2).all(), (op, L)
            assert any(n.startswith("k_utf8_cmp") for n in k)
        (got,), k = traced(lambda: project(ctx, arrays, [getattr(col(0), op)(col(1))]))
        assert (got == np.array([f(cmp3(x, y)) for x, y in zip(a, b)])).all(), op
        assert ("k_utf8_cmp<eq,col>" if op in ("eq", "not_eq") else "k_utf8_cmp<%s,col>" % op.strip("_")[:2]) in k
    # the same column on both sides, and a column against a copy of itself: every row equal
    (g1, g2), _ = traced(lambda: project(ctx, [binary(a), binary(a)], [col(0).eq(col(1)), col(0) <= col(1)]))
    assert g1.all() and g2.all()


PATTERNS = [("", "k_utf8_cmp<eq,lit>"), ("abc", "k_utf8_cmp<eq,lit>"), ("%", "k_utf8_like<prefix>"), ("%%", "k_utf8_like<prefix>"),
            ("abc%", "k_utf8_like<prefix>"), ("Elgin, %", "k_utf8_like<prefix>"), ("%the UK", "k_utf8_like<suffix>"),
            ("%\xc3\xa9", "k_utf8_like<suffix>"), ("%abc%", "k_utf8_like<contains>"), ("%Scotland%", "k_utf8_like<contains>"),
            ("%abcdefghijklmnopqrstuvwxyz%", "k_utf8_like<contains>"), ("_", "k_utf8_like<general>"),
            ("a_c", "k_utf8_like<general>"), ("%_%", "k_utf8_like<general>"), ("a%b%c", "k_utf8_like<general>"),
            ("%ab%x%", "k_utf8_like<general>"), ("_%_", "k_utf8_like<general>"), ("%\\%", "k_utf8_like<contains>"), ("%\\", "k_utf8_like<suffix>"),
            ("__\xf0\x9f\x98\x80%", "k_utf8_like<general>"), ("%Elgin%UK", "k_utf8_like<general>")]


@pytest.mark.parametrize("pattern,kernel", PATTERNS, ids=[p for p, _ in PATTERNS])
def test_like_and_not_like_every_class(ctx, pattern, kernel):
    pat = pattern.encode("latin-1")
    a = strings(4000, 3)
    ids = np.arange(len(a), dtype=np.int64)
    (g1, g2), k = traced(lambda: project(ctx, [binary(a)], [col(0).like(lit(pat)), col(0).not_like(lit(pat))]))
    assert (g1 == like_ref(a, pat)).all() and (g2 == like_ref(a, pat, True)).all()
    assert kernel in k
    # WHERE, and the same predicate on a slice of a longer array (offset != 0)
    (sel,), _ = traced(lambda: project(ctx, [binary(a), ids], [col(1)], pred=col(0).like(lit(pat))))
    assert (sel == ids[like_ref(a, pat)]).all()
    arr = binary(a).slice(37, 2500)
    (g,), _ = traced(lambda: project(ctx, [arr], [col(0).not_like(lit(pat))]))
    assert (g == like_ref(a[37:37 + 2500], pat, True)).all()


def test_edge_columns(ctx):
    for vals in ([None] * 100, [b""] * 100, [], [b"x" * 300, b"", None, b"x" * 299 + b"y", b"x" * 16, b"x" * 15, b"x" * 17]):
        arr = binary(vals)
        for e, ref in [(col(0).eq(lit(b"")), [cmp3(v, b"") == 0 for v in vals]),
                       (col(0) < lit(b"x" * 300), [cmp3(v, b"x" * 300) < 0 for v in vals]),
                       (col(0).like(lit(b"%x")), list(like_ref(vals, b"%x"))),
                       (col(0).not_like(lit(b"x%y")), list(like_ref(vals, b"x%y", True))),
                       (col(0).like(lit(b"%xxxxxxxxxxxxxxxxy%")), list(like_ref(vals, b"%xxxxxxxxxxxxxxxxy%")))]:
            (g,), _ = traced(lambda: project(ctx, [arr], [e]))
            assert list(g) == ref
    # strings that end exactly at the end of the byte buffer, of every length mod 16
    for n in range(1, 40):
        vals = [b"q" * n]
        (g1, g2), _ = traced(lambda: project(ctx, [binary(vals)], [col(0).like(lit(b"%q")), col(0) >= lit(b"q" * n)]))
        assert g1[0] and g2[0]


def test_mixed_with_numeric_predicates(ctx):
    a = strings(5000, 4)
    x = np.random.default_rng(5).random(5000)
    ids = np.arange(5000, dtype=np.int64)
    like = like_ref(a, b"%abc%")
    lt = np.array([cmp3(v, b"ab") < 0 for v in a])
    (sel,), k = traced(lambda: project(ctx, [binary(a), x, ids], [col(2)], pred=col(0).like("%abc%") & (col(1) > 0.5)))
    assert (sel == ids[like & (x > 0.5)]).all()
    (sel,), _ = traced(lambda: project(ctx, [binary(a), x, ids], [col(2)], pred=(col(1) > 0.9) | (col(0) < "ab") | col(0).like("%abc%")))
    assert (sel == ids[(x > 0.9) | lt | like]).all()
    (p1, p2), _ = traced(lambda: project(ctx, [binary(a), x], [col(0).like("%abc%") & (col(1) > 0.5), col(1) * 2.0],
                                         pred=col(0).not_like("%abc%") | (col(1) < 0.25)))
    keep = like_ref(a, b"%abc%", True) | (x < 0.25)
    assert (p1 == (like & (x > 0.5))[keep]).all() and (p2 == (x * 2.0)[keep]).all()


def agg(name, arg, distinct=False):
    return AggregateFunction(name, arg, distinct=distinct)


def aggregate(ctx, arrays, keys, aggs, pred=None):
    b = ctx.upload(arrays)
    try:
        r = ctx.aggregate([b], keys, aggs, 0, pred=pred)
        try:
            return r.columns()
        finally:
            r.free()
    finally:
        b.free()


def test_aggregate_fused_where(ctx):
    n = 20000
    a = strings(n, 6)
    rng = np.random.default_rng(7)
    k = rng.integers(0, 20, n).astype(np.int64)
    v = rng.integers(-50, 50, n).astype(np.int32)
    m = like_ref(a, b"%Scotland%")
    # integer key
    (gk, gc, gs), kern = traced(lambda: aggregate(ctx, [binary(a), k, v], [col(1)], [agg("count", col(2)), agg("sum", col(2))],
                                                  pred=col(0).like("%Scotland%")))
    exp = {int(key): (int((m & (k == key)).sum()), int(v[m & (k == key)].sum())) for key in np.unique(k[m])}
    assert {int(x): (int(c), int(s)) for x, c, s in zip(gk, gc, gs)} == exp
    assert "k_utf8_like<contains>" in kern
    # no GROUP BY, with AVG and COUNT(DISTINCT)
    (c, avg, dc), _ = traced(lambda: aggregate(ctx, [binary(a), k, v], [], [agg("count", col(2)), agg("avg", col(2)),
                                                                             agg("count", col(1), distinct=True)],
                                                pred=col(0).not_like("%Scotland%") & (col(2) > lit(0, A.INT32))))
    sel = like_ref(a, b"%Scotland%", True) & (v > 0)
    assert int(c[0]) == int(sel.sum()) and float(avg[0]) == pytest.approx(v[sel].mean(), rel=1e-12)
    assert int(dc[0]) == len(np.unique(k[sel]))
    # COUNT(DISTINCT) with a key
    (gk, dc), _ = traced(lambda: aggregate(ctx, [binary(a), k, v], [col(1)], [agg("count", col(2), distinct=True)], pred=col(0) >= "abc"))
    ge = np.array([cmp3(x, b"abc") >= 0 for x in a])
    assert {int(x): int(y) for x, y in zip(gk, dc)} == {int(key): len(np.unique(v[ge & (k == key)])) for key in np.unique(k[ge])}
    # the single Utf8 key, and a wide key (Utf8 + integer)
    names = ["Elgin", "Leeds", "Perth", "York", ""]
    cities = [names[int(i)] for i in rng.integers(0, len(names), n)]
    (gk, gc), kern = traced(lambda: aggregate(ctx, [pa.array(cities), v, binary(a)], [col(0)], [agg("count", col(1))],
                                              pred=col(2).like("%Scotland%")))
    exp = {}
    for c, ok in zip(cities, m):
        if ok:
            exp[c] = exp.get(c, 0) + 1
    assert {g: int(c) for g, c in zip(gk, gc)} == exp
    assert "k_utf8_like<contains>" in kern
    (g1, g2, gc), _ = traced(lambda: aggregate(ctx, [pa.array(cities), k, v, binary(a)], [col(0), col(1)], [agg("count", col(2))],
                                               pred=col(3).like("%Scotland%")))
    exp = {}
    for c, key, ok in zip(cities, k, m):
        if ok:
            exp[(c, int(key))] = exp.get((c, int(key)), 0) + 1
    assert {(x, int(y)): int(c) for x, y, c in zip(g1, g2, gc)} == exp


def test_aggregate_predicate_outlives_the_callers_program(ctx):
    """set_predicate copies the literal: the caller's bytes are overwritten and freed before three update calls."""
    L = engine.lib()
    a = strings(10000, 8)
    v = np.arange(10000, dtype=np.int64)
    keep = []
    aggarr = A.make_aggs([agg("sum", col(1)).lower([A.UTF8, A.INT64])], keep)
    st = C.c_void_p()
    engine.check(L.dfgpu_aggregate_create(ctx.h, None, None, 0, aggarr, 1, 0, C.byref(st)))
    try:
        buf = C.create_string_buffer(b"%abc%")
        prog = (A.Insn * 3)()
        prog[0].op, prog[0].col, prog[0].dtype = A.OP_COL, 0, A.UTF8
        prog[1].op, prog[1].col, prog[1].dtype = A.OP_LIT_UTF8, 5, A.UTF8
        prog[1].lit.str = C.addressof(buf)
        prog[2].op, prog[2].dtype = A.OP_LIKE, A.UTF8
        engine.check(L.dfgpu_aggregate_set_predicate(st, prog, 3))
        C.memset(buf, ord("z"), 5)
        del buf, prog
        batches = [ctx.upload([binary(a[i:i + 3400]), v[i:i + 3400]]) for i in range(0, 10000, 3400)]
        for b in batches:
            engine.check(L.dfgpu_aggregate_update(st, b.h))
        out = C.c_void_p()
        engine.check(L.dfgpu_aggregate_finish(st, C.byref(out)))
        (s,) = engine.Result(ctx, out).columns()
        assert int(s[0]) == int(v[like_ref(a, b"%abc%")].sum())
        for b in batches:
            b.free()
    finally:
        L.dfgpu_aggregate_free(st)


def test_sql_over_csv(ctx):
    hctx = host.ExecutionContext(0)
    try:
        fields = [("city", A.UTF8), ("lat", A.FLOAT64), ("lng", A.FLOAT64)]
        import csv
        with open(os.path.join(DATA, "uk_cities.csv")) as f:
            data = [(r[0], float(r[1]), float(r[2])) for r in csv.reader(f)][1:]  # the first line is read as a header
        hctx.register_csv("c1", os.path.join(DATA, "uk_cities.csv"), fields, 1024)
        got = rows(hctx.sql("SELECT city, lat FROM c1 WHERE city LIKE '%Scotland%'"))
        assert got == [(c, la) for c, la, _ in data if "Scotland" in c]
        hctx.register_csv("c2", os.path.join(DATA, "uk_cities.csv"), fields, 1024)
        got = rows(hctx.sql("SELECT lat FROM c2 WHERE city NOT LIKE '%, UK'"))
        assert [x for (x,) in got] == [la for c, la, _ in data if not c.endswith(", UK")]
        hctx.register_csv("c3", os.path.join(DATA, "uk_cities.csv"), fields, 1024)
        got = sorted(rows(hctx.sql("SELECT city, COUNT(lat) FROM c3 WHERE city LIKE '%Scotland%' GROUP BY city")))
        exp = {}
        for c, _, _ in data:
            if "Scotland" in c:
                exp[c] = exp.get(c, 0) + 1
        assert got == sorted(exp.items())
        hctx.register_csv("c4", os.path.join(DATA, "uk_cities.csv"), fields, 1024)
        got = rows(hctx.sql("SELECT lat FROM c4 WHERE city >= 'M' AND lat > 52.0"))
        assert [x for (x,) in got] == [la for c, la, _ in data if c.encode() >= b"M" and la > 52.0]
        pf = [("id", A.INT32), ("first_name", A.UTF8)]
        with open(os.path.join(DATA, "people.csv")) as f:
            people = [(int(r[0]), r[1]) for r in list(csv.reader(f))[1:]]
        hctx.register_csv("p1", os.path.join(DATA, "people.csv"), pf, 1024)
        got = rows(hctx.sql("SELECT id FROM p1 WHERE first_name = 'Andy'"))
        assert [x for (x,) in got] == [i for i, n in people if n == "Andy"]
        hctx.register_csv("p2", os.path.join(DATA, "people.csv"), pf, 1024)
        got = rows(hctx.sql("SELECT id FROM p2 WHERE first_name LIKE '_r%'"))
        assert [x for (x,) in got] == [i for i, n in people if len(n) >= 2 and n[1] == "r"]
    finally:
        hctx.close()


def test_host_paths_at_1e7_rows(ctx):
    n = 10_000_000
    rng = np.random.default_rng(11)
    words = np.array([b"Elgin, Scotland", b"Leeds, UK", b"abc", b"", b"Perth, Scotland, the UK", b"\xc3\xa9t\xc3\xa9"], dtype=object)
    idx = rng.integers(0, len(words), n)
    arr = pa.array(words[idx].tolist(), type=pa.binary())
    x = rng.random(n)
    m = np.isin(idx, [0, 4])
    r = ctx.filter_project_host([arr, x], pred=col(0).like("%Scotland%"), proj=[col(1)])
    try:
        (got,) = r.columns()
    finally:
        r.free()
    assert (got == x[m]).all()
    r = ctx.aggregate_host([arr, x], [], [agg("count", col(1)), agg("sum", col(1))], pred=col(0).like("%Scotland%") & (col(1) > 0.5))
    try:
        c, s = r.columns()
    finally:
        r.free()
    sel = m & (x > 0.5)
    assert int(c[0]) == int(sel.sum()) and float(s[0]) == pytest.approx(x[sel].sum(), rel=1e-9)


def test_queries_without_string_predicates_keep_their_kernels(ctx):
    x = np.random.default_rng(3).random(100_000)
    k = np.random.default_rng(4).integers(0, 10, 100_000).astype(np.int64)
    _, kern = traced(lambda: project(ctx, [x], [col(0)], pred=col(0) > 0.5))
    assert not any(n.startswith("k_utf8_cmp") or n.startswith("k_utf8_like") for n in kern)
    assert any(n.startswith("k_filter_project") for n in kern)
    _, kern = traced(lambda: aggregate(ctx, [k, x], [col(0)], [agg("sum", col(1))], pred=col(1) > 0.5))
    assert not any(n.startswith("k_utf8_cmp") or n.startswith("k_utf8_like") for n in kern)


def test_launch_counts_and_profile(ctx):
    a = strings(1000, 9)
    n0 = ctx.kernel_launches()
    ctx.profile_enable(True)
    project(ctx, [binary(a)], [col(0).like("%abc%"), col(0) < "b"])
    ms, launches = ctx.profile_get()
    ctx.profile_enable(False)
    assert ctx.kernel_launches() - n0 >= 3 and launches >= 3
