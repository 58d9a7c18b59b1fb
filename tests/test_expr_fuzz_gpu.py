"""The whole expression language, fuzzed at every kernel that interprets it, against the one reference of
tests/expr_ref.py.

Random typed trees of tests/fuzz_exprs.py (QueryGen(full=True): CASE, scalar functions, every numeric CAST, Utf8
comparisons and LIKE, Utf8 functions, guarded and unguarded divisions, trees at the stack-depth limit) over gen_table's
nullable columns, with garbage under their nulls, and Utf8 columns, 100 003 rows so that the last tile is ragged.  Each
site compares the engine with expr_ref bit for bit (transcendentals, only ever a projection's root, within
test_scalar_fn_gpu.within_ulps), and expects DivideByZero exactly when the reference's pending bits say the call raises:
filter/project without and with a WHERE on the TMA, direct and NULLS kernels; the chunked host call; GROUP BY on one
narrow key, packed composite keys and a wide key, the reduce, COUNT(DISTINCT) and AVG, with and without a fused WHERE,
and the front table; join and semi-join keys; sort keys and a sort's `keep`.  Every launch is traced, and the last test
asserts that the fuzz reached every kFnDepth and kCaseDepth instantiation and the Utf8 pre-pass kernels.  A failure
names the site, the seed, the query index and the repr of every expression."""
import os

import numpy as np
import pyarrow as pa
import pytest

import expr_ref as R
import fuzz_exprs as F
import groupby_ref as G
import sort_ref
from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import engine
from datafusion_archive_b200.expr import AggregateFunction, Case, col, fn, lit
from kernel_trace import traced_set
from join_ref import inner as ref_join, same_pairs
from test_join_gpu import gpu_pairs
from test_scalar_fn_gpu import within_ulps

pytestmark = pytest.mark.gpu

N = 100_003
LAUNCHED = set()


def traced(f):
    out, k = traced_set(f)
    LAUNCHED.update(k)
    return out


@pytest.fixture(scope="module")
def ctx():
    c = engine.GpuContext(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def dctx():
    """A context whose filter/project always takes the direct kernel (DFGPU_FP_KERNEL=direct, read at creation)."""
    old = os.environ.get("DFGPU_FP_KERNEL")
    os.environ["DFGPU_FP_KERNEL"] = "direct"
    try:
        c = engine.GpuContext(0)
    finally:
        if old is None:
            del os.environ["DFGPU_FP_KERNEL"]
        else:
            os.environ["DFGPU_FP_KERNEL"] = old
    yield c
    c.close()


def table(seed, n=N, profiles=None, dtypes=F.NUMERIC, strings=True, keys=()):
    rng = np.random.default_rng(seed)
    t = F.gen_table(rng, n, profiles=profiles, dtypes=dtypes)
    if strings:
        F.add_strings(rng, t, n)
    kc = F.add_keys(rng, t, keys, n) if keys else []
    if profiles == "nobitmap":  # the key columns too: the stored values, no bitmap
        for k in kc:
            t.arrays[k], t.valid[k], t.profile[k] = t.hidden[k], None, "nobitmap"
    return rng, t, kc


def what(site, seed, q, **exprs):
    return "%s seed %d query %d: %s" % (site, seed, q, "; ".join("%s = %r" % kv for kv in exprs.items()))


def expect_raise(f, msg):
    try:
        traced(f)
    except engine.DfGpuError as e:
        assert e.code == A.ERR_ARROW and "DivideByZero" in e.msg, "%s: expected DivideByZero, got %s" % (msg, e)
        return
    pytest.fail("%s: expected DivideByZero, the call returned" % msg)


def unpack(c):
    if isinstance(c, tuple):
        return np.asarray(c[0]), np.asarray(c[1], dtype=bool)
    return np.asarray(c), np.ones(len(c), dtype=bool)


def assert_column(got, e, v, msg):
    """got: an engine column; v: the reference Value over the same rows; bit for bit, or within 3 ulp for a
    transcendental root."""
    gv, gm = unpack(got)
    assert len(gv) == len(v.values), "%s: %d rows, expected %d" % (msg, len(gv), len(v.values))
    assert np.array_equal(gm, v.valid), "%s: validity differs in rows %s" % (msg, np.flatnonzero(gm != v.valid)[:8])
    ev = np.asarray(v.values)
    if R.is_approx(e):
        try:
            with np.errstate(all="ignore"):
                within_ulps(gv[gm], ev[gm])
        except AssertionError as err:
            raise AssertionError("%s: beyond 3 ulp: %s" % (msg, err)) from None
        return
    if ev.dtype == np.bool_:
        bad = np.flatnonzero(gv[gm].astype(bool) != ev[gm])
    else:
        bad = R.cast_ref.same(gv[gm], ev[gm].astype(gv.dtype))
    assert not len(bad), "%s: values differ in valid rows %s: %s, expected %s" % (msg, bad[:8], gv[gm][bad[:8]], ev[gm][bad[:8]])


def fp(c, batch, pred, proj):
    r = c.filter_project(batch, pred, proj)
    try:
        return r.columns()
    finally:
        r.free()


def check_fp(run, T, pred, proj, msg):
    """run(): the engine's columns of `proj` under `pred`."""
    bad, keep = R.raises(T, pred, proj)
    if bad:
        expect_raise(run, msg)
        return True
    got = traced(run)
    for i, e in enumerate(proj):
        v = R.evaluate(e, T, pred is None)
        assert_column(got[i], e, R.Value(v.values[keep], v.valid[keep], v.err[keep]), "%s, column %d" % (msg, i))
    return False


def gen_fp(rng, t, with_pred, want=None):
    """A full-language filter/project query; want: 'fn' (a scalar function and no CASE), 'case', or None."""
    for _ in range(400):
        seen = set()
        pred, proj = F.gen_fp_query(rng, t, with_pred=with_pred, full=True, seen=seen)
        progs = [p for e in proj + ([pred] if pred is not None else []) for p in e.program(t.dtype)]
        has_case = any(i.op == A.OP_CASE for i in progs)
        has_fn = any(i.op == A.OP_FN for i in progs)
        if want is None or (want == "case" and has_case) or (want == "fn" and has_fn and not has_case):
            return pred, proj
    raise AssertionError("no query of kind %s" % want)


def f64_only(exprs, schema):
    return all(i.op != A.OP_CAST and i.dtype in (A.FLOAT64, A.BOOL, 0) and (i.op != A.OP_COL or schema[i.col] in (A.FLOAT64, A.BOOL))
               for e in exprs for i in e.program(schema))


# ---- filter / project ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [11, 12])
def test_filter_project(ctx, dctx, seed):
    """Without a WHERE (bitmaps read) and with one, on the default context (TMA kernel when the inputs have no nulls,
    NULLS kernel when they do) and on the direct kernel; both kinds of instantiation."""
    ran = raised = 0
    for profiles in (None, "nobitmap"):
        rng, t, _ = table(seed, profiles=profiles)
        T = R.Table(t.arrays)
        b, bd = ctx.upload(t.arrays), dctx.upload(t.arrays)
        try:
            for q in range(16):
                pred, proj = gen_fp(rng, t, q % 2 == 1, want=("fn", "case", None, "case")[q % 4])
                for c, bb, name in ((ctx, b, "fp"), (dctx, bd, "fp direct")):
                    raised += check_fp(lambda: fp(c, bb, pred, proj), T, pred, proj, what(name, seed, q, pred=pred, proj=proj))
                    ran += 1
        finally:
            b.free()
            bd.free()
    assert raised <= ran // 3, (raised, ran)


def test_filter_project_float64_only(ctx):
    """Program sets over Float64 and Boolean operands alone take the F64ONLY TMA interpreter."""
    seed = 13
    rng, t, _ = table(seed, profiles="nobitmap", dtypes=[A.FLOAT64], strings=False)
    T = R.Table(t.arrays)
    b = ctx.upload(t.arrays)
    try:
        made = {"fn": 0, "case": 0}
        for q in range(2000):
            kind = "fn" if made["fn"] <= made["case"] else "case"
            pred, proj = gen_fp(rng, t, False, want=kind)
            if not f64_only(proj, t.dtype):
                continue
            check_fp(lambda: fp(ctx, b, pred, proj), T, pred, proj, what("fp f64", seed, q, proj=proj))
            made[kind] += 1
            if min(made.values()) >= 3:
                break
        assert min(made.values()) >= 3, made
    finally:
        b.free()


def test_chunked_host_call(ctx):
    """dfgpu_filter_project_host in small chunks over inputs without bitmaps: the chunk pipeline, and the resident
    operator for a projection with a CASE without ELSE."""
    seed = 14
    rng, t, _ = table(seed, profiles="nobitmap", strings=False)
    T = R.Table(t.arrays)
    no_else = 0
    for q in range(8):
        pred, proj = gen_fp(rng, t, q % 2 == 0, want="case")
        if q < 2:
            g = F.QueryGen(rng, t, range(len(t.dtype)), full=True, max_depth=3)
            d = t.dtype[t.values[A.FLOAT64]]
            proj = [Case([(g.boolean(1), g.numeric(d, 2))])] + proj[1:]
        no_else += any(i.op == A.OP_CASE and i.col % 2 == 0 for e in proj for i in e.program(t.dtype))

        def run():
            r = ctx.filter_project_host(t.arrays, pred, proj, chunk_rows=30_000)
            try:
                return r.columns()
            finally:
                r.free()
        check_fp(run, T, pred, proj, what("fp host", seed, q, pred=pred, proj=proj))
    assert no_else >= 2


# ---- aggregates ------------------------------------------------------------------------------------------------------
def check_agg(c, batches, T, pred, keys, aggs, msg):
    """The engine's GROUP BY / reduce against groupby_ref fed with the reference's keys and arguments.  Returns whether
    the call raised."""
    rb = pred is None
    bad, keep = R.raises(T, pred, keys + [a.arg for a in aggs])
    run = lambda: c.aggregate(batches, keys, aggs, 0, pred=pred).columns()  # noqa: E731
    if bad:
        expect_raise(run, msg)
        return True
    got = traced(run)
    kv = [R.evaluate(k, T, rb).values for k in keys]
    args = [(v.values, v.valid) for v in (R.evaluate(a.arg, T, rb) for a in aggs)]
    try:
        G.assert_matches(got, G.aggregate(kv, [(G.func_of(a), x) for a, x in zip(aggs, args)], where=keep))
    except AssertionError as err:
        raise AssertionError("%s: %s" % (msg, err)) from None
    return False


AGG_SHAPES = [  # (key dtypes, profiles, Utf8 columns): one narrow key, packed composite keys, a wide (> 64-bit) key,
    # no GROUP BY; with nullable inputs, and without bitmaps (where only a CASE without ELSE selects the NULLS kernels)
    ([A.INT32], None, True), ([A.INT8, A.UINT16, A.INT32], None, True), ([A.INT64, A.UINT64], None, True), ([], None, True),
    ([A.INT32], "nobitmap", False), ([A.INT64, A.INT64], "nobitmap", False), ([], "nobitmap", False),
]


@pytest.mark.parametrize("shape", range(len(AGG_SHAPES)))
def test_aggregates(ctx, shape):
    key_dtypes, profiles, strings = AGG_SHAPES[shape]
    wide = sum(np.dtype(A.NP_OF[d]).itemsize for d in key_dtypes) > 8  # COUNT(DISTINCT) takes keys of 64 bits at most
    seed = 20 + shape
    rng, t, kc = table(seed, profiles=profiles, keys=key_dtypes, strings=strings)
    T = R.Table(t.arrays)
    b = ctx.upload(t.arrays)
    ran = raised = 0
    try:
        for q in range(8):
            with_pred = q % 2 == 1
            while True:
                pred, keys, aggs = F.gen_agg_query(rng, t, kc, with_pred, False, distinct_avg=True, full=True)
                progs = [i for e in keys + [a.arg for a in aggs] + ([pred] if pred is not None else []) for i in e.program(t.dtype)]
                has_case = any(i.op == A.OP_CASE for i in progs)
                if wide and any(a.distinct for a in aggs):
                    continue
                if q % 4 == 1 and profiles == "nobitmap" and any(i.op == A.OP_CASE and i.col % 2 == 0 for i in progs):
                    continue  # every CASE with an ELSE: the kernels without NULLS
                if (q % 4 < 2) == has_case and (has_case or any(i.op == A.OP_FN for i in progs)):
                    break
            raised += check_agg(ctx, [b], T, pred, keys, aggs, what("aggregate", seed, q, pred=pred, keys=keys, args=[(a.name, a.distinct, a.arg) for a in aggs]))
            ran += 1
    finally:
        b.free()
    assert raised <= ran // 2, (raised, ran)


@pytest.mark.parametrize("kind", ["fn", "case"])
def test_aggregate_front_table(ctx, kind):
    """A first batch of 1.2 Mi rows over a few groups, then a ragged one: the second batch's scan takes the
    shared-memory front table."""
    seed = 30 + (kind == "case")
    m, n = 1_200_000, 1_300_003
    rng, t, kc = table(seed, n=n, profiles="nobitmap", strings=False, keys=[A.INT32])
    T = R.Table(t.arrays)
    g = F.QueryGen(rng, t, [t.values[A.FLOAT64], t.safe[A.FLOAT64]] + t.bools, max_depth=2, full=True)
    x, i = col(t.values[A.FLOAT64]), col(t.values[A.INT32])
    if kind == "fn":
        args = [fn("floor", x * lit(4.0)), fn("abs", i.cast(A.FLOAT64))]
    else:
        args = [Case([(g.boolean(1), i)], i + lit(1, A.INT32)), Case([(x > lit(0.0), fn("round", x))], x)]
    aggs = [AggregateFunction(f, a) for a in args for f in ("min", "max", "count")] + [AggregateFunction("sum", args[1])]
    batches = [ctx.upload([h[lo:hi] for h in t.hidden]) for lo, hi in ((0, m), (m, n))]
    try:
        check_agg(ctx, batches, T, None, [col(kc[0])], aggs, what("front table", seed, 0, args=args))
    finally:
        for b in batches:
            b.free()


# ---- join, semi-join, sort -------------------------------------------------------------------------------------------
def subset_gen(rng, t, keep, max_depth, strings=True):
    """A full-language QueryGen over 7 random numeric and Boolean columns, the columns `keep` and the Utf8 columns."""
    others = [i for i in range(len(t.dtype)) if t.dtype[i] != A.UTF8 and i not in keep]
    cols = set(rng.choice(others, 7, replace=False).tolist()) | set(keep) | (set(t.utf8) if strings else set())
    return F.QueryGen(rng, t, cols, max_depth=max_depth, full=True)


def key_array(v, dtype):
    return pa.array(np.asarray(v.values, dtype=A.NP_OF[dtype]), mask=~v.valid)


def test_join_and_semi_join_keys(ctx):
    seed = 40
    rng, t, kc = table(seed, profiles=None, keys=[A.INT64, A.INT32])
    T = R.Table(t.arrays)
    bt = F.gen_table(np.random.default_rng(41), 5_000)
    bk = F.add_keys(np.random.default_rng(42), bt, [A.INT64, A.INT32], 5_000)
    BT = R.Table(bt.arrays)
    for q in range(6):
        d = t.dtype[kc[q % 2]]
        while True:
            g = subset_gen(rng, t, [kc[q % 2]], 4, strings=q % 2 == 0)
            pkey = Case([(g.boolean(2), col(kc[q % 2]))], g.numeric(d, 2)) if q < 4 else g.numeric(d, 3)
            if F.fits([pkey], t.dtype):
                break
        bkey = col(bk[q % 2]) if q % 3 else col(bk[q % 2]) + lit(1, d)
        msg = what("join", seed, q, probe_key=pkey, build_key=bkey)
        pv, bv = R.evaluate(pkey, T), R.evaluate(bkey, BT)
        if pv.err.any():
            expect_raise(lambda: gpu_pairs(ctx, t.arrays, [pkey], bt.arrays, [bkey]), msg)
            continue
        got = traced(lambda: gpu_pairs(ctx, t.arrays, [pkey], bt.arrays, [bkey]))
        try:
            same_pairs(got, ref_join([key_array(pv, d)], [key_array(bv, d)]))
        except AssertionError:
            raise AssertionError("%s: the matching pairs differ" % msg) from None
        probe = ctx.upload(t.arrays + [np.arange(N, dtype=np.int64)])
        build = ctx.upload(bt.arrays)
        try:
            j = ctx.join_build(build, [bkey], keep_cols=[0])
            try:
                (rows,) = traced(lambda: j.semi(probe, [pkey], probe_cols=[len(t.arrays)]).columns())
            finally:
                j.free()
        finally:
            probe.free()
            build.free()
        bset = set(np.asarray(bv.values)[bv.valid].tolist())
        exp = np.flatnonzero(pv.valid & np.isin(pv.values, list(bset)))
        assert np.array_equal(rows, exp), "%s: semi-join rows differ (%d, expected %d)" % (msg, len(rows), len(exp))


def test_sort_keys_and_keep(ctx):
    seed = 50
    rng, t, _ = table(seed, profiles=None)
    T = R.Table(t.arrays)
    arrays = t.arrays + [np.arange(N, dtype=np.int64)]
    b = ctx.upload(arrays)
    try:
        for q in range(6):
            while True:
                g = subset_gen(rng, t, [], 3)
                keys = [g.utf8(2) if k == 0 and q % 2 == 0 else g.numeric(int(rng.choice(F.NUMERIC)), 2) for k in range(1 + q % 3)]
                keep = g.boolean(2) if q % 3 != 2 else None
                if F.fits(keys + ([keep] if keep is not None else []), t.dtype):
                    break
            desc = [bool(x) for x in rng.integers(0, 2, len(keys))]
            msg = what("sort", seed, q, keys=keys, desc=desc, keep=keep)
            vals = [R.evaluate(k, T) for k in keys]
            kv = R.evaluate(keep, T) if keep is not None else None
            if any(v.err.any() for v in vals) or (kv is not None and kv.err.any()):
                expect_raise(lambda: ctx.sort(b, keys, desc, keep).free(), msg)
                continue

            def run():
                r = ctx.sort(b, keys, desc, keep)
                try:
                    out = np.zeros(max(1, r.nrows), np.int64)
                    r.copy_into(len(arrays) - 1, out)
                    return out[:r.nrows]
                finally:
                    r.free()
            got = traced(run)
            spec = [(k.get_type(t.dtype), v.values, v.valid, dsc) for k, v, dsc in zip(keys, vals, desc)]
            exp = sort_ref.order(N, spec, None if kv is None else kv.values.astype(bool) & kv.valid)
            assert np.array_equal(got, exp), "%s: order differs (%d rows, expected %d)" % (msg, len(got), len(exp))
    finally:
        b.free()


# ---- coverage --------------------------------------------------------------------------------------------------------
def test_zz_every_interpreter_instantiation_was_reached():
    """Runs last in this file: the kernels the tests above launched include every kFnDepth and kCaseDepth
    instantiation of the expression-interpreting families, and the Utf8 pre-pass kernels."""
    want = set()
    for d in ("kFnDepth", "kCaseDepth"):
        want |= {"k_filter_project<%s,%d>" % (d, v) for v in (0, 1)}
        want |= {"k_filter_project_tma<%s,4,%d,0,0>" % (d, v) for v in (0, 1)}
        want |= {"k_hash_agg<%s,0,0>" % d, "k_hash_agg<%s,1,0>" % d, "k_hash_agg<%s,0,1>" % d}
        want |= {"k_hash_agg_wide<%s,%d>" % (d, v) for v in (0, 1)}
        want |= {"k_reduce<%s,%d>" % (d, v) for v in (0, 1)}
        want |= {"k_distinct_insert<%s,%d>" % (d, v) for v in (0, 1)}
    assert len(want) == 26
    missing = want - LAUNCHED
    assert not missing, sorted(missing)
    for prefix in ("k_utf8_cmp", "k_utf8_like", "k_utf8_view_len", "k_utf8_view_copy", "k_pack_bits"):
        assert any(k.startswith(prefix) for k in LAUNCHED), (prefix, sorted(LAUNCHED))
