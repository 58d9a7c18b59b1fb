"""Every GPU hash table under keys crafted to collide (tests/hash_ref.py): long probe chains, clusters that wrap from slot
cap - 1 to slot 0, front-table spills, tag aliases and the probe limit.

Random keys at a load of at most 1/2 make probe chains a few slots long that almost never cross the end of a table, so
the code that only runs on a long chain is reached by no other test.  Here each cluster is thousands of keys whose hashes
share their top 40 bits: all ones homes them at cap - 1 at every capacity, so the cluster wraps to slot 0, where a
second cluster (top bits zero) is homed and the wrapped one runs into it.  Every table also holds the key that equals the
empty marker and random background keys.  Results are compared exactly with groupby_ref and join_ref, as multisets where
the row order is unspecified.

The probe-limit cases double as the proof that the crafting reaches the device tables: AG_MAX_PROBE keys on one home
aggregate with no growth, and one more key makes the operator refuse the batch after at most one rebuild, which happens
only if the keys really share a home on the device."""
import numpy as np
import pyarrow as pa
import pytest

import groupby_ref as R
import hash_ref as H
import join_ref as J
from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import engine, host
from datafusion_archive_b200.expr import AggregateFunction, col, lit
from kernel_trace import traced
from test_join_gpu import gpu_pairs
from test_join_utf8_gpu import gpu_pairs as utf8_gpu_pairs
from test_semi_join_gpu import gpu_pass

pytestmark = pytest.mark.gpu

I64, U64 = np.int64, np.uint64
SENTINEL = np.uint64(H.EMPTY_KEY)
KINDS = {"semi": A.JOIN_SEMI, "anti": A.JOIN_ANTI, "anti_null_aware": A.JOIN_ANTI_NULL_AWARE}


@pytest.fixture(scope="module")
def ctx():
    c = engine.GpuContext(0)
    yield c
    c.close()


def aggregate(ctx, batches, keys, aggs, expected=0, pred=None):
    """The result columns of a GROUP BY over the given batches (lists of columns)."""
    bs = [ctx.upload(b) for b in batches]
    try:
        r = ctx.aggregate(bs, keys, aggs, expected, pred=pred)
        try:
            return r.columns()
        finally:
            r.free()
    finally:
        for b in bs:
            b.free()


def run_agg(ctx, batches, keys, aggs, expected=0, pred=None):
    """(result columns, kernels launched, in order)."""
    return traced(lambda: aggregate(ctx, batches, keys, aggs, expected, pred))


def run_agg_error(ctx, batches, keys, aggs):
    """The DfGpuError an aggregate raises, and the kernels it launched before."""
    def go():
        try:
            aggregate(ctx, batches, keys, aggs)
        except engine.DfGpuError as e:
            return e
        return None
    err, names = traced(go)
    assert err is not None, "the aggregate did not fail"
    return err, names


def launched(names, *want):
    canon = {n.replace(" ", "") for n in names}
    for w in want:
        assert w.replace(" ", "") in canon, (w, sorted(canon))


def crafted_pool(rng, wrapped=3000, at_zero=700, background=2000):
    """Key words: a cluster homed at cap - 1, a cluster homed at slot 0, random background keys and the empty-marker key."""
    k = np.concatenate([H.cluster_keys(rng, wrapped, "ones"), H.cluster_keys(rng, at_zero, "zeros"),
                        rng.integers(0, 2 ** 64, background, dtype=U64, endpoint=False), [SENTINEL]])
    return np.unique(k)


def draw(rng, pool, n):
    """n rows drawing every pool entry at least once."""
    k = pool[rng.integers(0, len(pool), n)]
    k[rng.choice(n, len(pool), replace=False)] = pool
    return k


def int_values(rng, n):
    return rng.integers(-10 ** 6, 10 ** 6, n).astype(I64)


def f64_values(rng, n):
    return rng.integers(-1000, 1000, n).astype(np.float64) * 0.25  # exact sums in any order


# ---- GROUP BY on one packed key word -----------------------------------------------------------------------------------
@pytest.mark.parametrize("kdt", [I64, U64], ids=["i64", "u64"])
def test_wrapped_cluster_through_every_scan(ctx, kdt):
    rng = np.random.default_rng(1 if kdt == I64 else 2)
    n = 200_001
    k = draw(rng, crafted_pool(rng), n).view(kdt)
    vi, vf, w = int_values(rng, n), f64_values(rng, n), rng.integers(-5, 5, n).astype(I64)
    # lean: SUM + COUNT of an Int64 column
    got, names = run_agg(ctx, [[k, vi]], [col(0)], [AggregateFunction("sum", col(1)), AggregateFunction("count", col(1))])
    launched(names, "k_hash_agg_lean<12, 3>")
    R.assert_matches(got, R.aggregate([k], [(R.SUM, vi), (R.COUNT, vi)]), "lean")
    # plain: MIN / MAX / SUM / COUNT / AVG
    funcs = [R.MIN, R.MAX, R.SUM, R.COUNT, R.AVG]
    got, names = run_agg(ctx, [[k, vf]], [col(0)], [AggregateFunction(f, col(1)) for f in funcs])
    launched(names, "k_hash_agg_plain<2, false>")
    R.assert_matches(got, R.aggregate([k], [(f, vf) for f in funcs]), "plain")
    # the interpreter: an expression argument
    got, names = run_agg(ctx, [[k, vf]], [col(0)], [AggregateFunction(f, col(1) * lit(1.0)) for f in funcs[:4]])
    launched(names, "k_hash_agg<1, false, false>")
    R.assert_matches(got, R.aggregate([k], [(f, vf) for f in funcs[:4]]), "interpreter")
    # NULLS: nullable arguments
    valid = rng.random(n) > 0.3
    got, names = run_agg(ctx, [[k, R.arrow_nullable(vi, valid)]], [col(0)], [AggregateFunction(f, col(1)) for f in funcs])
    launched(names, "k_hash_agg<8, false, true>")
    R.assert_matches(got, R.aggregate([k], [(f, (vi, valid)) for f in funcs]), "nulls")
    # a fused WHERE
    m = w >= -2
    got, names = run_agg(ctx, [[k, vi, w]], [col(0)], [AggregateFunction(f, col(1)) for f in funcs[:4]], pred=col(2) >= lit(-2))
    assert any(x.startswith("k_hash_agg_plain") for x in names), names
    R.assert_matches(got, R.aggregate([k], [(f, vi) for f in funcs[:4]], where=m), "where")


def test_packed_int32_pair_cluster(ctx):
    """(Int32, Int32) keys crafted as one packed word and split back: the packed word clusters, not the parts."""
    rng = np.random.default_rng(3)
    n = 200_001
    a, b = H.split_i32_pair(draw(rng, crafted_pool(rng), n))
    assert np.any((a == -1) & (b == -1))  # both parts all ones: the packed key is the empty marker
    v = int_values(rng, n)
    funcs = [R.MIN, R.MAX, R.SUM, R.COUNT]
    got, names = run_agg(ctx, [[a, b, v]], [col(0), col(1)], [AggregateFunction(f, col(2)) for f in funcs])
    launched(names, "k_hash_agg_plain<4, false>")
    R.assert_matches(got, R.aggregate([a, b], [(f, v) for f in funcs]), "packed pair")


def test_growth_replays_the_wrapped_cluster(ctx):
    """A hint of 1000 groups and 2.5 M more keys: the table refuses keys past its fill limit, k_compact / k_merge re-place
    the wrapped cluster in the grown table, and the refused rows are replayed into it."""
    rng = np.random.default_rng(4)
    k = np.unique(np.concatenate([crafted_pool(rng), rng.integers(0, 2 ** 64, 2_500_000, dtype=U64, endpoint=False)]))
    k = draw(rng, k, len(k) + 300_000).view(I64)
    v = int_values(rng, len(k))
    got, names = run_agg(ctx, [[k, v]], [col(0)], [AggregateFunction("sum", col(1)), AggregateFunction("count", col(1))],
                         expected=1000)
    launched(names, "k_merge", "k_hash_agg<1, false, false>")
    R.assert_matches(got, R.aggregate([k], [(R.SUM, v), (R.COUNT, v)]), "growth")


def test_line_layout_from_the_prefix_estimate(ctx):
    """A first batch of 5 M distinct keys: the prefix estimate rebuilds the table in line layout before the rest runs."""
    rng = np.random.default_rng(5)
    k = np.unique(np.concatenate([crafted_pool(rng), rng.integers(0, 2 ** 64, 5_000_000, dtype=U64, endpoint=False)]))
    k = k[rng.permutation(len(k))].view(I64)
    v = int_values(rng, len(k))
    got, names = run_agg(ctx, [[k, v]], [col(0)], [AggregateFunction("sum", col(1)), AggregateFunction("count", col(1))])
    launched(names, "k_hash_agg_lean<12, 3>", "k_merge", "k_hash_agg_plain<2, false>")
    assert names.index("k_hash_agg_plain<2, false>") > names.index("k_merge"), names
    R.assert_matches(got, R.aggregate([k], [(R.SUM, v), (R.COUNT, v)]), "line")


@pytest.mark.parametrize("groups", ["per_warp", "per_cta"])
def test_front_table_spills(ctx, groups):
    """A first batch of 1.1 M rows with few groups, then batches through the shared-memory front table whose groups put
    far more than AG_FRONT_PROBES keys on one front slot (the last one, so the front probe wraps to slot 0 too): the
    rows that find no front slot go to the global table."""
    rng = np.random.default_rng(6 if groups == "per_warp" else 7)
    if groups == "per_warp":  # <= 64 groups: one 256-slot table per warp
        pool = np.unique(np.concatenate([H.cluster_keys(rng, 40, "ones"), H.cluster_keys(rng, 12, "zeros"),
                                         rng.integers(0, 2 ** 64, 10, dtype=U64, endpoint=False), [SENTINEL]]))
        assert len(pool) <= 64
    else:  # <= 1024 groups: one 2048-slot table per CTA
        pool = crafted_pool(rng, wrapped=600, at_zero=150, background=250)
        assert len(pool) <= 1024
    fs = H.AG_FRONT_SLOTS // (H.AG_THREADS // 32) if groups == "per_warp" else H.AG_FRONT_SLOTS
    slots = H.front_slot(H.mix64(pool[pool != SENTINEL]), fs)
    assert np.bincount(slots.astype(np.int64)).max() > 4 * H.AG_FRONT_PROBES
    batches = []
    for n in (1_100_000, 400_001, 250_000):
        k = draw(rng, pool, n).view(I64)
        batches.append([k, f64_values(rng, n)])
    funcs = [R.MIN, R.MAX, R.COUNT, R.SUM]
    got, names = run_agg(ctx, batches, [col(0)], [AggregateFunction(f, col(1)) for f in funcs])
    launched(names, "k_hash_agg_plain<2, true>")
    k, v = (np.concatenate([b[i] for b in batches]) for i in range(2))
    R.assert_matches(got, R.aggregate([k], [(f, v) for f in funcs]), groups)


# ---- wide keys ---------------------------------------------------------------------------------------------------------
def wide_int_pool(rng):
    """(first, last) Int64 parts of distinct wide keys: 300 with one exact hash T, 300 with T ^ 1 (same tag), 100 each with
    hash EMPTY_KEY and EMPTY_KEY - 3 (same tag), 1500 more clustered at cap - 1, 400 at slot 0, random keys and (-1, -1)."""
    T = np.uint64(0xffffffffff7a5a13)
    hashes = [np.full(300, T), np.full(300, T ^ np.uint64(1)), np.full(100, SENTINEL), np.full(100, np.uint64(H.EMPTY_KEY - 3)),
              H.cluster_hashes(rng, 1500, "ones", exclude=[T, T ^ np.uint64(1), SENTINEL, np.uint64(H.EMPTY_KEY - 3)]),
              H.cluster_hashes(rng, 400, "zeros")]
    h = np.concatenate(hashes)
    first = rng.permutation(1 << 20)[:len(h)].astype(I64) - (1 << 19)
    last = H.wide_last_part([first], h).view(I64)
    assert np.array_equal(H.wide_hash([first, last]), h)
    rand = rng.integers(-2 ** 63, 2 ** 63 - 1, (2, 3000), dtype=I64)
    a = np.concatenate([first, rand[0], [-1]])
    b = np.concatenate([last, rand[1], [-1]])
    _, idx = np.unique(np.stack([a, b]), axis=1, return_index=True)
    return a[np.sort(idx)], b[np.sort(idx)]


def test_wide_int64_keys_with_one_hash(ctx):
    """Many distinct (Int64, Int64) keys with one exact hash and with aliased tags: every equal tag must be confirmed by
    comparing the parts.  Each key repeats over ~50 rows, so rows meet slots still being published (busy / deferred)."""
    rng = np.random.default_rng(8)
    a, b = wide_int_pool(rng)
    n = 300_001
    i = draw(rng, np.arange(len(a)), n)
    ka, kb, v = a[i], b[i], int_values(rng, n)
    funcs = [R.MIN, R.MAX, R.SUM, R.COUNT]
    got, names = run_agg(ctx, [[ka, kb, v]], [col(0), col(1)], [AggregateFunction(f, col(2)) for f in funcs])
    launched(names, "k_hash_agg_wide<8, false>")
    R.assert_matches(got, R.aggregate([ka, kb], [(f, v) for f in funcs]), "wide")


def test_wide_int64_growth_moves_the_clusters(ctx):
    """2.2 M more random wide keys: the table grows through k_wide_move with the crafted clusters in it, and a second
    batch finds every moved key again at its home in the grown table."""
    rng = np.random.default_rng(9)
    a, b = wide_int_pool(rng)
    ra = rng.integers(-2 ** 63, 2 ** 63 - 1, 2_200_000, dtype=I64)
    rb = rng.integers(-3, 3, len(ra)).astype(I64)
    again = rng.integers(0, len(ra), 200_000)
    ka = np.concatenate([a, ra, a, ra[again]])
    kb = np.concatenate([b, rb, b, rb[again]])
    v = int_values(rng, len(ka))
    cut = len(a) + len(ra)
    batches = [[ka[:cut], kb[:cut], v[:cut]], [ka[cut:], kb[cut:], v[cut:]]]
    got, names = run_agg(ctx, batches, [col(0), col(1)], [AggregateFunction("count", col(2)), AggregateFunction("sum", col(2))])
    launched(names, "k_wide_move")
    R.assert_matches(got, R.aggregate([ka, kb], [(R.COUNT, v), (R.SUM, v)]), "wide growth")


def utf8_codes(col_, strings):
    """Row codes of a Utf8 result column (a list, an arrow array or (values, valid)) in the order of `strings`."""
    vals = col_[0] if isinstance(col_, tuple) else col_
    vals = vals.to_pylist() if isinstance(vals, (pa.Array, pa.ChunkedArray)) else list(vals)
    at = {s: i for i, s in enumerate(strings)}
    return np.array([at[s.decode() if isinstance(s, bytes) else s] for s in vals], dtype=I64)


def test_wide_utf8_int64_keys_with_one_hash(ctx):
    """(Utf8, Int64) keys: distinct strings, each with the Int64 part that gives the key one exact hash, aliased tags and a
    cluster at cap - 1.  Equal tags are confirmed byte by byte against the strings of earlier batches."""
    rng = np.random.default_rng(10)
    strings = ["s%d" % i for i in range(400)] + ["", "x" * 40, "é"] + ["c%d" % i for i in range(600)]
    T = np.uint64(0xfffffffffff00f0e)
    h = np.concatenate([np.full(200, T), np.full(200, T ^ np.uint64(1)), [SENTINEL, np.uint64(H.EMPTY_KEY - 3), T],
                        H.cluster_hashes(rng, 600, "ones", exclude=[T, T ^ np.uint64(1), SENTINEL])])
    last = H.wide_last_part([H.utf8_hashes(strings)], h).view(I64)
    assert np.array_equal(H.wide_hash([H.utf8_hashes(strings), last.view(U64)]), h)
    batches, codes, ints = [], [], []
    for n in (100_000, 60_001):
        i = draw(rng, np.arange(len(strings)), n)
        batches.append([pa.array([strings[j] for j in i]), last[i], int_values(rng, n)])
        codes.append(i)
        ints.append(last[i])
    funcs = [R.MIN, R.MAX, R.SUM, R.COUNT]
    got, names = run_agg(ctx, batches, [col(0), col(1)], [AggregateFunction(f, col(2)) for f in funcs])
    launched(names, "k_hash_agg_wide<8, false>")
    v = np.concatenate([b[2] for b in batches])
    got = [utf8_codes(got[0], strings)] + list(got[1:])
    R.assert_matches(got, R.aggregate([np.concatenate(codes), np.concatenate(ints)], [(f, v) for f in funcs]), "utf8 wide")


# ---- COUNT(DISTINCT) pair sets ----------------------------------------------------------------------------------------
def clustered_pairs(rng, grouped):
    """(group keys, values) whose pair hashes cluster at the end of the 1 Mi-slot set and at its start, with pairs that
    have an EMPTY_KEY half (group key -1, or value -1) and the pair (-1, -1); without GROUP BY the key is 0."""
    ks, vs = [], []
    groups = [np.uint64(7), SENTINEL, np.uint64(123456789)] if grouped else [np.uint64(0)]
    for g in groups:
        for top, m in (("ones", 1500), ("zeros", 300)):
            vs.append(H.distinct_values_for(g, H.cluster_hashes(rng, m, top)))
            ks.append(np.full(m, g))
    if grouped:  # value -1 under many group keys, with their pairs at the end of the set
        kk = H.distinct_keys_for(SENTINEL, H.cluster_hashes(rng, 500, "ones"))
        ks.append(kk)
        vs.append(np.full(len(kk), SENTINEL))
        ks.append(np.array([SENTINEL]))
        vs.append(np.array([SENTINEL]))
    vs.append(np.array([SENTINEL]))  # value -1 with the first group key
    ks.append(np.array([groups[0]]))
    return np.concatenate(ks).view(I64), np.concatenate(vs).view(I64)


@pytest.mark.parametrize("grouped", [False, True], ids=["no_group_by", "group_by"])
def test_count_distinct_clustered_pairs(ctx, grouped):
    """Clustered pairs with random background pairs, in several batches; the background is big enough to grow the set
    by replay (k_set_move) with the clusters in it."""
    rng = np.random.default_rng(11 + grouped)
    ck, cv = clustered_pairs(rng, grouped)
    nb = 1_400_000
    bk = rng.integers(0, 50, nb).astype(I64) if grouped else np.zeros(nb, I64)
    bv = rng.permutation(nb).astype(I64) * 7919
    k, v = np.concatenate([ck, bk, ck]), np.concatenate([cv, bv, cv])
    p = rng.permutation(len(k))
    k, v = k[p], v[p]
    cut = np.linspace(0, len(k), 6).astype(int)
    batches = [[k[a:b], v[a:b]] for a, b in zip(cut[:-1], cut[1:])]
    aggs = [AggregateFunction("count", col(1), distinct=True), AggregateFunction("count", col(1))]
    got, names = run_agg(ctx, batches, [col(0)] if grouped else [], aggs)
    launched(names, "k_set_move")
    R.assert_matches(got, R.aggregate([k] if grouped else [], [(R.COUNT_DISTINCT, v), (R.COUNT, v)]), "distinct")


# ---- joins -------------------------------------------------------------------------------------------------------------
def join_int_keys(rng):
    """Build keys clustered at cap - 1 (which does not depend on cap = max(1024, 2n)) with duplicates, a cluster at slot 0,
    random keys and -1; probe keys: hits, misses homed inside the cluster (they walk all of it) and nulls."""
    wrapped = H.cluster_keys(rng, 3000, "ones").view(I64)
    build_keys = np.concatenate([wrapped[:2000], H.cluster_keys(rng, 500, "zeros").view(I64),
                                 rng.integers(-2 ** 62, 2 ** 62, 1000), [-1]])
    bk = np.concatenate([build_keys, build_keys[rng.integers(0, len(build_keys), 1500)]])  # duplicates
    miss = wrapped[2000:]
    pool = np.concatenate([build_keys, miss])
    pk = pool[rng.integers(0, len(pool), 40_000)]
    pk[:len(pool)] = pool
    return pk, bk


def test_join_clustered_build_inner(ctx):
    rng = np.random.default_rng(13)
    pk, bk = join_int_keys(rng)
    pcol = pa.array(pk, mask=rng.random(len(pk)) < 0.05)
    J.same_pairs(gpu_pairs(ctx, [pcol], [col(0)], [bk], [col(0)]), J.inner([pcol], [bk]))
    J.same_pairs(gpu_pairs(ctx, [bk], [col(0)], [pk], [col(0)]), J.inner([bk], [pk]))  # the sides swapped


@pytest.mark.parametrize("kind", list(KINDS.values()), ids=list(KINDS))
def test_join_clustered_build_semi_anti(ctx, kind):
    rng = np.random.default_rng(14)
    pk, bk = join_int_keys(rng)
    pcol = pa.array(pk, mask=rng.random(len(pk)) < 0.05)
    assert np.array_equal(gpu_pass(ctx, kind, [pcol], [col(0)], [bk], [col(0)]), J.passing(kind, [pcol], [bk]))


def join_utf8_keys(rng):
    """(Utf8, Int64) keys whose 64-bit tags are equal, the tags EMPTY_KEY and EMPTY_KEY - 1 (which alias), and a cluster
    at cap - 1.  Probe-only keys share those tags, so they must be told apart by their bytes and integer word."""
    T = np.uint64(0xffffffffffa0b0c1)
    strings = ["t%d" % i for i in range(300)] + ["", "é", "y" * 33] + ["e0", "e1"] + ["c%d" % i for i in range(500)]
    tags = np.concatenate([np.full(303, T), [SENTINEL, np.uint64(H.EMPTY_KEY - 1)],
                           H.cluster_hashes(rng, 500, "ones", exclude=[T, SENTINEL, np.uint64(H.EMPTY_KEY - 1)])])
    word = H.join_word_for_tag(strings, tags).view(I64)
    assert np.array_equal(H.join_utf8_tag(word, [H.utf8_hashes(strings)]),
                          np.where(tags == SENTINEL, np.uint64(H.EMPTY_KEY - 1), tags))
    probe_only = np.zeros(len(strings), bool)
    probe_only[250:303] = True  # equal tags, not in the build
    probe_only[304] = True      # tag EMPTY_KEY - 1, aliasing the build key of tag EMPTY_KEY
    probe_only[700:] = True
    return strings, word, probe_only


def utf8_side(rng, strings, word, pick, null_frac):
    s = pa.array([strings[j] for j in pick], mask=rng.random(len(pick)) < null_frac)
    return [s, pa.array(word[pick], mask=rng.random(len(pick)) < null_frac)]


@pytest.mark.parametrize("kind", [0, A.JOIN_SEMI, A.JOIN_ANTI], ids=["inner", "semi", "anti"])
def test_join_utf8_keys_with_equal_tags(ctx, kind, monkeypatch):
    monkeypatch.delenv("DFGPU_JOIN_TAG_BITS", raising=False)
    rng = np.random.default_rng(15)
    strings, word, probe_only = join_utf8_keys(rng)
    inb = np.flatnonzero(~probe_only)
    build = utf8_side(rng, strings, word, np.concatenate([inb, inb[rng.integers(0, len(inb), 400)]]), 0.02)
    pick = rng.integers(0, len(strings), 20_000)
    pick[:len(strings)] = np.arange(len(strings))
    probe = utf8_side(rng, strings, word, pick, 0.03)
    keys = [col(0), col(1)]
    if kind == 0:
        J.same_pairs(utf8_gpu_pairs(ctx, probe, keys, build, keys), J.inner(probe, build))
    else:
        assert np.array_equal(gpu_pass(ctx, kind, probe, keys, build, keys), J.passing(kind, probe, build))


# ---- SQL ---------------------------------------------------------------------------------------------------------------
def sql_rows(hctx, sql):
    out = []
    for b in hctx.sql(sql).collect():
        cols = [c if isinstance(c, list) else np.asarray(c).tolist() for c in b]
        out.extend(zip(*cols))
    return sorted(out)


def test_sql_over_crafted_keys():
    rng = np.random.default_rng(16)
    k = draw(rng, crafted_pool(rng, wrapped=2000, at_zero=400, background=500), 120_000).view(I64)
    v = int_values(rng, len(k))
    dk = np.concatenate([np.unique(k)[::3], H.cluster_keys(rng, 300, "ones").view(I64)])  # hits and clustered misses
    dw = np.arange(len(dk), dtype=I64)
    hctx = host.ExecutionContext(0)
    try:
        hctx.register_memory("t", [("k", k), ("v", v)], batch_size=25_000)
        hctx.register_memory("d", [("dk", dk), ("w", dw)], batch_size=500)
        got = sql_rows(hctx, "SELECT k, SUM(v), COUNT(v) FROM t GROUP BY k")
        e = R.aggregate([k], [(R.SUM, v), (R.COUNT, v)])
        assert got == sorted(zip(e.keys[0].tolist(), e.aggs[0]["values"].tolist(), e.aggs[1]["values"].tolist()))
        hctx.register_memory("t", [("k", k), ("v", v)], batch_size=25_000)  # the GROUP BY drained the table
        got = sql_rows(hctx, "SELECT v, w FROM t JOIN d ON k = dk")
        prow, brow = J.inner([k], [dk])
        assert got == sorted(zip(v[prow].tolist(), dw[brow].tolist()))
    finally:
        hctx.close()


# ---- the probe limit ---------------------------------------------------------------------------------------------------
def limit_hashes(rng, m):
    """m distinct hashes on one home (top 40 bits all ones) with bit 0 clear, so that no two share a wide tag."""
    low = rng.choice(1 << (H.LOW - 1), m, replace=False).astype(U64) << np.uint64(1)
    return low | np.uint64(((1 << H.TOP) - 1) << H.LOW)


def no_rebuild(names):
    return not {"k_merge", "k_wide_move", "k_set_move"} & set(names)


def assert_probe_limit_error(err, names, rebuild):
    assert err.code == A.ERR_NOT_IMPLEMENTED and "probe limit" in err.msg, (err.code, err.msg)
    assert names.count(rebuild) == 1, names  # one rebuild for the first refusal, then the error


@pytest.mark.parametrize("extra", [0, 1], ids=["at_limit", "past_limit"])
def test_probe_limit_group_table(ctx, extra):
    rng = np.random.default_rng(17)
    k = np.concatenate([H.keys_for_hashes(limit_hashes(rng, H.AG_MAX_PROBE + extra)), H.background_keys(rng, 500), [SENTINEL]])
    k = np.repeat(k, 2)[rng.permutation(2 * len(k))].view(I64)
    v = int_values(rng, len(k))
    aggs = [AggregateFunction("sum", col(1)), AggregateFunction("count", col(1))]
    if extra == 0:
        got, names = run_agg(ctx, [[k, v]], [col(0)], aggs)
        assert no_rebuild(names), names
        R.assert_matches(got, R.aggregate([k], [(R.SUM, v), (R.COUNT, v)]), "at the probe limit")
    else:
        assert_probe_limit_error(*run_agg_error(ctx, [[k, v]], [col(0)], aggs), "k_merge")


@pytest.mark.parametrize("extra", [0, 1], ids=["at_limit", "past_limit"])
def test_probe_limit_wide_table(ctx, extra):
    rng = np.random.default_rng(18)
    h = limit_hashes(rng, H.AG_MAX_PROBE + extra)
    a = rng.permutation(1 << 22)[:len(h)].astype(I64)
    b = H.wide_last_part([a], h).view(I64)
    ba = rng.integers(-2 ** 40, 2 ** 40, 300)
    bb = H.wide_last_part([ba], H.background_hashes(rng, 300)).view(I64)
    assert int(H.wide_hash([np.array([-1]), np.array([-1])])[0]) >> 62 in (1, 2)  # (-1, -1) homes in the middle half too
    a, b = np.concatenate([a, ba, [-1]]), np.concatenate([b, bb, [-1]])
    v = int_values(rng, len(a))
    aggs = [AggregateFunction("count", col(2)), AggregateFunction("max", col(2))]
    if extra == 0:
        got, names = run_agg(ctx, [[a, b, v]], [col(0), col(1)], aggs)
        assert no_rebuild(names), names
        R.assert_matches(got, R.aggregate([a, b], [(R.COUNT, v), (R.MAX, v)]), "wide at the probe limit")
    else:
        assert_probe_limit_error(*run_agg_error(ctx, [[a, b, v]], [col(0), col(1)], aggs), "k_wide_move")


@pytest.mark.parametrize("extra", [0, 1], ids=["at_limit", "past_limit"])
def test_probe_limit_pair_set(ctx, extra):
    rng = np.random.default_rng(19)
    v = np.concatenate([H.distinct_values_for(0, limit_hashes(rng, H.AG_MAX_PROBE + extra)),
                        H.distinct_values_for(0, H.background_hashes(rng, 500))]).view(I64)
    v = np.repeat(v, 2)[rng.permutation(2 * len(v))]
    aggs = [AggregateFunction("count", col(0), distinct=True)]
    if extra == 0:
        got, names = run_agg(ctx, [[v]], [], aggs)
        assert no_rebuild(names), names
        R.assert_matches(got, R.aggregate([], [(R.COUNT_DISTINCT, v)]), "set at the probe limit")
    else:
        assert_probe_limit_error(*run_agg_error(ctx, [[v]], [], aggs), "k_set_move")
