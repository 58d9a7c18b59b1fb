#!/usr/bin/env python
"""Workload for compute-sanitizer (memcheck / racecheck): one pass through every hand-rolled synchronisation
protocol of the engine at sizes a sanitizer finishes in minutes, each result checked against numpy.
  compute-sanitizer --tool racecheck python profiles/sanitize_cases.py
  compute-sanitizer --tool memcheck  python profiles/sanitize_cases.py
Covers: the mbarrier / cp.async.bulk pipeline of k_filter_project_tma (full, ragged and single tiles, lagged
scan, dual ring), the direct filter kernel, the CAS / RED table of k_hash_agg_lean / _plain / interpreter, table
growth with overflow replay, the shared-memory front tables, wide-key slots (busy / ready publication) and the
chunked host pipelines, and the
join's build, probe and gathers, and CASE in the extended interpreter: its validity bytes under a WHERE (out_vbytes,
k_pack_bits), the null-aware reduce, the group scan and the TMA interpreter loop."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from datafusion_archive_b200 import _abi as A  # noqa: E402
from datafusion_archive_b200 import engine, workloads  # noqa: E402
from datafusion_archive_b200.expr import AggregateFunction, case, col, lit  # noqa: E402

ctx = engine.GpuContext(0)
rng = np.random.default_rng(1)


def fp(arrays, pred, proj):
    b = ctx.upload(arrays)
    r = ctx.filter_project(b, pred, proj)
    out = r.columns()
    r.free(); b.free()
    return out


def agg(arrays, keys, aggs, nb=1, pred=None, expected=0):
    n = len(arrays[0])
    bounds = [int(x) for x in np.linspace(0, n, nb + 1)]
    bs = [ctx.upload([a[bounds[i]:bounds[i + 1]] for a in arrays]) for i in range(nb)]
    r = ctx.aggregate(bs, keys, aggs, expected, pred=pred)
    out = r.columns()
    r.free()
    for b in bs:
        b.free()
    return out


# 1. TMA filter pipeline: sizes around tile boundaries, C2 and C3 shapes
for n in [1, 4095, 4096, 4097, 700_001]:
    a = rng.random(n)
    out = fp([a], col(0) > lit(0.5), [col(0)])[0]
    assert np.array_equal(out, a[a > 0.5]), n
arrays, pred, proj = workloads.c3(300_000)
o = fp(arrays, pred, proj)
m = arrays[1] < arrays[0]
assert np.array_equal(o[0], (arrays[0] + arrays[1])[m]) and np.array_equal(o[1], (arrays[0] * arrays[1])[m])
# lean consumer loop: Int64 comparison against a column, 64-bit integer arithmetic, two projections; generic FAST loop: two terms
ki = rng.integers(-50, 50, 300_001, dtype=np.int64)
kj = rng.integers(-50, 50, 300_001, dtype=np.int64)
o = fp([ki, kj], col(0) <= col(1), [col(0) * col(1), col(1)])
assert np.array_equal(o[0], (ki * kj)[ki <= kj]) and np.array_equal(o[1], kj[ki <= kj])
a1 = rng.random(300_001)
o = fp([a1], (col(0) > lit(0.25)) & (col(0) < lit(0.75)), [col(0)])
assert np.array_equal(o[0], a1[(a1 > 0.25) & (a1 < 0.75)])
# generic interpreter (direct kernel shapes)
o = fp([arrays[0]], (col(0) * col(0)) < lit(0.3), [(col(0) + col(0)) * (col(0) - lit(1.0)) / (col(0) + lit(2.0))])
a0 = arrays[0]
assert np.array_equal(o[0], ((a0 + a0) * (a0 - 1.0) / (a0 + 2.0))[a0 * a0 < 0.3])
print("filter/project ok", flush=True)

# 2. hash aggregate: lean (SUM, COUNT / MIN, MAX, SUM), plain (with WHERE), interpreter (expression key)
n = 400_000
k = workloads.mix_keys(rng.integers(0, 3000, n, dtype=np.int64))
v = rng.random(n)
uk, inv = np.unique(k, return_inverse=True)
got = agg([k, v], [col(0)], [AggregateFunction("sum", col(1)), AggregateFunction("count", col(1))], nb=2)
o = np.argsort(got[0])
assert np.array_equal(got[0][o], uk) and np.array_equal(got[2][o], np.bincount(inv).astype(np.uint64))
got = agg([k, v], [col(0)], [AggregateFunction("min", col(1)), AggregateFunction("max", col(1)), AggregateFunction("sum", col(1))])
o = np.argsort(got[0])
mn = np.full(len(uk), np.inf); np.minimum.at(mn, inv, v)
assert np.array_equal(got[1][o], mn)
got = agg([k, v], [col(0)], [AggregateFunction("max", col(1))], pred=col(1) < lit(0.5))
assert len(got[0]) == len(np.unique(k[v < 0.5]))
got = agg([k, v], [col(0) + lit(1)], [AggregateFunction("sum", col(1) * lit(2.0))])
assert len(got[0]) == len(uk)
print("hash aggregate ok", flush=True)

# 3. table growth with overflow replay (more distinct keys than half the initial table)
n = 2_300_000
kk = workloads.mix_keys(np.arange(n, dtype=np.int64))
got = agg([kk, np.ones(n)], [col(0)], [AggregateFunction("count", col(1))])
assert len(got[0]) == n and int(got[1].sum()) == n
print("growth ok", flush=True)

# 4. front tables (few groups, > 4 Mi rows so that the sampled prefix switches them on)
n = 4_500_000
for g in [3, 500]:
    kf = workloads.mix_keys(rng.integers(0, g, n, dtype=np.int64))
    vf = rng.random(n)
    got = agg([kf, vf], [col(0)], [AggregateFunction("sum", col(1)), AggregateFunction("count", col(1)), AggregateFunction("max", col(1))])
    assert len(got[0]) == g and int(got[2].sum()) == n
print("front tables ok", flush=True)

# 5. wide keys: busy / ready publication under contention, and growth by moving slots
n = 600_000
h1 = rng.integers(0, 3, n, dtype=np.int64) * (2 ** 40)
h2 = rng.integers(0, 2, n, dtype=np.int64) - 1
got = agg([h1, h2, rng.random(n)], [col(0), col(1)], [AggregateFunction("count", col(2))])
assert len(got[0]) == 6 and int(got[2].sum()) == n
s1 = ["k%d" % i for i in rng.integers(0, 50, 100_000)]
k3 = rng.integers(0, 4, 100_000, dtype=np.int32)
got = agg([s1, k3, rng.random(100_000)], [col(0), col(1)], [AggregateFunction("sum", col(2))], nb=2)
assert len(got[0]) == len(set(zip(s1, k3.tolist())))
print("wide keys ok", flush=True)

# 6. chunked host pipelines
a = rng.random(9_000_000)
r = ctx.filter_project_host([a], col(0) > lit(0.5), [col(0)], chunk_rows=2_000_000)
assert r.nrows == int((a > 0.5).sum())
r.free()
kh = workloads.mix_keys(rng.integers(0, 1000, 9_000_000, dtype=np.int64))
r = ctx.aggregate_host([kh, a], [col(0)], [AggregateFunction("sum", col(1))], chunk_rows=2_000_000)
assert r.nrows == 1000
r.free()
print("host pipelines ok", flush=True)

# 7. COUNT(DISTINCT): 128-bit CAS pair sets, their growth with overflow replay, and the count at finish
kd = rng.integers(-1, 300, 1_500_000).astype(np.int64)
vd = rng.integers(-1, 5000, 1_500_000).astype(np.int64)
got = agg([kd, vd], [col(0)], [AggregateFunction("count", col(1), distinct=True)], nb=2)
pairs = np.unique(np.stack([kd, vd], 1), axis=0)
assert int(got[1].sum()) == len(pairs) and len(got[0]) == len(np.unique(kd))
got = agg([vd], [], [AggregateFunction("count", col(0), distinct=True)])
assert int(got[0][0]) == len(np.unique(vd))
print("count distinct ok", flush=True)

# 8. AVG: the converting fold with nulls, the lean f64 scan, k_avg_finish's bitmap, and the scalar reduce
import pyarrow as pa  # noqa: E402
ka = rng.integers(0, 1000, 1_000_003).astype(np.int64)
va = rng.integers(-100, 100, 1_000_003).astype(np.int32)
ok = (rng.random(len(va)) < 0.5) & (ka != 3)
got = agg([ka, pa.array(va, mask=~ok)], [col(0)], [AggregateFunction("avg", col(1))])
vals, valid = got[1]
assert len(got[0]) == len(np.unique(ka)) and not valid[np.asarray(got[0]) == 3].any()
got = agg([ka, va.astype(np.float64)], [col(0)], [AggregateFunction("avg", col(1))])
assert len(got[0]) == len(np.unique(ka))
got = agg([va], [], [AggregateFunction("avg", col(0))])
assert float(got[0][0]) == float(np.float64(va.astype(np.int64).sum()) / len(va))
print("avg ok", flush=True)

# 9. Utf8 functions: k_utf8_view_len / k_utf8_view_copy over every row, over selected rows, the case-only path, a
# predicate over a view, and an Int64 length as a GROUP BY key (strings straddle 16-byte words; one is > 4 KiB)
from datafusion_archive_b200.expr import utf8_fn  # noqa: E402
sv = [None if i % 11 == 0 else (b" " * (i % 3) + b"ab\xc3\xa9Xy" * (i % 7) + b" " * (i % 2)) for i in range(200_003)] + [b"q" * 5000]
sa = pa.array(sv, type=pa.binary())
sx = rng.random(len(sv))
o = fp([sa, sx], col(1) > lit(0.5), [utf8_fn("upper", utf8_fn("trim", utf8_fn("substr", col(0), 2))), utf8_fn("length", col(0))])
assert len(o[0]) == int((sx > 0.5).sum())
o = fp([pa.array([v or b"" for v in sv], type=pa.binary())], None, [utf8_fn("lower", col(0))])
assert o[0][5] == sv[5].lower().decode()
o = fp([sa, sx], utf8_fn("lower", col(0)).like(lit(b"%abx%")), [col(1)])
assert len(o[0]) == sum(1 for v in sv if v is not None and b"abx" in v.strip(b" ").lower())
got = agg([sa, sx], [utf8_fn("length", col(0))], [AggregateFunction("count", col(1))])
assert int(np.asarray(got[1]).sum()) == len(sv)
print("utf8 functions ok", flush=True)
# 10. Inner join: k_join_build's CAS claims and warp-aggregated counts (a hot key, the key that equals the empty marker,
# null keys), k_join_scatter, the u32 -> u64 scan, k_join_count, k_join_emit's per-tile search (a skewed key and
# one-match rows), and every gather: fixed width, the ballot-based bit gather (validity, Boolean) and Utf8
jn = 50_003
jbk = np.concatenate([np.full(5000, 3, np.int64), np.full(7, -1, np.int64), rng.integers(0, 20_000, jn - 5007)])
jbv = rng.random(jn) > 0.05
jbool = pa.array(rng.random(jn) > 0.5, mask=rng.random(jn) < 0.1)
jpk = np.concatenate([np.array([3, -1, 3], np.int64), rng.integers(0, 40_000, 70_000)])
jps = pa.array(["r%d" % (i % 97) * (i % 5) for i in range(len(jpk))], mask=rng.random(len(jpk)) < 0.1)
jbb = ctx.upload([pa.array(jbk, mask=~jbv), np.arange(jn, dtype=np.int32), jbool])
jpb = ctx.upload([jpk, jps, rng.random(len(jpk))])
jj = ctx.join_build(jbb, [col(0)], keep_cols=[1, 2])
jbb.free()
jr = jj.probe(jpb, [col(0)], probe_cols=[1, 2], build_cols=[1, 2])
jo = jr.columns()
jcnt = {}
for k, v in zip(jbk.tolist(), jbv.tolist()):
    if v:
        jcnt[k] = jcnt.get(k, 0) + 1
assert jr.nrows == sum(jcnt.get(k, 0) for k in jpk.tolist())
jr.free(); jj.free(); jpb.free()
print("join ok", flush=True)
# 11. Inner join on Utf8 keys: k_join_utf8_place's claims, k_join_utf8_verify's byte compare of each row against its
# slot's representative and its list of rows for the next round, and k_join_utf8_count's confirmation against the
# join's copy of the build keys (strings at every alignment, a string ending at its buffer's end, a lower() key); then
# the same under 2-bit tags, where many distinct strings share a tag and the build runs many rounds
jwords = ["w%d" % i * (1 + i % 7) for i in range(400)] + ["", "x" * 40]
jus = pa.array([jwords[i] for i in rng.integers(0, len(jwords), 20_000)], mask=rng.random(20_000) < 0.05)
jup = pa.array([jwords[i].upper() for i in rng.integers(0, len(jwords), 30_000)] + ["X" * 40])
jcount = {}
for v in jus.to_pylist():
    if v is not None:
        jcount[v] = jcount.get(v, 0) + 1
for bits in (None, "2"):
    if bits:
        os.environ["DFGPU_JOIN_TAG_BITS"] = bits
    jbb = ctx.upload([jus, np.arange(20_000, dtype=np.int32)])
    jpb = ctx.upload([jup])
    jj = ctx.join_build(jbb, [col(0)], keep_cols=[0, 1])
    jbb.free()
    jr = jj.probe(jpb, [utf8_fn("lower", col(0))], probe_cols=[0], build_cols=[0, 1])
    jr.columns()
    assert jr.nrows == sum(jcount.get(v.lower(), 0) for v in jup.to_pylist())
    jr.free(); jj.free(); jpb.free()
    os.environ.pop("DFGPU_JOIN_TAG_BITS", None)
print("utf8 join ok", flush=True)
# 12. Semi / anti join: k_join_mark's ballots and tile counts, k_join_select's prefix over the mask words (a ragged last
# tile, every kind, nulls on both sides), and k_join_utf8_mark's confirmation under 2-bit tags
spk = pa.array(rng.integers(0, 300, 9_001), mask=rng.random(9_001) < 0.05)
sbk = pa.array(rng.integers(0, 600, 200), mask=rng.random(200) < 0.01)
sset = {v for v in sbk.to_pylist() if v is not None}
for kind in (A.JOIN_SEMI, A.JOIN_ANTI, A.JOIN_ANTI_NULL_AWARE):
    sbb, spb = ctx.upload([sbk]), ctx.upload([spk, np.arange(9_001, dtype=np.int64)])
    sj = ctx.join_build(sbb, [col(0)], keep_cols=[])
    sr = sj.semi(spb, [col(0)], kind, probe_cols=[1])
    got = sr.columns()[0] if sr.nrows else np.zeros(0, np.int64)
    pl = spk.to_pylist()
    if kind == A.JOIN_SEMI:
        exp = [i for i, v in enumerate(pl) if v is not None and v in sset]
    elif kind == A.JOIN_ANTI:
        exp = [i for i, v in enumerate(pl) if v is None or v not in sset]
    else:
        exp = [] if sbk.null_count else [i for i, v in enumerate(pl) if v is not None and v not in sset]
    assert list(got) == exp, kind
    sr.free(); sj.free(); sbb.free(); spb.free()
os.environ["DFGPU_JOIN_TAG_BITS"] = "2"
sbb, spb = ctx.upload([jus]), ctx.upload([jup, np.arange(len(jup), dtype=np.int64)])
sj = ctx.join_build(sbb, [col(0)], keep_cols=[])
sr = sj.semi(spb, [utf8_fn("lower", col(0))], A.JOIN_SEMI, probe_cols=[1])
assert sr.nrows == sum(1 for v in jup.to_pylist() if v.lower() in jcount)
sr.free(); sj.free(); sbb.free(); spb.free()
os.environ.pop("DFGPU_JOIN_TAG_BITS", None)
print("semi join ok", flush=True)

# 13. CASE: the direct kernel's validity bytes of a CASE without ELSE under a WHERE and k_pack_bits's ballots and zero
# count (a ragged last word), the NULLS kernel without a WHERE, the TMA interpreter loop (CASE with ELSE), and the reduce
# and group scan counting CASE-made nulls under a fused WHERE
for n in [1, 31, 33, 300_001]:
    a = rng.random(n)
    nn = case([(col(0) > lit(0.5), col(0))])
    v, ok = (lambda c: c if isinstance(c, tuple) else (c, np.ones(len(c), bool)))(fp([a], col(0) < lit(0.9), [nn])[0])
    sel = a < 0.9
    assert np.array_equal(ok, a[sel] > 0.5) and np.array_equal(v[ok], a[sel][a[sel] > 0.5]), n
    c = fp([a], None, [nn])[0]
    c = c if isinstance(c, tuple) else (c, np.ones(len(c), bool))
    assert np.array_equal(c[1], a > 0.5), n
    o = fp([a], None, [case([(col(0) > lit(0.5), col(0))], lit(0.0))])[0]
    assert np.array_equal(o, np.where(a > 0.5, a, 0.0)), n
kc = rng.integers(0, 1000, 300_001, dtype=np.int64)
vc = rng.random(300_001)
cnt = agg([kc, vc], [], [AggregateFunction("count", case([(col(1) > lit(0.5), col(1))]))], nb=2, pred=col(0) > lit(100))
assert cnt[0][0] == np.count_nonzero((vc > 0.5) & (kc > 100))
g = agg([kc, vc], [col(0)], [AggregateFunction("count", case([(col(1) > lit(0.5), col(1))]))], pred=col(0) > lit(100))
exp = np.bincount(kc[(vc > 0.5) & (kc > 100)], minlength=1000)
assert np.array_equal(np.asarray(g[1]), exp[np.asarray(g[0])])
print("case ok", flush=True)
# 14. ORDER BY / LIMIT / HAVING (dfgpu_sort): the keep mask's ragged last tile, a nullable Utf8 key's MSD rounds and
# null pass, a skipped digit, the stable scatter's partial chunk and tile, and the gathers of a LIMIT inside a tile
for n in [1, 33, 4097, 100_003]:
    ks = pa.array(["k%d" % (i % 37) * (1 + i % 3) for i in range(n)], type=pa.string(), mask=np.arange(n) % 11 == 0)
    kv = rng.integers(0, 300, n, dtype=np.int64)
    keep = pa.array(np.arange(n) % 5 != 0, mask=np.arange(n) % 7 == 0)
    b = ctx.upload([ks, kv, np.arange(n, dtype=np.int64), keep])
    r = ctx.sort(b, keys=[col(0), col(1)], desc=[True, False], keep=col(3), limit=n // 2)
    assert r.nrows == min(n // 2, int(np.count_nonzero((np.arange(n) % 5 != 0) & (np.arange(n) % 7 != 0)))), n
    r.free(); b.free()
print("sort ok", flush=True)
# 15. window functions (dfgpu_window): the segmented scan's ragged last tile, a nullable Utf8 partition key, one row,
# and the rank, MIN / AVG and integer SUM outputs of a partial validity word
for n in [1, 33, 2049, 100_003]:
    ks = pa.array(["k%d" % (i % 37) for i in range(n)], type=pa.string(), mask=np.arange(n) % 11 == 0)
    b = ctx.upload([ks, rng.integers(0, 300, n, dtype=np.int64), pa.array(rng.standard_normal(n), mask=np.arange(n) % 5 == 0)])
    r = ctx.window(b, [(A.WIN_RANK, None, 0), (A.AGG_MIN, col(2), 0), (A.AGG_AVG, col(2), 0), (A.AGG_SUM, col(1), 0)], partition=[col(0)],
                   order=[col(1)], desc=[True])
    assert r.nrows == n, n
    r.free(); b.free()
print("window ok", flush=True)
ctx.close()
print("SANITIZE_CASES_OK")
