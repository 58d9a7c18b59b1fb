"""The order of the kernel launches through which a batch reaches the group table and the COUNT(DISTINCT) sets.

Cases: the prefix sample of a first big batch and the table or set sizing it leads to; growth and replay of the group
table; growth and replay of the sets; and how the group scan and the set insert of each row range interleave.  Each case
runs the updates of an aggregate under DFGPU_TRACE, compares the kernels they launched, in order, with the sequence the
operator produces for that input, and checks the result against numpy.  Every input is far from the fill limits it meets,
so the number of replay rounds does not depend on how the CTAs of a launch interleave."""
import ctypes as C

import numpy as np
import pytest

from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import engine
from datafusion_archive_b200.expr import AggregateFunction, col
from kernel_trace import traced

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = engine.GpuContext(0)
    yield c
    c.close()


def aggregate(ctx, arrays, keys, aggs, expected_groups=0, batches=1):
    """(result columns, kernels launched by the updates) of one aggregate over `arrays`, cut into `batches` strided
    batches.  Nullable result columns come back as their values."""
    bs = [ctx.upload([a[i::batches] for a in arrays]) for i in range(batches)]
    keep = []
    kptrs, klens, nk = A.make_programs([k.program(bs[0].schema) for k in keys], keep)
    aggarr = A.make_aggs([a.lower(bs[0].schema) for a in aggs], keep)
    st = C.c_void_p()
    engine.check(engine.lib().dfgpu_aggregate_create(ctx.h, kptrs, klens, nk, aggarr, len(aggs), expected_groups, C.byref(st)))
    try:
        def update():
            for b in bs:
                engine.check(engine.lib().dfgpu_aggregate_update(st, b.h))
        _, names = traced(update)
        out = C.c_void_p()
        engine.check(engine.lib().dfgpu_aggregate_finish(st, C.byref(out)))
        r = engine.Result(ctx, out)
        try:
            cols = r.columns()
        finally:
            r.free()
    finally:
        engine.lib().dfgpu_aggregate_free(st)
        for b in bs:
            b.free()
    return [c[0] if isinstance(c, tuple) else c for c in cols], names


def sorted_by_key(cols):
    order = np.argsort(cols[0], kind="stable")
    return [np.asarray(c)[order] for c in cols]


# Kernel names as the library traces them.  Every input below is integer, null-free and unfiltered, so the first scan of a
# range is the plain or lean kernel and every replay, which reads a row list, takes the interpreter.
LEAN_SUM_COUNT = "k_hash_agg_lean<12, 3>"  # SUM + COUNT of an Int64 column, hybrid table layout
LEAN_SUM = "k_hash_agg_lean<4, 3>"
PLAIN = "k_hash_agg_plain<2, false>"
PLAIN_FRONT = "k_hash_agg_plain<2, true>"  # through the shared-memory front table: few groups so far
SCAN_REPLAY = "k_hash_agg<1, false, false>"
INSERT = "k_distinct_insert_plain<2>"
INSERT_REPLAY = "k_distinct_insert<2, false>"
REBUILD = ["k_table_init", "k_compact", "k_merge"]  # table_grow: new table, raw compaction, merge
SET_MOVE = "k_set_move"  # a set grows, x4 or to the size the prefix estimates


def test_prefix_sizes_the_group_table(ctx):
    """First GROUP BY batch, no hint, 5 M distinct keys: the 1 Mi-row prefix estimates 5 M groups, more than the 4 Mi-slot
    table takes, so the table is rebuilt for them (in line layout, where the lean kernel does not apply) before the rest of
    the batch is scanned, with no replay."""
    rng = np.random.default_rng(21)
    n = 5_000_000
    k = rng.permutation(n).astype(np.int64)
    v = rng.integers(-1000, 1000, n).astype(np.int64)
    (gk, s, c), names = aggregate(ctx, [k, v], [col(0)], [AggregateFunction("sum", col(1)), AggregateFunction("count", col(1))])
    assert names == ["k_table_init", LEAN_SUM_COUNT] + REBUILD + [PLAIN]
    gk, s, c = sorted_by_key([gk, s, c])
    assert np.array_equal(gk, np.arange(n)) and np.array_equal(s, v[np.argsort(k)]) and np.all(c == 1)


def test_group_table_grows_and_replays(ctx):
    """An expected_groups hint of 1000, so no prefix sample, and 3 M distinct keys: the 4 Mi-slot table refuses the keys
    beyond half full, grows x4, and the refused rows are replayed once."""
    rng = np.random.default_rng(22)
    n = 3_000_000
    k = rng.permutation(n).astype(np.int64) * 3 - 7
    v = rng.integers(-1000, 1000, n).astype(np.int64)
    (gk, s, c), names = aggregate(ctx, [k, v], [col(0)], [AggregateFunction("sum", col(1)), AggregateFunction("count", col(1))],
                                  expected_groups=1000)
    assert names == ["k_table_init", LEAN_SUM_COUNT] + REBUILD + [SCAN_REPLAY]
    gk, s, c = sorted_by_key([gk, s, c])
    order = np.argsort(k)
    assert np.array_equal(gk, k[order]) and np.array_equal(s, v[order]) and np.all(c == 1)


def test_prefix_sizes_the_set(ctx):
    """No GROUP BY, COUNT(x) and COUNT(DISTINCT x) over one first batch of 10.5 M distinct values: the reduce runs once
    over the whole batch; the prefix insert fills the 1 Mi-slot set, which grows x4 for one replay; the set is then sized
    for the estimate, and the rest of the batch needs no growth."""
    rng = np.random.default_rng(11)
    n = 10_500_000
    v = rng.permutation(n).astype(np.int64)
    (cnt, dis), names = aggregate(ctx, [v], [], [AggregateFunction("count", col(0)), AggregateFunction("count", col(0), distinct=True)])
    assert names == ["k_table_init", "k_reduce<1, false>", INSERT, SET_MOVE, INSERT_REPLAY, SET_MOVE, INSERT]
    assert int(cnt[0]) == n and int(dis[0]) == n


def test_scan_and_insert_interleave(ctx):
    """GROUP BY with SUM(v) and COUNT(DISTINCT v) over one first batch of 6 M distinct values in 3 M groups: the group scan
    of each range finishes before the sets insert it, and after the prefix the set is sized before the table."""
    rng = np.random.default_rng(23)
    n = 6_000_000
    v = rng.permutation(n).astype(np.int64)
    k = v // 2
    (gk, s, d), names = aggregate(ctx, [k, v], [col(0)], [AggregateFunction("sum", col(1)), AggregateFunction("count", col(1), distinct=True)])
    prefix = [LEAN_SUM, INSERT, SET_MOVE, INSERT_REPLAY]
    assert names == ["k_table_init"] + prefix + [SET_MOVE] + REBUILD + [PLAIN, INSERT]
    gk, s, d = sorted_by_key([gk, s, d])
    g = np.arange(n // 2)
    assert np.array_equal(gk, g) and np.array_equal(s, 4 * g + 1) and np.all(d == 2)


def test_sets_grow_by_replay(ctx):
    """test_count_distinct_gpu's set growth input: 10.5 M distinct values in 5 batches, each too small for a prefix sample,
    grouped by value % 1000.  The set grows x4 under the first batch (twice) and the fourth, each time followed by one
    replay; from the second batch on, the 1000 groups go through the front table."""
    rng = np.random.default_rng(11)
    n = 10_500_000
    v = rng.permutation(n).astype(np.int64)
    k = (v % 1000).astype(np.int32)
    (gk, d), names = aggregate(ctx, [k, v], [col(0)], [AggregateFunction("count", col(1), distinct=True)], batches=5)
    grow = [SET_MOVE, INSERT_REPLAY]
    assert names == (["k_table_init", PLAIN, INSERT] + grow + grow + [PLAIN_FRONT, INSERT] + [PLAIN_FRONT, INSERT] +
                     [PLAIN_FRONT, INSERT] + grow + [PLAIN_FRONT, INSERT])
    gk, d = sorted_by_key([gk, d])
    assert np.array_equal(gk, np.arange(1000)) and np.array_equal(d, np.bincount(k))
