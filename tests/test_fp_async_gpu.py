"""Stream-ordered filter/project: calls that return once their kernel is queued, with the row count read on first use.

A query with a WHERE clause over null-free columns, numeric outputs and no division returns before its kernel has
finished; the kernel writes the row count into words the result owns.  These cases queue many such calls behind a
busy stream, free results while their kernels can still be running, and close a context with results pending, and
check every result bit for bit against numpy.  A division keeps the call synchronous, so that DivideByZero still
comes from the call itself.  Under DFGPU_TRACE the library names the calls that return stream-ordered; the C2 and C3
shapes are asserted to be among them."""
import numpy as np
import pytest

from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import engine
from datafusion_archive_b200.expr import col, lit

pytestmark = pytest.mark.gpu

ASYNC_LINE = "[dfgpu trace] filter_project returns stream-ordered"


@pytest.fixture(scope="module")
def ctx():
    c = engine.GpuContext(0)
    yield c
    c.close()


def hold_stream(ctx, n=100):
    """Queue n 128 MB memsets (about 50 us each on an H100) ahead of what follows, so that the calls after them
    return while their kernels are still waiting to run."""
    for _ in range(n):
        ctx.flush_l2()


def c2_like(ctx, n, t, seed):
    a = np.random.default_rng(seed).random(n)
    return ctx.upload([a]), (col(0) > lit(t)), [col(0)], lambda: [a[a > t]]


def c3_like(ctx, n, seed):
    a, b = (np.random.default_rng(seed + i).random(n) for i in range(2))
    m = b < a
    return ctx.upload([a, b]), (col(1) < col(0)), [col(0) + col(1), col(0) * col(1)], lambda: [(a + b)[m], (a * b)[m]]


def i64_like(ctx, n, t, seed):
    k = np.random.default_rng(seed).integers(-1000, 1000, n, dtype=np.int64)
    return ctx.upload([k]), (col(0) > lit(t)), [col(0) * lit(3), col(0)], lambda: [k[k > t] * np.int64(3), k[k > t]]


def f32_like(ctx, n, t, seed):
    v = np.random.default_rng(seed).random(n).astype(np.float32)
    return ctx.upload([v]), (col(0) < lit(t, A.FLOAT32)), [col(0)], lambda: [v[v < np.float32(t)]]


def check(r, want):
    got = r.columns()
    assert r.nrows == len(want[0])
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g.dtype == w.dtype
        assert np.array_equal(g.view(np.uint8), w.view(np.uint8))


def queries(ctx):
    """Ten queries over different batches, each selecting a different number of rows."""
    qs = [c2_like(ctx, 3_000_017 + 101 * i, t, seed=i) for i, t in enumerate([0.5, 0.1, 0.9, 0.33])]
    qs.append(c3_like(ctx, 2_500_009, seed=20))
    qs.append(c3_like(ctx, 1_000_003, seed=30))
    qs.append(i64_like(ctx, 2_000_003, 100, seed=40))
    qs.append(i64_like(ctx, 1_500_001, -700, seed=41))
    qs.append(f32_like(ctx, 2_200_001, 0.25, seed=50))
    qs.append(c2_like(ctx, 4_096, 0.75, seed=60))  # one tile
    counts = [len(want()[0]) for _, _, _, want in qs]
    assert len(set(counts)) == len(counts)
    return qs


def test_back_to_back_calls_keep_their_own_counts(ctx, capfd, monkeypatch):
    qs = queries(ctx)
    monkeypatch.setenv("DFGPU_TRACE", "1")
    capfd.readouterr()
    hold_stream(ctx)
    results = [ctx.filter_project(b, pred, proj) for b, pred, proj, _ in qs]
    assert capfd.readouterr().err.count(ASYNC_LINE) == len(qs)
    monkeypatch.delenv("DFGPU_TRACE")
    for r, (_, _, _, want) in zip(results, qs):
        check(r, want())
    # the same calls again, read in reverse order
    hold_stream(ctx)
    results = [ctx.filter_project(b, pred, proj) for b, pred, proj, _ in qs]
    for r, (_, _, _, want) in reversed(list(zip(results, qs))):
        check(r, want())
    for r in results:
        r.free()
    for b, _, _, _ in qs:
        b.free()


def test_results_freed_while_their_kernels_run(ctx):
    qs = queries(ctx)
    # freed right after the call
    hold_stream(ctx)
    for b, pred, proj, _ in qs:
        ctx.filter_project(b, pred, proj).free()
    # freed in reverse order, then interleaved with reads of the ones kept
    hold_stream(ctx)
    results = [ctx.filter_project(b, pred, proj) for b, pred, proj, _ in qs]
    for r in reversed(results):
        r.free()
    hold_stream(ctx)
    results = [ctx.filter_project(b, pred, proj) for b, pred, proj, _ in qs]
    for i, r in enumerate(results):
        if i % 2 == 0:
            r.free()
    for i, (r, (_, _, _, want)) in enumerate(zip(results, qs)):
        if i % 2:
            check(r, want())
            r.free()
    # later results reuse the freed buffers and count words
    hold_stream(ctx)
    results = [ctx.filter_project(b, pred, proj) for b, pred, proj, _ in qs]
    for r, (_, _, _, want) in zip(results, qs):
        check(r, want())
        r.free()
    for b, _, _, _ in qs:
        b.free()


def test_more_pending_results_than_one_slab(ctx):
    """150 results pending at once, a third of them freed unread: the count words grow instead of being shared."""
    n = 50_000
    a = np.random.default_rng(7).random(n)
    b = ctx.upload([a])
    ts = np.linspace(0.01, 0.99, 150)
    hold_stream(ctx, 600)
    results = [ctx.filter_project(b, col(0) > lit(float(t)), [col(0)]) for t in ts]
    for i in range(0, 150, 3):
        results[i].free()
    for i, t in enumerate(ts):
        if i % 3:
            check(results[i], [a[a > t]])
            results[i].free()
    b.free()


def test_division_by_zero_raises_from_the_call(ctx, capfd, monkeypatch):
    n = 1_000_003
    rng = np.random.default_rng(3)
    x, y = rng.random(n), rng.random(n) + 1.0
    y[n // 2] = 0.0
    x[n // 2] = 0.75  # survives the filter
    k, d = rng.integers(1, 100, n, dtype=np.int64), rng.integers(1, 5, n, dtype=np.int64)
    d[17] = 0
    k[17] = 50
    b = ctx.upload([x, y, k, d])
    monkeypatch.setenv("DFGPU_TRACE", "1")
    capfd.readouterr()
    for pred, proj in [(col(0) > lit(0.5), [col(0) / col(1)]), (col(2) > lit(10), [col(2) / col(3)]),
                       (col(0) > lit(0.5), [col(0), lit(1.0) / col(1)])]:
        with pytest.raises(engine.DfGpuError) as e:
            ctx.filter_project(b, pred, proj)
        assert e.value.code == A.ERR_ARROW and "DivideByZero" in e.value.msg
    assert ASYNC_LINE not in capfd.readouterr().err
    # the context is still usable, and a stream-ordered call after the failed ones is exact
    r = ctx.filter_project(b, col(0) > lit(0.5), [col(0) + col(1)])
    assert ASYNC_LINE in capfd.readouterr().err
    check(r, [(x + y)[x > 0.5]])
    r.free()
    b.free()


def test_close_with_results_pending():
    c = engine.GpuContext(0)
    qs = queries(c)
    hold_stream(c)
    results = [c.filter_project(b, pred, proj) for b, pred, proj, _ in qs]
    c.close()
    # closing waited for the kernels: the row counts were kept with the results
    for r, (_, _, _, want) in zip(results, qs):
        assert r.nrows == len(want()[0])
        r.free()


def test_dispatch_of_the_stream_ordered_path(ctx, capfd, monkeypatch):
    """C2 and C3 return stream-ordered; shapes whose count the host needs after the kernel do not."""
    n = 100_003
    rng = np.random.default_rng(11)
    a, b2 = rng.random(n), rng.random(n)
    flags = rng.random(n) < 0.5
    import pyarrow as pa
    nullable = pa.array(np.where(rng.random(n) < 0.1, np.nan, a), from_pandas=True)
    names = pa.array(["s%d" % (i % 13) for i in range(n)])
    batch = ctx.upload([a, b2, flags, nullable, names])
    monkeypatch.setenv("DFGPU_TRACE", "1")
    cases = [
        ("C2", col(0) > lit(0.5), [col(0)], True),
        ("C3", col(1) < col(0), [col(0) + col(1), col(0) * col(1)], True),
        ("Utf8 predicate, numeric output", col(4).eq(lit("s3")), [col(0)], True),
        ("no predicate", None, [col(0)], False),
        ("division", col(0) > lit(0.5), [col(0) / lit(2.0)], False),
        ("Boolean output", col(0) > lit(0.5), [col(1) < lit(0.5)], False),
        ("Utf8 output", col(0) > lit(0.5), [col(4)], False),
        ("Boolean input", col(2), [col(0)], True),
        ("nullable input", col(3) > lit(0.5), [col(0)], False),
    ]
    for name, pred, proj, stream_ordered in cases:
        capfd.readouterr()
        r = ctx.filter_project(batch, pred, proj)
        assert (ASYNC_LINE in capfd.readouterr().err) == stream_ordered, name
        assert r.nrows >= 0
        r.free()
    batch.free()
