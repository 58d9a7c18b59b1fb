"""Filter/project over many waves of the persistent TMA kernel (one wave = one tile per CTA): the offset
exchange between CTAs, run at every tile size the host picks, bit-exact against numpy.  Selectivity varies by
region, so some waves select nothing, some everything and some a mix; the sizes leave the last wave partial
and the last tile ragged, and the small sizes leave CTAs with fewer tiles than the pipeline is deep."""
import numpy as np
import pytest

from datafusion_archive_b200 import engine
from datafusion_archive_b200.expr import col, lit

pytestmark = pytest.mark.gpu

REGION = 300_007  # rows per selectivity region: not a multiple of any tile or wave


@pytest.fixture(scope="module")
def ctx():
    c = engine.GpuContext(0)
    yield c
    c.close()


def run(ctx, arrays, pred, proj):
    b = ctx.upload(arrays)
    try:
        r = ctx.filter_project(b, pred, proj)
        try:
            return r.columns()
        finally:
            r.free()
    finally:
        b.free()


def regional(n, seed):
    """a in [0, 1) with a per-region pattern for `a > 0.5`: none, all, mixed, sparse."""
    rng = np.random.default_rng(seed)
    a = rng.random(n)
    region = (np.arange(n) // REGION) % 4
    a[region == 0] *= 0.5                          # nothing selected
    a[region == 1] = 0.5 + 0.5 * a[region == 1] + 1e-9  # everything selected
    a[region == 3] = np.where(a[region == 3] < 0.99, a[region == 3] * 0.5, a[region == 3])  # about 1 %
    return a, region


def delay_env(monkeypatch, delay):
    if delay is not None:
        monkeypatch.setenv("DFGPU_FP_DELAY", str(delay))
        monkeypatch.setenv("DFGPU_FP_LAG", str(delay + 1))


# C2 shape: 8-byte predicate and projection column, 4096-row tiles; 22e6 rows are over 40 waves on 132 SMs
@pytest.mark.parametrize("n", [22_000_003, 1_130_000])
@pytest.mark.parametrize("delay", [None, 1, 3])
def test_c2_shape_many_waves(ctx, monkeypatch, n, delay):
    delay_env(monkeypatch, delay)
    a, _ = regional(n, seed=n)
    got = run(ctx, [a], col(0) > lit(0.5), [col(0)])
    exp = a[a > 0.5]
    assert got[0].shape == exp.shape
    assert np.array_equal(got[0].view(np.uint64), exp.view(np.uint64))


# C3 shape: two predicate columns, two arithmetic projections, 2048-row tiles
@pytest.mark.parametrize("n", [11_000_001, 560_000])
@pytest.mark.parametrize("delay", [None, 2])
def test_c3_shape_many_waves(ctx, monkeypatch, n, delay):
    delay_env(monkeypatch, delay)
    a, region = regional(n, seed=n + 1)
    b = np.random.default_rng(n + 2).random(n)
    b[region == 0] = a[region == 0] + 1.0  # b < a nowhere
    b[region == 1] = a[region == 1] - 1.0  # b < a everywhere
    got = run(ctx, [a, b], col(1) < col(0), [col(0) + col(1), col(0) * col(1)])
    m = b < a
    for g, e in zip(got, [(a + b)[m], (a * b)[m]]):
        assert g.shape == e.shape
        assert np.array_equal(g.view(np.uint64), e.view(np.uint64))


# six projected columns: 1024-row tiles
@pytest.mark.parametrize("n", [5_500_007, 290_000])
def test_six_columns_many_waves(ctx, n):
    a, _ = regional(n, seed=n + 3)
    rng = np.random.default_rng(n + 4)
    cols = [a] + [rng.random(n) for _ in range(5)]
    got = run(ctx, cols, col(0) > lit(0.5), [col(i) for i in range(6)])
    m = a > 0.5
    for g, c in zip(got, cols):
        assert np.array_equal(g.view(np.uint64), c[m].view(np.uint64))
