"""Every filter/project dispatch shape, bit for bit against numpy, with the kernel instantiation it is named for.

Each case runs with DFGPU_TRACE set, reads the names of the kernels the library launched, and asserts the
`k_filter_project_tma<DEPTH, K, F64ONLY, FAST, LEAN>` or `k_filter_project<DEPTH, NULLS>` it expects, so a change in
how expression shapes are recognised cannot silently move a query onto another kernel.  K follows from the bytes
per row the predicate and the projections read (DESIGN §4.2): 8 rows per lane up to 16 bytes, 4 up to 32."""

import numpy as np
import pytest

from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import engine
from datafusion_archive_b200.expr import col, lit
from kernel_trace import capfd_launched

pytestmark = pytest.mark.gpu

N = 1_000_003  # the last tile is ragged at every tile size


@pytest.fixture(scope="module")
def ctx():
    c = engine.GpuContext(0)
    yield c
    c.close()


@pytest.fixture
def launched(monkeypatch, capfd):
    """Returns a function that yields the canonical names of the kernels launched since the last call:
    `k_filter_project_tma<1, 8, true, true, 1>` -> `k_filter_project_tma<1,8,1,1,1>`."""
    return capfd_launched(monkeypatch, capfd)


def f64s(rng, n, nan=True):
    """[0, 1) with ±0.0 and exact comparison edges sprinkled in, and NaN / ±inf unless the values feed arithmetic
    (NaN payloads from the GPU's arithmetic differ from the host's)."""
    x = rng.random(n)
    idx = rng.choice(n, 64, replace=False)
    special = [np.nan, -0.0, 0.0, np.inf, -np.inf, 0.5, 0.25, 1e-300] if nan else [-0.0, 0.0, 0.5, 0.25, 1e-300, 0.9, 0.1, 0.05]
    x[idx] = np.array(special * 8)
    return x


def ints(rng, dt, n):
    """Small values (so comparisons find equal ones) with the type's extremes sprinkled in."""
    info = np.iinfo(dt)
    x = rng.integers(max(info.min, -8), 8, n).astype(dt)
    idx = rng.choice(n, 40, replace=False)
    x[idx] = np.array([info.min, info.max, 0, info.max - 1, info.min + 1] * 8, dtype=dt)
    return x


def f32s(rng, n):
    x = (rng.integers(-8, 8, n) * 0.5).astype(np.float32)
    idx = rng.choice(n, 24, replace=False)
    x[idx] = np.array([np.nan, -0.0, 0.0, np.inf, -np.inf, 3.5] * 4, dtype=np.float32)
    return x


def deep(c, depth):
    """An Int64 expression equal to col(c) whose register stack depth is `depth` (>= 2)."""
    e = col(c) - col(c)
    for _ in range(depth - 2):
        e = (col(c) - col(c)) + e
    return col(c) + e


CMP = {"lt": (lambda e, r: e < r, np.less), "le": (lambda e, r: e <= r, np.less_equal),
       "gt": (lambda e, r: e > r, np.greater), "ge": (lambda e, r: e >= r, np.greater_equal),
       "eq": (lambda e, r: e.eq(r), np.equal), "ne": (lambda e, r: e.not_eq(r), np.not_equal)}

# Each case: (kernel, columns(rng), predicate, projections, reference(columns) -> (mask, projected arrays)).
CASES = {
    # ---- lean consumer loop: one comparison over 8-byte operands, one or two 8-byte projections
    "lean_c2": ("k_filter_project_tma<1,8,1,1,1>", lambda rng: [f64s(rng, N)],
                col(0) > lit(0.5), [col(0)], lambda c: (c[0] > 0.5, [c[0]])),
    "lean_c3": ("k_filter_project_tma<1,4,1,1,2>", lambda rng: [f64s(rng, N, nan=False), f64s(rng, N, nan=False)],
                col(1) < col(0), [col(0) + col(1), col(0) * col(1)], lambda c: (c[1] < c[0], [c[0] + c[1], c[0] * c[1]])),
    "lean_i64": ("k_filter_project_tma<1,4,1,1,2>", lambda rng: [ints(rng, np.int64, N), ints(rng, np.int64, N)],
                 col(0) > lit(-3), [col(0) * lit(3), col(0) - col(1)], lambda c: (c[0] > -3, [c[0] * np.int64(3), c[0] - c[1]])),
    "lean_u64": ("k_filter_project_tma<1,4,1,1,1>", lambda rng: [ints(rng, np.uint64, N), ints(rng, np.uint64, N)],
                 col(0) >= col(1), [col(0) + col(1)], lambda c: (c[0] >= c[1], [c[0] + c[1]])),
    # ---- generic FAST loop, every column Float64
    "fast_f64_copy_no_pred": ("k_filter_project_tma<1,8,1,1,0>", lambda rng: [f64s(rng, N)],
                              None, [col(0)], lambda c: (np.ones(N, bool), [c[0]])),
    "fast_f64_and2": ("k_filter_project_tma<1,4,1,1,0>", lambda rng: [f64s(rng, N), f64s(rng, N)],
                      (col(0) > lit(0.25)) & (col(1) < lit(0.75)), [col(0)], lambda c: ((c[0] > 0.25) & (c[1] < 0.75), [c[0]])),
    "fast_f64_or3": ("k_filter_project_tma<1,4,1,1,0>", lambda rng: [f64s(rng, N), f64s(rng, N)],
                     ((col(0) > lit(0.9)) | (col(1) <= lit(0.1))) & col(0).not_eq(col(1)), [col(1)],
                     lambda c: (((c[0] > 0.9) | (c[1] <= 0.1)) & (c[0] != c[1]), [c[1]])),
    "fast_f64_chain4": ("k_filter_project_tma<1,4,1,1,0>", lambda rng: [f64s(rng, N), f64s(rng, N)],
                        (((col(0) >= lit(0.2)) & (col(1) < col(0))) | col(0).eq(lit(0.5))) & (col(1) > lit(0.05)), [col(0)],
                        lambda c: ((((c[0] >= 0.2) & (c[1] < c[0])) | (c[0] == 0.5)) & (c[1] > 0.05), [c[0]])),
    "fast_f64_three_proj": ("k_filter_project_tma<1,4,1,1,0>", lambda rng: [f64s(rng, N, nan=False), f64s(rng, N, nan=False)],
                            col(0) > lit(0.5), [col(0), col(1) / lit(4.0), col(0) - col(1)],
                            lambda c: (c[0] > 0.5, [c[0], c[1] / 4.0, c[0] - c[1]])),
    # ---- interpreter: f64_only (every operand Float64 / Boolean, no CAST) and generic
    "interp_f64_chain5": ("k_filter_project_tma<2,4,1,0,0>", lambda rng: [f64s(rng, N), f64s(rng, N)],
                          ((((col(0) > lit(0.1)) & (col(1) < lit(0.9))) | (col(0) < lit(0.05))) & (col(1) > lit(0.2))) | col(0).eq(col(1)),
                          [col(0)], lambda c: (((((c[0] > 0.1) & (c[1] < 0.9)) | (c[0] < 0.05)) & (c[1] > 0.2)) | (c[0] == c[1]), [c[0]])),
    "interp_cast": ("k_filter_project_tma<2,8,0,0,0>", lambda rng: [f64s(rng, N), ints(rng, np.int32, N)],
                    col(0) > lit(0.5), [col(1).cast(A.FLOAT64)], lambda c: (c[0] > 0.5, [c[1].astype(np.float64)])),
    "interp_mixed_dtypes": ("k_filter_project_tma<2,4,0,0,0>", lambda rng: [ints(rng, np.int32, N), ints(rng, np.int64, N)],
                            col(0).cast(A.INT64) < col(1), [col(1)], lambda c: (c[0].astype(np.int64) < c[1], [c[1]])),
    "interp_narrow_arith": ("k_filter_project_tma<2,8,0,0,0>", lambda rng: [ints(rng, np.int32, N), ints(rng, np.int16, N)],
                            col(0) > lit(-5, A.INT32), [col(0) + lit(7, A.INT32), col(1) * col(1)],
                            lambda c: (c[0] > -5, [c[0] + np.int32(7), c[1] * c[1]])),
    # ---- direct-load kernel
    "direct_depth5": ("k_filter_project<8,0>", lambda rng: [ints(rng, np.int64, N)],
                      col(0) > lit(0), [deep(0, 5)], lambda c: (c[0] > 0, [c[0]])),
}


# FAST loop, mixed types: Float32 / Int32 / UInt32 comparisons against a column and an immediate, an Int32 copy
def mixed_case(dt, code, v, op, rhs_col):
    make = lambda rng: [f32s(rng, N) if dt == np.float32 else ints(rng, dt, N) for _ in range(2)] + [ints(rng, np.int32, N)]  # noqa: E731
    expr, f = CMP[op]
    pred = expr(col(0), col(1) if rhs_col else lit(v, code))
    return ("k_filter_project_tma<1,8,0,1,0>", make, pred, [col(2)], lambda c: (f(c[0], c[1] if rhs_col else dt(v)), [c[2]]))


for _name, _dt, _code, _v in [("f32", np.float32, A.FLOAT32, -1.5), ("i32", np.int32, A.INT32, -3), ("u32", np.uint32, A.UINT32, 3)]:
    for _op in sorted(CMP):
        for _rhs_col in (True, False):
            CASES["fast_mixed_%s_%s_%s" % (_name, _op, "col" if _rhs_col else "imm")] = mixed_case(_dt, _code, _v, _op, _rhs_col)


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


@pytest.mark.parametrize("case", sorted(CASES))
def test_dispatch(ctx, launched, case):
    kernel, make, pred, proj, ref = CASES[case]
    cols = make(np.random.default_rng(sum(map(ord, case))))
    got = run(ctx, cols, pred, proj)
    names = launched()
    assert kernel in names, (case, sorted(names))
    with np.errstate(all="ignore"):
        mask, exp = ref(cols)
    assert len(got) == len(exp)
    for g, e in zip(got, exp):
        e = e[mask]
        assert g.dtype == e.dtype and g.shape == e.shape, (case, g.dtype, e.dtype, g.shape, e.shape)
        assert np.array_equal(g.view(np.uint8), e.view(np.uint8)), case


def test_direct_nullable(ctx, launched):
    import groupby_ref as R
    rng = np.random.default_rng(5)
    a, b, valid = f64s(rng, N), f64s(rng, N), rng.random(N) > 0.3
    # a null left operand of `>` compares false (arrow 0.12); with a predicate the projections lose their bitmaps
    got = run(ctx, [R.arrow_nullable(a, valid), b], col(0) > lit(0.5), [col(0), col(1)])
    names = launched()
    assert "k_filter_project<8,1>" in names, sorted(names)
    m = valid & (a > 0.5)
    for g, e in zip(got, [a[m], b[m]]):
        assert np.array_equal(g.view(np.uint8), e.view(np.uint8))
