"""Binary arithmetic `+ - * /` over the ten numeric dtypes on the GPU, against the exact reference of
tests/arith_ref.py, at every site that evaluates it: the TMA interpreter (K = 8 and 4, register-stack depth 2 and 4,
the all-Float64 instantiation), the FAST leaf loop, both lean loops, the direct kernel at every depth, the null-aware
direct kernel with and without a WHERE, the chunked host path; stack-mode `V_RSUB` / `V_RDIV` at the last spill slot of
every depth; predicates over arithmetic; the aggregate's keys, arguments and fused WHERE; join keys; SQL.

Integer arithmetic wraps at the operand width, `/` truncates toward zero and `MIN / -1 = MIN`; a zero divisor raises
DivideByZero only in a row that survives the WHERE.  Bit for bit; NaNs compare as a class.  Each ABI case runs with
DFGPU_TRACE set and asserts the kernel it is about, so a case cannot silently land on another instantiation."""
import math
import os
from fractions import Fraction

import numpy as np
import pytest

import arith_ref as AR
import cast_ref as CR
import groupby_ref as R
from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import engine, host
from datafusion_archive_b200.expr import AggregateFunction, col, lit
from kernel_trace import traced_set as traced
from test_cast_gpu import assert_same, launched, sql_batches

pytestmark = pytest.mark.gpu

N = 1_000_003  # the last tile is ragged at every tile size
NUMERIC = AR.NUMERIC
NAME = {np.dtype(d): np.dtype(d).name for d in NUMERIC}
F32, F64, I64, U64, U8 = np.float32, np.float64, np.int64, np.uint64, np.uint8
EXPR = {"+": lambda x, y: x + y, "-": lambda x, y: x - y, "*": lambda x, y: x * y, "/": lambda x, y: x / y}
CMP = {"eq": (lambda e, r: e.eq(r), np.equal), "ne": (lambda e, r: e.not_eq(r), np.not_equal), "lt": (lambda e, r: e < r, np.less),
       "le": (lambda e, r: e <= r, np.less_equal), "gt": (lambda e, r: e > r, np.greater), "ge": (lambda e, r: e >= r, np.greater_equal)}


def code(dt):
    return CR.CODE[np.dtype(dt)]


def L(v, dt):
    return lit(float(v) if AR.is_float(dt) else int(v), code(dt))


def w8(dt):
    return np.dtype(dt).itemsize


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


def run_fp(ctx, arrays, pred, proj):
    b = ctx.upload(arrays)
    try:
        r = ctx.filter_project(b, pred, proj)
        try:
            return r.columns()
        finally:
            r.free()
    finally:
        b.free()


def fp(ctx, arrays, pred, proj):
    return traced(lambda: run_fp(ctx, arrays, pred, proj))


def raises_dbz(fn, want):
    """fn() (an untraced run_*) raises DivideByZero, and the kernel `want` ran before it was raised."""
    def go():
        try:
            fn()
        except engine.DfGpuError as e:
            return e
        return None
    e, names = traced(go)
    assert e is not None, ("no DivideByZero", want)
    assert e.code == A.ERR_ARROW and "DivideByZero" in e.msg, (e.code, e.msg)
    launched(names, want)


# ---- the projection matrix ------------------------------------------------------------------------------------------
def lits(dt):
    """A literal per operator, chosen where the operator wraps or rounds: a op L and L op b."""
    dt = np.dtype(dt)
    if AR.is_float(dt):
        f = np.finfo(dt)
        return {"+": float(f.max), "-": float(f.tiny), "*": 0.5, "/": 3.0}
    lo, hi = AR.int_bounds(dt)
    h = 1 << (4 * dt.itemsize)
    return {"+": hi, "-": lo if lo else 1, "*": h + 1, "/": -1 if lo else 3}


def matrix(dt):
    """The 12 projections a op b, a op L, L op b and their exact values over the rows of data(dt)."""
    exprs, refs = [], []
    a, b, _ = data(dt)
    for op in AR.OPS:
        lv = np.dtype(dt).type(lits(dt)[op])
        exprs += [EXPR[op](col(0), col(1)), EXPR[op](col(0), L(lv, dt)), EXPR[op](L(lv, dt), col(1))]
        refs += [AR.arith(op, a, b)[0], AR.arith(op, a, lv)[0], AR.arith(op, lv, b)[0]]
    return exprs, refs


_DATA = {}


def data(dt):
    """(a, b, keep) of N rows: the operand pairs of AR.operands, keep = the rows a WHERE keeps (never a zero b)."""
    key = np.dtype(dt)
    if key not in _DATA:
        rng = np.random.default_rng(500 + key.num)
        a, b = AR.operands(rng, dt, N)
        keep = (rng.random(N) < 0.8) & (b != 0)
        _DATA[key] = (a, b, keep)
    return _DATA[key]


_MATRIX = {}


def cached_matrix(dt):
    """(expressions, exact values, exact values of the rows data(dt) keeps)"""
    key = np.dtype(dt)
    if key not in _MATRIX:
        exprs, refs = matrix(dt)
        keep = data(dt)[2]
        _MATRIX[key] = (exprs, refs, [r[keep] for r in refs])
    return _MATRIX[key]


def u8_where(keep):
    """A UInt8 column and the predicate `w < 200` that keeps exactly `keep`."""
    rng = np.random.default_rng(9)
    w = np.where(keep, rng.integers(0, 200, len(keep)), rng.integers(200, 256, len(keep))).astype(U8)
    return w, col(2) < lit(200, A.UINT8)


def deep(d):
    """A tree over columns 0 and 1 of register-stack depth d (2, 3 or 5) without a division; deep_value() is its value."""
    e = col(0) * col(1)
    for i in range(d - 1):
        e = (col(1) if i % 2 == 0 else col(0)) - e
    return e


_DEEP = {}


def deep_value(a, b, d):
    """The exact value of deep(d) over the columns (a, b) = data(dt)[:2], computed once per (dtype, d)."""
    key = (a.dtype, d)
    if key not in _DEEP:
        v = AR.value("*", a, b)
        for i in range(d - 1):
            v = AR.value("-", b if i % 2 == 0 else a, v)
        _DEEP[key] = v
    return _DEEP[key]


def check_matrix(got, refs, what):
    for i, (g, e) in enumerate(zip(got, refs)):
        assert_same(g, e, (what, AR.OPS[i // 3], ["a op b", "a op L", "L op b"][i % 3]))


@pytest.mark.parametrize("dt", NUMERIC, ids=NAME.get)
def test_projection_tma_k8(ctx, dt):
    a, b, keep = data(dt)
    exprs, refs, kept = cached_matrix(dt)
    if w8(dt) <= 4:
        # UInt8 predicate + two operands: at most 9 bytes a row, 8 rows per lane
        w, pred = u8_where(keep)
        got, names = fp(ctx, [a, b, w], pred, exprs)
        launched(names, "k_filter_project_tma<2,8,0,0,0>")
        check_matrix(got, kept, "k8")
    else:
        # two 8-byte operands fill the 16 bytes of K = 8 alone: no WHERE, so the rows with a zero divisor are left out
        nz = b != 0
        got, names = fp(ctx, [a[nz], b[nz]], None, exprs)
        launched(names, "k_filter_project_tma<2,8,%d,0,0>" % (np.dtype(dt) == F64))
        check_matrix(got, [r[nz] for r in refs], "k8 no where")


@pytest.mark.parametrize("dt", NUMERIC, ids=NAME.get)
def test_projection_tma_k4(ctx, dt):
    # two Float64 predicate columns + two operands: 18 to 32 bytes a row, 4 rows per lane; all-Float64 programs take
    # the F64ONLY interpreter
    a, b, keep = data(dt)
    exprs, refs, kept = cached_matrix(dt)
    rng = np.random.default_rng(2)
    p = np.where(keep, rng.random(N) * 0.75, 0.8 + rng.random(N) * 0.2)
    q = rng.random(N) * 0.5 + 0.2
    got, names = fp(ctx, [a, b, p, q], (col(2) < lit(0.75)) & (col(3) > lit(0.1)), exprs)
    launched(names, "k_filter_project_tma<2,4,%d,0,0>" % (np.dtype(dt) == F64))
    check_matrix(got, kept, "k4")


@pytest.mark.parametrize("dt", NUMERIC, ids=NAME.get)
def test_projection_tma_depth4(ctx, dt):
    a, b, keep = data(dt)
    exprs, refs, kept = cached_matrix(dt)
    w, pred = u8_where(keep)
    e3 = deep(3)
    got, names = fp(ctx, [a, b, w], pred, exprs + [e3])
    launched(names, "k_filter_project_tma<4,4,0,0,0>")
    check_matrix(got[:-1], kept, "depth 4")
    assert_same(got[-1], deep_value(a, b, 3)[keep], "depth-3 tree")


@pytest.mark.parametrize("depth", [1, 2, 4, 8])
@pytest.mark.parametrize("dt", NUMERIC, ids=NAME.get)
def test_projection_direct(ctx, dctx, dt, depth):
    a, b, keep = data(dt)
    exprs, refs, kept = cached_matrix(dt)
    w, pred = u8_where(keep)
    extra = {1: [], 2: [deep(2)], 4: [deep(3)], 8: [deep(5)]}[depth]
    got, names = fp(ctx if depth == 8 else dctx, [a, b, w], pred, exprs + extra)
    launched(names, "k_filter_project<%d,0>" % depth)
    check_matrix(got[:12], kept, "direct %d" % depth)
    if extra:
        assert_same(got[12], deep_value(a, b, {2: 2, 4: 3, 8: 5}[depth])[keep], "deep")


@pytest.mark.parametrize("dt", NUMERIC, ids=NAME.get)
def test_projection_direct_nullable(ctx, dt):
    a, b, keep = data(dt)
    exprs, refs, kept = cached_matrix(dt)
    rng = np.random.default_rng(3)
    va, vb = rng.random(N) > 0.2, rng.random(N) > 0.2
    # without a WHERE: null where an operand is null, value 0 there; a zero divisor under a null does not raise
    vb &= b != 0
    got, names = fp(ctx, [R.arrow_nullable(a, va), R.arrow_nullable(b, vb)], None, exprs)
    launched(names, "k_filter_project<8,1>")
    zero = np.zeros(1, dtype=dt)
    for i, g in enumerate(got):
        valid = [va & vb, va, vb][i % 3]
        assert isinstance(g, tuple), i
        v, m = g
        assert np.array_equal(m, valid), i
        assert_same(v, np.where(valid, refs[i], zero), ("nulls", AR.OPS[i // 3], i % 3))
    # under a WHERE the bitmap is dropped and a surviving null slot's value is an operand like any other
    w, pred = u8_where(keep)
    got, names = fp(ctx, [R.arrow_nullable(a, va), R.arrow_nullable(b, vb), w], pred, exprs)
    launched(names, "k_filter_project<8,1>")
    assert not any(isinstance(g, tuple) for g in got)
    check_matrix(got, kept, "nulls + where")


@pytest.mark.parametrize("dt", NUMERIC, ids=NAME.get)
def test_projection_host_chunks(ctx, dt):
    a, b, keep = data(dt)
    exprs, refs, kept = cached_matrix(dt)
    w, pred = u8_where(keep)

    def go():
        r = ctx.filter_project_host([a, b, w], pred, exprs, chunk_rows=131_071)
        try:
            return [r.host_view(i).copy() for i in range(len(exprs))]
        finally:
            r.free()
    got, names = traced(go)
    launched(names, "k_filter_project_tma<2,%d,0,0,0>" % (8 if w8(dt) <= 4 else 4))
    check_matrix(got, kept, "host")


# ---- the interpreter-free loops -------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F32, F64, I64, U64], ids=NAME.get)
def test_fast_leaf_loop(ctx, dt):
    # every projection one `a op b` / `a op L` leaf (integer division is never a leaf); a comparison predicate over a
    # column of the operands' dtype drops every zero divisor
    a, b, keep = data(dt)
    ops = AR.OPS if AR.is_float(dt) else "+-*"
    lv = {op: np.dtype(dt).type(lits(dt)[op]) for op in ops}
    exprs = [EXPR[op](col(0), col(1)) for op in ops] + [EXPR[op](col(0), L(lv[op], dt)) for op in ops]
    refs = [AR.arith(op, a, b)[0] for op in ops] + [AR.arith(op, a, lv[op])[0] for op in ops]
    p = np.where(keep, 1, 0).astype(dt)
    got, names = fp(ctx, [a, b, p], col(2) > L(0, dt), exprs)
    k = 8 if np.dtype(dt) == F32 else 4
    launched(names, "k_filter_project_tma<1,%d,%d,1,0>" % (k, np.dtype(dt) == F64))
    for g, e, x in zip(got, refs, exprs):
        assert_same(g, e[keep], ("fast", repr(x)))
    # without a WHERE (the rows with a zero divisor left out): 8 rows per lane for every dtype
    nz = b != 0
    got, names = fp(ctx, [a[nz], b[nz]], None, exprs)
    launched(names, "k_filter_project_tma<1,8,%d,1,0>" % (np.dtype(dt) == F64))
    for g, e, x in zip(got, refs, exprs):
        assert_same(g, e[nz], ("fast no where", repr(x)))


LEAN = [(I64, "+", "-"), (U64, "-", "*"), (I64, "*", "+"), (F64, "/", "-"), (F64, "*", "+"), (U64, "+", "-")]


@pytest.mark.parametrize("dt,op1,op2", LEAN, ids=["%s_%s%s" % (NAME[np.dtype(d)], {"+": "add", "-": "sub", "*": "mul", "/": "div"}[x],
                                                                  {"+": "add", "-": "sub", "*": "mul", "/": "div"}[y]) for d, x, y in LEAN])
def test_lean_loop(ctx, dt, op1, op2):
    a, b, keep = data(dt)
    # two projections: a predicate over a third 8-byte column, 24 bytes a row, 4 rows per lane
    p = np.where(keep, 1, 0).astype(dt)
    got, names = fp(ctx, [a, b, p], col(2) > L(0, dt), [EXPR[op1](col(0), col(1)), EXPR[op2](col(0), col(1))])
    launched(names, "k_filter_project_tma<1,4,1,1,2>")
    assert_same(got[0], AR.arith(op1, a, b)[0][keep], ("lean 2", op1))
    assert_same(got[1], AR.arith(op2, a, b)[0][keep], ("lean 2", op2))
    # one projection over the predicate's own column: 16 bytes a row, 8 rows per lane
    lv = np.dtype(dt).type(lits(dt)[op1])
    thr = a[len(a) // 2]
    thr = thr if not (AR.is_float(dt) and math.isnan(thr)) else np.dtype(dt).type(1)
    got, names = fp(ctx, [a], col(0) > L(thr, dt), [EXPR[op1](col(0), L(lv, dt))])
    launched(names, "k_filter_project_tma<1,8,1,1,1>")
    with np.errstate(invalid="ignore"):
        m = a > thr
    assert_same(got[0], AR.arith(op1, a, lv)[0][m], ("lean 1", op1))


# ---- b. stack mode --------------------------------------------------------------------------------------------------
def nested(d, last):
    """x1 op1 (x2 op2 (... (x_d op_d x_{d+1}))) over columns 0..3 (x_i = column i % 4): register-stack depth d, with
    `last` (- or /) as op_{d-1}, the stack-mode instruction that pops the deepest spill slot; the other operators
    cycle through + * - /.  Returns (expression, [op_1 .. op_d])."""
    cyc = "+*-/"
    ops = [cyc[i % 4] for i in range(d)]
    ops[d - 2] = last
    ops[d - 1] = "-" if last == "/" else "+"
    e = EXPR[ops[d - 1]](col((d - 1) % 4), col(d % 4))
    for i in range(d - 2, -1, -1):
        e = EXPR[ops[i]](col(i % 4), e)
    return e, ops


def nested_value(cols, d, ops):
    v, bad = AR.arith(ops[d - 1], cols[(d - 1) % 4], cols[d % 4])
    for i in range(d - 2, -1, -1):
        v, z = AR.arith(ops[i], cols[i % 4], v)
        bad |= z
    return v, bad


STACK = [(d, last, direct) for d in (2, 4, 8) for last in "-/" for direct in (False, True) if not (d == 8 and direct)]


@pytest.mark.parametrize("dt", NUMERIC, ids=NAME.get)
def test_stack_mode(ctx, dctx, dt):
    n = 60_013
    rng = np.random.default_rng(np.dtype(dt).num + 600)
    # 4 columns drawn from 3000 distinct rows of edge and random values (the reference runs once per distinct row)
    pool = np.concatenate([AR.edges(dt), AR.pool(rng, dt, 200)])
    rows = pool[rng.integers(0, len(pool), (3000, 4))]
    rows[:len(pool), 0] = pool
    cols = list(rows[rng.integers(0, 3000, n)].T.copy())
    # Float64 runs once more under a Float64 predicate, which makes the program set all-Float64: the F64ONLY interpreter
    f64 = [False, True] if np.dtype(dt) == F64 else [False]
    for (d, last, direct), f64_pred in [(x, f) for x in STACK for f in f64 if not (f and (x[2] or x[0] == 8))]:
        e, ops = nested(d, last)
        v, bad = nested_value(cols, d, ops)
        keep = ~bad & (rng.random(n) < 0.9)
        if f64_pred:
            w, pred = np.where(keep, 1.0, 2.0), col(4) < lit(1.5)
        else:
            w, pred = np.where(keep, 1, 2).astype(U8), col(4) < lit(2, A.UINT8)
        got, names = fp(dctx if direct else ctx, cols + [w], pred, [e])
        if direct or d == 8:
            want = "k_filter_project<%d,0>" % d
        else:
            rowb = min(d + 1, 4) * w8(dt) + w.dtype.itemsize  # the columns the tree reads and the predicate's
            k = 8 if d <= 2 and rowb <= 16 else 4 if rowb <= 33 else 2
            want = "k_filter_project_tma<%d,%d,%d,0,0>" % (d, k, f64_pred)
        launched(names, want)
        assert_same(got[0], v[keep], (d, last, direct, f64_pred, ops))
    # depth 9 is refused
    e, _ = nested(9, "-")
    b = ctx.upload(cols)
    try:
        with pytest.raises(engine.DfGpuError) as ex:
            ctx.filter_project(b, None, [e])
        assert "expression too deep" in ex.value.msg
    finally:
        b.free()


# ---- c. predicates over arithmetic ----------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [np.int8, np.uint16, np.int32, np.uint64, F32], ids=NAME.get)
def test_predicates(ctx, dt):
    n = 50_003
    rng = np.random.default_rng(np.dtype(dt).num + 700)
    a, b = AR.operands(rng, dt, n, k=32)
    b = np.where(b == 0, np.dtype(dt).type(1), b)  # a WHERE evaluates every row: no zero divisor anywhere
    c = AR.operands(rng, dt, n, k=32)[0]
    rid = np.arange(n, dtype=np.int32)
    if np.dtype(dt) == np.int8:  # the wrapped sum flips the sign: 100 + 100 < 0
        a[:10], b[:10], c[:10] = 100, 100, 0
    if np.dtype(dt) == np.uint16:  # 0 - 1 > 0
        a[:10], b[:10], c[:10] = 0, 1, 0
    for op in AR.OPS:
        v = AR.value(op, a, b)
        fin = v[~np.isnan(v)] if AR.is_float(dt) else v
        lv = np.unique(fin)[len(np.unique(fin)) // 3]
        for name, (mk, f) in CMP.items():
            for rhs_col in (False, True):
                pred = mk(EXPR[op](col(0), col(1)), col(2) if rhs_col else L(lv, dt))
                with np.errstate(invalid="ignore"):
                    m = f(v, c if rhs_col else lv)
                for direct in (False, True):
                    e = deep(5)
                    got, names = fp(ctx, [a, b, c, rid], pred, [col(3)] + ([e] if direct else []))
                    if direct:
                        launched(names, "k_filter_project<8,0>")
                    else:
                        # predicate columns a, b (and c), projection column rid (4 bytes)
                        k = 8 if (3 if rhs_col else 2) * w8(dt) + 4 <= 16 else 4
                        launched(names, "k_filter_project_tma<2,%d,0,0,0>" % k)
                    assert np.array_equal(got[0], rid[m]), (op, name, rhs_col, direct)
    if np.dtype(dt) in (np.dtype(np.int8), np.dtype(np.uint16)):
        got, _ = fp(ctx, [a, b, c, rid], (col(0) + col(1) < col(2)) if np.dtype(dt) == np.int8 else (col(0) - col(1) > col(2)), [col(3)])
        assert set(range(10)) <= set(got[0].tolist())


# ---- d. no fused multiply-add ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [F32, F64], ids=NAME.get)
def test_no_fused_multiply_add(ctx, dt):
    n = 200_003
    rng = np.random.default_rng(np.dtype(dt).num + 800)
    p = np.finfo(dt).nmant + 1
    # a = 1 + 2^-k, b = 1 - 2^-k: a*b = 1 - 2^-2k rounds to 1 for 2k > p, so a*b - 1 is 0 with two roundings and -2^-2k
    # with one; random scales and signs keep the pairs apart, the rest are random
    k = rng.integers(p // 2 + 1, p - 1, n)
    s = rng.choice([-1.0, 1.0], n) * 2.0 ** rng.integers(-20, 20, n)
    s2 = rng.choice([-1.0, 1.0], n) * 2.0 ** rng.integers(-20, 20, n)
    a = (s * (1 + 2.0 ** -k)).astype(dt)
    b = (s2 * (1 - 2.0 ** -k)).astype(dt)
    c = (-s * s2).astype(dt)  # -round(a*b): two roundings give 0, one gives -s*s2*2^-2k
    r = rng.random(n) < 0.3
    a[r], b[r], c[r] = AR.pool(rng, dt, r.sum()), AR.pool(rng, dt, r.sum()), AR.pool(rng, dt, r.sum())
    t = rng.integers(0, 3000, n)  # 3000 distinct triples: the exact reference runs once per distinct row
    a, b, c = a[t], b[t], c[t]
    ab = AR.value("*", a, b)
    add, sub = AR.value("+", ab, c), AR.value("-", ab, -c)
    fused = np.array([float("nan") if not (math.isfinite(x) and math.isfinite(y) and math.isfinite(z)) else
                      AR.round_float(Fraction(x) * Fraction(y) + Fraction(z), dt) for x, y, z in zip(a[:2000].tolist(), b[:2000].tolist(), c[:2000].tolist())], dtype=dt)
    assert len(AR.same(fused, add[:2000])) > 500  # the test tells the two apart
    exprs = [col(0) * col(1) + col(2), col(0) * col(1) - col(3)]
    for direct in (False, True):
        got, names = fp(ctx, [a, b, c, -c], None, exprs + ([deep(5)] if direct else []))
        if direct:
            launched(names, "k_filter_project<8,0>")
        else:  # four columns: 16 bytes a row for Float32 (K = 8), 32 for Float64 (K = 4, all-Float64)
            launched(names, "k_filter_project_tma<2,8,0,0,0>" if np.dtype(dt) == F32 else "k_filter_project_tma<2,4,1,0,0>")
        assert_same(got[0], add, ("a*b + c", direct))
        assert_same(got[1], sub, ("a*b - c", direct))


# ---- e. aggregates --------------------------------------------------------------------------------------------------
def run_agg(ctx, arrays, keys, aggs, pred=None):
    b = ctx.upload(arrays)
    try:
        r = ctx.aggregate([b], keys, aggs, 0, pred=pred)
        try:
            return r.columns()
        finally:
            r.free()
    finally:
        b.free()


def agg(ctx, arrays, keys, aggs, pred=None):
    return traced(lambda: run_agg(ctx, arrays, keys, aggs, pred))


@pytest.mark.parametrize("dt", AR.INTS, ids=NAME.get)
def test_group_by_arithmetic_key(ctx, dt):
    n = 300_001
    rng = np.random.default_rng(np.dtype(dt).num + 900)
    a, b = AR.operands(rng, dt, n, k=12)
    b = np.where(b == 0, np.dtype(dt).type(1), b)
    v = rng.integers(-1000, 1000, n).astype(I64)
    spec = [R.COUNT, R.SUM, R.MIN, R.MAX]
    for op in AR.OPS:
        kv = AR.value(op, a, b)
        got, names = agg(ctx, [a, b, v], [EXPR[op](col(0), col(1))], [AggregateFunction(f, col(2)) for f in spec])
        launched(names, "k_hash_agg<1,0,0>")
        R.assert_matches(got, R.aggregate([kv], [(f, v) for f in spec]), ("key", op))
        # composite: the arithmetic key and the column a
        got, names = agg(ctx, [a, b, v], [EXPR[op](col(0), col(1)), col(0)], [AggregateFunction(f, col(2)) for f in spec])
        launched(names, "k_hash_agg<1,0,0>" if w8(dt) <= 4 else "k_hash_agg_wide<8,0>")
        R.assert_matches(got, R.aggregate([kv, a], [(f, v) for f in spec]), ("two keys", op))
        # the same with a nullable argument: the null-aware kernels
        valid = rng.random(n) > 0.25
        got, names = agg(ctx, [a, b, R.arrow_nullable(v, valid)], [EXPR[op](col(0), col(1)), col(0)], [AggregateFunction(f, col(2)) for f in spec])
        launched(names, "k_hash_agg<8,0,1>" if w8(dt) <= 4 else "k_hash_agg_wide<8,1>")
        R.assert_matches(got, R.aggregate([kv, a], [(f, (v, valid)) for f in spec]), ("two keys, nulls", op))


def check_avg(got, v, k, what):
    """AVG of an integer argument: the f64 sum of the values, each rounded to f64, over the count: within
    (count + 2) ulps of sum|v| / count, plus the division's rounding, of the exact mean."""
    if k is None:
        groups, g = [np.arange(len(v))], [float(got[0][0])]
    else:
        order = np.argsort(got[0])
        assert np.array_equal(got[0][order], np.unique(k)), what
        groups, g = [np.flatnonzero(k == u) for u in got[0][order]], got[1][order].tolist()
    for x, rows in zip(g, groups):
        vals = [int(t) for t in v[rows].tolist()]
        c = len(vals)
        mean = Fraction(sum(vals), c)
        bound = Fraction(sum(abs(t) for t in vals), c) * Fraction(c + 2, 2 ** 52) + abs(mean) / 2 ** 52
        assert abs(Fraction(x) - mean) <= bound, (what, x, float(mean))


@pytest.mark.parametrize("dt", NUMERIC, ids=NAME.get)
def test_aggregates_of_arithmetic(ctx, dt):
    # integer SUM wraps in the operand type; float SUM depends on the order of the additions (and Float32 SUM flushes
    # subnormals, DESIGN §7), so floats are checked through MIN / MAX / COUNT
    n = 300_001
    rng = np.random.default_rng(np.dtype(dt).num + 1000)
    a, b = AR.operands(rng, dt, n, k=24)
    b = np.where(b == 0, np.dtype(dt).type(1), b)
    k = rng.integers(0, 61, n).astype(np.int32)
    valid = rng.random(n) > 0.3
    spec = [R.MIN, R.MAX, R.COUNT] + ([] if AR.is_float(dt) else [R.SUM])
    for op in AR.OPS:
        v = AR.value(op, a, b)
        arg = EXPR[op](col(1), col(2))
        for keys, kv, kern in (([col(0)], [k], "k_hash_agg<1,0,0>"), ([], [], "k_reduce<1,0>")):
            got, names = agg(ctx, [k, a, b], keys, [AggregateFunction(f, arg) for f in spec])
            launched(names, kern)
            R.assert_matches(got, R.aggregate(kv, [(f, v) for f in spec]), ("aggs", op, len(keys)))
            # a nullable operand: null where it is, value 0 there (read by GROUP BY, skipped by a reduction)
            got, names = agg(ctx, [k, R.arrow_nullable(a, valid), b], keys, [AggregateFunction(f, arg) for f in spec])
            launched(names, "k_hash_agg<8,0,1>" if keys else "k_reduce<8,1>")
            R.assert_matches(got, R.aggregate(kv, [(f, (np.where(valid, v, np.zeros(1, dtype=dt)), valid)) for f in spec]), ("aggs nulls", op, len(keys)))
            if not AR.is_float(dt):
                got, _ = agg(ctx, [k, a, b], keys, [AggregateFunction("avg", arg)])
                check_avg([np.asarray(c) for c in got], v, k if keys else None, ("avg", op))
        # COUNT(DISTINCT a op b)
        got, names = agg(ctx, [k, a, b], [], [AggregateFunction("count", arg, distinct=True)])
        launched(names, "k_distinct_insert<2,0>")
        if AR.is_float(dt):
            fin = v[~np.isnan(v)]
            want = len(np.unique(np.where(fin == 0, np.dtype(dt).type(0), fin))) + int(np.isnan(v).any())
        else:
            want = len(np.unique(v))
        assert int(got[0][0]) == want, ("distinct", op)
        if not AR.is_float(dt):
            got, names = agg(ctx, [k, R.arrow_nullable(a, valid), b], [], [AggregateFunction("count", arg, distinct=True)])
            launched(names, "k_distinct_insert<8,1>")
            assert int(got[0][0]) == len(np.unique(v[valid])), ("distinct nulls", op)


@pytest.mark.parametrize("dt", [np.int8, np.uint16, I64, U64, F32, F64], ids=NAME.get)
def test_fused_where_over_arithmetic(ctx, dt):
    n = 300_001
    rng = np.random.default_rng(np.dtype(dt).num + 1100)
    a, b = AR.operands(rng, dt, n, k=24)
    b = np.where(b == 0, np.dtype(dt).type(1), b)  # the WHERE reads every row
    c = AR.operands(rng, dt, n, k=24)[0]
    k = rng.integers(0, 50, n).astype(np.int32)
    v = rng.integers(-1000, 1000, n).astype(I64)
    spec = [R.SUM, R.COUNT, R.MIN]
    for op in AR.OPS:
        with np.errstate(invalid="ignore"):
            m = AR.value(op, a, b) > c
        pred = EXPR[op](col(1), col(2)) > col(3)
        got, names = agg(ctx, [k, a, b, c, v], [col(0)], [AggregateFunction(f, col(4)) for f in spec], pred=pred)
        launched(names, "k_hash_agg<1,0,0>")
        R.assert_matches(got, R.aggregate([k[m]], [(f, v[m]) for f in spec]), ("where", op))
        got, names = agg(ctx, [k, a, b, c, v], [], [AggregateFunction(f, col(4)) for f in spec], pred=pred)
        launched(names, "k_reduce<1,0>")
        R.assert_matches(got, R.aggregate([], [(f, v[m]) for f in spec]), ("reduce where", op))


# ---- f. join keys ---------------------------------------------------------------------------------------------------
def run_join(ctx, build, bkeys, probe, pkeys):
    """(probe row, build row) of every match of probe keys pkeys against build keys bkeys."""
    pb = ctx.upload(probe + [np.arange(len(probe[0]), dtype=I64)])
    try:
        bb = ctx.upload(build + [np.arange(len(build[0]), dtype=I64)])
        try:
            j = ctx.join_build(bb, bkeys, keep_cols=[len(build)])
            try:
                r = j.probe(pb, pkeys, probe_cols=[len(probe)], build_cols=[len(build)])
                try:
                    return r.columns()
                finally:
                    r.free()
            finally:
                j.free()
        finally:
            bb.free()
    finally:
        pb.free()


def join(ctx, build, bkeys, probe, pkeys):
    return traced(lambda: run_join(ctx, build, bkeys, probe, pkeys))


def key_kernel(dt, leaf):
    """The filter/project instantiation that evaluates a join key of dtype dt over at most 16 bytes a row: the FAST
    leaf loop for a 64-bit `a + b` / `a * lit` (leaf), the interpreter otherwise (narrow types, integer division)."""
    return "k_filter_project_tma<1,8,0,1,0>" if leaf and w8(dt) == 8 else "k_filter_project_tma<2,8,0,0,0>"


@pytest.mark.parametrize("dt", [np.int8, np.uint8, np.int16, np.int32, np.uint32, I64, U64], ids=NAME.get)
def test_join_arithmetic_keys(ctx, dt):
    rng = np.random.default_rng(np.dtype(dt).num + 1200)
    lo, hi = AR.int_bounds(dt)
    ba, bb = AR.operands(rng, dt, 3000, k=20)
    pa, pb = AR.operands(rng, dt, 50_003, k=20)
    lv = np.dtype(dt).type(lits(dt)["*"])
    bk = AR.value("+", ba, bb)
    for pkey, pv in ((col(0) + col(1), AR.value("+", pa, pb)), (col(0) * L(lv, dt), AR.value("*", pa, lv))):
        got, names = join(ctx, [ba, bb], [col(0) + col(1)], [pa, pb], [pkey])
        for want in (key_kernel(dt, True), "k_join_build", "k_join_count", "k_join_emit"):
            launched(names, want)
        pos = {}
        for j, x in enumerate(bk.tolist()):
            pos.setdefault(x, []).append(j)
        exp = sorted((i, j) for i, x in enumerate(pv.tolist()) for j in pos.get(x, []))
        assert sorted(zip(got[0].tolist(), got[1].tolist())) == exp
    # keys equal only after wrapping: MAX + 1 on the build side meets MIN + 0 on the probe side
    got, _ = join(ctx, [np.array([hi], dtype=dt), np.array([1], dtype=dt)], [col(0) + col(1)],
                  [np.array([lo, 0], dtype=dt), np.array([0, 1], dtype=dt)], [col(0) + col(1)])
    assert got[0].tolist() == [0] and got[1].tolist() == [0]


# ---- g. DivideByZero ------------------------------------------------------------------------------------------------
def dbz_sites(dt):
    """(context, projections, name) of the filter/project sites that divide: (kernel with the UInt8 / Float32 / 8-byte
    WHERE of the site, kernel without a WHERE)."""
    w, f64 = w8(dt), int(np.dtype(dt) == F64)
    sites = [("ctx", [col(0) / col(1), col(0) + L(1, dt), L(2, dt) - col(0)], "u8",
              "k_filter_project_tma<2,%d,0,0,0>" % (8 if 2 * w + 1 <= 16 else 4), "k_filter_project_tma<2,8,%d,0,0>" % f64),
             ("dctx", [col(0) / col(1)], "u8", "k_filter_project<1,0>", "k_filter_project<1,0>"),
             ("ctx", [col(0) / col(1), deep(5)], "u8", "k_filter_project<8,0>", "k_filter_project<8,0>")]
    if AR.is_float(dt):  # every projection a leaf: the FAST loop
        sites.append(("ctx", [col(0) / col(1), col(0) - col(1), col(0) * col(1)], "f32",
                      "k_filter_project_tma<1,%d,0,1,0>" % (8 if 2 * w + 4 <= 16 else 4), "k_filter_project_tma<1,8,%d,1,0>" % f64))
    if f64:  # one Float64 comparison and one division: the lean loop
        sites.append(("ctx", [col(0) / col(1)], "same", "k_filter_project_tma<1,4,1,1,1>", "k_filter_project_tma<1,8,1,1,0>"))
    return sites


@pytest.mark.parametrize("dt", NUMERIC, ids=NAME.get)
def test_divide_by_zero(ctx, dctx, dt):
    n = 100_003
    rng = np.random.default_rng(np.dtype(dt).num + 1300)
    t = np.dtype(dt).type
    zeros = [t(0.0), t(-0.0)] if AR.is_float(dt) else [t(0)]
    a = AR.pool(rng, dt, n)
    z_row = n // 2 + 7
    ctxs = {"ctx": ctx, "dctx": dctx}
    u8 = col(2) < lit(1, A.UINT8)
    for z in zeros:
        b = np.full(n, t(3), dtype=dt)
        b[z_row] = z  # one zero divisor
        drop = np.zeros(n, dtype=bool)
        drop[z_row] = True
        for c, proj, where, kern, kern_nowhere in dbz_sites(dt):
            c = ctxs[c]
            # a WHERE column that keeps every row but `drop`'s, or every row
            if where == "u8":
                pred, wcol = u8, lambda m: m.astype(U8)
            elif where == "f32":
                pred, wcol = col(2) > lit(0.5, A.FLOAT32), lambda m: np.where(m, 0, 1).astype(F32)
            else:
                pred, wcol = col(2) > L(0, dt), lambda m: np.where(m, -1, 1).astype(dt)
            # the zero survives the WHERE: raised
            raises_dbz(lambda: run_fp(c, [a, b, wcol(np.zeros(n, dtype=bool))], pred, proj), kern)
            # the zero is dropped: no error
            got, names = fp(c, [a, b, wcol(drop)], pred, proj)
            launched(names, kern)
            assert len(got[0]) == n - 1
            # no WHERE: raised
            raises_dbz(lambda: run_fp(c, [a, b], None, proj), kern_nowhere)
        # nulls: without a WHERE a zero under a null does not raise, and does in a non-null row
        vb, va = ~drop, np.arange(n) != 3
        got, names = fp(ctx, [a, R.arrow_nullable(b, vb)], None, [col(0) / col(1)])
        launched(names, "k_filter_project<8,1>")
        assert not got[0][1][z_row]
        raises_dbz(lambda: run_fp(ctx, [R.arrow_nullable(a, va), b], None, [col(0) / col(1)]), "k_filter_project<8,1>")
        # with a WHERE the surviving null slot's zero is a value like any other: raised; dropped: not raised
        raises_dbz(lambda: run_fp(ctx, [a, R.arrow_nullable(b, vb), np.zeros(n, dtype=U8)], u8, [col(0) / col(1)]), "k_filter_project<8,1>")
        got, names = fp(ctx, [a, R.arrow_nullable(b, vb), drop.astype(U8)], u8, [col(0) / col(1)])
        launched(names, "k_filter_project<8,1>")
        # a WHERE reads every row: a zero divisor in the predicate raises even where the row is dropped
        rowb = 2 * w8(dt) + 1 + w8(dt)  # predicate columns a, b, w; projection column a
        raises_dbz(lambda: run_fp(ctx, [a, b, drop.astype(U8)], (col(0) / col(1) > L(0, dt)) & u8, [col(0)]),
                   "k_filter_project_tma<2,%d,0,0,0>" % (8 if rowb <= 16 else 4))
        # aggregates: the argument (grouped and reduce), the fused WHERE, COUNT(DISTINCT), then a nullable divisor
        kcol = (np.arange(n) % 7).astype(np.int32)
        mx = [AggregateFunction("max", col(0) / col(1))]
        for keys, kern, kern_n, kern_d in (([col(3)], "k_hash_agg<1,0,0>", "k_hash_agg<8,0,1>", "k_distinct_insert<2,0>"),
                                           ([], "k_reduce<1,0>", "k_reduce<8,1>", "k_distinct_insert<2,0>")):
            raises_dbz(lambda: run_agg(ctx, [a, b, drop.astype(U8), kcol], keys, mx), kern)
            got, names = agg(ctx, [a, b, drop.astype(U8), kcol], keys, mx, pred=u8)
            launched(names, kern)
            raises_dbz(lambda: run_agg(ctx, [a, b, np.zeros(n, dtype=U8), kcol], keys, mx, pred=u8), kern)
            raises_dbz(lambda: run_agg(ctx, [a, b, drop.astype(U8), kcol], keys, [AggregateFunction("count", col(0))],
                                       pred=col(0) / col(1) > L(0, dt)), kern)
            raises_dbz(lambda: run_agg(ctx, [a, b, drop.astype(U8), kcol], keys, [AggregateFunction("count", col(0) / col(1), distinct=True)]),
                       kern_d)
            # a nullable divisor: a zero under a null does not raise without a WHERE, does under one
            got, names = agg(ctx, [a, R.arrow_nullable(b, vb), drop.astype(U8), kcol], keys, mx)
            launched(names, kern_n)
            raises_dbz(lambda: run_agg(ctx, [a, R.arrow_nullable(b, vb), np.zeros(n, dtype=U8), kcol], keys, mx, pred=u8), kern_n)
        if not AR.is_float(dt):
            # an integer GROUP BY key
            raises_dbz(lambda: run_agg(ctx, [a, b], [col(0) / col(1)], [AggregateFunction("count", col(0))]), "k_hash_agg<1,0,0>")
            got, names = agg(ctx, [a, b, drop.astype(U8)], [col(0) / col(1)], [AggregateFunction("count", col(0))], pred=u8)
            launched(names, "k_hash_agg<1,0,0>")
            # join keys, build and probe side (integer division is never a leaf: the interpreter)
            small = [a[:5].copy(), np.full(5, t(1), dtype=dt)]
            raises_dbz(lambda: run_join(ctx, [a, b], [col(0) / col(1)], small, [col(0)]), key_kernel(dt, False))
            raises_dbz(lambda: run_join(ctx, small, [col(0)], [a, b], [col(0) / col(1)]), key_kernel(dt, False))
            got, names = join(ctx, [a, np.full(n, t(1), dtype=dt)], [col(0) / col(1)], small, [col(0) / col(1)])
            launched(names, key_kernel(dt, False))
            assert len(got[0]) >= 5


# ---- h. SQL ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def typed():
    rng = np.random.default_rng(14)
    n = 20_011
    cols = {}
    for d in NUMERIC:
        a = AR.operands(rng, d, n, k=40)[0]
        cols["c_" + NAME[np.dtype(d)]] = np.where(a == 0, np.dtype(d).type(1), a)  # a divisor everywhere
    hctx = host.ExecutionContext(0)
    yield hctx, cols
    hctx.close()


def one_col(hctx, cols, sql):
    bs = sql_batches(hctx, {"t": cols}, sql)
    return np.concatenate([np.asarray(b[0]) for b in bs]) if bs else None


@pytest.mark.parametrize("src", NUMERIC, ids=NAME.get)
def test_sql_arithmetic(typed, src):
    hctx, cols = typed
    name = "c_" + NAME[np.dtype(src)]
    x = cols[name]
    planned = 0
    for litx in ("3", "-7", "0.5", "-0.1"):
        is_f = "." in litx or "e" in litx
        st = CR.DTYPE[host.supertype(code(src), A.FLOAT64 if is_f else A.INT64)]
        lv = float(litx) if is_f else int(litx)
        for op in AR.OPS:
            for sql, left in (("%s %s %s" % (name, op, litx), True), ("%s %s %s" % (litx, op, name), False),
                              ("(%s %s %s) %s %s" % (name, op, litx, op, name), None)):
                q = "SELECT %s FROM t" % sql
                if not CR.can_coerce_from(st, src) or (not is_f and st == np.dtype(F32)):
                    with pytest.raises(host.ExecutionError):
                        one_col(hctx, cols, q)
                    continue
                cx = CR.cast(x, st) if np.dtype(st) != x.dtype else x
                lc = np.dtype(st).type(CR.cast(np.array([lv], dtype=F64 if is_f else I64), st)[0])
                if left is None:
                    ref = AR.arith(op, AR.arith(op, cx, lc)[0], cx)
                else:
                    ref = AR.arith(op, cx, lc) if left else AR.arith(op, lc, cx)
                if ref[1].any():
                    with pytest.raises(host.ExecutionError) as e:
                        one_col(hctx, cols, q)
                    assert "DivideByZero" in e.value.msg
                    continue
                assert_same(one_col(hctx, cols, q), ref[0], (q,))
                planned += 1
    assert planned > 0
    # INT64_MIN, computed
    assert one_col(hctx, cols, "SELECT c_int64 - c_int64 + (-9223372036854775807 - 1) FROM t").tolist() == [-(2 ** 63)] * len(x)
    assert one_col(hctx, cols, "SELECT (-9223372036854775807 - 1) / -1 + c_int64 * 0 FROM t").tolist() == [-(2 ** 63)] * len(x)
