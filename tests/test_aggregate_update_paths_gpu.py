"""Host-side rules of the aggregate operator that no kernel test reaches: how the first batch types the operator, the
checks on later batches, the order of the ABI calls, and the Utf8-key aggregate limit.  Each case asserts the error
code and message a caller sees."""
import numpy as np
import pytest

from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import engine
from datafusion_archive_b200.expr import AggregateFunction, col

pytestmark = pytest.mark.gpu

KEY_TYPES_CHANGED = "GROUP BY key types changed between batches"
ALREADY_FINISHED = "aggregate already finished"


@pytest.fixture(scope="module")
def ctx():
    c = engine.GpuContext(0)
    yield c
    c.close()


class Agg:
    """One aggregate operator driven call by call through the C ABI."""

    def __init__(self, ctx, schema, keys, aggs, expected_groups=0):
        self.ctx, self.keep = ctx, []
        kptrs, klens, nk = A.make_programs([k.program(schema) for k in keys], self.keep)
        aggarr = A.make_aggs([a.lower(schema) for a in aggs], self.keep)
        self.schema, self.st = schema, engine.C.c_void_p()
        engine.check(engine.lib().dfgpu_aggregate_create(ctx.h, kptrs, klens, nk, aggarr, len(aggs), expected_groups,
                                                         engine.C.byref(self.st)))

    def set_predicate(self, pred):
        prog = pred.program(self.schema)
        engine.check(engine.lib().dfgpu_aggregate_set_predicate(self.st, (A.Insn * len(prog))(*prog), len(prog)))

    def update(self, arrays):
        b = self.ctx.upload(arrays)
        try:
            engine.check(engine.lib().dfgpu_aggregate_update(self.st, b.h))
        finally:
            b.free()

    def finish(self):
        out = engine.C.c_void_p()
        engine.check(engine.lib().dfgpu_aggregate_finish(self.st, engine.C.byref(out)))
        r = engine.Result(self.ctx, out)
        try:
            return r.columns()
        finally:
            r.free()

    def free(self):
        engine.lib().dfgpu_aggregate_free(self.st)


def dtypes(arrays):
    return [A.UTF8 if isinstance(a, list) else A.DTYPE_OF_NP[np.asarray(a).dtype] for a in arrays]


def expect_error(code, msg, fn, *args):
    with pytest.raises(engine.DfGpuError) as e:
        fn(*args)
    assert e.value.code == code and msg in e.value.msg, (e.value.code, e.value.msg)


def run(ctx, batches, keys, aggs):
    a = Agg(ctx, dtypes(batches[0]), keys, aggs)
    try:
        for b in batches:
            a.update(b)
        return a.finish()
    finally:
        a.free()


def i64(*v):
    return np.array(v, dtype=np.int64)


def f64(*v):
    return np.array(v, dtype=np.float64)


# (first batch, second batch, GROUP BY): the second batch's key columns have other types than the first's
KEY_CHANGES = {
    "narrow": ([i64(1, 2), f64(1, 2)], [np.array([1, 2], np.int32), f64(1, 2)], [col(0)]),
    "utf8_then_int": ([["a", "b"], f64(1, 2)], [i64(1, 2), f64(1, 2)], [col(0)]),
    "int_then_utf8": ([i64(1, 2), f64(1, 2)], [["a", "b"], f64(1, 2)], [col(0)]),
    "wide": ([i64(1, 2), i64(3, 4), f64(1, 2)], [i64(1, 2), np.array([3, 4], np.int32), f64(1, 2)], [col(0), col(1)]),
    "wide_utf8_part": ([["a", "b"], np.array([3, 4], np.int32), f64(1, 2)], [i64(1, 2), np.array([3, 4], np.int32), f64(1, 2)],
                       [col(0), col(1)]),
}


@pytest.mark.parametrize("case", sorted(KEY_CHANGES))
def test_key_types_changed_between_batches(ctx, case):
    first, second, keys = KEY_CHANGES[case]
    a = Agg(ctx, dtypes(first), keys, [AggregateFunction("sum", col(len(first) - 1))])
    try:
        a.update(first)
        expect_error(A.ERR_GENERAL, KEY_TYPES_CHANGED, a.update, second)
    finally:
        a.free()


@pytest.mark.parametrize("nkeys", [0, 1])
def test_argument_types_changed_between_batches(ctx, nkeys):
    # COUNT: its output type is UInt64 whatever the argument, so only the argument type check can fire
    keys = [col(0)] * nkeys
    a = Agg(ctx, [A.INT64, A.FLOAT64], keys, [AggregateFunction("count", col(1))])
    try:
        a.update([i64(1, 2), f64(1, 2)])
        expect_error(A.ERR_GENERAL, "aggregate argument types changed between batches", a.update, [i64(1, 2), i64(1, 2)])
    finally:
        a.free()


@pytest.mark.parametrize("first_rows", [0, 2])
def test_predicate_after_first_batch(ctx, first_rows):
    # a zero-row batch already types the operator, so it too closes the predicate
    a = Agg(ctx, [A.INT64, A.FLOAT64], [col(0)], [AggregateFunction("sum", col(1))])
    try:
        a.update([i64(*range(first_rows)), f64(*range(first_rows))])
        expect_error(A.ERR_GENERAL, "the predicate must be set before the first batch", a.set_predicate, col(1) > 0.5)
    finally:
        a.free()


def test_finish_is_one_shot(ctx):
    a = Agg(ctx, [A.INT64, A.FLOAT64], [col(0)], [AggregateFunction("sum", col(1))])
    try:
        a.update([i64(1, 1, 2), f64(1, 2, 3)])
        k, s = a.finish()
        assert sorted(zip(k.tolist(), s.tolist())) == [(1, 3.0), (2, 3.0)]
        expect_error(A.ERR_GENERAL, ALREADY_FINISHED, a.finish)
        expect_error(A.ERR_GENERAL, ALREADY_FINISHED, a.update, [i64(1), f64(1)])
    finally:
        a.free()


def test_finish_group_by_without_batch(ctx):
    a = Agg(ctx, [A.INT64, A.FLOAT64], [col(0)], [AggregateFunction("sum", col(1))])
    try:
        expect_error(A.ERR_GENERAL, "aggregate finished before any input batch was provided", a.finish)
    finally:
        a.free()


def test_finish_reduce_without_batch_or_output_type(ctx):
    a = Agg(ctx, [A.FLOAT64], [], [AggregateFunction("sum", col(0), return_type=0)])
    try:
        expect_error(A.ERR_GENERAL, "aggregate output type must be given when there is no input", a.finish)
    finally:
        a.free()


@pytest.mark.parametrize("nkeys", [0, 1, 2])
def test_zero_row_first_batch_types_the_aggregate(ctx, nkeys):
    keys = [col(k) for k in range(nkeys)]
    aggs = [AggregateFunction("sum", col(nkeys)), AggregateFunction("min", col(nkeys)), AggregateFunction("count", col(nkeys))]
    empty = [i64() for _ in range(nkeys)] + [f64()]
    data = [i64(3, 1, 3, 1) for _ in range(nkeys)] + [f64(1.5, 2.0, -4.0, 8.0)]
    got = run(ctx, [empty, data], keys, aggs)
    exp = run(ctx, [data], keys, aggs)
    order_got, order_exp = np.argsort(got[0]), np.argsort(exp[0])
    for g, e in zip(got, exp):
        assert np.array_equal(np.asarray(g)[order_got], np.asarray(e)[order_exp])
    if nkeys:
        # the empty batch fixed the key types: a later batch of other key types is refused
        a = Agg(ctx, dtypes(empty), keys, aggs)
        try:
            a.update(empty)
            other = [np.array([1, 2], np.int32) for _ in range(nkeys)] + [f64(1, 2)]
            expect_error(A.ERR_GENERAL, KEY_TYPES_CHANGED, a.update, other)
        finally:
            a.free()


@pytest.mark.parametrize("naggs", [7, 8])
def test_utf8_key_aggregate_limit(ctx, naggs):
    # a single Utf8 key holds one hidden aggregate (the representative row of each group), so it leaves room for
    # one aggregate less than the operator's limit of 8
    keys = ["x", "y", "x", "z", "y", "x"]
    v = f64(1, 2, 3, 4, 5, 6)
    funcs = ["sum", "min", "max", "count"]
    aggs = [AggregateFunction(funcs[i % 4], col(1)) for i in range(naggs)]
    if naggs == 8:
        a = Agg(ctx, [A.UTF8, A.FLOAT64], [col(0)], aggs)
        try:
            expect_error(A.ERR_NOT_IMPLEMENTED, "Utf8 GROUP BY key with 8 aggregates", a.update, [keys, v])
        finally:
            a.free()
        return
    got = run(ctx, [[keys, v]], [col(0)], aggs)
    rows = sorted(zip(*[c if isinstance(c, list) else c.tolist() for c in got]))
    want = {"sum": {"x": 10.0, "y": 7.0, "z": 4.0}, "min": {"x": 1.0, "y": 2.0, "z": 4.0},
            "max": {"x": 6.0, "y": 5.0, "z": 4.0}, "count": {"x": 3, "y": 2, "z": 1}}
    assert rows == [(k,) + tuple(want[funcs[i % 4]][k] for i in range(naggs)) for k in ["x", "y", "z"]]
