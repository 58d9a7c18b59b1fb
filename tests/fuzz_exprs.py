"""Random expression trees obeying the reference's typing rules (identical operand dtypes for math /
compare, boolean operands for And / Or), for GPU-vs-oracle fuzzing."""
import numpy as np

from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200.expr import AggregateFunction, BinaryExpr, Case, Literal, col, fn, lit, utf8_fn

MATH = [A.OP_ADD, A.OP_SUB, A.OP_MUL, A.OP_DIV]
CMP = [A.OP_EQ, A.OP_NE, A.OP_LT, A.OP_LE, A.OP_GT, A.OP_GE]


def gen_numeric(rng, schema, dtype, depth):
    """Expression of type `dtype`."""
    cols = [i for i, d in enumerate(schema) if d == dtype]
    if depth <= 0 or rng.random() < 0.3:
        if cols and rng.random() < 0.75:
            return col(int(rng.choice(cols)))
        if dtype in (A.FLOAT64, A.FLOAT32):
            return lit(float(np.round(rng.random() * 4 - 2, 3)) or 0.5, dtype)
        return lit(int(rng.integers(-5, 6)) or 3, dtype)
    op = int(rng.choice(MATH if dtype in (A.FLOAT64, A.FLOAT32) else MATH[:3]))  # integer division: zero divisors are data dependent
    left = gen_numeric(rng, schema, dtype, depth - 1)
    right = gen_numeric(rng, schema, dtype, depth - 1)
    if op == A.OP_DIV:
        right = lit(float(rng.choice([0.5, 2.0, -3.0, 7.25])), dtype)  # never a zero divisor
    return BinaryExpr(left, op, right)


def gen_bool(rng, schema, depth):
    if depth <= 0 or rng.random() < 0.45:
        dtype = int(rng.choice(sorted(set(schema))))
        return BinaryExpr(gen_numeric(rng, schema, dtype, max(0, depth - 1)), int(rng.choice(CMP)), gen_numeric(rng, schema, dtype, max(0, depth - 1)))
    return BinaryExpr(gen_bool(rng, schema, depth - 1), int(rng.choice([A.OP_AND, A.OP_OR])), gen_bool(rng, schema, depth - 1))


def gen_query(rng, schema, max_depth=3, has_literal_only_ok=False):
    pred = gen_bool(rng, schema, int(rng.integers(0, max_depth + 1))) if rng.random() < 0.85 else None
    nproj = int(rng.integers(1, 4))
    proj = []
    for _ in range(nproj):
        dtype = int(rng.choice(sorted(set(schema))))
        e = gen_numeric(rng, schema, dtype, int(rng.integers(0, max_depth + 1)))
        proj.append(e)
    return pred, proj


def references_column(e):
    from datafusion_archive_b200.expr import Column, Cast, ScalarFunction, Utf8Function
    if isinstance(e, Column):
        return True
    if isinstance(e, BinaryExpr):
        return references_column(e.left) or references_column(e.right)
    if isinstance(e, Cast):
        return references_column(e.expr)
    if isinstance(e, (ScalarFunction, Utf8Function)):
        return any(references_column(a) for a in e.args)
    if isinstance(e, Case):
        return any(references_column(x) for w in e.whens for x in w) or (e.else_ is not None and references_column(e.else_))
    return False


# ---- nullable tables over all ten numeric dtypes and Boolean columns ---------------------------------------------
# gen_table writes every column with pa.Array.from_buffers over our own buffers and puts deliberate garbage under
# each null slot (type extremes, NaN, -0.0, infinities; bit 1 under a Boolean null), so that a kernel that reads 0
# there, skips the row, or reads the hidden value gives a different answer each way.  Integer division is the one
# operation that can fail: its divisors are plain columns made for it ("safe": zeros only under nulls; "gated": every
# zero, null or not, in a row where the gate column is 0) or nonzero literals, and never -1, so MIN / -1 cannot occur.
NUMERIC = [A.INT8, A.INT16, A.INT32, A.INT64, A.UINT8, A.UINT16, A.UINT32, A.UINT64, A.FLOAT32, A.FLOAT64]
FLOATS = (A.FLOAT32, A.FLOAT64)
PROFILES = ("bitmap", "nulls", "allnull", "nobitmap")  # null fraction 0 with a bitmap, ~30 %, all null, no bitmap


def garbage(dtype):
    """Values written under null slots (Float32: no subnormal, and sums of them cannot overflow at the test sizes)."""
    if dtype == A.FLOAT64:
        return np.array([np.nan, -0.0, np.inf, -np.inf, 1e200, -1e200], dtype=np.float64)
    if dtype == A.FLOAT32:
        return np.array([np.nan, -0.0, np.inf, -np.inf, 1e15, -1e15], dtype=np.float32)
    info = np.iinfo(A.NP_OF[dtype])
    return np.array(sorted({info.min, info.max, info.max - 1, info.min + 1 if info.min else 7}), dtype=A.NP_OF[dtype])


def _values(rng, dtype, n, divisor):
    """Valid-slot values: small magnitudes with a few type extremes; Float32 clear of subnormals; a divisor column
    never holds 0 or -1."""
    npd = A.NP_OF[dtype]
    if dtype in FLOATS:
        v = (rng.random(n) * 3.75 + 0.25) * rng.choice([-1.0, 1.0], n)
        if not divisor:
            v[rng.random(n) < 0.02] = -0.0
        return v.astype(npd)
    info = np.iinfo(npd)
    lo = max(info.min, -20)
    v = rng.integers(lo, 21, n, dtype=np.int64).astype(npd)
    edge = rng.random(n) < 0.01
    v[edge] = rng.choice(garbage(dtype), int(edge.sum()))
    if divisor:
        v[(v == 0) | ((v == -1) if info.min < 0 else False)] = 3
    return v


def column(values, valid):
    """Arrow array over our buffers; valid=None: no bitmap.  Boolean values are packed LSB first."""
    import pyarrow as pa
    n = len(values)
    bits = None if valid is None else pa.py_buffer(np.packbits(np.asarray(valid, dtype=bool), bitorder="little").tobytes())
    if values.dtype == np.bool_:
        return pa.Array.from_buffers(pa.bool_(), n, [bits, pa.py_buffer(np.packbits(values, bitorder="little").tobytes())])
    return pa.Array.from_buffers(pa.from_numpy_dtype(values.dtype), n, [bits, pa.py_buffer(np.ascontiguousarray(values).tobytes())])


def validity(rng, n, profile):
    if profile == "nobitmap":
        return None
    if profile == "bitmap":
        return np.ones(n, dtype=bool)
    if profile == "allnull":
        return np.zeros(n, dtype=bool)
    return rng.random(n) >= 0.3


class Table:
    """Columns (pyarrow arrays) with their roles.  dtype[i]: the column's dtype code; valid[i]: its validity (None: no
    bitmap); hidden[i]: its raw values.  gate: an Int32 column of 0 / 1 without nulls; a WHERE of a generated query
    is `gate > 0 AND ...`, so the rows with gate 0 are the ones every WHERE drops.  safe[d] / gated[d]: the divisor
    columns of dtype d."""

    def __init__(self):
        self.arrays, self.dtype, self.valid, self.hidden, self.profile = [], [], [], [], []
        self.values, self.bools, self.safe, self.gated, self.gate, self.utf8 = {}, [], {}, {}, None, []

    def add(self, values, valid, profile):
        self.arrays.append(column(values, valid))
        self.dtype.append(A.BOOL if values.dtype == np.bool_ else A.DTYPE_OF_NP[values.dtype])
        self.valid.append(valid)
        self.hidden.append(values)
        self.profile.append(profile)
        return len(self.arrays) - 1


def gen_table(rng, n, profiles=None, gate_frac=0.8, surviving_zero=False, dtypes=NUMERIC):
    """A table of n rows: the gate, per dtype a value column, a safe and a gated divisor column, and two Boolean
    columns.  profiles: a profile for every nullable column (default: random).  surviving_zero: also put zeros under
    the nulls of the safe divisors in rows that pass the gate (a WHERE evaluates its keys and arguments as over
    bitmap-free arrays, so such a row must raise DivideByZero)."""
    pick = (lambda: profiles) if isinstance(profiles, str) else (lambda: PROFILES[int(rng.integers(0, len(PROFILES)))] if profiles is None else profiles)
    t = Table()
    gate = (rng.random(n) < gate_frac).astype(np.int32)
    t.gate = t.add(gate, None, "nobitmap")
    for d in dtypes:
        g = garbage(d)
        for role in ("values", "safe", "gated"):
            prof = pick()
            valid = validity(rng, n, prof)
            v = _values(rng, d, n, role != "values")
            nulls = np.zeros(n, dtype=bool) if valid is None else ~valid
            hidden = g[rng.integers(0, len(g), n)]
            if role != "values":  # a divisor's zeros are placed below, and it never holds -1
                hidden = np.where((hidden == -1) | (hidden == 0), hidden.dtype.type(7), hidden)
            v = np.where(nulls, hidden, v).astype(A.NP_OF[d])
            if role == "safe":
                zero = nulls & (rng.random(n) < 0.5) & ((gate == 0) | surviving_zero)
                v[zero] = 0
            elif role == "gated":
                zero = (gate == 0) & (rng.random(n) < 0.5)
                v[zero] = 0
            i = t.add(v, valid, prof)
            getattr(t, role)[d] = i
    for _ in range(2):
        prof = pick()
        valid = validity(rng, n, prof)
        v = rng.random(n) < 0.5
        if valid is not None:
            v[~valid] = True  # hidden bit 1 under every null
        t.bools.append(t.add(v, valid, prof))
    return t


def _cap(e):
    """(instructions, tree depth) of an expression."""
    from datafusion_archive_b200.expr import Cast
    if isinstance(e, BinaryExpr):
        (a, da), (b, db) = _cap(e.left), _cap(e.right)
        return a + b + 1, 1 + max(da, db)
    if isinstance(e, Cast):
        a, d = _cap(e.expr)
        return a + 1, d + 1
    return 1, 0


def add_strings(rng, t, n, k=2):
    """k nullable Utf8 columns of utf8_fn_ref.random_strings (multi-byte and invalid bytes, spaces at either end, '')
    with a `\\0` put into about one string in twenty, appended to the table; returns their indices."""
    import pyarrow as pa
    import utf8_fn_ref
    out = []
    for _ in range(k):
        vals = utf8_fn_ref.random_strings(n, int(rng.integers(0, 1 << 30)), null_frac=0.15)
        zero = rng.random(n) < 0.05
        vals = [v if v is None or not z else v[:len(v) // 2] + b"\0" + v[len(v) // 2:] for v, z in zip(vals, zero)]
        t.arrays.append(pa.array(vals, type=pa.binary()))
        t.dtype.append(A.UTF8)
        t.valid.append(np.array([v is not None for v in vals]))
        t.hidden.append(vals)
        t.profile.append("nulls")
        t.utf8.append(len(t.arrays) - 1)
        out.append(len(t.arrays) - 1)
    return out


# The full language (QueryGen(full=True)): every node kind, typed as the C ABI types it (it casts nothing).
FULL_KINDS = ("case", "fn", "cast", "utf8_cmp", "like", "utf8_fn", "length", "transcendental", "guarded_div", "unguarded_div")
EXACT_FNS = ["sqrt", "abs", "floor", "ceil", "trunc", "round", "signum"]
TRANSCENDENTAL = ["exp", "ln", "log2", "log10", "sin", "cos", "tan", "asin", "acos", "atan", "power", "atan2"]
LIKE_PATTERNS = [b"%", b"a%", b"%a", b"%a%", b"_", b"__%", b"%_", b"Hello%", b"%\xc3\xa9%", b"_\xf0\x9f\x98\x80%", b"%  ", b" %",
                 b"%0123%", b"a_c", b"", b"%\0%"]
UTF8_LITERALS = [b"", b"a", b"Hello", b"abc", b" ", b"\xc3\xa9", b"Z", b"\0", b"\xff"]


class QueryGen:
    """Random expressions over a Table, typed as the reference types them (identical operand dtypes, Boolean operands
    of And / Or), with CAST only where the oracle implements it: a column to Int16 / Int32, an Int64 literal to
    Float64.  `cols`: the columns a query may read (the engine reads at most 12 distinct columns per query).

    full=True: the whole language, typed as the C ABI requires: CASE (1-4 WHENs, with and without ELSE, nested, as a
    value and as a Boolean), the exact scalar functions at any depth over Float64 (other dtypes cast to it), CASTs
    between every numeric dtype, Utf8 comparisons and LIKE over Utf8 columns and nests of upper / lower / trim /
    substr (Int64 literal bounds), length / octet_length as Int64 leaves, and divisions guarded by a CASE over their
    zero divisor beside a share of unguarded ones.  `seen` collects the node kinds made."""

    def __init__(self, rng, table, cols, max_depth=8, full=False):
        self.rng, self.t, self.max_depth, self.full = rng, table, max_depth, full
        self.cols = set(cols)
        self.divisor_role = "safe"
        self.seen = set()

    def _lit(self, d, nonzero=False):
        r = self.rng
        if d in FLOATS:
            return lit(float(r.choice([0.5, 2.0, -3.0, 7.25, 1.5])), d)
        lo = 0 if d in (A.UINT8, A.UINT16, A.UINT32, A.UINT64) else -5
        x = int(r.integers(lo, 6))
        if nonzero and x in (0, -1):
            x = 3
        return lit(x, d)

    def _leaf(self, d):
        r = self.rng
        if d in (A.INT16, A.INT32) and r.random() < 0.2:  # CAST(column AS Int16 / Int32) from any numeric column
            src = [c for c in self.cols if self.t.dtype[c] in NUMERIC]
            if src:
                return col(int(r.choice(sorted(src)))).cast(d)
        if d == A.FLOAT64 and r.random() < 0.1:
            return lit(int(r.integers(-5, 6)), A.INT64).cast(A.FLOAT64)
        own = [c for c in self.cols if self.t.dtype[c] == d and c != self.t.gate]
        if own and r.random() < 0.8:
            return col(int(r.choice(sorted(own))))
        return self._lit(d)

    # ---- the full language ----------------------------------------------------------------------------------------
    def _utf8_cols(self):
        return sorted(c for c in self.cols if self.t.dtype[c] == A.UTF8)

    def utf8(self, depth):
        """A Utf8 column or a nest of upper / lower / trim / ltrim / rtrim / substr over one."""
        r = self.rng
        if depth <= 0 or r.random() < 0.4:
            return col(int(r.choice(self._utf8_cols())))
        self.seen.add("utf8_fn")
        name = str(r.choice(["upper", "lower", "trim", "ltrim", "rtrim", "substr", "substr"]))
        inner = self.utf8(depth - 1)
        if name != "substr":
            return utf8_fn(name, inner)
        start = lit(int(r.choice([-3, -1, 0, 1, 2, 3, 5])), A.INT64)
        if r.random() < 0.4:
            return utf8_fn("substr", inner, start)
        return utf8_fn("substr", inner, start, lit(int(r.choice([0, 1, 2, 4, 9])), A.INT64))

    def utf8_predicate(self):
        r = self.rng
        s = self.utf8(int(r.integers(0, 4)))
        if r.random() < 0.4:
            self.seen.add("like")
            return BinaryExpr(s, int(r.choice([A.OP_LIKE, A.OP_NOT_LIKE])), lit(bytes(r.choice(LIKE_PATTERNS)), A.UTF8))
        self.seen.add("utf8_cmp")
        op = int(r.choice(CMP))
        other = self.utf8(1) if r.random() < 0.3 else lit(bytes(r.choice(UTF8_LITERALS)), A.UTF8)
        if isinstance(other, Literal) and r.random() < 0.3:
            return BinaryExpr(other, op, s)  # a literal on the left
        return BinaryExpr(s, op, other)

    def _case(self, depth, value):
        """CASE with 1-4 WHENs, with or without ELSE, whose values are made by value(depth)."""
        r = self.rng
        self.seen.add("case")
        whens = [(self.boolean(max(0, depth - 1)), value(depth - 1)) for _ in range(int(r.integers(1, 5)))]
        if any(isinstance(e, Case) for _, e in whens):
            self.seen.add("nested_case")
        return Case(whens, value(depth - 1) if r.random() < 0.6 else None)

    def _divide(self, d, depth):
        """x / y over a divisor that may be zero: guarded by a CASE on `y <> 0` (never raises) or, rarely, unguarded over
        a value column (raises when a zero lands in a row that is evaluated)."""
        r = self.rng
        x = self.numeric(d, depth - 1)
        own = sorted(c for c in self.cols if self.t.dtype[c] == d and c != self.t.gate)
        if not own:
            return BinaryExpr(x, A.OP_DIV, self._lit(d, nonzero=True))
        y = col(int(r.choice(own)))
        if r.random() < 0.12:
            self.seen.add("unguarded_div")
            return BinaryExpr(x, A.OP_DIV, y)
        self.seen.add("guarded_div")
        zero = lit(0.0 if d in FLOATS else 0, d)
        return Case([(y.not_eq(zero), BinaryExpr(x, A.OP_DIV, y))], self.numeric(d, depth - 1) if r.random() < 0.7 else None)

    def _full_numeric(self, d, depth):
        r = self.rng
        src = sorted(c for c in self.cols if self.t.dtype[c] in NUMERIC and self.t.dtype[c] != d)
        if depth <= 0 or r.random() < 0.2:
            if d == A.INT64 and self._utf8_cols() and r.random() < 0.15:
                self.seen.add("length")
                return utf8_fn(str(r.choice(["length", "octet_length", "char_length"])), self.utf8(int(r.integers(0, 3))))
            if src and r.random() < 0.2:  # the C ABI casts columns (and Int64 literals to Float64) only
                self.seen.add("cast")
                return col(int(r.choice(src))).cast(d)
            return self._leaf(d)
        k = r.random()
        if k < 0.2:
            return self._case(depth, lambda dd: self.numeric(d, dd))
        if k < 0.3 and src:
            self.seen.add("cast")
            return BinaryExpr(col(int(r.choice(src))).cast(d), int(r.choice([A.OP_ADD, A.OP_SUB, A.OP_MUL])), self.numeric(d, depth - 1))
        if k < 0.5 and d == A.FLOAT64:
            self.seen.add("fn")
            return fn(str(r.choice(EXACT_FNS)), self.numeric(A.FLOAT64, depth - 1))
        if k < 0.56:
            return self._divide(d, depth)
        op = int(r.choice([A.OP_ADD, A.OP_SUB, A.OP_MUL]))
        left = self.numeric(d, depth - 1)
        right = self.numeric(d, depth - 1) if r.random() < 0.6 else self._leaf(d)
        return BinaryExpr(left, op, right)

    def _full_boolean(self, depth):
        r = self.rng
        k = r.random()
        if self._utf8_cols() and k < 0.2:
            return self.utf8_predicate()
        if depth > 0 and k < 0.3:
            self.seen.add("bool_case")
            return self._case(depth, lambda dd: self.boolean(max(0, dd)))
        return None

    def deep(self, d):
        """A right-nested chain `l1 op (l2 op (.. (CASE ..)))` whose stack depth is exactly 8, the limit: the entries
        below the top are spilled, and their operands are small CASEs and guarded divisions, so the spilled entries
        carry validity and DivideByZero bits."""
        import expr_ref
        r = self.rng
        self.seen.add("deep")
        small = lambda: self._case(1, lambda dd: self._leaf(d)) if r.random() < 0.4 else self._divide(d, 1) if r.random() < 0.4 else self._leaf(d)  # noqa: E731
        e = self._case(1, lambda dd: self._leaf(d))
        while expr_ref.stack_depth(e, self.t.dtype) < 8:
            e = BinaryExpr(small(), int(r.choice([A.OP_ADD, A.OP_SUB, A.OP_MUL])), e)
        return e

    def transcendental(self):
        """A transcendental function of Float64 operands: only ever the root of a projection."""
        r = self.rng
        self.seen.add("transcendental")
        name = str(r.choice(TRANSCENDENTAL))
        args = [self.numeric(A.FLOAT64, int(r.integers(0, 3))) for _ in range(2 if name in ("power", "atan2") else 1)]
        return fn(name, *args)

    def numeric(self, d, depth):
        r = self.rng
        if self.full:
            return self._full_numeric(d, depth)
        if depth <= 0 or r.random() < 0.25:
            return self._leaf(d)
        op = int(r.choice(MATH))
        left = self.numeric(d, depth - 1)
        if op == A.OP_DIV:
            role = getattr(self.t, self.divisor_role)
            if d in role and role[d] in self.cols and r.random() < 0.7:
                right = col(role[d])
            else:
                right = self._lit(d, nonzero=True)
        elif r.random() < 0.5:  # right-nested subtrees push the evaluator's register stack deep
            right = self.numeric(d, depth - 1)
        else:
            right = self._leaf(d)
        return BinaryExpr(left, op, right)

    def boolean(self, depth):
        r = self.rng
        if self.full:
            b = self._full_boolean(depth)
            if b is not None:
                return b
        bools = [c for c in self.cols if self.t.dtype[c] == A.BOOL]
        if depth <= 0 or r.random() < 0.35:
            if bools and r.random() < 0.3:
                return col(int(r.choice(sorted(bools))))
            ds = sorted({self.t.dtype[c] for c in self.cols if self.t.dtype[c] in NUMERIC})
            d = int(r.choice(ds))
            sub = max(0, depth - 1)
            return BinaryExpr(self.numeric(d, int(r.integers(0, sub + 1))), int(r.choice(CMP)), self.numeric(d, int(r.integers(0, sub + 1))))
        return BinaryExpr(self.boolean(depth - 1), int(r.choice([A.OP_AND, A.OP_OR])), self.boolean(depth - 1))

    def predicate(self):
        """`gate > 0 AND <random Boolean>` (the predicate is null-aware: its divisors are the safe columns)."""
        self.divisor_role = "safe"
        b = self.boolean(int(self.rng.integers(0, self.max_depth + 1)))
        return BinaryExpr(col(self.t.gate) > lit(0, A.INT32), A.OP_AND, b)

    def value(self, d, under_where):
        """A numeric expression of dtype d for a projection or an aggregate argument.  Under a WHERE the gated
        divisors apply (their zeros sit only in rows the WHERE drops), else the safe ones."""
        self.divisor_role = "gated" if under_where else "safe"
        return self.numeric(d, int(self.rng.integers(0, self.max_depth + 1)))


def _synthetic_slots(e, schema):
    """The synthetic columns the compiler makes for `e`: one per Utf8 predicate and per Int64 Utf8 function nest."""
    from datafusion_archive_b200.expr import Cast, ScalarFunction, Utf8Function
    if isinstance(e, Utf8Function):
        return 1 if e.dtype == A.INT64 else 0
    if isinstance(e, BinaryExpr):
        if e.op in (A.OP_LIKE, A.OP_NOT_LIKE) or e.left.get_type(schema) == A.UTF8:
            return 1
        return _synthetic_slots(e.left, schema) + _synthetic_slots(e.right, schema)
    if isinstance(e, Cast):
        return _synthetic_slots(e.expr, schema)
    if isinstance(e, ScalarFunction):
        return sum(_synthetic_slots(a, schema) for a in e.args)
    if isinstance(e, Case):
        return sum(_synthetic_slots(x, schema) for w in e.whens for x in w) + (_synthetic_slots(e.else_, schema) if e.else_ is not None else 0)
    return 0


def fits(exprs, schema):
    """Whether a query of these programs fits the engine's program-set limits (96 instructions, 12 columns, synthetic
    ones included, stack depth 8)."""
    import expr_ref
    n, cols, synth = 0, set(), 0
    for e in exprs:
        prog = e.program(schema)
        n += len(prog)
        cols |= {i.col for i in prog if i.op == A.OP_COL and schema[i.col] != A.UTF8}
        synth += _synthetic_slots(e, schema)
    return n <= 96 and len(cols) + synth <= 12 and all(expr_ref.stack_depth(e, schema) <= 8 for e in exprs)


def gen_fp_query(rng, table, ncols=8, with_pred=True, full=False, seen=None):
    """(pred, projections) for filter / project over a random subset of the table's columns (gate always included):
    1-3 numeric projections and sometimes a Boolean one.  Retries until the query fits the engine's limits.
    full: the whole language (QueryGen(full=True)), every Utf8 column readable, and sometimes a transcendental
    projection; `seen` (a set) collects the node kinds made."""
    schema = table.dtype
    while True:
        others = [i for i in range(len(schema)) if i != table.gate and schema[i] != A.UTF8]
        cols = set(rng.choice(others, size=min(ncols, len(others)), replace=False).tolist()) | {table.gate}
        if full:
            cols |= set(table.utf8)
        g = QueryGen(rng, table, cols, full=full, max_depth=8 if not full else 6)
        pred = g.predicate() if with_pred else None
        ds = sorted({schema[c] for c in cols if schema[c] in NUMERIC})
        proj = [g.value(int(rng.choice(ds)), with_pred) for _ in range(int(rng.integers(1, 4)))]
        if rng.random() < 0.2:
            g.divisor_role = "safe" if not with_pred else "gated"
            proj.append(g.boolean(2))
        if full and rng.random() < 0.25:
            proj.append(g.transcendental())
        if full and rng.random() < 0.25:
            proj[0] = g.deep(int(rng.choice(ds)))
        if full and pred is not None and rng.random() < 0.15:
            d = int(rng.choice(ds))
            pred = BinaryExpr(pred, A.OP_AND, BinaryExpr(g.deep(d), A.OP_GT, g._lit(d)))
        if fits(proj + ([pred] if pred is not None else []), schema) and any(references_column(e) for e in proj):
            if seen is not None:
                seen |= g.seen
            return pred, proj


def add_keys(rng, t, key_dtypes, n):
    """Integer key columns with few distinct values, garbage under their nulls (the bytes under a null key are its
    value), appended to the table; returns their indices."""
    out = []
    for d in key_dtypes:
        prof = PROFILES[int(rng.integers(0, len(PROFILES)))]
        valid = validity(rng, n, prof)
        v = rng.integers(0, 6, n).astype(A.NP_OF[d])
        if valid is not None:
            g = garbage(d)
            v = np.where(valid, v, g[rng.integers(0, len(g), n)]).astype(A.NP_OF[d])
        out.append(t.add(v, valid, prof))
    return out


def gen_agg_query(rng, t, key_cols, with_pred, plain_args, distinct_avg=False, full=False, seen=None):
    """(pred, keys, aggs): the keys are the key columns or expressions of them; 1-4 of MIN / MAX / SUM / COUNT (and
    AVG / COUNT(DISTINCT) when asked) over plain columns or random expressions.  full: the whole language in the
    arguments and the WHERE, and keys that are sometimes a CASE over the key column."""
    while True:
        others = [i for i in range(len(t.dtype)) if i != t.gate and i not in key_cols and t.dtype[i] not in (A.BOOL, A.UTF8)]
        cols = set(rng.choice(others, size=min(6, len(others)), replace=False).tolist()) | {t.gate} | set(t.bools)
        if full:
            cols |= set(t.utf8)
        g = QueryGen(rng, t, cols, max_depth=(8 if not full else 5) if not plain_args else 4, full=full)
        pred = g.predicate() if with_pred else None
        keys = []
        for k in key_cols:
            e = col(k)
            if full and rng.random() < 0.4:
                g.seen.add("case")
                e = Case([(g.boolean(1), e)], e + lit(1, t.dtype[k]) if rng.random() < 0.7 else None)
            elif rng.random() < 0.4:
                e = e + lit(int(rng.integers(1, 9)), t.dtype[k]) if rng.random() < 0.5 else e * lit(3, t.dtype[k])
            keys.append(e)
        funcs = ["min", "max", "sum", "count"] + (["avg", "distinct"] if distinct_avg else [])
        aggs = []
        for _ in range(int(rng.integers(1, 5))):
            c = int(rng.choice(sorted(cols - {t.gate} - set(t.bools) - set(t.utf8))))
            arg = col(c) if plain_args else g.deep(t.dtype[c]) if full and rng.random() < 0.2 else g.value(t.dtype[c], with_pred)
            f = str(rng.choice(funcs))
            aggs.append(AggregateFunction("count", arg, distinct=True) if f == "distinct" else AggregateFunction(f, arg))
        exprs = keys + [a.arg for a in aggs] + ([pred] if pred is not None else [])
        if fits(exprs, t.dtype):
            if seen is not None:
                seen |= g.seen
            return pred, keys, aggs
