"""Python reference of the Utf8 functions (include/dfgpu.h "Utf8 functions"), over bytes, and a builder of the same nest
as an engine expression.  A nest is a tuple (name, operand, *int arguments) whose innermost operand is the string "s"
(column `c`).  A character starts at the first byte and at every later byte that is not 10xxxxxx."""
import numpy as np

from datafusion_archive_b200.expr import col, utf8_fn

I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1


def chars(s):
    starts = [i for i in range(len(s)) if i == 0 or (s[i] & 0xC0) != 0x80]
    return [s[a:b] for a, b in zip(starts, starts[1:] + [len(s)])]


def apply(name, s, *args):
    name = name.lower()
    if name == "upper":
        return bytes(c - 32 if 97 <= c <= 122 else c for c in s)
    if name == "lower":
        return bytes(c + 32 if 65 <= c <= 90 else c for c in s)
    if name == "trim":
        return s.strip(b" ")
    if name == "ltrim":
        return s.lstrip(b" ")
    if name == "rtrim":
        return s.rstrip(b" ")
    if name == "substr":
        cs = chars(s)
        start = args[0]
        lo = max(start, 1)
        hi = start + args[1] if len(args) > 1 else I64_MAX  # unbounded ints: no overflow, as the engine's saturation
        return b"" if hi <= lo else b"".join(cs[lo - 1:hi - 1])
    if name in ("length", "char_length"):
        return len(chars(s))
    if name == "octet_length":
        return len(s)
    raise KeyError(name)


def ev(nest, s):
    """The value of `nest` for one string (None for a null)."""
    if isinstance(nest, str):
        return s
    inner = ev(nest[1], s)
    return None if inner is None else apply(nest[0], inner, *nest[2:])


def build(nest, c=0):
    if isinstance(nest, str):
        return col(c)
    return utf8_fn(nest[0], build(nest[1], c), *nest[2:])


def is_int(nest):
    return not isinstance(nest, str) and nest[0] in ("length", "char_length", "octet_length")


def random_strings(n, seed, null_frac=0.0, max_pieces=8):
    """Byte strings with 1-4 byte characters, stray continuation bytes, invalid bytes, runs of spaces at either end,
    and ''."""
    rng = np.random.default_rng(seed)
    pieces = [b"a", b"Z", b"abc", b"Hello", b" ", b"  ", b"\xc3\xa9", b"\xc3\x89", b"\xe2\x82\xac", b"\xf0\x9f\x98\x80", b"\x80",
              b"\xbf\xbf", b"\xff", b"\xc3", b"_", b"%", b"\t", b"0123456789"]
    out = []
    for _ in range(n):
        if rng.random() < null_frac:
            out.append(None)
            continue
        k = int(rng.integers(0, max_pieces + 1))
        out.append(b"".join(pieces[int(i)] for i in rng.integers(0, len(pieces), k)))
    return out


NESTS = [
    ("upper", "s"), ("lower", "s"), ("trim", "s"), ("ltrim", "s"), ("rtrim", "s"),
    ("substr", "s", 2), ("substr", "s", 0, 3), ("substr", "s", -2, 4), ("substr", "s", 3, 0), ("substr", "s", 1, 1),
    ("length", "s"), ("char_length", "s"), ("octet_length", "s"),
    ("upper", ("trim", ("substr", "s", 2))), ("length", ("lower", "s")), ("octet_length", ("trim", "s")),
    ("lower", ("upper", ("ltrim", "s"))), ("substr", ("substr", ("rtrim", "s"), 2, 5), 2), ("length", ("substr", ("trim", "s"), 2, 3)),
]
EDGE_STARTS = [I64_MIN, -1, 0, 1, 2, 5, I64_MAX]
EDGE_COUNTS = [0, 1, 3, I64_MAX]
