"""Utf8 comparisons and LIKE / NOT LIKE without a GPU: the C ABI's type check of DFGPU_OP_LIT_UTF8, DFGPU_OP_LIKE and
DFGPU_OP_NOT_LIKE (every accepted shape, every refused one with its code and message, malformed literals), the plan text
of the SQL front-end, and the engine's LIKE pattern compiler and matcher against an independent Python matcher."""
import ctypes as C
import re

import pytest

from datafusion_archive_b200 import _abi as A
from datafusion_archive_b200 import engine, host
from datafusion_archive_b200.expr import col, lit

U, I, F = A.UTF8, A.INT64, A.FLOAT64


def check_err(schema, e):
    with pytest.raises(engine.DfGpuError) as ei:
        engine.check_program(schema, e)
    return ei.value


class Raw:
    """A postfix program given instruction by instruction: (op, col, dtype, lit.str) tuples."""

    def __init__(self, *insns):
        self.insns = insns

    def program(self, schema):
        out = []
        for op, c, dt, s in self.insns:
            i = A.Insn()
            i.op, i.col, i.dtype = op, c, dt
            i.lit.u64 = s
            out.append(i)
        return out


@pytest.mark.parametrize("op", ["eq", "not_eq", "__lt__", "__le__", "__gt__", "__ge__"])
def test_comparison_shapes_type_boolean(op):
    assert engine.check_program([U], getattr(col(0), op)(lit("CO"))) == A.BOOL
    assert engine.check_program([U], getattr(lit("CO"), op)(col(0))) == A.BOOL
    assert engine.check_program([U, U], getattr(col(0), op)(col(1))) == A.BOOL
    assert engine.check_program([U], getattr(col(0), op)(lit(""))) == A.BOOL


def test_like_shapes_and_mixed_trees_type_boolean():
    assert engine.check_program([U], col(0).like("%UK")) == A.BOOL
    assert engine.check_program([U], col(0).not_like("a_c%")) == A.BOOL
    assert engine.check_program([U], col(0).like("")) == A.BOOL
    assert engine.check_program([U, F], col(0).like("a%") & (col(1) > 1.0)) == A.BOOL
    assert engine.check_program([U, F, U], (col(0) < col(2)) | col(0).eq("x") & (col(1) > 1.0)) == A.BOOL
    # two string predicates in one tree
    assert engine.check_program([U], col(0).like("a%") | col(0).not_like("%b")) == A.BOOL
    # the longest literal
    assert engine.check_program([U], col(0).like("x" * A.UTF8_LITERAL_MAX)) == A.BOOL


def test_refused_shapes():
    e = check_err([U], lit("x"))
    assert e.code == A.ERR_EXECUTION and e.msg == 'No support for literal type Utf8("x")'
    e = check_err([U], lit("a") + lit("b"))
    assert e.code == A.ERR_EXECUTION and e.msg == 'No support for literal type Utf8("a")'
    e = check_err([F], col(0) + lit("b"))
    assert e.code == A.ERR_EXECUTION and e.msg == 'No support for literal type Utf8("b")'
    e = check_err([U], lit("x").cast(F))
    assert e.code == A.ERR_EXECUTION and "No support for literal type Utf8" in e.msg
    e = check_err([U], lit("a").eq(lit("b")))
    assert e.code == A.ERR_NOT_IMPLEMENTED
    e = check_err([U], lit("a").like("a%"))
    assert e.code == A.ERR_NOT_IMPLEMENTED
    e = check_err([U, U], col(0).like(col(1)))
    assert e.code == A.ERR_NOT_IMPLEMENTED and "not a literal" in e.msg
    e = check_err([I], col(0).like("1%"))
    assert e.code == A.ERR_EXECUTION and "Like" in e.msg
    e = check_err([U], col(0).not_like(lit(1)))
    assert e.code == A.ERR_EXECUTION and "NotLike" in e.msg
    # Utf8 against a number keeps comparison_ops
    e = check_err([U, I], col(0).eq(col(1)))
    assert e.code == A.ERR_EXECUTION and e.msg == "comparison_ops"
    e = check_err([I], col(0) < lit("5"))
    assert e.code == A.ERR_EXECUTION and e.msg == "comparison_ops"
    # DFGPU_OP_LIT with dtype Utf8 keeps its error and never reads lit
    e = check_err([U], Raw((A.OP_COL, 0, U, 0), (A.OP_LIT, 0, U, 0xDEADBEEF), (A.OP_EQ, 0, U, 0)))
    assert e.code == A.ERR_EXECUTION and e.msg == "No support for literal type Utf8"
    e = check_err([U], col(0).like("x" * (A.UTF8_LITERAL_MAX + 1)))
    assert e.code == A.ERR_NOT_IMPLEMENTED


def test_malformed_literals_are_errors_not_crashes():
    buf = C.create_string_buffer(b"abc")
    for c, dt, s in [(-1, U, C.addressof(buf)), (3, U, 0), (2, I, C.addressof(buf)), (-(2**31), U, 0xDEADBEEF)]:
        e = check_err([U], Raw((A.OP_COL, 0, U, 0), (A.OP_LIT_UTF8, c, dt, s), (A.OP_EQ, 0, U, 0)))
        assert e.code == A.ERR_GENERAL and e.msg == "malformed expression program"
    # an empty literal may have a null address
    assert engine.check_program([U], Raw((A.OP_COL, 0, U, 0), (A.OP_LIT_UTF8, 0, U, 0), (A.OP_LE, 0, U, 0))) == A.BOOL


def test_plan_text():
    host.build()
    c = host.Catalog()
    c.add_table("uk_cities", [("city", A.UTF8), ("lat", A.FLOAT64), ("lng", A.FLOAT64)])
    assert c.plan("SELECT city FROM uk_cities WHERE city LIKE '%UK'") == (
        'Projection: #0\n  Selection: #0 Like Utf8("%UK")\n    TableScan: uk_cities projection=None')
    assert c.plan("SELECT lat FROM uk_cities WHERE city NOT LIKE '%UK'") == (
        'Projection: #1\n  Selection: #0 NotLike Utf8("%UK")\n    TableScan: uk_cities projection=None')


# ---- LIKE: an independent matcher ------------------------------------------------------------------------------------
def py_like(s: bytes, p: bytes) -> bool:
    """`%` any run of bytes, `_` one byte and the continuation bytes after it (possessively), anything else itself."""
    rx = b"".join(b"[\\x00-\\xff]*" if ch == 0x25 else b"[\\x00-\\xff][\\x80-\\xbf]*+" if ch == 0x5F else re.escape(bytes([ch]))
                  for ch in p)
    return re.fullmatch(rx, s, re.DOTALL) is not None


PATTERNS = ["", "%", "_", "%%", "a%b%c", "a_c", "%_%", "abc", "abc%", "%abc", "%abc%", "%%abc%%", "a%", "%a", "%a%", "_%", "%_",
            "__", "a__", "%b_", "_é_", "é%", "%é", "%é%", "%😀%", "_😀", "😀_", "%\\%", "a\\_b", "%a%a%", "a%%c", "%ab%ab%",
            "abcdefghijklmnopqrstuvwxyz%", "%klmnopqrstuvwxyz0123456789", "%x_y%z", "Elgin%", "%UK", "%, the UK", "%Scotland%"]
STRINGS = ["", "a", "ab", "abc", "abcabc", "xabcx", "ac", "abbc", "aXc", "aéc", "a😀c", "é", "éé", "😀", "x😀y", "abxc", "aabc",
           "a\\b", "a\\_b", "a_b", "\\", "%", "_", "abab", "ababab", "xyz", "x1yz", "xyyz", "abcdefghijklmnopqrstuvwxyz0123456789",
           "Elgin, Scotland, the UK", "Solihull, Birmingham, UK", "aaa", "aa", "\x80abc", "ab\xc3"]


def test_pattern_compiler_and_matcher_agree_with_python():
    bad = []
    for p in PATTERNS:
        for s in STRINGS + ["x" * 300 + "abc", "abc" + "y" * 300]:
            sb = s.encode("utf-8", "surrogatepass") if not s.startswith("\x80") and not s.endswith("\xc3") else s.encode("latin-1")
            got, _ = engine.utf8_like_host(sb, p)
            if got != py_like(sb, p.encode()):
                bad.append((s, p, got))
    assert not bad, bad[:10]


def test_pattern_longer_than_the_string_and_classes():
    assert engine.utf8_like_host("ab", "abc%") == (False, 1)
    assert engine.utf8_like_host("ab", "%abc") == (False, 2)
    assert engine.utf8_like_host("ab", "%abc%") == (False, 3)
    assert engine.utf8_like_host("ab", "a_c") == (False, 4)
    assert engine.utf8_like_host("ab", "abc") == (False, 0)
    assert engine.utf8_like_host("", "") == (True, 0)
    assert engine.utf8_like_host("", "%") == (True, 1)
    assert engine.utf8_like_host("", "%%") == (True, 1)
    assert engine.utf8_like_host("", "_") == (False, 4)
    assert engine.utf8_like_host("é", "_") == (True, 4)
    assert engine.utf8_like_host("é", "__") == (False, 4)
    assert engine.utf8_like_host("x", "%_%") == (True, 4)
    assert engine.utf8_like_host("xaybzc", "%a%b%c") == (True, 4)


def test_header_constants_match_python():
    hdr = open(A.repo_root() + "/include/dfgpu.h").read()
    for name, val in [("DFGPU_OP_LIT_UTF8", A.OP_LIT_UTF8), ("DFGPU_OP_LIKE", A.OP_LIKE), ("DFGPU_OP_NOT_LIKE", A.OP_NOT_LIKE)]:
        assert re.search(r"\b%s = %d\b" % (name, val), hdr), name
    assert re.search(r"#define DFGPU_UTF8_LITERAL_MAX %d\b" % A.UTF8_LITERAL_MAX, hdr)
    assert C.sizeof(A.Insn) == 24
