"""VARCHAR operations of expression programs without a GPU: the generated FilterAndProject kernels compile for sm_90a over nullable and
non-nullable UTF8 channels in every form, the new structs have gcc's layout, and the refusals answer at create."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

from trino_b200 import abi
from trino_b200 import operators as ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B, BOOL, S = abi.V_BIGINT, abi.V_BOOLEAN, abi.V_VARCHAR
C0, C1, C2 = ops.Col(0, S), ops.Col(1, S), ops.Col(2, B)
TYPES = [abi.UTF8, abi.UTF8, abi.INT64, abi.INT32]

EVERY_OP = [ops.Call(op, C0, ops.Const("MAIL", S)) for op in (abi.EX_EQ, abi.EX_NE, abi.EX_LT, abi.EX_LE, abi.EX_GT, abi.EX_GE)] + [
    ops.Call(abi.EX_EQ, C0, C1), ops.Call(abi.EX_LT, C1, C0),
    ops.Call(abi.EX_BETWEEN, C0, ops.Const("AIR", S), ops.Const("SHIP", S)),
    ops.Call(abi.EX_IN, C1, in_list=["MAIL", "SHIP", b"DELIVER IN PERSON"]),
    ops.Call(abi.EX_IS_NULL, C0), ops.Call(abi.EX_IS_NOT_NULL, C1), ops.Call(abi.EX_EQ, C0, ops.Null(S)),
    ops.Call(abi.EX_LIKE, C0, pattern="%special%requests%"),         # FJS
    ops.Call(abi.EX_LIKE, C1, pattern="a_b%c"),                       # DFA
    ops.Call(abi.EX_LIKE, C0, pattern="%x%y_z"),                      # NFA
    ops.Call(abi.EX_LIKE, C1, pattern="MEDIUM POLISHED%"),            # prefix only
    ops.Call(abi.EX_LIKE, C1, pattern="x$%%", escape="$"),
]


def _selftest(prog, nullable_mask, types=TYPES):
    lib = abi.load_library()
    t = (C.c_int32 * len(types))(*types)
    n = C.c_int64()
    buf = C.create_string_buffer(1 << 20)
    st = lib.tgpu_jit_selftest_filter_project(C.byref(prog.struct), t, len(types), nullable_mask, C.byref(n), buf, len(buf))
    return st, n.value, buf.value.decode(errors="replace")


def _filter(exprs):
    f = exprs[0]
    for e in exprs[1:]:
        f = ops.Call(abi.EX_OR, f, e)
    return f


@pytest.mark.parametrize("nullable_mask", [0, 0b0011, 0b1111])
@pytest.mark.parametrize("form", ["chunked", "selection_vector", "no_filter"])
def test_every_string_op_compiles(form, nullable_mask):
    for k in range(0, len(EVERY_OP), 4):                    # four operations per program: within the 8 temporaries
        group = EVERY_OP[k:k + 4]
        if form == "chunked":
            prog = ops.PageProcessorProgram(_filter(group[:2]), [3, 2] + group[2:])
        elif form == "selection_vector":
            prog = ops.PageProcessorProgram(_filter(group[:2]), [0, 3] + group[2:])      # a VARCHAR pass-through channel
        else:
            prog = ops.PageProcessorProgram(None, group + [1])
        st, size, src = _selftest(prog, nullable_mask)
        if st == abi.ERR_NOT_SUPPORTED and "nvrtc" in src.lower():
            pytest.skip("NVRTC not installed: " + src)
        assert st == 0, src[-3000:]
        assert size > 1000
        assert ("tg_fp_project_chunks_jit" in src) == (form == "chunked")
        assert "tg_fp_filter_jit" in src and "tg_fp_project_jit" in src
        assert ("tg_valid(cols.cols[0].validity" in src) == bool(nullable_mask & 1) or "s0" not in src


def test_generated_code_decides_on_length_and_packed_words():
    prog = ops.PageProcessorProgram(ops.Call(abi.EX_EQ, C0, ops.Const("DELIVER IN PERSON", S)), [3])
    st, _, src = _selftest(prog, 0)
    if st == abi.ERR_NOT_SUPPORTED and "nvrtc" in src.lower():
        pytest.skip("NVRTC not installed")
    assert st == 0, src[-3000:]
    assert "a.len == 17 && tg_ld_bytes(a.p + 0, 8) == 0x20524556494c4544ULL" in src     # "DELIVER " little-endian
    prog = ops.PageProcessorProgram(ops.Call(abi.EX_LIKE, C0, pattern="%special%requests%"), [3])
    st, _, src = _selftest(prog, 0)
    assert st == 0, src[-3000:]
    assert "bool tg_like_0(StrRef s)" in src and "if (s.len < 15) return false;" in src and "return tg_like_fjs(" in src


_PAIRS = [("tgpu_bytes", "Bytes"), ("tgpu_like_pattern", "LikePattern"), ("tgpu_expr_program", "ExprProgram")]


def test_new_structs_have_the_layout_gcc_gives_the_header(tmp_path):
    gcc = shutil.which("gcc") or shutil.which("cc")
    if not gcc:
        pytest.skip("no C compiler")
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "trino_gpu.h")).read(), flags=re.S)
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "trino_gpu.h"', "int main(void) {"]
    names = {}
    for cname, _ in _PAIRS:
        body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (cname, cname), text, flags=re.S).group(1)
        names[cname] = [re.search(r"([A-Za-z_][A-Za-z0-9_]*)\s*$", d.strip()).group(1) for d in body.split(";") if d.strip()]
        lines.append('printf("%%zu", sizeof(%s));' % cname)
        lines += ['printf(" %%zu", offsetof(%s, %s));' % (cname, f) for f in names[cname]]
        lines.append('printf("\\n");')
    lines.append("return 0; }")
    (tmp_path / "l.c").write_text("\n".join(lines))
    subprocess.run([gcc, "-I", os.path.join(ROOT, "include"), str(tmp_path / "l.c"), "-o", str(tmp_path / "l")], check=True)
    out = subprocess.run([str(tmp_path / "l")], check=True, capture_output=True, text=True).stdout.split("\n")
    for line, (cname, py) in zip(out, _PAIRS):
        size, *offs = [int(x) for x in line.split()]
        st = getattr(abi, py)
        assert C.sizeof(st) == size, cname
        assert [f[0] for f in st._fields_] == names[cname], cname
        assert [getattr(st, f[0]).offset for f in st._fields_] == offs, cname


def _status(prog):
    st, _, src = _selftest(prog, 0)
    return st, src


def _raw_program(insns, strings=(), likes=(), in_lists=()):
    """a tgpu_expr_program built by hand, for the arguments PageProcessorProgram never produces"""
    p = ops.PageProcessorProgram(ops.Call(abi.EX_IS_NULL, C0), [3])
    arr = (abi.ExprInsn * len(insns))()
    for i, (op, vt, dst, a, b) in enumerate(insns):
        arr[i].op, arr[i].vtype, arr[i].dst = op, vt, dst
        arr[i].a.kind, arr[i].a.index, arr[i].a.imm.i64 = a
        arr[i].b.kind, arr[i].b.index, arr[i].b.imm.i64 = b
    p._keep = [arr]
    p.struct.num_insns, p.struct.insns, p.struct.filter_temp, p.struct.num_filter_insns = len(insns), C.cast(arr, C.POINTER(abi.ExprInsn)), 0, len(insns)
    return p


def test_refusals():
    lib = abi.load_library()
    # invalid escape uses (TestLikeFunctions.java:266-278) and an escape of more than one character: NOT_SUPPORTED
    for pat, esc in [("#", "#"), ("abc#abc", "#"), ("abc#", "#"), ("a", "ab"), ("a", "\U0001F600")]:
        st, src = _status(ops.PageProcessorProgram(ops.Call(abi.EX_LIKE, C0, pattern=pat, escape=esc), [3]))
        assert st == abi.ERR_NOT_SUPPORTED, (pat, esc, src)
    # limits, each exceeded by one
    st, _ = _status(ops.PageProcessorProgram(ops.Call(abi.EX_IN, C0, in_list=[str(i) for i in range(abi.MAX_STRINGS)]), [3]))
    assert st == 0
    st, _ = _status(ops.PageProcessorProgram(ops.Call(abi.EX_IN, C0, in_list=[str(i) for i in range(abi.MAX_STRINGS + 1)]), [3]))
    assert st in (abi.ERR_NOT_SUPPORTED,)
    big = "x" * (abi.MAX_STRING_BYTES // 2)
    st, _ = _status(ops.PageProcessorProgram(ops.Call(abi.EX_IN, C0, in_list=[big, big[:-1] + "y"]), [3]))
    assert st == 0
    st, _ = _status(ops.PageProcessorProgram(ops.Call(abi.EX_IN, C0, in_list=[big, big + "y"]), [3]))
    assert st == abi.ERR_NOT_SUPPORTED
    many = [ops.Call(abi.EX_LIKE, C0, pattern=f"%{i}%") for i in range(abi.MAX_LIKE_PATTERNS + 1)]
    st, _ = _status(ops.PageProcessorProgram(_filter(many[:abi.MAX_LIKE_PATTERNS]), [3]))
    assert st == 0
    st, _ = _status(ops.PageProcessorProgram(_filter(many), [3]))
    assert st == abi.ERR_NOT_SUPPORTED
    st, src = _status(ops.PageProcessorProgram(ops.Call(abi.EX_LIKE, C0, pattern="%a" + "_" * 62 + "b"), [3]))  # NFA: 63 states + accept
    assert st == 0, src[-2000:]
    st, _ = _status(ops.PageProcessorProgram(ops.Call(abi.EX_LIKE, C0, pattern="%a" + "_" * 63 + "b"), [3]))
    assert st == abi.ERR_NOT_SUPPORTED
    # a string pre-stage in the aggregation kernel generator
    keys = (C.c_int32 * 1)(3)
    fns = (abi.AggFn * 1)()
    fns[0].function, fns[0].input_channel, fns[0].mask_channel = abi.AGG_COUNT_STAR, -1, -1
    pre = ops.PageProcessorProgram(ops.Call(abi.EX_LIKE, C0, pattern="%a%"), [3])
    spec = abi.AggSpec(1, C.cast(keys, C.POINTER(C.c_int32)), abi.STEP_SINGLE, 1, C.cast(fns, C.POINTER(abi.AggFn)), 16, 0, C.pointer(pre.struct))
    t = (C.c_int32 * 4)(*TYPES)
    n = C.c_int64()
    buf = C.create_string_buffer(1 << 16)
    assert lib.tgpu_jit_selftest_agg(C.byref(spec), t, 4, 0, C.byref(n), buf, len(buf)) == abi.ERR_NOT_SUPPORTED
    # INVALID_ARGUMENT: a VARCHAR temp, pool and pattern indices out of range
    CONST, COL, TEMP = abi.OPND_CONST, abi.OPND_COLUMN, abi.OPND_TEMP
    p = _raw_program([(abi.EX_EQ, S, 0, (COL, 0, 0), (TEMP, 1, 0))])
    assert _status(p)[0] == abi.ERR_INVALID_ARGUMENT
    p = ops.PageProcessorProgram(ops.Call(abi.EX_EQ, C0, ops.Const("a", S)), [3])
    p._insns[0].b.imm.i64 = 1
    assert _status(p)[0] == abi.ERR_INVALID_ARGUMENT
    p = ops.PageProcessorProgram(ops.Call(abi.EX_LIKE, C0, pattern="a%"), [3])
    p._insns[0].b.imm.i64 = 1
    assert _status(p)[0] == abi.ERR_INVALID_ARGUMENT
    p = ops.PageProcessorProgram(ops.Call(abi.EX_IN, C0, in_list=["a"]), [3])
    p._list_bufs[0][0] = 5
    assert _status(p)[0] == abi.ERR_INVALID_ARGUMENT
    p = ops.PageProcessorProgram(ops.Call(abi.EX_LIKE, ops.Col(2, B), pattern="a%"), [3])     # LIKE needs VARCHAR operands
    assert _status(p)[0] == abi.ERR_INVALID_ARGUMENT


def test_long_constants_compile():
    """a constant of several KB (its comparison reads the pool's copy) in =, IN, BETWEEN and a LIKE prefix"""
    long = "q" * 3000
    prog = ops.PageProcessorProgram(ops.Call(abi.EX_OR, ops.Call(abi.EX_EQ, C0, ops.Const(long, S)), ops.Call(abi.EX_IN, C1, in_list=[long, "a"])),
                                    [3, ops.Call(abi.EX_BETWEEN, C0, ops.Const("a", S), ops.Const(long, S)),
                                     ops.Call(abi.EX_LIKE, C1, pattern="q" * 900 + "%")])
    st, _, src = _selftest(prog, 0b11)
    if st == abi.ERR_NOT_SUPPORTED and "nvrtc" in src.lower():
        pytest.skip("NVRTC not installed")
    assert st == 0, src[-3000:]
    assert "a.len == 3000 && tg_str_eq(a, StrRef{(const uint8_t*)tg_pool + 0, 3000})" in src
