"""DECIMAL operations of expression programs without a GPU: the generated FilterAndProject kernels compile for sm_90a for every decimal
operation over every short / long combination of operands and result, nullable and not, in every form; the new structs have gcc's
layout; the refusals answer at create; and programs without DECIMAL generate the same source as before decimals existed."""
import ctypes as C
import json
import os
import re
import shutil
import subprocess

import pytest

from trino_b200 import abi
from trino_b200 import operators as ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_SOURCES = os.path.join(ROOT, "tests", "golden", "fp_sources_without_decimal.json")
B, D, BOOL, S, DEC = abi.V_BIGINT, abi.V_DOUBLE, abi.V_BOOLEAN, abi.V_VARCHAR, getattr(abi, "V_DECIMAL", 4)


def _selftest(prog, nullable_mask, types):
    lib = abi.load_library()
    t = (C.c_int32 * len(types))(*types)
    n = C.c_int64()
    buf = C.create_string_buffer(1 << 21)
    st = lib.tgpu_jit_selftest_filter_project(C.byref(prog.struct), t, len(types), nullable_mask, C.byref(n), buf, len(buf))
    return st, n.value, buf.value.decode(errors="replace")


def source_programs():
    """numeric and string programs whose generated source is pinned (name, program, channel types, nullable mask)"""
    import q1
    import q6
    q1_types = [abi.INT32, abi.INT8, abi.INT8, abi.FLOAT64, abi.FLOAT64, abi.FLOAT64, abi.FLOAT64]
    q6_types = [abi.INT32, abi.FLOAT64, abi.FLOAT64, abi.FLOAT64, abi.FLOAT64, abi.FLOAT64]
    mixed = ops.PageProcessorProgram(
        ops.Call(abi.EX_OR, ops.Call(abi.EX_AND, ops.Call(abi.EX_GT, ops.Call(abi.EX_DIV, ops.Col(0, B), ops.Col(1, B)), ops.Const(3, B)),
                                     ops.Call(abi.EX_IN, ops.Col(2, D), in_list=[1.5, 2.5])),
                 ops.Call(abi.EX_BETWEEN, ops.Col(0, B), ops.Const(-4, B), ops.Null(B))),
        [1, ops.Call(abi.EX_CAST_BIGINT_TO_DOUBLE, ops.Call(abi.EX_NEG, ops.Col(0, B))), ops.Call(abi.EX_CAST_DOUBLE_TO_BIGINT, ops.Col(2, D)),
         ops.Call(abi.EX_IS_NULL, ops.Col(1, B))])
    strings = ops.PageProcessorProgram(
        ops.Call(abi.EX_OR, ops.Call(abi.EX_LIKE, ops.Col(3, S), pattern="%special%requests%"),
                 ops.Call(abi.EX_IN, ops.Col(3, S), in_list=["MAIL", "SHIP"])),
        [3, ops.Call(abi.EX_BETWEEN, ops.Col(3, S), ops.Const("A", S), ops.Const("M", S)), ops.Call(abi.EX_MUL, ops.Col(0, B), ops.Const(7, B))])
    mixed_types = [abi.INT64, abi.INT32, abi.FLOAT64, abi.UTF8]
    return [
        ("q1", q1.q1_program(), q1_types, 0),
        ("q1_nullable", q1.q1_program(), q1_types, 0x7F),
        ("q6", q6.q6_program(), q6_types, 0),
        ("mixed", mixed, mixed_types, 0b0111),
        ("mixed_no_filter", ops.PageProcessorProgram(None, [ops.Call(abi.EX_ADD, ops.Col(0, B), ops.Col(1, B)), 2]), mixed_types, 0),
        ("strings", strings, mixed_types, 0b1001),
    ]


def test_programs_without_decimal_generate_the_same_source():
    golden = json.load(open(GOLDEN_SOURCES))
    for name, prog, types, mask in source_programs():
        st, _, src = _selftest(prog, mask, types)
        if st == abi.ERR_NOT_SUPPORTED and "nvrtc" in src.lower():
            pytest.skip("NVRTC not installed")
        assert st == 0, src[-2000:]
        assert src == golden[name], name


def _case_groups(size=6):
    """every decimal operation over short and long operands and results, `size` per program: each operand type reads its own channel
    (a channel is read with one type throughout a program).  Yields (expressions, channel types)."""
    import test_gpu_decimal_expressions as g
    cases = list(g.CASES) + [(abi.EX_IN, DEC, [(12, 2)], None), (abi.EX_IN, DEC, [(38, 6)], None)]
    for k in range(0, len(cases), size):
        chan = {}
        exprs = []
        for op, vt, types, rt in cases[k:k + size]:
            args = [ops.Col(chan.setdefault((vt, t), len(chan)), vt, t) for t in types]
            if op == abi.EX_IN:
                exprs.append(ops.Call(op, *args, in_list=[0, 150, -99, 10 ** types[0][0] - 1]))
            else:
                exprs.append(ops.Call(op, *args, **({"result_dtype": rt} if rt else {})))
        ctypes_ = [abi.INT128 if vt == DEC and t[0] > 18 else abi.INT64 for vt, t in chan]
        yield exprs, ctypes_


@pytest.mark.parametrize("nullable_mask", [0, 0xFFFF])
@pytest.mark.parametrize("form", ["chunked", "selection_vector", "no_filter"])
def test_every_decimal_op_compiles(form, nullable_mask):
    for exprs, types in _case_groups():
        flag = len(types)
        types = types + [abi.INT64, abi.INT128]     # the filter's BIGINT channel, a long DECIMAL pass-through channel
        flt = ops.Call(abi.EX_NE, ops.Col(flag, B), ops.Const(0, B)) if form != "no_filter" else None
        projs = ([flag + 1] if form == "selection_vector" else [flag]) + exprs
        prog = ops.PageProcessorProgram(flt, projs)
        st, size, src = _selftest(prog, nullable_mask, types)
        if st == abi.ERR_NOT_SUPPORTED and "nvrtc" in src.lower():
            pytest.skip("NVRTC not installed: " + src)
        assert st == 0, src[-3000:]
        assert size > 1000
        assert "vm_apply_dec(" in src
        assert ("tg_fp_project_chunks_jit" in src) == (form != "no_filter")


def test_short_paths_stay_64_bit():
    """short + short -> short has no high-word temps; a long result declares them"""
    prog = ops.PageProcessorProgram(None, [ops.Call(abi.EX_ADD, ops.Col(0, DEC, (12, 2)), ops.Col(1, DEC, (12, 4)))])
    st, _, src = _selftest(prog, 0, [abi.INT64, abi.INT64])
    if st == abi.ERR_NOT_SUPPORTED and "nvrtc" in src.lower():
        pytest.skip("NVRTC not installed")
    assert st == 0, src[-2000:]
    assert "long long th" not in src and "100LL, 1LL" in src
    prog = ops.PageProcessorProgram(None, [ops.Call(abi.EX_MUL, ops.Col(0, DEC, (12, 2)), ops.Col(1, DEC, (12, 4)))])
    st, _, src = _selftest(prog, 0, [abi.INT64, abi.INT64])
    assert st == 0 and "long long th" in src and "TGD_V_DECIMAL_LONG" in src


_PAIRS = [("tgpu_decimal_type", "DecimalType"), ("tgpu_decimal_signature", "DecimalSignature"), ("tgpu_expr_program", "ExprProgram")]


def test_new_structs_have_the_layout_gcc_gives_the_header(tmp_path):
    gcc = shutil.which("gcc") or shutil.which("cc")
    if not gcc:
        pytest.skip("no C compiler")
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "trino_gpu.h")).read(), flags=re.S)
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "trino_gpu.h"', "int main(void) {"]
    names = {}
    for cname, _ in _PAIRS:
        body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (cname, cname), text, flags=re.S).group(1)
        fields = []
        for decl in body.split(";"):
            decl = decl.strip()
            if not decl:
                continue
            head = re.match(r"(.*?)([A-Za-z_][A-Za-z0-9_]*(\s*,\s*[A-Za-z_][A-Za-z0-9_]*)*)\s*$", decl, flags=re.S)
            fields += [f.strip() for f in head.group(2).split(",")]
        names[cname] = fields
        lines.append('printf("%%zu", sizeof(%s));' % cname)
        lines += ['printf(" %%zu", offsetof(%s, %s));' % (cname, f) for f in fields]
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
    st, _, src = _selftest(prog, 0, [abi.INT64, abi.INT64, abi.INT128, abi.FLOAT64])
    return st, src


def test_refusals():
    lib = abi.load_library()
    c0, c2 = ops.Col(0, DEC, (12, 2)), ops.Col(2, DEC, (38, 6))
    # NOT_SUPPORTED: DECIMAL %, CAST(DOUBLE AS DECIMAL)
    assert _status(ops.PageProcessorProgram(None, [ops.Call(abi.EX_MOD, c0, c0, result_dtype=(12, 2))]))[0] == abi.ERR_NOT_SUPPORTED
    assert _status(ops.PageProcessorProgram(None, [ops.Call(abi.EX_CAST_TO_DECIMAL, ops.Col(3, D), result_dtype=(12, 2))]))[0] == abi.ERR_NOT_SUPPORTED
    # INVALID_ARGUMENT: bad types, comparisons of different types, a constant past its precision, no signatures
    bad = [
        ops.Call(abi.EX_ADD, ops.Col(0, DEC, (12, 13)), c0),
        ops.Call(abi.EX_ADD, ops.Col(0, DEC, (39, 2)), c0),
        ops.Call(abi.EX_EQ, c0, ops.Col(1, DEC, (12, 3))),
        ops.Call(abi.EX_ADD, c0, ops.Const(10 ** 12, DEC, (12, 2))),
        ops.Call(abi.EX_NEG, c0, result_dtype=(13, 2)),
        ops.Call(abi.EX_ADD, c2, c2, result_dtype=(18, 6)),
    ]
    for e in bad:
        assert _status(ops.PageProcessorProgram(None, [e]))[0] == abi.ERR_INVALID_ARGUMENT, e.op
    p = ops.PageProcessorProgram(None, [ops.Call(abi.EX_ADD, c0, c0)])
    p.struct.decimal_signatures = None
    assert _status(p)[0] == abi.ERR_INVALID_ARGUMENT
    # a column read as DECIMAL and as BIGINT
    p = ops.PageProcessorProgram(ops.Call(abi.EX_GT, ops.Col(0, B), ops.Const(0, B)), [ops.Call(abi.EX_NEG, c0)])
    assert _status(p)[0] == abi.ERR_INVALID_ARGUMENT
    # the fused aggregation pre-stage and join filters refuse DECIMAL programs
    keys = (C.c_int32 * 1)(1)
    fns = (abi.AggFn * 1)()
    fns[0].function, fns[0].input_channel, fns[0].mask_channel = abi.AGG_COUNT_STAR, -1, -1
    pre = ops.PageProcessorProgram(ops.Call(abi.EX_GT, c0, ops.Const(5, DEC, (12, 2))), [1])
    spec = abi.AggSpec(1, C.cast(keys, C.POINTER(C.c_int32)), abi.STEP_SINGLE, 1, C.cast(fns, C.POINTER(abi.AggFn)), 16, 0, C.pointer(pre.struct))
    t = (C.c_int32 * 2)(abi.INT64, abi.INT64)
    n = C.c_int64()
    buf = C.create_string_buffer(1 << 16)
    assert lib.tgpu_jit_selftest_agg(C.byref(spec), t, 2, 0, C.byref(n), buf, len(buf)) == abi.ERR_NOT_SUPPORTED
    jf = ops.PageProcessorProgram(ops.Call(abi.EX_GT, c0, ops.Col(1, DEC, (12, 2))), [])
    assert lib.tgpu_jit_selftest_join_filter(C.byref(jf.struct), 1, t, 2, 0, C.byref(n), buf, len(buf)) == abi.ERR_NOT_SUPPORTED
