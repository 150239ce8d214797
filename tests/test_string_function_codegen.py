"""String functions of expression programs without a GPU: every new operation compiles with NVRTC for sm_90a as a filter, a chunked
projection and a selection-vector projection, over nullable and non-nullable channels, with operands from channels, constants and view
temps; the refusals answer at create; programs without the new operations generate the source they did before."""
import ctypes as C
import json
import os

import pytest

from trino_b200 import abi
from trino_b200 import operators as ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B, BOOL, S = abi.V_BIGINT, abi.V_BOOLEAN, abi.V_VARCHAR
C0, C1, C2, C3 = ops.Col(0, S), ops.Col(1, S), ops.Col(2, B), ops.Col(3, B)
K = lambda v: ops.Const(v, B)
T = lambda v: ops.Const(v, S)
call = ops.Call
TYPES = [abi.UTF8, abi.UTF8, abi.INT64, abi.INT32]

# each a VARCHAR (or BIGINT) valued expression over channels, constants and view temps
VALUES = [
    call(abi.EX_LENGTH, C0), call(abi.EX_LENGTH, T("x")), call(abi.EX_SUBSTR, C0, C2), call(abi.EX_SUBSTR, C1, C2, C3),
    call(abi.EX_SUBSTR, T("Quadratically"), K(5), K(6)), call(abi.EX_LTRIM, C0), call(abi.EX_RTRIM, T("  a  ")), call(abi.EX_TRIM, C1),
    ops.concat(C0, C1), ops.concat(T("store"), C1, T("-"), C0),
    call(abi.EX_LENGTH, call(abi.EX_TRIM, call(abi.EX_SUBSTR, C0, K(-5)))),
    ops.concat(C0, T("-"), call(abi.EX_SUBSTR, C1, K(2), K(3))),
    call(abi.EX_SUBSTR, call(abi.EX_RTRIM, C0), call(abi.EX_LENGTH, C1)),
]
# filters over the new operations (a VARCHAR view read by every kind of predicate)
FILTERS = [
    call(abi.EX_IN, call(abi.EX_SUBSTR, C0, K(1), K(2)), in_list=["13", "31"]),
    call(abi.EX_GT, call(abi.EX_LENGTH, call(abi.EX_TRIM, C1)), K(0)),
    call(abi.EX_LIKE, call(abi.EX_LTRIM, C0), pattern="%a_b%"),
    call(abi.EX_BETWEEN, call(abi.EX_RTRIM, C1), T("a"), call(abi.EX_SUBSTR, C0, K(2))),
    call(abi.EX_AND, call(abi.EX_IS_NOT_NULL, call(abi.EX_SUBSTR, C1, C2)), call(abi.EX_NE, call(abi.EX_TRIM, C0), T("x"))),
]


def _selftest(prog, nullable_mask, types=TYPES):
    lib = abi.load_library()
    t = (C.c_int32 * len(types))(*types)
    n = C.c_int64()
    buf = C.create_string_buffer(1 << 21)
    st = lib.tgpu_jit_selftest_filter_project(C.byref(prog.struct), t, len(types), nullable_mask, C.byref(n), buf, len(buf))
    return st, n.value, buf.value.decode(errors="replace")


def _ok(st, src):
    if st == abi.ERR_NOT_SUPPORTED and "nvrtc" in src.lower():
        pytest.skip("NVRTC not installed: " + src)
    assert st == 0, src[-3000:]


@pytest.mark.parametrize("nullable_mask", [0, 0b0101, 0b1111])
@pytest.mark.parametrize("form", ["chunked", "selection_vector", "no_filter"])
def test_every_function_compiles(form, nullable_mask):
    for k in range(0, len(VALUES), 3):
        group = VALUES[k:k + 3]
        filt = FILTERS[(k // 3) % len(FILTERS)]
        if form == "chunked":
            prog = ops.PageProcessorProgram(filt, [3, 2] + group)
        elif form == "selection_vector":
            prog = ops.PageProcessorProgram(filt, [0, 3] + group)      # a VARCHAR pass-through channel
        else:
            prog = ops.PageProcessorProgram(None, group + [1])
        st, size, src = _selftest(prog, nullable_mask)
        _ok(st, src)
        assert size > 1000
        assert ("tg_fp_project_chunks_jit" in src) == (form == "chunked")
        assert "out.str_desc[0]" in src or all(e.vtype != S for e in group)


def test_every_filter_compiles():
    for f in FILTERS:
        st, _, src = _selftest(ops.PageProcessorProgram(f, [3]), 0b11)
        _ok(st, src)


def test_views_and_pieces_in_generated_code():
    prog = ops.PageProcessorProgram(None, [ops.concat(C0, T("-"), call(abi.EX_SUBSTR, C1, K(2), K(3)))])
    st, _, src = _selftest(prog, 0)
    _ok(st, src)
    assert "tg_substr(a, b.bits, true, c.bits)" in src
    assert "q0 = s0;" in src and "q1 = StrRef{(const uint8_t*)tg_pool + 0, 1};" in src and "q2 = v" in src
    assert "tot > TGD_MAX_CONCAT_BYTES" in src
    assert "out.str_desc[0] + j * 3" in src


def test_struct_layout_unchanged():
    """the new operations add no field to the public structs"""
    assert C.sizeof(abi.ExprInsn) == 64 and C.sizeof(abi.Projection) == 12


def test_programs_without_string_functions_generate_the_same_source():
    """the captured sources of programs without DECIMAL (and without string functions) come out byte for byte as before"""
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "fp_sources_without_decimal.json")))
    assert golden
    prog = ops.PageProcessorProgram(call(abi.EX_EQ, C0, T("DELIVER IN PERSON")), [3])
    st, _, src = _selftest(prog, 0)
    _ok(st, src)
    assert "StrRef v0" not in src and "str_desc" not in src


CONST, COL, TEMP, NONE = abi.OPND_CONST, abi.OPND_COLUMN, abi.OPND_TEMP, abi.OPND_NONE


def _raw_program(insns, projections=((0, 3, 0),)):
    """a tgpu_expr_program built by hand, for the arguments PageProcessorProgram never produces"""
    p = ops.PageProcessorProgram(None, [3])
    arr = (abi.ExprInsn * len(insns))()
    for i, (op, vt, dst, a, b, c) in enumerate(insns):
        arr[i].op, arr[i].vtype, arr[i].dst = op, vt, dst
        for fld, o in (("a", a), ("b", b), ("c", c)):
            f = getattr(arr[i], fld)
            f.kind, f.index, f.imm.i64 = o
    projs = (abi.Projection * len(projections))()
    for i, (k, idx, vt) in enumerate(projections):
        projs[i].kind, projs[i].index, projs[i].vtype = k, idx, vt
    p._keep = [arr, projs]
    p.struct.num_insns, p.struct.insns = len(insns), C.cast(arr, C.POINTER(abi.ExprInsn))
    p.struct.filter_temp, p.struct.num_filter_insns = -1, 0
    p.struct.num_projections, p.struct.projections = len(projections), C.cast(projs, C.POINTER(abi.Projection))
    return p


def test_refusals():
    st = lambda p: _selftest(p, 0)[0]
    # a concatenation read by anything but a concatenation or a projection: NOT_SUPPORTED
    for e in (call(abi.EX_EQ, ops.concat(C0, C1), T("x")), call(abi.EX_LIKE, ops.concat(C0, C1), pattern="a%"),
              call(abi.EX_GT, call(abi.EX_LENGTH, ops.concat(C0, C1)), K(1))):
        assert st(ops.PageProcessorProgram(e, [3])) == abi.ERR_NOT_SUPPORTED
    assert st(ops.PageProcessorProgram(None, [call(abi.EX_SUBSTR, ops.concat(C0, C1), K(1))])) == abi.ERR_NOT_SUPPORTED
    assert st(ops.PageProcessorProgram(None, [call(abi.EX_TRIM, ops.concat(C0, C1))])) == abi.ERR_NOT_SUPPORTED
    # eight pieces compile, a ninth is refused
    assert st(ops.PageProcessorProgram(None, [ops.concat(*([C0, C1] * 4))])) == 0
    assert st(ops.PageProcessorProgram(None, [ops.concat(*([C0, C1] * 4 + [C0]))])) == abi.ERR_NOT_SUPPORTED
    # a VARCHAR temp read before it is written: INVALID_ARGUMENT
    assert st(_raw_program([(abi.EX_LENGTH, S, 0, (TEMP, 1, 0), (NONE, 0, 0), (NONE, 0, 0))])) == abi.ERR_INVALID_ARGUMENT
    # a temp holding a BIGINT read as VARCHAR, and a VARCHAR temp read as a number
    assert st(_raw_program([(abi.EX_LENGTH, S, 1, (COL, 0, 0), (NONE, 0, 0), (NONE, 0, 0)),
                            (abi.EX_TRIM, S, 0, (TEMP, 1, 0), (NONE, 0, 0), (NONE, 0, 0))])) == abi.ERR_INVALID_ARGUMENT
    assert st(_raw_program([(abi.EX_TRIM, S, 1, (COL, 0, 0), (NONE, 0, 0), (NONE, 0, 0)),
                            (abi.EX_ADD, B, 0, (TEMP, 1, 0), (CONST, 0, 1), (NONE, 0, 0))])) == abi.ERR_INVALID_ARGUMENT
    # SUBSTR with a start that is not BIGINT (a DOUBLE temp)
    prog = ops.PageProcessorProgram(None, [call(abi.EX_SUBSTR, C0, call(abi.EX_CAST_BIGINT_TO_DOUBLE, C2))])
    assert st(prog) == abi.ERR_INVALID_ARGUMENT
    # a VARCHAR projection of a temp that holds no VARCHAR, and a BIGINT projection of a view
    assert st(_raw_program([(abi.EX_LENGTH, S, 0, (COL, 0, 0), (NONE, 0, 0), (NONE, 0, 0))], [(1, 0, S)])) == abi.ERR_INVALID_ARGUMENT
    assert st(_raw_program([(abi.EX_TRIM, S, 0, (COL, 0, 0), (NONE, 0, 0), (NONE, 0, 0))], [(1, 0, B)])) == abi.ERR_INVALID_ARGUMENT
    # more than 8 VARCHAR projections
    trim = [(abi.EX_TRIM, S, 0, (COL, 0, 0), (NONE, 0, 0), (NONE, 0, 0))]
    assert st(_raw_program(trim, [(1, 0, S)] * 8)) == 0
    assert st(_raw_program(trim, [(1, 0, S)] * 9)) == abi.ERR_NOT_SUPPORTED
    # string functions in the fused aggregation pre-stage and in join filters keep NOT_SUPPORTED
    lib = abi.load_library()
    keys = (C.c_int32 * 1)(0)
    fns = (abi.AggFn * 1)()
    fns[0].function, fns[0].input_channel, fns[0].mask_channel = abi.AGG_COUNT_STAR, -1, -1
    pre = ops.PageProcessorProgram(call(abi.EX_GT, call(abi.EX_LENGTH, C0), K(3)), [3])
    spec = abi.AggSpec(1, C.cast(keys, C.POINTER(C.c_int32)), abi.STEP_SINGLE, 1, C.cast(fns, C.POINTER(abi.AggFn)), 16, 0, C.pointer(pre.struct))
    t = (C.c_int32 * 4)(*TYPES)
    n = C.c_int64()
    buf = C.create_string_buffer(1 << 16)
    assert lib.tgpu_jit_selftest_agg(C.byref(spec), t, 4, 0, C.byref(n), buf, len(buf)) == abi.ERR_NOT_SUPPORTED
    jf = ops.PageProcessorProgram(call(abi.EX_EQ, call(abi.EX_SUBSTR, C0, K(1), K(2)), T("ab")), [])
    assert lib.tgpu_jit_selftest_join_filter(C.byref(jf.struct), 2, t, 4, 0, C.byref(n), buf, len(buf)) == abi.ERR_NOT_SUPPORTED


def test_status_name():
    lib = abi.load_library()
    assert lib.tgpu_status_name(abi.ERR_INVALID_FUNCTION_ARGUMENT) == b"INVALID_FUNCTION_ARGUMENT"
