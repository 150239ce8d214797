"""IF and COALESCE without a GPU: every accepted vtype (BIGINT, DOUBLE, BOOLEAN, short and long DECIMAL), over nullable and non-nullable
channels, compiles with NVRTC for sm_90a in the chunked, selection-vector and no-filter FilterAndProject forms, and the numeric ones in
the fused aggregation pre-stage (tg_agg_small_jit / tg_agg_general_jit and tg_agg_global_jit); the refusals answer at create; the
lowering of CASE, the simple CASE, NULLIF and COALESCE shares temps and frees them after their last reader."""
import ctypes as C
import os
import re

import pytest

from trino_b200 import abi
from trino_b200 import operators as ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B, D, BOOL, S, DEC = abi.V_BIGINT, abi.V_DOUBLE, abi.V_BOOLEAN, abi.V_VARCHAR, abi.V_DECIMAL
call = ops.Call
K = lambda v, vt=B, dt=None: ops.Const(v, vt, dt)
# channels: BIGINT, DOUBLE, BOOLEAN, DECIMAL(12, 2), DECIMAL(38, 6), VARCHAR, BIGINT
TYPES = [abi.INT64, abi.FLOAT64, abi.INT8, abi.INT64, abi.INT128, abi.UTF8, abi.INT64]
X, F, P, SD, LD, V, Y = (ops.Col(0, B), ops.Col(1, D), ops.Col(2, BOOL), ops.Col(3, DEC, (12, 2)), ops.Col(4, DEC, (38, 6)),
                         ops.Col(5, S), ops.Col(6, B))
POS = call(abi.EX_GT, X, K(0))
PROMO = call(abi.EX_LIKE, V, pattern="PROMO%")

# per vtype: IF and COALESCE over channels, constants, NULL and temps; conditions over numbers, BOOLEAN channels and VARCHAR predicates
VALUES = {
    "bigint": [ops.If(POS, call(abi.EX_DIV, Y, X)), ops.Coalesce(X, Y, K(0)), ops.If(PROMO, X, K(0)),
               call(abi.EX_ADD, ops.Case([(P, X), (POS, Y)], K(1)), K(1)), ops.Switch(X, [(K(1), Y), (K(2), K(3))], X), ops.NullIf(Y, X)],
    "double": [ops.If(P, F, K(0.0, D)), ops.Coalesce(F, call(abi.EX_CAST_BIGINT_TO_DOUBLE, X)), ops.NullIf(X, F, compare_as=D),
               call(abi.EX_DIV, K(1.0, D), ops.NullIf(F, K(0.0, D)))],
    "boolean": [ops.If(POS, P, K(False, BOOL)), ops.Coalesce(P, call(abi.EX_GT, X, Y)), ops.If(P, ops.Null(BOOL), call(abi.EX_IS_NULL, F))],
    "short_decimal": [ops.If(POS, SD, K(0, DEC, (12, 2))), ops.Coalesce(SD, ops.Const(5, DEC, (12, 2))), ops.NullIf(SD, K(0, DEC, (12, 2))),
                      ops.If(PROMO, call(abi.EX_ADD, SD, SD), ops.Null(DEC, (13, 2)))],
    "long_decimal": [ops.If(P, LD, ops.Null(DEC, (38, 6))), ops.Coalesce(LD, ops.Const(10 ** 30, DEC, (38, 6))),
                     ops.If(POS, call(abi.EX_MUL, SD, SD), K(0, DEC, (25, 4))), ops.NullIf(LD, ops.Const(-1, DEC, (38, 6)))],
}
FILTERS = [call(abi.EX_GT, ops.Coalesce(X, K(0)), K(1)), ops.If(P, call(abi.EX_LT, F, K(2.0, D)), PROMO),
           call(abi.EX_GT, ops.If(POS, SD, ops.Const(0, DEC, (12, 2))), ops.Const(100, DEC, (12, 2)))]


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


@pytest.mark.parametrize("nullable_mask", [0, 0b1111111])
@pytest.mark.parametrize("form", ["chunked", "selection_vector", "no_filter"])
@pytest.mark.parametrize("vt", sorted(VALUES))
def test_every_vtype_compiles(vt, form, nullable_mask):
    exprs = VALUES[vt]
    filt = FILTERS[len(vt) % len(FILTERS)]
    if form == "chunked":
        prog = ops.PageProcessorProgram(filt, [0, 3] + exprs)
    elif form == "selection_vector":
        prog = ops.PageProcessorProgram(filt, [5] + exprs)      # a VARCHAR pass-through channel: the selection-vector form only
    else:
        prog = ops.PageProcessorProgram(None, exprs + [1])
    assert any(op in (abi.EX_IF, abi.EX_COALESCE) for op, *_ in prog.insns)
    st, size, src = _selftest(prog, nullable_mask)
    _ok(st, src)
    assert size > 1000
    assert ("tg_fp_project_chunks_jit" in src) == (form == "chunked")
    n_if = sum(1 for op, *_ in prog.insns if op == abi.EX_IF)
    n_dec = sum(1 for i, (op, *_r) in enumerate(prog.insns) if op == abi.EX_IF and prog.signatures[i] is not None)
    assert src.count("vm_apply(%d, " % abi.EX_IF) + src.count("vm_apply_dec(%d, " % abi.EX_IF) >= n_if * (2 if form == "chunked" else 1)
    if vt == "long_decimal":
        assert "th" in src and n_dec


def test_decimal_condition_is_read_as_a_word():
    """the BOOLEAN condition of a DECIMAL IF is a plain word (la = 0), never a (high, low) pair of the decimal operand loader.  This checks
    the generated source only; test_gpu_conditionals.test_boolean_channel_condition_of_decimal_if runs the same shape through create and
    add_input (whose channel checks the self-test does not reach) in every form"""
    prog = ops.PageProcessorProgram(None, [ops.If(P, LD, ops.Null(DEC, (38, 6)))])
    st, _, src = _selftest(prog, 0b10100)
    _ok(st, src)
    assert "DVal{u128_sx(c2), c2n}" in src and "ch2" not in src
    assert "DVal{U128{(unsigned long long)ch4, (unsigned long long)c4}, c4n}" in src
    assert re.search(r"const DDec dd = \{1, 0, 1, 1, 1,", src)


def _agg_selftest(pre, num_keys, aggs, types, nullable_mask):
    lib = abi.load_library()
    keys = (C.c_int32 * 1)(0)
    fns = (abi.AggFn * len(aggs))()
    for i, (f, ch) in enumerate(aggs):
        fns[i].function, fns[i].input_channel, fns[i].mask_channel = f, ch, -1
    spec = abi.AggSpec(num_keys, C.cast(keys, C.POINTER(C.c_int32)) if num_keys else None, abi.STEP_SINGLE, len(aggs),
                       C.cast(fns, C.POINTER(abi.AggFn)), 16, 0, C.pointer(pre.struct))
    t = (C.c_int32 * len(types))(*types)
    n = C.c_int64()
    buf = C.create_string_buffer(1 << 20)
    st = lib.tgpu_jit_selftest_agg(C.byref(spec), t, len(types), nullable_mask, C.byref(n), buf, len(buf))
    return st, buf.value.decode(errors="replace")


PRE_TYPES = [abi.INT8, abi.INT64, abi.FLOAT64, abi.INT8, abi.INT64]          # key, BIGINT, DOUBLE, BOOLEAN, BIGINT
PK, PX, PF, PP, PY = ops.Col(0, B), ops.Col(1, B), ops.Col(2, D), ops.Col(3, BOOL), ops.Col(4, B)


@pytest.mark.parametrize("vec", [False, True])
@pytest.mark.parametrize("nullable_mask", [0, 0b11110])
@pytest.mark.parametrize("kernel", ["keyed", "global"])
def test_pre_stage_compiles(monkeypatch, kernel, nullable_mask, vec):
    """sum(IF(x > 5, f, 0.0)), count(COALESCE(x, y)), min(IF(p, x, NULL)) and count(IF(...BOOLEAN...)) behind a filter with a COALESCE:
    tg_agg_small_jit with tg_agg_general_jit (one source), or tg_agg_global_jit"""
    if vec:
        monkeypatch.setenv("TGPU_JIT_SELFTEST_VEC", "1")
    else:
        monkeypatch.delenv("TGPU_JIT_SELFTEST_VEC", raising=False)
    projs = [ops.If(call(abi.EX_GT, PX, K(5)), PF, K(0.0, D)), ops.Coalesce(PX, PY), ops.If(PP, PX), ops.Coalesce(PP, call(abi.EX_LT, PX, PY))]
    pre = ops.PageProcessorProgram(call(abi.EX_GE, ops.Coalesce(PY, K(0)), K(-5)), ([0] if kernel == "keyed" else []) + projs)
    base = 1 if kernel == "keyed" else 0
    aggs = [(abi.AGG_SUM, base), (abi.AGG_COUNT, base + 1), (abi.AGG_MIN, base + 2), (abi.AGG_COUNT, base + 3)]
    st, src = _agg_selftest(pre, 1 if kernel == "keyed" else 0, aggs, PRE_TYPES, nullable_mask)
    _ok(st, src)
    names = ("tg_agg_small_jit", "tg_agg_general_jit") if kernel == "keyed" else ("tg_agg_global_jit",)
    assert all(n in src for n in names)
    assert "vm_apply(%d, " % abi.EX_IF in src and "vm_apply(%d, " % abi.EX_COALESCE in src


def _count_aliased(src):
    """number of ACC_NONNULL accumulators the generated kernel keeps (count(x) over a never-NULL x aliases count(*) instead)"""
    acc = re.search(r"void accumulate\(.*?\n  \}\n", src, flags=re.S).group(0)
    return sum(1 for k in re.findall(r"acc_update_private\((\d+), ", acc) if int(k) == 1)


@pytest.mark.parametrize("case", ["if_both_never_null", "if_else_null", "if_then_nullable", "coalesce_one_never_null", "coalesce_both_nullable"])
def test_never_null_rule(case):
    """count(IF(c, a, b)) may alias count(*) only when a and b are never NULL; count(COALESCE(a, b)) when either is never NULL"""
    e, nullable_mask, aliased = {
        "if_both_never_null": (ops.If(PP, PX, PY), 0, True),
        "if_else_null": (ops.If(PP, PX), 0, False),
        "if_then_nullable": (ops.If(PP, PX, PY), 0b00010, False),
        "coalesce_one_never_null": (ops.Coalesce(PX, PY), 0b00010, True),
        "coalesce_both_nullable": (ops.Coalesce(PX, PY), 0b10010, False),
    }[case]
    pre = ops.PageProcessorProgram(None, [0, e])
    st, src = _agg_selftest(pre, 1, [(abi.AGG_COUNT, 1)], PRE_TYPES, nullable_mask)
    _ok(st, src)
    assert _count_aliased(src) == (0 if aliased else 1), src[-2000:]


# ---- refusals ----------------------------------------------------------------------------------------------------------------------
CONST, COL, TEMP, NONE, NUL = abi.OPND_CONST, abi.OPND_COLUMN, abi.OPND_TEMP, abi.OPND_NONE, abi.OPND_NULL


def _raw_program(insns, projections=((1, 0, B),)):
    p = ops.PageProcessorProgram(None, [0])
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
    # a VARCHAR result: NOT_SUPPORTED (a view has one static source), for IF and COALESCE alike
    assert st(_raw_program([(abi.EX_IF, S, 0, (COL, 2, 0), (COL, 5, 0), (NUL, 0, 0))], [(1, 0, S)])) == abi.ERR_NOT_SUPPORTED
    assert st(_raw_program([(abi.EX_COALESCE, S, 0, (COL, 5, 0), (CONST, 0, 0), (NONE, 0, 0))], [(1, 0, S)])) == abi.ERR_NOT_SUPPORTED
    # a condition that is not BOOLEAN, and a branch temp of another type: INVALID_ARGUMENT
    assert st(ops.PageProcessorProgram(None, [ops.If(call(abi.EX_ADD, X, K(1)), X, Y)])) == abi.ERR_INVALID_ARGUMENT
    assert st(_raw_program([(abi.EX_CAST_BIGINT_TO_DOUBLE, B, 1, (COL, 0, 0), (NONE, 0, 0), (NONE, 0, 0)),
                            (abi.EX_IF, B, 0, (COL, 2, 0), (TEMP, 1, 0), (COL, 0, 0))])) == abi.ERR_INVALID_ARGUMENT
    assert st(_raw_program([(abi.EX_COALESCE, B, 0, (COL, 0, 0), (NONE, 0, 0), (NONE, 0, 0))])) == abi.ERR_INVALID_ARGUMENT
    # DECIMAL branches of two types, or a result of a third: INVALID_ARGUMENT
    assert st(ops.PageProcessorProgram(None, [ops.If(P, SD, ops.Const(1, DEC, (12, 3)))])) == abi.ERR_INVALID_ARGUMENT
    assert st(ops.PageProcessorProgram(None, [ops.Coalesce(SD, ops.Const(1, DEC, (13, 2)))])) == abi.ERR_INVALID_ARGUMENT
    assert st(ops.PageProcessorProgram(None, [ops.If(P, LD, SD)])) == abi.ERR_INVALID_ARGUMENT
    # a DECIMAL condition is not BOOLEAN
    assert st(ops.PageProcessorProgram(None, [ops.If(call(abi.EX_ADD, SD, SD), X, Y)])) == abi.ERR_INVALID_ARGUMENT
    # the pre-stage refuses DECIMAL (NOT_SUPPORTED), join filters refuse IF and COALESCE (NOT_SUPPORTED)
    pre = ops.PageProcessorProgram(None, [0, ops.If(PP, ops.Col(1, DEC, (12, 2)), ops.Const(0, DEC, (12, 2)))])
    assert _agg_selftest(pre, 1, [(abi.AGG_COUNT, 1)], PRE_TYPES, 0)[0] == abi.ERR_NOT_SUPPORTED
    lib = abi.load_library()
    t = (C.c_int32 * len(PRE_TYPES))(*PRE_TYPES)
    n = C.c_int64()
    buf = C.create_string_buffer(1 << 16)
    for f in (call(abi.EX_GT, ops.If(PP, PX, PY), K(3)), call(abi.EX_EQ, ops.Coalesce(PX, PY), PY)):
        jf = ops.PageProcessorProgram(f, [])
        assert lib.tgpu_jit_selftest_join_filter(C.byref(jf.struct), 2, t, len(PRE_TYPES), 0, C.byref(n), buf, len(buf)) == abi.ERR_NOT_SUPPORTED
    # numeric IF / COALESCE in a join filter is refused, not wrongly evaluated, also at create
    ctx_free = ops.PageProcessorProgram(call(abi.EX_GT, ops.Coalesce(PX, PY), K(3)), [])
    assert lib.tgpu_jit_selftest_join_filter(C.byref(ctx_free.struct), 2, t, len(PRE_TYPES), 0, C.byref(n), buf, len(buf)) == abi.ERR_NOT_SUPPORTED


# ---- lowering ------------------------------------------------------------------------------------------------------------------------
def test_switch_value_is_emitted_once_and_read_by_every_eq():
    v = call(abi.EX_ADD, X, Y)
    prog = ops.PageProcessorProgram(None, [ops.Switch(v, [(K(1), K(10)), (K(2), K(20)), (K(3), K(30))], K(0))])
    adds = [i for i in prog.insns if i[0] == abi.EX_ADD]
    assert len(adds) == 1
    t = adds[0][2]
    eqs = [i for i in prog.insns if i[0] == abi.EX_EQ]
    assert len(eqs) == 3 and all(i[3] == (TEMP, t, 0) for i in eqs)       # value is the FIRST operand of each EQ
    # the temp is not overwritten before its last reader
    last = max(k for k, i in enumerate(prog.insns) if i[0] == abi.EX_EQ)
    assert all(i[2] != t for i in prog.insns[1:last])


def test_nullif_reads_its_first_argument_twice():
    a = call(abi.EX_MUL, X, Y)
    prog = ops.PageProcessorProgram(None, [ops.NullIf(a, F, compare_as=D)])
    ops_ = [i[0] for i in prog.insns]
    assert ops_ == [abi.EX_MUL, abi.EX_CAST_BIGINT_TO_DOUBLE, abi.EX_EQ, abi.EX_IF]
    t = prog.insns[0][2]
    assert prog.insns[1][3] == (TEMP, t, 0) and prog.insns[3][5] == (TEMP, t, 0) and prog.insns[3][4] == (NUL, 0, 0)
    assert prog.insns[1][2] != t and prog.insns[2][2] != t


def test_temps_are_freed_after_the_last_reader():
    """a temp read twice stays live between its readers; read once, it is free for the next instruction as before"""
    v = call(abi.EX_ADD, X, Y)
    prog = ops.PageProcessorProgram(None, [call(abi.EX_MUL, call(abi.EX_SUB, v, K(1)), call(abi.EX_ADD, v, K(2)))])
    assert [i[0] for i in prog.insns] == [abi.EX_ADD, abi.EX_SUB, abi.EX_ADD, abi.EX_MUL]
    t = prog.insns[0][2]
    assert prog.insns[1][2] != t                  # v is still needed by the second reader
    assert prog.insns[2][3] == (TEMP, t, 0)
    one_reader = ops.PageProcessorProgram(None, [call(abi.EX_SUB, call(abi.EX_ADD, X, Y), K(1))])
    assert one_reader.insns[1][2] == one_reader.insns[0][2]


def test_long_case_hits_the_temp_limit():
    whens = [(call(abi.EX_GT, X, K(k)), call(abi.EX_ADD, Y, K(k))) for k in range(3)]
    ops.PageProcessorProgram(None, [ops.Case(whens, K(0))])
    whens = [(call(abi.EX_GT, X, K(k)), call(abi.EX_ADD, Y, K(k))) for k in range(5)]
    with pytest.raises(ValueError):
        ops.PageProcessorProgram(None, [ops.Case(whens, K(0))])


def test_program_past_64_instructions_is_refused():
    e = X
    for k in range(65):
        e = call(abi.EX_ADD, e, K(k))
    with pytest.raises(ValueError):
        ops.PageProcessorProgram(None, [e])


def test_abi_values_match_the_header():
    header = open(os.path.join(ROOT, "include", "trino_gpu.h")).read()
    assert int(re.search(r"TGPU_EX_IF = (\d+)", header).group(1)) == abi.EX_IF
    assert int(re.search(r"TGPU_EX_COALESCE = (\d+)", header).group(1)) == abi.EX_COALESCE
    lib_src = open(os.path.join(ROOT, "trino_b200", "csrc", "device_lib.cuh")).read()
    assert "TGD_EX_IF = %d, TGD_EX_COALESCE = %d" % (abi.EX_IF, abi.EX_COALESCE) in lib_src
