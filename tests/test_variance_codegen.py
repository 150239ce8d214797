"""The variance family in the global aggregation kernel (tg_agg_global_jit) needs no GPU to generate and compile: every argument type, with
and without a mask and a NULL-able input, the state input of FINAL / INTERMEDIATE steps, and a variance over a fused pre-stage temp.
The keyed path-S kernel likewise.  REAL, VARCHAR and long-DECIMAL arguments are refused before any source is generated."""
import ctypes as C
import re

import pytest

from trino_b200 import abi
from trino_b200 import operators as ops

A = ops.Aggregator
VAR_FNS = (abi.AGG_VAR_SAMP, abi.AGG_VAR_POP, abi.AGG_STDDEV_SAMP, abi.AGG_STDDEV_POP)
ACC_VAR_F64, ACC_VAR_I64, ACC_VAR_STATE = 10, 11, 12          # device_lib.cuh AccKind


def _selftest(types, aggs, step=abi.STEP_SINGLE, nullable_mask=0, keys=(), pre=None):
    lib = abi.load_library()
    fns = (abi.AggFn * len(aggs))()
    for i, a in enumerate(aggs):
        fns[i].function, fns[i].input_channel, fns[i].mask_channel = a.function, a.input_channel, a.mask_channel
    kc = (C.c_int32 * max(1, len(keys)))(*keys)
    spec = abi.AggSpec(len(keys), C.cast(kc, C.POINTER(C.c_int32)) if keys else None, step, len(aggs), C.cast(fns, C.POINTER(abi.AggFn)), 1, 0,
                       C.pointer(pre.struct) if pre is not None else None)
    ct = (C.c_int32 * len(types))(*types)
    n = C.c_int64()
    buf = C.create_string_buffer(1 << 17)
    st = lib.tgpu_jit_selftest_agg(C.byref(spec), ct, len(types), nullable_mask, C.byref(n), buf, len(buf))
    return st, n.value, buf.value.decode()


def _ok(st, src):
    if st == abi.ERR_NOT_SUPPORTED and "NVRTC" in src:
        pytest.skip("NVRTC not installed: " + src)
    assert st == 0, src


@pytest.mark.parametrize("arg_type", [abi.INT64, abi.INT32, abi.INT16, abi.INT8, abi.FLOAT64])
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("nullable", [False, True])
def test_every_argument_type_compiles(monkeypatch, arg_type, masked, nullable):
    monkeypatch.setenv("TGPU_JIT_SELFTEST_VEC", "1")
    mask = 1 if masked else -1
    st, size, src = _selftest([arg_type, abi.INT8], [A(f, 0, mask) for f in VAR_FNS], nullable_mask=0b11 if nullable else 0)
    _ok(st, src)
    assert size > 1000 and "tg_agg_global_jit" in src
    kind = ACC_VAR_F64 if arg_type == abi.FLOAT64 else ACC_VAR_I64
    # the four functions share ONE three-word accumulator: one update per row
    updates = re.findall(r"if \((.*)\) acc_update_private\((\d+), acc \+ (\d+) \* T, T, v(\d+)\);", src)
    assert [(int(k), int(w)) for _, k, w, _ in updates] == [(kind, 0)], src
    cond, v = updates[0][0], updates[0][3]
    assert "v%s = c0;" % v in src
    assert (" != 0" in cond) == masked
    assert ("!vn%s" % v in cond.replace("(!vn%s && v%s != 0)" % (1 - int(v), 1 - int(v)), "")) == nullable
    assert re.search(r"case 1: return 13;\n\s+case 2: return 14;", src)


@pytest.mark.parametrize("step", [abi.STEP_FINAL, abi.STEP_INTERMEDIATE])
@pytest.mark.parametrize("nullable", [False, True])
def test_state_input_merges_count_mean_and_m2(step, nullable):
    # state columns: count BIGINT, m2 DOUBLE, mean DOUBLE
    st, _, src = _selftest([abi.INT64, abi.FLOAT64, abi.FLOAT64], [A(f, 0) for f in VAR_FNS], step=step, nullable_mask=0b111 if nullable else 0)
    _ok(st, src)
    calls = re.findall(r"if \((.*)\) acc_var_merge_private\(acc \+ 0 \* T, T, v0, v(\d), v(\d)\);", src)
    assert len(calls) == 1, src
    cond, mean_src, m2_src = calls[0]
    assert ("!vn0" in cond) == nullable
    # sources are numbered in the order they are read: count (channel 0), m2 (channel 1), mean (channel 2)
    assert "v1 = c1;" in src and "v2 = c2;" in src
    assert (mean_src, m2_src) == ("2", "1")
    assert "acc_update_private" not in src


def test_over_a_fused_pre_stage_temp():
    """var_pop(l_extendedprice * (1 - l_discount)) behind a filter on l_quantity: the projected DOUBLE temp feeds the accumulator"""
    X = ops
    prog = X.PageProcessorProgram(X.Call(abi.EX_LT, X.Col(0, abi.V_DOUBLE), X.Const(24.0, abi.V_DOUBLE)),
                                  [X.Call(abi.EX_MUL, X.Col(1, abi.V_DOUBLE), X.Call(abi.EX_SUB, X.Const(1.0, abi.V_DOUBLE), X.Col(2, abi.V_DOUBLE))),
                                   X.Col(3, abi.V_BIGINT)])
    st, _, src = _selftest([abi.FLOAT64, abi.FLOAT64, abi.FLOAT64, abi.INT64], [A(abi.AGG_VAR_POP, 0), A(abi.AGG_STDDEV_SAMP, 1)], pre=prog)
    _ok(st, src)
    ups = re.findall(r"acc_update_private\((\d+), acc \+ (\d+) \* T, T, v(\d+)\);", src)
    assert [int(k) for k, _, _ in ups] == [ACC_VAR_F64, ACC_VAR_I64], src
    assert [int(w) for _, w, _ in ups] == [0, 3]


@pytest.mark.parametrize("arg_type", [abi.FLOAT32, abi.UTF8, abi.INT128])
def test_real_varchar_and_long_decimal_arguments_are_refused(arg_type):
    st, _, src = _selftest([arg_type], [A(abi.AGG_VAR_SAMP, 0)])
    assert st == abi.ERR_NOT_SUPPORTED and src == ""


@pytest.mark.parametrize("arg_type", [abi.INT64, abi.INT16, abi.FLOAT64])
@pytest.mark.parametrize("step", [abi.STEP_SINGLE, abi.STEP_FINAL])
def test_keyed_path_s_kernel_compiles(step, arg_type):
    """tg_agg_small_jit: the same accumulator, at the slot's stride T; the fused-G record form carries no variance (the plan never takes it)"""
    types = [abi.INT64, arg_type] if step == abi.STEP_SINGLE else [abi.INT64, abi.INT64, abi.FLOAT64, abi.FLOAT64]
    st, _, src = _selftest(types, [A(f, 1) for f in VAR_FNS], step=step, keys=(0,))
    _ok(st, src)
    assert "tg_agg_small_jit" in src
    if step == abi.STEP_SINGLE:
        kind = ACC_VAR_F64 if arg_type == abi.FLOAT64 else ACC_VAR_I64
        assert len(re.findall(r"acc_update_private\(%d, acc \+ 0 \* T, T, v\d+\);" % kind, src)) == 1, src
    else:
        assert len(re.findall(r"acc_var_merge_private\(acc \+ 0 \* T, T, v\d+, v\d+, v\d+\);", src)) == 1, src
    assert "atomic" not in _function(src, "accumulate_global")


def _function(src, name):
    m = re.search(r"void %s\(.*?\n  \}\n" % name, src, flags=re.S)
    assert m, name
    return m.group(0)


def test_state_channels_of_the_wrong_types_are_refused():
    st, _, _ = _selftest([abi.INT64, abi.INT64, abi.FLOAT64], [A(abi.AGG_VAR_POP, 0)], step=abi.STEP_FINAL)
    assert st == abi.ERR_INVALID_ARGUMENT
