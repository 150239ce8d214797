"""The global aggregation kernel (tg_agg_global_jit, AggregationOperator) needs no GPU to compile: generate it for the TPC-H Q6 spec
(num_keys = 0) and compile it for sm_90a with NVRTC, with and without the vector loader and with NULL-able channels.  The keyed kernel
(tg_agg_small_jit, num_keys = 1) likewise, over every argument type."""
import ctypes as C
import re

import pytest

from q6 import INPUT_TYPES, q6_aggregators, q6_program
from trino_b200 import abi


def _selftest(nullable_mask, step=abi.STEP_SINGLE, aggs=None):
    lib = abi.load_library()
    prog = q6_program()
    aggs = aggs or q6_aggregators()
    fns = (abi.AggFn * len(aggs))()
    for i, a in enumerate(aggs):
        fns[i].function, fns[i].input_channel, fns[i].mask_channel = a.function, a.input_channel, a.mask_channel
    spec = abi.AggSpec(0, None, step, len(aggs), C.cast(fns, C.POINTER(abi.AggFn)), 1, 0, C.pointer(prog.struct))
    types = (C.c_int32 * 7)(*INPUT_TYPES)
    n = C.c_int64()
    buf = C.create_string_buffer(1 << 17)
    st = lib.tgpu_jit_selftest_agg(C.byref(spec), types, 7, nullable_mask, C.byref(n), buf, len(buf))
    return st, n.value, buf.value.decode()


def _function(src, name):
    m = re.search(r"void %s\(.*?\n  \}\n" % name, src, flags=re.S)
    assert m, name
    return m.group(0)


@pytest.mark.parametrize("vec", [False, True])
@pytest.mark.parametrize("nullable_mask", [0, 0b0111000])
def test_q6_global_kernel_compiles(monkeypatch, vec, nullable_mask):
    if vec:
        monkeypatch.setenv("TGPU_JIT_SELFTEST_VEC", "1")
    st, size, src = _selftest(nullable_mask)
    if st == abi.ERR_NOT_SUPPORTED:
        pytest.skip("NVRTC not installed: " + src)
    assert st == 0, src
    assert size > 1000
    assert "tg_agg_global_jit" in src and "agg_global_body" in src
    assert ("VEC = true" in src) == vec
    if nullable_mask:
        assert "tg_valid(cols.cols[4].validity" in src


def test_global_kernel_has_no_table_and_no_atomics():
    st, _, src = _selftest(0)
    if st == abi.ERR_NOT_SUPPORTED:
        pytest.skip("NVRTC not installed")
    assert st == 0, src
    for word in ("tkeys", "smem", "__shared__", "atomic", "agg_small_body", "agg_general_body", "tg_agg_small_jit", "accumulate_global", "TGD_EMPTY_KEY", "*pk ="):
        assert word not in src, word
    # register accumulators: every update indexes the accumulator array with a constant at stride 1
    assert re.search(r"acc_update_private\(\d+, acc \+ \d+ \* T, T, ", src)


def test_refuses_what_the_operator_refuses():
    """The hook builds the operator as tgpu_aggregation_create does, so a spec the operator refuses is refused before any source is
    generated: here Q6's sum(revenue) behind a fused pre-stage on a FINAL step, whose input is accumulator state rather than raw rows
    (the kernel itself would plan and compile)"""
    st, _, src = _selftest(0, step=abi.STEP_FINAL, aggs=q6_aggregators()[:1])
    assert st == abi.ERR_INVALID_ARGUMENT
    assert src == ""


# ---- the keyed kernel (tg_agg_small_jit, HashAggregationOperator's path S) over every argument type ----------------------------------
_ELEM = {abi.INT8: 1, abi.INT16: 2, abi.INT32: 4, abi.INT64: 8, abi.FLOAT64: 8}
_LOAD4 = {1: "char4 a = *(const char4*)((const char*)cols.cols[1].data", 2: "short4 a = *(const short4*)((const char*)cols.cols[1].data",
          4: "int4 a = *(const int4*)((const char*)cols.cols[1].data", 8: "const longlong2* p = (const longlong2*)((const char*)cols.cols[1].data"}
# accumulator kinds (device_lib.cuh ACC_*) of each function over an integer / a DOUBLE argument
_KINDS = {abi.AGG_COUNT_STAR: (0, 0), abi.AGG_COUNT: (1, 1), abi.AGG_SUM: (3, 2), abi.AGG_AVG: (9, 2), abi.AGG_MIN: (7, 5), abi.AGG_MAX: (8, 6)}


def _keyed_selftest(arg_type, masked, nullable):
    """page [BIGINT key, argument, BOOLEAN mask]; count(*), count, sum, avg, min and max of the argument, all masked or none"""
    lib = abi.load_library()
    keys = (C.c_int32 * 1)(0)
    fns = (abi.AggFn * len(_KINDS))()
    for i, f in enumerate(_KINDS):
        fns[i].function, fns[i].input_channel, fns[i].mask_channel = f, -1 if f == abi.AGG_COUNT_STAR else 1, 2 if masked else -1
    spec = abi.AggSpec(1, C.cast(keys, C.POINTER(C.c_int32)), abi.STEP_SINGLE, len(_KINDS), C.cast(fns, C.POINTER(abi.AggFn)), 16, 0, None)
    types = (C.c_int32 * 3)(abi.INT64, arg_type, abi.INT8)
    n = C.c_int64()
    buf = C.create_string_buffer(1 << 17)
    st = lib.tgpu_jit_selftest_agg(C.byref(spec), types, 3, 0b110 if nullable else 0, C.byref(n), buf, len(buf))
    return st, buf.value.decode()


@pytest.mark.parametrize("vec", [False, True])
@pytest.mark.parametrize("nullable", [False, True])
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("arg_type", [abi.INT8, abi.INT16, abi.INT32, abi.INT64, abi.FLOAT64], ids=["tinyint", "smallint", "integer", "bigint", "double"])
def test_keyed_kernel_loads_every_argument_type_at_its_width(monkeypatch, arg_type, masked, nullable, vec):
    """tg_agg_small_jit compiles for every argument type, with and without a mask, a validity buffer and the four-row loader; one kernel
    holds all six functions (a compile per function would repeat the same loads 240 times).  The argument is read at its own width
    (tg_load_elem<w>; char4 / short4 / int4 / longlong2 in load4): a load of another width reads the neighbouring rows, and a narrow
    load through an unsigned vector type loses the sign."""
    if vec:
        monkeypatch.setenv("TGPU_JIT_SELFTEST_VEC", "1")
    else:
        monkeypatch.delenv("TGPU_JIT_SELFTEST_VEC", raising=False)
    st, src = _keyed_selftest(arg_type, masked, nullable)
    if st == abi.ERR_NOT_SUPPORTED:
        pytest.skip("NVRTC not installed: " + src)
    assert st == 0, src
    w = _ELEM[arg_type]
    assert "tg_agg_small_jit" in src and ("VEC = true" in src) == vec
    assert "r.c1 = tg_load_elem<%d>(cols.cols[1].data, row);" % w in src
    load4 = _function(src, "load4")
    assert _LOAD4[w] in load4
    assert all(_LOAD4[o] not in load4 for o in _LOAD4 if o != w)
    assert ("r.c1n = !tg_valid(cols.cols[1].validity, row)" in src) == nullable
    acc = re.search(r"void accumulate\(.*?\n  \}\n", src, flags=re.S).group(0)
    updates = re.findall(r"if \((.*)\) acc_update_private\((\d+), ", acc)
    kinds = {int(k) for _, k in updates}
    dbl = arg_type == abi.FLOAT64
    for f, (ki, kd) in _KINDS.items():
        if f == abi.AGG_COUNT and not nullable:
            assert 1 not in kinds          # the non-NULL counter of an argument without NULLs is the row counter
        else:
            assert (kd if dbl else ki) in kinds, (f, kinds)
    for cond, kind in updates:
        assert ("!= 0" in cond) == masked, cond
        assert (" && !vn" in cond) == (nullable and int(kind) != 0), cond


def test_deferred_loads_follow_the_filter():
    """shipdate, quantity and discount feed the filter; extendedprice is read only by the projection, so it is loaded after the filter"""
    st, _, src = _selftest(0)
    if st == abi.ERR_NOT_SUPPORTED:
        pytest.skip("NVRTC not installed")
    assert st == 0, src
    early, late = _function(src, "load_early"), _function(src, "load_late")
    early4, late4 = _function(src, "load4_early"), _function(src, "load4_late")
    for body in (early, early4):
        assert "cols.cols[0]" in body and "cols.cols[3]" in body and "cols.cols[5]" in body and "cols.cols[4]" not in body
    for body in (late, late4):
        assert "cols.cols[4]" in body and "cols.cols[0]" not in body and "cols.cols[5]" not in body
    # the filter function reads only the early columns and returns the filter's verdict
    flt = re.search(r"bool filter\(.*?\n  \}\n", src, flags=re.S).group(0)
    assert "r.c4" not in flt and "return !(tn" in flt
