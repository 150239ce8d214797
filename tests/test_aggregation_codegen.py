"""The global aggregation kernel (tg_agg_global_jit, AggregationOperator) needs no GPU to compile: generate it for the TPC-H Q6 spec
(num_keys = 0) and compile it for sm_90a with NVRTC, with and without the vector loader and with NULL-able channels."""
import ctypes as C
import re

import pytest

from q6 import INPUT_TYPES, q6_aggregators, q6_program
from trino_b200 import abi


def _selftest(nullable_mask):
    lib = abi.load_library()
    prog = q6_program()
    aggs = q6_aggregators()
    fns = (abi.AggFn * len(aggs))()
    for i, a in enumerate(aggs):
        fns[i].function, fns[i].input_channel, fns[i].mask_channel = a.function, a.input_channel, a.mask_channel
    spec = abi.AggSpec(0, None, abi.STEP_SINGLE, len(aggs), C.cast(fns, C.POINTER(abi.AggFn)), 1, 0, C.pointer(prog.struct))
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
