"""The NVRTC specialisation path needs no GPU to compile: generate the fused Q1 kernel (and variants with NULL-able
channels) and compile it for sm_90a on the CPU box.  The launch itself is covered by the -m gpu suites."""
import ctypes as C

import pytest

from q1 import q1_aggregators, q1_program
from trino_b200 import abi


def _selftest(nullable_mask, with_pre=True, aggs=None):
    lib = abi.load_library()
    prog = q1_program()
    aggs = aggs or q1_aggregators()
    keys = (C.c_int32 * 2)(0, 1) if with_pre else (C.c_int32 * 2)(1, 2)
    fns = (abi.AggFn * len(aggs))()
    for i, a in enumerate(aggs):
        fns[i].function, fns[i].input_channel, fns[i].mask_channel = a.function, a.input_channel, a.mask_channel
    spec = abi.AggSpec(2, C.cast(keys, C.POINTER(C.c_int32)), abi.STEP_SINGLE, len(aggs), C.cast(fns, C.POINTER(abi.AggFn)), 16, 0,
                       C.pointer(prog.struct) if with_pre else None)
    types = (C.c_int32 * 7)(abi.INT32, abi.INT8, abi.INT8, abi.FLOAT64, abi.FLOAT64, abi.FLOAT64, abi.FLOAT64)
    n = C.c_int64()
    buf = C.create_string_buffer(1 << 16)
    st = lib.tgpu_jit_selftest_agg(C.byref(spec), types, 7, nullable_mask, C.byref(n), buf, len(buf))
    return st, n.value, buf.value.decode()


def test_q1_kernel_compiles_and_drops_redundant_counters():
    st, size, src = _selftest(0)
    if st == abi.ERR_NOT_SUPPORTED:
        pytest.skip("NVRTC not installed: " + src)
    assert st == 0, src
    assert size > 10_000
    assert "A = 6" in src                      # 5 sums + count(*): the 5 non-null counters alias the row counter
    assert "tg_agg_small_jit" in src and "vm_apply(3, 1" in src


def test_vector_loader_variant_compiles(monkeypatch):
    # the kernel launched for 16-byte aligned columns: four consecutive rows per thread through 16-byte loads
    monkeypatch.setenv("TGPU_JIT_SELFTEST_VEC", "1")
    for mask in (0, 0b1111000):
        st, size, src = _selftest(mask)
        if st == abi.ERR_NOT_SUPPORTED:
            pytest.skip("NVRTC not installed")
        assert st == 0, src
        assert "VEC = true" in src and "load4" in src and "const longlong2* p" in src


def test_nullable_channels_keep_their_counters():
    st, size, src = _selftest(0b1111000)      # quantity, extendedprice, discount, tax carry NULLs
    if st == abi.ERR_NOT_SUPPORTED:
        pytest.skip("NVRTC not installed")
    assert st == 0, src
    assert "A = 11" in src
    assert "tg_valid(cols.cols[4].validity" in src


def test_unfused_plan_compiles_too():
    from trino_b200.operators import Aggregator as A
    st, size, src = _selftest(0, with_pre=False, aggs=[A(abi.AGG_SUM, 3), A(abi.AGG_MIN, 4), A(abi.AGG_MAX, 0), A(abi.AGG_COUNT_STAR), A(abi.AGG_AVG, 0)])
    if st == abi.ERR_NOT_SUPPORTED:
        pytest.skip("NVRTC not installed")
    assert st == 0, src


def test_filter_project_kernels_compile():
    lib = abi.load_library()
    prog = q1_program()
    types = (C.c_int32 * 7)(abi.INT32, abi.INT8, abi.INT8, abi.FLOAT64, abi.FLOAT64, abi.FLOAT64, abi.FLOAT64)
    n = C.c_int64()
    buf = C.create_string_buffer(1 << 16)
    st = lib.tgpu_jit_selftest_filter_project(C.byref(prog.struct), types, 7, 0b0010000, C.byref(n), buf, len(buf))
    src = buf.value.decode()
    if st == abi.ERR_NOT_SUPPORTED:
        pytest.skip("NVRTC not installed: " + src)
    assert st == 0, src
    assert "tg_fp_filter_jit" in src and "tg_fp_project_jit" in src
    # fixed-width pass-through channels + a filter: the chunked two-pass form (no selection vector) is generated as well
    assert "tg_fp_filter_chunks_jit" in src and "tg_fp_project_chunks_jit" in src and "out.pass_data[1]" in src
    assert "tg_valid(cols.cols[4].validity" in src and "tg_valid(cols.cols[5].validity" not in src
