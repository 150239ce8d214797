"""The join filter kernels specialised with NVRTC (tg_jf_positions_jit / tg_jf_pairs_jit) compile for sm_90a without a GPU.
A join filter reads the join-sources layout: build channels at the build position, probe channels at the probe row.  The launches
are covered by tests/test_gpu_join_filter.py."""
import ctypes as C

import pytest

from trino_b200 import abi
from trino_b200 import operators as ops

B, D, BOOL = abi.V_BIGINT, abi.V_DOUBLE, abi.V_BOOLEAN

# build layout: [orderkey BIGINT, orderdate INTEGER, totalprice DOUBLE]; probe layout: [orderkey BIGINT, shipdate INTEGER, flag BOOLEAN, qty DOUBLE]
TYPES = (abi.INT64, abi.INT32, abi.FLOAT64, abi.INT64, abi.INT32, abi.INT8, abi.FLOAT64)
NB = 3


def _selftest(filt, nullable_mask, num_build_channels=NB, types=TYPES, projections=()):
    lib = abi.load_library()
    prog = ops.PageProcessorProgram(filt, list(projections))
    t = (C.c_int32 * len(types))(*types)
    n = C.c_int64()
    buf = C.create_string_buffer(1 << 16)
    st = lib.tgpu_jit_selftest_join_filter(C.byref(prog.struct), num_build_channels, t, len(types), nullable_mask, C.byref(n), buf, len(buf))
    return st, n.value, buf.value.decode()


def _date_window():
    # l_shipdate - o_orderdate BETWEEN 0 AND 121
    return ops.Call(abi.EX_BETWEEN, ops.Call(abi.EX_SUB, ops.Col(4, B), ops.Col(1, B)), ops.Const(0, B), ops.Const(121, B))


def _mixed():
    # (l_quantity < 0.2 * o_totalprice AND flag) OR l_orderkey <> o_orderkey
    lhs = ops.Call(abi.EX_AND, ops.Call(abi.EX_LT, ops.Col(6, D), ops.Call(abi.EX_MUL, ops.Const(0.2, D), ops.Col(2, D))), ops.Col(5, BOOL))
    return ops.Call(abi.EX_OR, lhs, ops.Call(abi.EX_NE, ops.Col(3, B), ops.Col(0, B)))


@pytest.mark.parametrize("nullable_mask", [0, 0b0000010, 0b0010000, 0b1111111])
def test_join_filter_kernels_compile(nullable_mask):
    st, size, src = _selftest(_date_window(), nullable_mask)
    if st == abi.ERR_NOT_SUPPORTED:
        pytest.skip("NVRTC not installed: " + src)
    assert st == 0, src
    assert size > 1000
    assert "tg_jf_positions_jit" in src and "tg_jf_pairs_jit" in src
    # build channel 1 at the build position, probe channel 4 - 3 = 1 at the probe row
    assert "tg_load_elem<4>(cols.cols[1].data, b)" in src and "tg_load_elem<4>(cols.cols[4].data, p)" in src
    assert ("tg_valid(cols.cols[1].validity, b)" in src) == bool(nullable_mask & 0b10)
    assert ("tg_valid(cols.cols[4].validity, p)" in src) == bool(nullable_mask & 0b10000)
    assert "cols.cols[0]" not in src and "cols.cols[3]" not in src     # channels the filter does not read are not loaded


@pytest.mark.parametrize("nullable_mask", [0, 0b1100101])
def test_mixed_filter_reads_both_sides(nullable_mask):
    st, size, src = _selftest(_mixed(), nullable_mask)
    if st == abi.ERR_NOT_SUPPORTED:
        pytest.skip("NVRTC not installed: " + src)
    assert st == 0, src
    for c, side, elem in ((0, "b", 8), (2, "b", 8), (3, "p", 8), (5, "p", 1), (6, "p", 8)):
        assert f"tg_load_elem<{elem}>(cols.cols[{c}].data, {side})" in src
        assert (f"tg_valid(cols.cols[{c}].validity, {side})" in src) == bool(nullable_mask >> c & 1)


def test_probe_only_and_build_only_layouts():
    # every channel a probe channel (num_build_channels = 0), and every channel a build channel
    filt = ops.Call(abi.EX_GT, ops.Col(1, B), ops.Const(7, B))
    for nb, side in ((0, "p"), (len(TYPES), "b")):
        st, _, src = _selftest(filt, 0b10, num_build_channels=nb)
        if st == abi.ERR_NOT_SUPPORTED:
            pytest.skip("NVRTC not installed: " + src)
        assert st == 0, src
        assert f"tg_load_elem<4>(cols.cols[1].data, {side})" in src


def test_invalid_programs_are_refused():
    st, _, _ = _selftest(_date_window(), 0, projections=[0])
    assert st == abi.ERR_INVALID_ARGUMENT                     # projections
    st, _, _ = _selftest(_date_window(), 0, num_build_channels=-1)
    assert st == abi.ERR_INVALID_ARGUMENT
    st, _, _ = _selftest(ops.Call(abi.EX_GT, ops.Col(9, B), ops.Const(7, B)), 0)
    assert st == abi.ERR_INVALID_ARGUMENT                     # channel outside the layout
    lib = abi.load_library()
    prog = ops.PageProcessorProgram(None, [ops.Call(abi.EX_ADD, ops.Col(1, B), ops.Const(1, B))])
    t = (C.c_int32 * len(TYPES))(*TYPES)
    n = C.c_int64()
    prog.struct.num_projections = 0                           # no filter_temp
    assert lib.tgpu_jit_selftest_join_filter(C.byref(prog.struct), NB, t, len(TYPES), 0, C.byref(n), None, 0) == abi.ERR_INVALID_ARGUMENT
