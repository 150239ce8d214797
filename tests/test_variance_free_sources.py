"""Aggregation programs without a variance aggregate generate the same NVRTC sources as before the variance family existed: the sha256
of the source (and the status) of every spec below, global and keyed, raw and state steps, with and without the vector loader and
NULL-able channels, is pinned in tests/golden/agg_sources_without_variance.json (generated from the library as it was before)."""
import ctypes as C
import hashlib
import json
import os

import pytest

from q6 import INPUT_TYPES, q6_aggregators, q6_program
from trino_b200 import abi
from trino_b200 import operators as ops

A = ops.Aggregator
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "agg_sources_without_variance.json")


def specs():
    out = [("q6", (), INPUT_TYPES, q6_aggregators(), q6_program(), abi.STEP_SINGLE)]
    for t in (abi.INT64, abi.INT32, abi.INT16, abi.INT8, abi.FLOAT64):
        for m in (-1, 2):
            for step in (abi.STEP_SINGLE, abi.STEP_PARTIAL):
                out.append((f"keyed-{t}-{m}-{step}", (0,), [abi.INT64, t, abi.INT8], [A(f, 1, m) for f in range(6)], None, step))
    for t in (abi.INT64, abi.FLOAT64):
        for m in (-1, 1):
            out.append((f"global-{t}-{m}", (), [t, abi.INT8], [A(f, 0, m) for f in (1, 2, 3, 4, 5)], None, abi.STEP_SINGLE))
    out.append(("keyed-final-avg", (0,), [abi.INT64, abi.INT64, abi.FLOAT64], [A(abi.AGG_AVG, 1)], None, abi.STEP_FINAL))
    return out


def generate():
    lib = abi.load_library()
    res = {}
    for vec in (False, True):
        if vec:
            os.environ["TGPU_JIT_SELFTEST_VEC"] = "1"
        else:
            os.environ.pop("TGPU_JIT_SELFTEST_VEC", None)
        for name, keys, types, aggs, pre, step in specs():
            for nm in (0, 0b111):
                fns = (abi.AggFn * len(aggs))()
                for i, a in enumerate(aggs):
                    fns[i].function, fns[i].input_channel, fns[i].mask_channel = a.function, a.input_channel, a.mask_channel
                kc = (C.c_int32 * max(1, len(keys)))(*keys)
                spec = abi.AggSpec(len(keys), C.cast(kc, C.POINTER(C.c_int32)) if keys else None, step, len(aggs), C.cast(fns, C.POINTER(abi.AggFn)),
                                   1, 0, C.pointer(pre.struct) if pre is not None else None)
                ct = (C.c_int32 * len(types))(*types)
                n = C.c_int64()
                buf = C.create_string_buffer(1 << 18)
                st = lib.tgpu_jit_selftest_agg(C.byref(spec), ct, len(types), nm, C.byref(n), buf, len(buf))
                res[f"{name}-vec{int(vec)}-null{nm}"] = [st, hashlib.sha256(buf.value).hexdigest()]
    os.environ.pop("TGPU_JIT_SELFTEST_VEC", None)
    return res


def test_variance_free_sources_are_unchanged():
    want = json.load(open(GOLDEN))["sources"]
    got = generate()
    if all(st == abi.ERR_NOT_SUPPORTED for st, _ in got.values()):
        pytest.skip("NVRTC not installed")
    assert got == want

