"""CPU-side checks of the C-ABI library: it loads, exports every symbol include/trino_gpu.h declares, and fails
loudly (no CPU fallback) when there is no CUDA device.  No compute calls are made here."""
import ctypes as C
import os
import re

import pytest

from trino_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "trino_gpu.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(tgpu_[a-z0-9_]+)\s*\(", text)))


def test_library_is_built_in_tree():
    assert os.path.exists(abi.LIB_PATH), "run python -m trino_b200._build"


def test_every_declared_symbol_is_exported_and_bound():
    lib = abi.load_library()
    declared = _declared_symbols()
    assert len(declared) >= 45
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in trino_gpu.h but not exported"
        assert name in abi.SIGNATURES, f"{name} has no ctypes signature"
    for name in abi.SIGNATURES:
        assert name in declared, f"{name} bound in abi.py but not declared in trino_gpu.h"


def test_struct_layouts_match_header_expectations():
    assert C.sizeof(abi.Column) == 48
    assert C.sizeof(abi.Page) == 24
    assert C.sizeof(abi.Operand) == 16
    assert C.sizeof(abi.ExprInsn) == 64
    assert C.sizeof(abi.AggFn) == 16


_PAIRS = [("tgpu_column", "Column"), ("tgpu_page", "Page"), ("tgpu_operand", "Operand"), ("tgpu_expr_insn", "ExprInsn"), ("tgpu_in_list", "InList"),
          ("tgpu_projection", "Projection"), ("tgpu_expr_program", "ExprProgram"), ("tgpu_agg_fn", "AggFn"), ("tgpu_agg_spec", "AggSpec"),
          ("tgpu_join_build_spec", "JoinBuildSpec"), ("tgpu_join_probe_spec", "JoinProbeSpec"), ("tgpu_partition_spec", "PartitionSpec"), ("tgpu_domain", "Domain")]


def test_ctypes_structs_have_the_layout_the_c_compiler_gives_the_header(tmp_path):
    """Every struct of include/trino_gpu.h as gcc lays it out (size and the offset of every field, in declaration order) against the ctypes
    mirror in trino_b200/abi.py: a field added to one side only, or in another position, fails here and not as a wild pointer on the GPU box."""
    import shutil
    import subprocess
    gcc = shutil.which("gcc") or shutil.which("cc")
    if not gcc:
        pytest.skip("no C compiler")
    header = open(os.path.join(ROOT, "include", "trino_gpu.h")).read()
    text = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "trino_gpu.h"', "int main(void) {"]
    fields = {}
    for cname, _ in _PAIRS:
        m = re.search(r"typedef struct %s \{(.*?)\} %s;" % (cname, cname), text, flags=re.S)
        assert m, cname
        names = []
        body = re.sub(r"\{[^{}]*\}", "", m.group(1))          # an anonymous union keeps only its member name
        for decl in body.split(";"):
            decl = decl.strip()
            if not decl:
                continue
            for part in decl.split(","):                     # `tgpu_operand a, b, c`
                name = re.search(r"([A-Za-z_][A-Za-z0-9_]*)\s*(\[[^\]]*\])?$", part.strip())
                assert name, (cname, decl)
                names.append(name.group(1))
        fields[cname] = names
        lines.append('printf("%s %%zu", sizeof(%s));' % (cname, cname))
        for f in names:
            lines.append('printf(" %%zu", offsetof(%s, %s));' % (cname, f))
        lines.append('printf("\\n");')
    lines.append("return 0; }")
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run([gcc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.strip().splitlines()
    assert len(out) == len(_PAIRS)
    for line, (cname, pyname) in zip(out, _PAIRS):
        parts = line.split()
        assert parts[0] == cname
        size, offsets = int(parts[1]), [int(x) for x in parts[2:]]
        st = getattr(abi, pyname)
        assert C.sizeof(st) == size, (cname, C.sizeof(st), size)
        py_fields = [f[0] for f in st._fields_]
        assert len(py_fields) == len(fields[cname]), (cname, py_fields, fields[cname])
        assert [getattr(st, f).offset for f in py_fields] == offsets, (cname, py_fields, fields[cname])


def test_status_names_are_trino_error_codes():
    lib = abi.load_library()
    assert lib.tgpu_status_name(abi.ERR_INSUFFICIENT_RESOURCES) == b"GENERIC_INSUFFICIENT_RESOURCES"
    assert lib.tgpu_status_name(abi.ERR_NUMERIC_VALUE_OUT_OF_RANGE) == b"NUMERIC_VALUE_OUT_OF_RANGE"
    assert lib.tgpu_status_name(abi.ERR_DIVISION_BY_ZERO) == b"DIVISION_BY_ZERO"
    assert lib.tgpu_status_name(abi.ERR_INVALID_CAST_ARGUMENT) == b"INVALID_CAST_ARGUMENT"


def test_no_cpu_fallback_without_device():
    lib = abi.load_library()
    if lib.tgpu_device_count() > 0:
        pytest.skip("a CUDA device is present")
    h = C.c_void_p()
    st = lib.tgpu_ctx_create(0, C.byref(h))
    assert st == abi.ERR_CUDA and not h.value
    assert b"no CPU fallback" in lib.tgpu_last_error(None)
    from trino_b200.operators import Context
    with pytest.raises(abi.TrinoGpuError):
        Context(0)


def test_product_does_not_reference_the_oracle():
    # the product path must never import, link or call anything under oracle/
    for dirpath, _, files in os.walk(os.path.join(ROOT, "trino_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
                text = open(os.path.join(dirpath, f), errors="ignore").read()
                assert "liboracle" not in text and "oracle_lib" not in text and "oracle/oracle" not in text, os.path.join(dirpath, f)
    out = os.popen(f"ldd {abi.LIB_PATH}").read()
    assert "oracle" not in out
