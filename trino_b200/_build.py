"""Build recipe for libtrino_gpu.so (sm_90a).

`python -m trino_b200._build` or `__graft_entry__.build()`.  nvcc cross-compiles without a GPU.
The library is built IN-TREE (trino_b200/libtrino_gpu.so) so that the package imports from the repository tree.
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "trino_b200", "csrc")
LIB = os.path.join(ROOT, "trino_b200", "libtrino_gpu.so")
SOURCES = ["core.cu", "join.cu", "groupby.cu", "expr.cu", "partition.cu", "synth.cu", "jit.cu", "serde.cu", "dynfilter.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-fmad=false",            # Java never contracts a*b+c (M/type/DoubleOperators.java:66-86)
    "-Xcompiler", "-fPIC",
    "-I", os.path.join(ROOT, "build"),
    "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
]


def _newer(target, deps):
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(d) <= t for d in deps)


def build_gpu(force=False, verbose=False):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(ROOT, "include", "trino_gpu.h")]
    if not force and _newer(LIB, deps):
        return LIB
    objs = []
    procs = []
    os.makedirs(os.path.join(ROOT, "build"), exist_ok=True)
    # device_lib.cuh is also the prelude of every NVRTC-specialised kernel: embed it as a string literal
    with open(os.path.join(CSRC, "device_lib.cuh")) as f:
        text = f.read()
    assert ')TGJIT"' not in text
    chunks = [text[i:i + 12000] for i in range(0, len(text), 12000)]   # stay under the 64 KiB literal limit
    with open(os.path.join(ROOT, "build", "device_lib_str.inc"), "w") as f:
        f.write("\n".join('R"TGJIT(' + c + ')TGJIT"' for c in chunks) + "\n")
    for src in SOURCES:
        obj = os.path.join(ROOT, "build", src.replace(".cu", ".o"))
        objs.append(obj)
        cmd = [nvcc, *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write(f"--- nvcc {src} failed ---\n{out}\n")
        elif verbose:
            sys.stderr.write(f"--- nvcc {src} ---\n{out}\n")
    if failed:
        raise RuntimeError("nvcc failed")
    cmd = [nvcc, "-shared", "-o", LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a", "-ldl"]
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    build_gpu(force="--force" in sys.argv, verbose=True)
    print(LIB)
