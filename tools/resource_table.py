#!/usr/bin/env python
"""`cuobjdump -res-usage` of the library as a markdown table.  usage: tools/resource_table.py > resources.md"""
import re
import subprocess

txt = subprocess.run(["cuobjdump", "-res-usage", "trino_b200/libtrino_gpu.so"], capture_output=True, text=True).stdout
rows, fn = [], None
for line in txt.splitlines():
    m = re.search(r"Function (\S+):", line)
    if m:
        fn = m.group(1)
        continue
    m = re.search(r"REG:(\d+) STACK:(\d+) SHARED:(\d+)", line)
    if m and fn:
        rows.append((fn, int(m.group(1)), int(m.group(2)), int(m.group(3))))
        fn = None
names = subprocess.run(["c++filt"] + [r[0] for r in rows], capture_output=True, text=True).stdout.splitlines()
out = []
for (fn, reg, stack, sh), nm in zip(rows, names):
    nm = nm.replace("(anonymous namespace)::", "").split("(")[0].replace("void ", "")
    out.append((nm, reg, stack, sh))
print("# static resource usage (`cuobjdump -res-usage trino_b200/libtrino_gpu.so`, sm_90a, nvcc 12.9 -O3 -fmad=false)\n")
print("Registers, local stack and static shared memory per kernel, and how many 256-thread CTAs the register file (64 K x 32-bit per SM) admits.  "
      "NVRTC kernels (`tg_agg_small_jit`: 76 registers + 49.2 KB dynamic smem for the Q1 program; `tg_agg_general_jit`: `__launch_bounds__(256, 4)`; "
      "`tg_fp_*_jit`: 19 / 32 registers) are compiled at run time and appear in `r02_kernels.md` instead.\n")
print("| kernel | registers | stack B | static smem B | max CTAs/SM by registers (256 thr) |\n|---|---:|---:|---:|---:|")
seen = set()
for nm, reg, stack, sh in sorted(out):
    if nm in seen or nm.startswith("cub::") or nm.startswith("thrust::"):
        continue
    seen.add(nm)
    print("| `%s` | %d | %d | %d | %d |" % (nm, reg, stack, sh, min(8, 65536 // (max(reg, 1) * 256))))
