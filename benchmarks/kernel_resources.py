"""Registers / stack (spills) / static shared memory of every kernel in the shipped library (cuobjdump -res-usage).
    python benchmarks/kernel_resources.py > profiles/r2_kernel_resources.md"""
import re
import subprocess
from pathlib import Path

LIB = Path(__file__).resolve().parent.parent / "fadtk_b200" / "csrc" / "libfadtk_b200.so"
txt = subprocess.run(["cuobjdump", "-res-usage", str(LIB)], capture_output=True, text=True).stdout
rows, cur = [], None
for line in txt.splitlines():
    m = re.search(r"Function (\S+):", line)
    if m:
        cur = m.group(1)
        continue
    m = re.search(r"REG:(\d+) STACK:(\d+) SHARED:(\d+)", line)
    if m and cur:
        rows.append((cur, int(m.group(1)), int(m.group(2)), int(m.group(3))))
        cur = None
names = subprocess.run(["c++filt"] + [r[0] for r in rows], capture_output=True, text=True).stdout.splitlines()
print("# Kernel resource audit (`cuobjdump -res-usage fadtk_b200/csrc/libfadtk_b200.so`, sm_90a)\n")
print("Registers per thread, stack bytes (spills / local arrays), static shared memory; dynamic shared memory (conv_gemm,")
print("attention_wgmma, logmel) is set at launch.  The fp64 tensor-pipe kernels (`dgemm_strided_kernel`,")
print("`stats_dmma_kernel<__half | double>`, `song_stats_dmma_kernel`) stay at <= 128 registers for two CTAs per SM.\n")
print("| kernel | registers | stack bytes | static smem |\n|---|---|---|---|")
for (m, r, st, sh), n in sorted(zip(rows, names), key=lambda t: t[1]):
    n = re.sub(r"\(.*", "", n.replace("(anonymous namespace)::", "")).replace("void ", "")
    print(f"| `{n}` | {r} | {st} | {sh} |")
