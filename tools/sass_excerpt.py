#!/usr/bin/env python
"""SASS evidence: which tensor-core / TMA / warp-reduction instructions the shipped kernels contain.
usage: python tools/sass_excerpt.py [path/to/libcosdata_b200.so]
For each kernel of interest (one instantiation per form) prints the count of every interesting mnemonic and the first
full SASS line it occurs in (cuobjdump -sass of the sm_90a cubin inside the .so)."""
import collections
import re
import subprocess
import sys

SO = sys.argv[1] if len(sys.argv) > 1 else "cosdata_b200/libcosdata_b200.so"
PICK = [
    ("tensor_scan_kernel<4 stages, NG=16, no degenerate rows, f16>  (C2 headline prefilter)", r"tensor_scan_kernelILi4ELi16ELb0ELi0E"),
    ("tensor_scan_kernel<4 stages, NG=16, u8>  (C4 exact integer scores)", r"tensor_scan_kernelILi4ELi16ELb0ELi1E"),
    ("hnsw_search_warp_kernel<f16 chain, no profiling>  (C3/C5)", r"hnsw_search_warp_kernelILi1ELb0E"),
    ("scan_f32_kernel<QB=1>  (exact f32 scan, B=1)", r"scan_f32_kernelILi1ELi2E"),
    ("tc_probe_kernel<u8>  (measured integer tensor peak)", r"tc_probe_kernelILb1E"),
]
WANT = re.compile(r"\b(HGMMA|IGMMA|WARPGROUP|USETMAXREG|UTMALDG|UTMACCTL|UTMAPF|UBLKCP|UBLKPF|SYNCS|REDUX|CREDUX|UCGABAR|FMNMX3?|LDG|LDS|ATOMS|ATOMG|RED|CCTL|PREFETCH|F2FP|HADD2|HFMA2|FFMA|I2FP|I2F|IDP|POPC|SHFL|VOTE|MATCH|NANOSLEEP|BAR|WARPSYNC|MEMBAR|FENCE|ELECT|PLOP3|UCLEA|ACQBULK|ARRIVES)(\.[A-Z0-9_.]+)?")

sass = subprocess.run(["cuobjdump", "-sass", SO], capture_output=True, text=True, check=True).stdout
funcs = collections.OrderedDict()
cur = None
for line in sass.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = m.group(1)
        funcs[cur] = []
    elif cur and "/*" in line and ";" in line:
        funcs[cur].append(line.strip())
print(f"# cuobjdump -sass {SO}: {len(funcs)} kernels, sm_90a\n")
for title, pat in PICK:
    hits = [f for f in funcs if re.search(pat, f)]
    if not hits:
        print(f"## {title}\n   (no such instantiation)\n")
        continue
    f = hits[0]
    counts, first = collections.Counter(), {}
    for ln in funcs[f]:
        body = re.sub(r"/\*[0-9a-f]+\*/", "", ln).strip()
        m = WANT.search(body)
        if m:
            key = m.group(0)
            counts[key] += 1
            first.setdefault(key, body.rstrip(" ;"))
    print(f"## {title}\n   {f}   ({len(funcs[f])} instructions)")
    for key in sorted(counts, key=lambda k: (not k.startswith(("HGMMA", "IGMMA", "WARPGROUP", "USETMAXREG", "UTM", "UBLK", "SYNCS", "REDUX", "CREDUX", "UCGA")), k)):
        print(f"   {counts[key]:5d}  {key:34s} {first[key][:110]}")
    print()
