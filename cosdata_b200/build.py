"""Builds libcosdata_b200.so (sm_90a, H100) in-tree with nvcc.

    python -m cosdata_b200.build [--force] [--verbose]

The shared object and the object files are git-ignored build products.  cudart
is linked statically (nvcc default), so the library shares the primary CUDA
context with any torch in the same process without sharing a runtime instance.
"""
import concurrent.futures
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libcosdata_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
HOST_CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"

GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]   # wgmma, TMA and setmaxnreg: Hopper-only, no other target
FLAGS = [
    "-O3", "-std=c++17", *GENCODE, "-lineinfo",
    "-ccbin", HOST_CXX, "-Xcompiler", "-fPIC,-O2,-Wall", "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
]


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _headers_mtime():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hs.append(os.path.join(HERE, "..", "include", "cosdata_b200.h"))
    return max(os.path.getmtime(h) for h in hs)


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    # objects compiled with other flags (another architecture) are never reused
    stamp = os.path.join(OBJ, "flags.txt")
    want = " ".join([NVCC] + FLAGS)
    if not os.path.exists(stamp) or open(stamp).read() != want:
        force = True
    hm = _headers_mtime()
    jobs = []
    for src in _sources():
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJ, src[:-3] + ".o")
        if force or not os.path.exists(o) or os.path.getmtime(o) < max(os.path.getmtime(s), hm):
            jobs.append((s, o))

    def compile_one(job):
        s, o = job
        cmd = [NVCC] + FLAGS + ["-c", s, "-o", o]
        r = subprocess.run(cmd, capture_output=True, text=True)
        return job, r

    failed = False
    with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        for (s, o), r in ex.map(compile_one, jobs):
            log = os.path.join(OBJ, os.path.basename(s) + ".log")
            with open(log, "w") as f:
                f.write(r.stdout + r.stderr)
            if r.returncode != 0:
                failed = True
                sys.stderr.write(r.stdout + r.stderr)
            elif verbose:
                sys.stderr.write(r.stderr)
    if failed:
        raise RuntimeError("nvcc failed")
    objs = [os.path.join(OBJ, src[:-3] + ".o") for src in _sources()]
    if jobs or force or not os.path.exists(LIB):
        cmd = [NVCC, "-shared", "-ccbin", HOST_CXX, *GENCODE, "-o", LIB] + objs
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed")
    with open(stamp, "w") as f:
        f.write(want)
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(LIB)
