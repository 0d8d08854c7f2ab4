"""Build liborp_b200.so IN-TREE with nvcc for sm_90a (H100; no JIT cache, no torch extension machinery).

    python -m orientedreppoints_b200.build [--force] [--verbose]

The shared library is a plain C-ABI library (include/orp_b200.h); the built file lands in
orientedreppoints_b200/lib/, which is git-ignored.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "lib")
LIB = os.path.join(OUT, "liborp_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
         "-Xptxas", "-v", "--threads", "2"]


def _sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _headers():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hs.append(os.path.join(HERE, "..", "include", "orp_b200.h"))
    hs.append(os.path.join(HERE, "..", "include", "orp_b200_dcnv2.h"))
    hs.append(os.path.join(HERE, "..", "include", "orp_b200_swin.h"))
    hs.append(os.path.join(HERE, "..", "include", "orp_b200_group.h"))
    hs.append(os.path.join(HERE, "..", "include", "orp_b200_hrnet.h"))
    hs.append(os.path.join(HERE, "..", "include", "orp_b200_attention.h"))
    hs.append(os.path.join(HERE, "..", "include", "orp_b200_context.h"))
    hs.append(os.path.join(HERE, "..", "include", "orp_b200_carafe.h"))
    return hs


def build(force=False, verbose=False):
    os.makedirs(OUT, exist_ok=True)
    objdir = os.path.join(OUT, "obj")
    os.makedirs(objdir, exist_ok=True)
    hdr_m = max(os.path.getmtime(h) for h in _headers())
    jobs = []
    objs = []
    for src in _sources():
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        if force or not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(src), hdr_m):
            jobs.append((src, obj))

    def compile_one(job):
        src, obj = job
        cmd = [NVCC] + ARCH + FLAGS + ["-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        log = obj[:-2] + ".ptxas.log"
        with open(log, "w") as f:
            f.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s" % (src, r.stdout + r.stderr))
        if verbose:
            print("compiled", os.path.basename(src))
        return obj

    if jobs:
        with ThreadPoolExecutor(max_workers=min(4, len(jobs))) as ex:
            list(ex.map(compile_one, jobs))
    if jobs or force or not os.path.exists(LIB):
        cmd = [NVCC] + ARCH + ["-shared", "-o", LIB] + objs + ["-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n" + r.stdout + r.stderr)
        if verbose:
            print("linked", LIB)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
