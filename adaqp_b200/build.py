"""Build libadaqp_b200.so (sm_90a, H100) in-tree with nvcc.

The shared library is the C-ABI boundary declared in include/adaqp_b200.h.  It is
built next to this file (git-ignored build product).
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(CSRC, "_build")
LIB = os.path.join(HERE, "libadaqp_b200.so")
SOURCES = ["runtime.cu", "quant.cu", "exchange.cu", "spmm.cu", "gemm.cu", "norm.cu", "partition.cu", "gat.cu", "sage_pool.cu",
           "gatv2.cu", "cs.cu"]
HEADERS = [os.path.join(CSRC, "common.cuh"), os.path.join(CSRC, "attn.cuh"),
           os.path.join(os.path.dirname(HERE), "include", "adaqp_b200.h")]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
         "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(verbose: bool = False, force: bool = False, ptxas_info: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    jobs = []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJ, src.replace(".cu", ".o"))
        if force or _stale(o, [s] + HEADERS):
            cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if ptxas_info else []) + ["-c", s, "-o", o]
            jobs.append(cmd)
    def run(cmd):
        if verbose:
            print(" ".join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed:\n{' '.join(cmd)}\n{r.stdout}\n{r.stderr}")
        return r.stderr
    if jobs:
        with ThreadPoolExecutor(max_workers=min(4, len(jobs))) as ex:
            outs = list(ex.map(run, jobs))
        if ptxas_info:
            for o in outs:
                print(o)
    objs = [os.path.join(OBJ, s.replace(".cu", ".o")) for s in SOURCES]
    if force or jobs or _stale(LIB, objs):
        run([NVCC, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"])
    return LIB


if __name__ == "__main__":
    print(build(verbose=True, force="--force" in sys.argv, ptxas_info="--ptxas" in sys.argv))
