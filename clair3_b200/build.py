"""Build libclair3b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python -m clair3_b200.build [--force]

The shared object and the object files are build products (git-ignored).
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libclair3b200.so")
OBJ_DIR = os.path.join(HERE, "csrc", "_obj")
SOURCES = ["c3b_api.cu", "kernels_common.cu", "kernels_fp32.cu", "lstm_tc.cu", "fa_tc.cu", "pconv_tc.cu", "decode.cu", "proj_tc.cu", "tail_tc.cu", "plp_counts.cu", "plp_alt_text.cu", "fa_tensor.cu", "fa_alt_text.cu", "bam_decode.cu", "cascade.cu", "phase.cu"]
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = GENCODE + ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC"]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build_library(force=False, verbose=False):
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    for h in ("clair3_b200.h", "clair3_b200_debug.h", "clair3_b200_pileup.h", "clair3_b200_fa.h", "clair3_b200_bam.h", "clair3_b200_cascade.h", "clair3_b200_phase.h"):
        headers.append(os.path.join(os.path.dirname(HERE), "include", h))
    os.makedirs(OBJ_DIR, exist_ok=True)
    nvcc = _nvcc()
    jobs = []
    objs = []
    for src in SOURCES:
        sp = os.path.join(CSRC, src)
        op = os.path.join(OBJ_DIR, src.replace(".cu", ".o"))
        objs.append(op)
        if force or _stale(op, [sp] + headers):
            cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", sp, "-o", op]
            jobs.append(cmd)

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed: %s\n%s\n%s" % (" ".join(cmd), r.stdout, r.stderr))
        return r.stderr

    if jobs:
        with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 4)) as ex:
            for out in ex.map(run, jobs):
                if verbose and out:
                    print(out)
    if jobs or force or _stale(LIB, objs):
        run([nvcc, "-shared", "-o", LIB] + objs + GENCODE + ["-ldl"])
    return LIB


if __name__ == "__main__":
    path = build_library(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(path)
