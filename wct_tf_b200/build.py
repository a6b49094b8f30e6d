"""Build libwctb200.so in-tree with nvcc for sm_90a (H100; no GPU needed: cross-compiles)."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libwctb200.so")
SOURCES = ["capi.cu", "layers.cu", "conv_tc.cu", "cov_tc.cu", "wct.cu", "image_ops.cu", "conv_tail_tc.cu", "conv_head_tc.cu", "matfun_tc.cu",
           "flow.cu", "mst.cu", "efdm.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden"]
NVCC_FLAGS += os.environ.get("WCTB_NVCC_EXTRA", "").split()      # experiments, e.g. -DWCTB_MBAR_TEST_WAIT


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _newer(src, dst):
    return (not os.path.exists(dst)) or os.path.getmtime(src) > os.path.getmtime(dst)


def build(force=False, verbose=False):
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    deps = [os.path.join(CSRC, "common.cuh"), os.path.join(CSRC, "jacobi_common.cuh"), os.path.join(CSRC, "wctb200_debug.h"),
            os.path.join(os.path.dirname(HERE), "include", "wctb200.h")]
    objs, relink = [], force or not os.path.exists(LIB)
    procs = []
    for s in SOURCES:
        src = os.path.join(CSRC, s)
        obj = os.path.join(objdir, s.replace(".cu", ".o"))
        objs.append(obj)
        if force or _newer(src, obj) or any(_newer(d, obj) for d in deps):
            cmd = [_nvcc()] + NVCC_FLAGS + ["-c", src, "-o", obj]
            if verbose:
                print(" ".join(cmd))
            procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
            relink = True
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError("nvcc failed on %s:\n%s" % (s, out.decode()))
        if verbose and out:
            print(out.decode())
    if relink:
        cmd = [_nvcc(), "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC"]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s" % r.stdout.decode())
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
