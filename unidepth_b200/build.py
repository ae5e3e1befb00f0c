"""Build libudb.so (the sm_90a kernels + C ABI) in-tree with nvcc.

    python -m unidepth_b200.build        # or  __graft_entry__.build()

nvcc cross-compiles for sm_90a without a GPU; the library and its objects are git-ignored build products.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libudb.so")
SOURCES = ["common.cu", "gemm.cu", "conv_halo.cu", "attention.cu", "elementwise.cu", "camera.cu", "metrics.cu", "v1_kernels.cu", "engine.cu", "engine_v1.cu", "engine_v2old.cu", "p2p.cu"]
HEADERS = ["common.h", "cuda_core.cuh", "ptx.cuh", "engine_common.h", os.path.join("..", "..", "include", "udb.h")]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
         "-Xcompiler", "-fPIC", "-Xptxas", "-v", "--expt-relaxed-constexpr"]


def _digest() -> str:
    h = hashlib.sha256()
    for f in SOURCES + HEADERS:
        with open(os.path.join(CSRC, f), "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    stamp = LIB + ".stamp"
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == dig:
        return LIB
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(CSRC, src.replace(".cu", ".o"))
        objs.append(obj)
        cmd = [NVCC, *FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    for src, pr in procs:
        out, _ = pr.communicate()
        log.append(out)
        if pr.returncode != 0:
            sys.stderr.write(out)
            raise RuntimeError(f"nvcc failed on {src}")
    with open(os.path.join(CSRC, "build.log"), "w") as fh:
        fh.write("\n".join(log))
    if verbose:
        print("\n".join(log))
    cmd = [NVCC, "-shared", *FLAGS[:2], "-o", LIB, *objs, "-lcudart"]
    subprocess.check_call(cmd)
    with open(stamp, "w") as fh:
        fh.write(dig)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
