"""Build recipe: compile csrc/*.cu for sm_90a (H100) into ONE in-tree shared library with a C ABI.

    python -m macvo_b200.build        (or  __graft_entry__.build())

No torch extension machinery: plain `nvcc -shared`; the Python side binds it with ctypes, so the same
library can be bound from any host language (INTEGRATION.md).
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
LIB_DIR = os.path.join(PKG_DIR, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libmacvo_b200.so")
SOURCES = ["corr_build.cu", "corr_build_simt.cu", "corr_build_tc.cu", "corr_lookup.cu", "dense_select.cu",
           "cov2to3.cu", "pgo.cu", "nn_kernels.cu", "decoder_fused.cu", "observe.cu", "decoder_token.cu", "motion_interp.cu",
           "gru_conv_tc.cu", "conv_tc.cu", "posenet.cu", "mlp_tc.cu",
           "patch_tokens_tc.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "--use_fast_math=false"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found (CUDA 12.9 toolkit expected at /usr/local/cuda)")


def _fingerprint() -> str:
    h = hashlib.sha256()
    for name in sorted(os.listdir(CSRC)) + ["../../include/macvo_b200.h"]:
        with open(os.path.join(CSRC, name), "rb") as f:
            h.update(name.encode())
            h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = True) -> str:
    os.makedirs(LIB_DIR, exist_ok=True)
    stamp = os.path.join(LIB_DIR, "libmacvo_b200.stamp")
    fp = _fingerprint()
    if not force and os.path.exists(LIB_PATH) and os.path.exists(stamp) and open(stamp).read() == fp:
        return LIB_PATH
    nvcc = _nvcc()
    flags = [f for f in NVCC_FLAGS if f != "--use_fast_math=false"]
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(LIB_DIR, src.replace(".cu", ".o"))
        objs.append(obj)
        cmd = [nvcc, *flags, "-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{out}")
        if verbose and out.strip():
            print(out, file=sys.stderr)
    link = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB_PATH, *objs, "-lcuda" if False else "-lcudart_static",
            "-Xlinker", "--no-undefined", "-lpthread", "-ldl", "-lrt"]
    r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}")
    with open(stamp, "w") as f:
        f.write(fp)
    if verbose:
        print(f"built {LIB_PATH}", file=sys.stderr)
    return LIB_PATH


if __name__ == "__main__":
    build(force="--force" in sys.argv)
