"""Build libhairfast_sm90.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python -m hairfastgan_b200.build [--force]
"""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(CSRC, "libhairfast_sm90.so")
SOURCES = ["hf_api.cu", "hf_ops.cu", "hf_conv_tc.cu", "hf_generator.cu", "hf_enc_ops.cu", "hf_enc_api.cu",
           "hf_seg_ops.cu", "hf_glue_ops.cu"]
HEADERS = ["hf_common.cuh", "hf_kernels.cuh", os.path.join("..", "..", "include", "hairfast_b200.h")]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    objs = []
    flags = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
             "-Xcompiler", "-fPIC", "--use_fast_math=false"]
    flags = [f for f in flags if f != "--use_fast_math=false"]
    if verbose:
        flags += ["-Xptxas", "-v"]
    procs = []
    for s in SOURCES:
        obj = os.path.join(CSRC, s.replace(".cu", ".o"))
        objs.append(obj)
        cmd = [_nvcc(), *flags, "-c", os.path.join(CSRC, s), "-o", obj]
        procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for cmd, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError("nvcc failed: %s\n%s" % (" ".join(cmd), out))
        if verbose and out:
            print(out)
    cmd = [_nvcc(), "-shared", "-o", LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed: %s\n%s" % (" ".join(cmd), r.stdout))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
