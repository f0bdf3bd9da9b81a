# -*- coding: utf-8 -*-
"""Builds libstoke_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python stoke_b200/csrc/build.py [--force] [--verbose]
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.dirname(HERE)
LIB = os.path.join(PKG, "libstoke_b200.so")
SOURCES = ["ctx.cu", "vmm.cu", "k1_reduce.cu", "k1_bulk.cu", "k1_nvls.cu", "k1_norm.cu", "k2_optim.cu", "k2_adafactor.cu",
           "k2_layerwise.cu", "collectives.cu", "sampler.cu", "bn_act.cu"]
HEADERS = ["common.cuh", "ctx.cuh", "k1_common.cuh", os.path.join("..", "..", "include", "stoke_b200.h")]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + [
    "-lineinfo", "-O3", "-std=c++17", "--use_fast_math", "-Xcompiler", "-fPIC", "-cudart", "static",
]
# --use_fast_math would change division / sqrt rounding in the optimizer kernel; keep IEEE there
NVCC_FLAGS.remove("--use_fast_math")


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _stamp():
    h = hashlib.sha256()
    for f in SOURCES + HEADERS:
        with open(os.path.join(HERE, f), "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    stamp_file = LIB + ".stamp"
    stamp = _stamp()
    if not force and os.path.exists(LIB) and os.path.exists(stamp_file) and open(stamp_file).read() == stamp:
        return LIB
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(HERE, src.replace(".cu", ".o"))
        cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", os.path.join(HERE, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            sys.stderr.write(f"---- {src} ----\n{out}\n")
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed (see output above)")
    link = [_nvcc(), "-shared"] + ARCH + ["-cudart", "static", "-o", LIB] + objs
    subprocess.check_call(link)
    with open(stamp_file, "w") as f:
        f.write(stamp)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
