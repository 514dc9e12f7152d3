"""Builds runbooks_b200/libb200w.so (CUDA kernels + C ABI) in-tree with nvcc for sm_90a (H100).

In-tree so that the package imports from the repository tree with its library beside it.
No torch cpp_extension: the library has no
torch types in its ABI (include/b200w.h), so a plain nvcc -shared is all it needs.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libb200w.so")
SOURCES = ["host_common.cu", "gemm.cu", "attention.cu", "ops.cu", "engine.cu", "kv_cache.cu", "kv_attention.cu",
           "logits.cu", "wq.cu", "infer.cu", "op_hooks.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
]


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: libb200w.so cannot be built")


def _digest() -> str:
    h = hashlib.sha256()
    for root in (CSRC, os.path.join(HERE, "..", "include")):
        for name in sorted(os.listdir(root)):
            if name.endswith((".cu", ".cuh", ".h")):
                with open(os.path.join(root, name), "rb") as f:
                    h.update(name.encode())
                    h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(BUILD, exist_ok=True)
    stamp = os.path.join(BUILD, "stamp")
    digest = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp):
        with open(stamp) as f:
            if f.read().strip() == digest:
                return LIB
    nvcc = _nvcc()

    def compile_one(src: str) -> None:
        obj = os.path.join(BUILD, src.replace(".cu", ".o"))
        cmd = [nvcc, *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        if verbose or r.returncode:
            sys.stderr.write(r.stdout + r.stderr)
        if r.returncode:
            raise RuntimeError(f"nvcc failed on {src}")

    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        list(ex.map(compile_one, SOURCES))
    objs = [os.path.join(BUILD, s.replace(".cu", ".o")) for s in SOURCES]
    r = subprocess.run([nvcc, "-shared", "-o", LIB, *objs, "-ldl", "-Xcompiler", "-fPIC"],
                       capture_output=True, text=True)
    if r.returncode:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("link of libb200w.so failed")
    with open(stamp, "w") as f:
        f.write(digest)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
