"""Builds libsdxl_b200.so (hand-written sm_90a CUDA + C++ host, C ABI in include/sdxl_b200.h) and libsdxl_b200_testing.so
(the same kernel objects behind the test-only entry points of csrc/testing.cu, bound by sdxl_b200/_testing.py).

In-tree build with plain nvcc (cross-compiles on a machine without a GPU). The .so is git-ignored but
travels with the repo snapshot to the GPU box. `python build.py` or `build_library()`.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "sdxl_b200", "libsdxl_b200.so")
TEST_LIB = os.path.join(HERE, "sdxl_b200", "libsdxl_b200_testing.so")
KERNEL_SOURCES = ["igemm.cu", "attention.cu", "norm.cu", "elementwise.cu", "vae_kernels.cu", "clip_kernels.cu", "t2i_kernels.cu", "freeu.cu"]
SOURCES = KERNEL_SOURCES + ["engine.cu", "vae.cu", "clip.cu", "tokenizer.cpp", "mpk.cpp"]
TEST_SOURCES = ["testing.cu"]
HEADERS = ["common.cuh", "kernels.h", "engine_core.h", "schedule.h", "unicode_tables.h", os.path.join("..", "..", "include", "sdxl_b200.h")]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
]


def _digest() -> str:
    h = hashlib.sha256()
    for f in SOURCES + TEST_SOURCES + HEADERS:
        with open(os.path.join(CSRC, f), "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def build_library(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(BUILD, exist_ok=True)
    stamp = os.path.join(BUILD, "stamp")
    dg = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(TEST_LIB) and os.path.exists(stamp) and open(stamp).read() == dg:
        return LIB

    def cc(src: str) -> str:
        obj = os.path.join(BUILD, os.path.splitext(src)[0] + ".o")
        cmd = [NVCC, *FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            print(" ".join(cmd), file=sys.stderr)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        return obj

    with ThreadPoolExecutor(max_workers=len(SOURCES + TEST_SOURCES)) as ex:
        objs = dict(zip(SOURCES + TEST_SOURCES, ex.map(cc, SOURCES + TEST_SOURCES)))

    def link(out: str, srcs: list, extra: tuple = ()) -> None:
        cmd = [NVCC, "-shared", "-o", out, *(objs[s] for s in srcs), "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler",
               "-fPIC", "-ldl", *extra]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link of {os.path.basename(out)} failed:\n{r.stdout}\n{r.stderr}")

    link(LIB, SOURCES)
    # the kernels alone, without the engine: an unresolved symbol is a link error rather than a dlopen failure on the GPU host
    link(TEST_LIB, TEST_SOURCES + KERNEL_SOURCES, ("-Xlinker", "--no-undefined"))
    with open(stamp, "w") as fh:
        fh.write(dg)
    return LIB


if __name__ == "__main__":
    print(build_library(force="--force" in sys.argv, verbose=True))
