#!/usr/bin/env python
"""Builds libdfft.so (the C-ABI library), the distFFT driver and the developer tools, in-tree.

    python -m distributedfft_b200.build [--force] [--tools]

Everything is compiled for sm_90a (H100) only:  nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo.
The resulting .so and executables are git-ignored build products.
"""
from __future__ import annotations

import concurrent.futures as cf
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libdfft.so")
DRIVER = os.path.join(HERE, "distFFT")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-ccbin", "/usr/bin/g++"]

LIB_SOURCES = ["dfft_api.cu", "dfft_kernels_common.cu", "dfft_kernels_generic.cu", "dfft_kernels_f64.cu", "dfft_kernels_f32.cu", "dfft_kernels_tma.cu"]
HEADERS = ["fft_core.cuh", "fft_passes.cuh", "fft_real.cuh", "fft_generic.cuh", "fft_tma.cuh", "fft_plane.cuh", "dfft_kernels.cuh", "dfft_kernels_inst.cuh", "dfft_launch.cuh", os.path.join("..", "..", "include", "dfft.h")]


def _newer(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def _run(cmd):
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        raise RuntimeError("build step failed: " + " ".join(cmd[:3]))
    return r.stdout + r.stderr


def build(force: bool = False, tools: bool = False, verbose: bool = False, experiments: bool = False) -> str:
    os.makedirs(BUILD, exist_ok=True)
    common = COMMON + (["-DDFFT_EXPERIMENTS"] if experiments else [])
    stamp = os.path.join(BUILD, "experiments.stamp")
    if experiments != os.path.exists(stamp):   # switching the flavour rebuilds everything
        force = True
        if experiments:
            open(stamp, "w").close()
        elif os.path.exists(stamp):
            os.remove(stamp)
    hdrs = [os.path.join(CSRC, h) for h in HEADERS]
    jobs = []
    objs = []
    for src in LIB_SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(BUILD, src.replace(".cu", ".o"))
        objs.append(o)
        if force or _newer(o, [s] + hdrs):
            jobs.append([NVCC] + ARCH + common + ["-c", s, "-o", o])
    if jobs:
        with cf.ThreadPoolExecutor(max_workers=min(4, len(jobs))) as ex:
            for out in ex.map(_run, jobs):
                if verbose and out.strip():
                    print(out)
    if force or jobs or _newer(LIB, objs):
        # link to a temporary name and rename: a snapshot taken while we build never sees a half-written library
        _run([NVCC] + ARCH + ["-shared", "-o", LIB + ".tmp"] + objs + ["-ldl", "-lpthread", "-ccbin", "/usr/bin/g++"])
        os.replace(LIB + ".tmp", LIB)
    drv = os.path.join(HERE, "driver", "distFFT.cpp")
    if os.path.exists(drv) and (force or _newer(DRIVER, [drv, LIB, os.path.join(HERE, "..", "include", "fft_mpi_3d_api.h")])):
        _run([NVCC] + ARCH + ["-O2", "-std=c++17", "-ccbin", "/usr/bin/g++", "-I", os.path.join(HERE, "..", "include"), drv, "-o", DRIVER,
              "-L", HERE, "-ldfft", "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN", "-lpthread"])
    bdrv = os.path.join(HERE, "driver", "batchFFT.cpp")
    bout = os.path.join(HERE, "batchFFT")
    if os.path.exists(bdrv) and (force or _newer(bout, [bdrv, LIB, os.path.join(HERE, "..", "include", "dfft.h")])):
        _run([NVCC] + ARCH + ["-O2", "-std=c++17", "-ccbin", "/usr/bin/g++", "-I", os.path.join(HERE, "..", "include"), bdrv, "-o", bout,
              "-L", HERE, "-ldfft", "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN"])
    if tools:
        kb = os.path.join(CSRC, "tools", "kbench.cu")
        out = os.path.join(CSRC, "tools", "kbench")
        if force or _newer(out, [kb] + hdrs):
            _run([NVCC] + ARCH + COMMON + [kb, "-o", out])
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv, tools="--tools" in sys.argv, verbose=True, experiments="--experiments" in sys.argv)
    print("built", LIB)
