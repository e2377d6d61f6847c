"""Build recipe for the in-tree native libraries (explicit nvcc / g++ commands, no JIT cache).

  hector_slam_b200/lib/libhsb200.so        CUDA kernels + C-ABI (include/hector_slam_b200.h), sm_90a only
  hector_slam_b200/lib/libhsb200_host.so   C wrapper around the C++ host façade (host/), links libhsb200.so
  hector_slam_b200/lib/libhsb200_probe.so  the kernels' scalar device functions one by one (tests/device/hsb_probe.cu),
                                           for the tests only: nothing in the package loads it

nvcc cross-compiles without a GPU, so this runs on a CPU-only build machine; the .so files are
git-ignored build products.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
HOST = os.path.join(PKG, "host")
LIBDIR = os.path.join(PKG, "lib")
LIB = os.path.join(LIBDIR, "libhsb200.so")
HOST_LIB = os.path.join(LIBDIR, "libhsb200_host.so")
PROBE_SRC = os.path.join(ROOT, "tests", "device", "hsb_probe.cu")
PROBE_LIB = os.path.join(LIBDIR, "libhsb200_probe.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    # no implicit FMA contraction anywhere (nvcc AND ptxas): the map-coordinate arithmetic must round
    # like the reference's.  Fused operations are written explicitly (fmaf) where they are wanted.
    "-fmad=false",
    # host code too: the bit-exact host arithmetic (affine maps, beam table) must not be contracted on
    # targets whose baseline ISA has FMA (aarch64); GCC defaults to -ffp-contract=fast
    "-Xcompiler", "-ffp-contract=off",
    "-Xcompiler", "-fPIC", "-shared",
    "-cudart", "static",
]


def _newer(target: str, sources: list[str]) -> bool:
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(s) <= t for s in sources if os.path.exists(s))


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def build_cuda(force: bool = False, verbose: bool = False, extra: list[str] | None = None, out: str | None = None) -> str:
    """`extra` / `out`: a variant build (e.g. -DHSB_TLD4_OFFSET=0) next to the product library, for A/B comparisons
    (scripts/alt_compare.py); load it with HSB_LIB_PATH."""
    out = out or LIB
    srcs = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(ROOT, "include", "hector_slam_b200.h")]
    if not force and _newer(out, srcs):
        return out
    os.makedirs(LIBDIR, exist_ok=True)
    cmd = [_nvcc()] + NVCC_FLAGS + (extra or []) + (["-Xptxas", "-v"] if verbose else []) + [
        "-o", out, os.path.join(CSRC, "hsb_api.cu")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed: " + " ".join(cmd))
    return out


def build_host(force: bool = False) -> str | None:
    src = os.path.join(HOST, "host_capi.cpp")
    if not os.path.exists(src):
        return None
    srcs = [os.path.join(HOST, f) for f in os.listdir(HOST)] + [LIB]
    if not force and _newer(HOST_LIB, srcs):
        return HOST_LIB
    cxx = shutil.which("g++") or "g++"
    cmd = [cxx, "-std=c++14", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-I", os.path.join(ROOT, "include"), "-I", HOST, src,
           "-o", HOST_LIB, "-L", LIBDIR, "-lhsb200", "-Wl,-rpath,$ORIGIN"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("host build failed: " + " ".join(cmd))
    return HOST_LIB


def probe_command() -> list[str]:
    """nvcc command of the probe library: the product library's NVCC_FLAGS unchanged, so the probed functions are
    compiled as the kernels compile them (-fmad=false above all)"""
    return [_nvcc()] + NVCC_FLAGS + ["-I", CSRC, "-o", PROBE_LIB, PROBE_SRC]


def build_probe(force: bool = False) -> str | None:
    if not os.path.exists(PROBE_SRC):
        return None
    srcs = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(ROOT, "include", "hector_slam_b200.h"), PROBE_SRC]
    if not force and _newer(PROBE_LIB, srcs):
        return PROBE_LIB
    os.makedirs(LIBDIR, exist_ok=True)
    cmd = probe_command()
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("nvcc failed: " + " ".join(cmd))
    return PROBE_LIB


def build_all(force: bool = False, verbose: bool = False):
    build_cuda(force, verbose)
    build_host(force)
    build_probe(force)


if __name__ == "__main__":
    build_all(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(LIB)
