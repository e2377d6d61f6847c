"""Host side of the exhaustive fp32 sweeps: tests/device/libm_sweep.cpp compiled with g++ at test time, loaded with
ctypes.  Each call runs the whole chunk on every CPU in C++ threads (ctypes releases the GIL while it runs).

The running libm is the reference for sinf / cosf / expf.  csrc/sincosf_glibc.h transcribes glibc 2.39's FMA build,
which libm selects through ifunc on every AVX2+FMA host; on a host without FMA libm takes another code path, so
`skip_reason()` names that case and the callers skip."""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "device", "libm_sweep.cpp")
CSRC = os.path.join(ROOT, "hector_slam_b200", "csrc")
MAX_BAD = 8
ALL = 1 << 32

_vp, _ll, _u32, _i = C.c_void_p, C.c_longlong, C.c_uint32, C.c_int


def skip_reason() -> str | None:
    if not shutil.which("g++"):
        return "no g++"
    flags = open("/proc/cpuinfo").read()
    if " fma" not in flags or " avx2" not in flags:
        return "host CPU without FMA/AVX2: libm does not run the code path the header transcribes"
    return None


def threads() -> int:
    return len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)


def _ptr(a) -> int:
    return a.ctypes.data


class Sweep:
    """lx_* of libm_sweep.cpp; every check returns (counts (K,), lowest mismatching argument bits (K, MAX_BAD))"""

    def __init__(self, path: str):
        self.lib = C.CDLL(path)
        L = self.lib
        L.lx_check_trig.argtypes = [_u32, _ll, _vp, _vp, _vp, _vp, _i, _i, _vp, _vp]
        L.lx_check_exp.argtypes = [_u32, _ll, _vp, _i, _i, _vp, _vp]
        L.lx_compare.argtypes = [_u32, _ll, _vp, _vp, _i, _i, _vp, _vp]
        L.lx_host_trig.argtypes = [_u32, _ll, _i, _i, _vp, _vp]
        L.lx_host_exp.argtypes = [_u32, _ll, _i, _i, _vp, _vp]
        L.lx_power.argtypes = [_u32, _ll, _ll, _i, _i, _vp, _vp]
        L.lx_check_pack.argtypes = [_u32, _ll, _vp, _vp, _vp, _u32, _i, C.c_ulonglong, _i, _i, _vp, _vp]
        L.lx_inverse3_fma.argtypes = [_vp, _vp, _ll, _vp, _i]
        L.lx_inverse3_fma.restype = _ll
        self.threads = threads()

    def _run(self, fn, k, *args):
        counts, bad = np.zeros(k, np.int64), np.zeros((k, MAX_BAD), np.uint32)
        fn(*args, self.threads, MAX_BAD, _ptr(counts), _ptr(bad))
        return counts, bad

    def check_trig(self, first, s, c, ss, sc):
        return self._run(self.lib.lx_check_trig, 6, first, s.size, _ptr(s), _ptr(c), _ptr(ss), _ptr(sc))

    def check_exp(self, first, e):
        return self._run(self.lib.lx_check_exp, 1, first, e.size, _ptr(e))

    def compare(self, first, x, y):
        assert x.size == y.size
        return self._run(self.lib.lx_compare, 1, first, x.size, _ptr(x), _ptr(y))

    def host_trig(self, first, n):
        return self._run(self.lib.lx_host_trig, 4, first, n)

    def host_exp(self, first, n):
        return self._run(self.lib.lx_host_exp, 1, first, n)

    def power(self, first, n, stride):
        return self._run(self.lib.lx_power, 2, first, n, stride)

    def check_pack(self, first, packed, score, index_out, index, prev):
        return self._run(self.lib.lx_check_pack, 4, first, packed.size, _ptr(packed), _ptr(score), _ptr(index_out),
                         index, int(prev is not None), int(prev or 0))

    def inverse3_fma(self, m9, v3, port3) -> int:
        return int(self.lib.lx_inverse3_fma(_ptr(m9), _ptr(v3), m9.shape[0], _ptr(port3), self.threads))


def build(out_dir) -> Sweep:
    """compile the helper into out_dir (g++ -O2, no FMA contraction) and load it"""
    so = os.path.join(str(out_dir), "liblibm_sweep.so")
    subprocess.run([shutil.which("g++") or "g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-pthread",
                    "-I", CSRC, SRC, "-o", so, "-lm"], check=True, capture_output=True)
    return Sweep(so)


def chunks(size: int):
    """(first, n) over all 2^32 bit patterns"""
    for first in range(0, ALL, size):
        yield first, min(size, ALL - first)


def report_bad(names, counts, bad) -> str:
    """'name: count mismatches, first at 0x........ (value)' for each nonzero count"""
    out = []
    for name, c, b in zip(names, counts, bad):
        if c:
            args = ", ".join(f"0x{int(a):08x} ({float(np.uint32(a).view(np.float32))!r})" for a in b[:min(int(c), MAX_BAD)])
            out.append(f"{name}: {int(c)} mismatches, first at {args}")
    return "; ".join(out)
