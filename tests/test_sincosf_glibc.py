"""CPU: hector_slam_b200/csrc/sincosf_glibc.h (the sinf/cosf the kernels use for the pose angle)
against the running libm, bit for bit.  The header transcribes glibc 2.39's FMA build, which libm
selects through ifunc on every AVX2+FMA host; on a host without FMA libm takes another code path
and the comparison is skipped.

The sampled cases below aim at the reductions' edges; test_*_every_argument then compares the host build with libm on
all 2^32 bit patterns (tests/libm_sweep.py), so the transcription is right everywhere and the device sweep
(test_gpu_scalar_functions.py) only has to show that nvcc compiles it to the same bits.  Cost: the two exhaustive
tests take about 45-60 s of wall time on an 8-thread x86-64 CPU (the sweep uses every CPU the process may run on)."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import ROOT

SRC = r'''
#include <cstdio>
#include <cmath>
#include <cstring>
#include <cstdint>
#include <cfloat>
#include "sincosf_glibc.h"
static bool same(float a, float b) { uint32_t x, y; memcpy(&x, &a, 4); memcpy(&y, &b, 4); return x == y || (a != a && b != b); }
static long n = 0, bad = 0, bad_large = 0;
static void check(float x) {
  ++n;
  float sc, cc; hsb::sincosf_glibc(x, &sc, &cc);
  const float s = sinf(x), c = cosf(x);
  const long b = !same(hsb::sinf_glibc(x), s) + !same(hsb::cosf_glibc(x), c) + (!same(sc, s) || !same(cc, c));
  bad += b;
  if (!(fabsf(x) < 120.f)) bad_large += b;
}
static float from_bits(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
int main() {
  unsigned s = 2463534242u;
  for (long i = 0; i < 12000000; ++i) {
    s = s * 1664525u + 1013904223u;
    float u = (float)(s >> 8) / 16777216.0f * 2.f - 1.f;
    check((i % 3 == 0) ? u * 3.1415927f : (i % 3 == 1) ? u * 119.9f : ldexpf(u, -(int)(i % 40)));
  }
  const float edge[] = {0.f, -0.f, 0.78539816f, 0.785398185f, 0.78539822f, 1.5707963f, 3.1415927f, -3.1415927f, 6.2831855f,
                        2.4414062e-4f, 2.4414065e-4f, 119.99999f, 120.f, -120.f, FLT_MAX, -FLT_MAX, INFINITY, -INFINITY, NAN,
                        -NAN, 3.4e38f, -3.4e38f};
  for (float x : edge) check(x);
  // glibc's large-argument reduction: random bit patterns with 120 <= |y| < inf, every exponent, both signs
  uint64_t r = 88172645463325252ull;
  for (long i = 0; i < 6000000; ++i) {
    r ^= r << 13; r ^= r >> 7; r ^= r << 17;
    const uint32_t lo = 0x42f00000u, hi = 0x7f800000u;   // 120.f .. inf
    check(from_bits((uint32_t)(lo + (r >> 8) % (hi - lo)) | (uint32_t)(r & 1) << 31));
  }
  // every float in [119.99, 120.01], both signs: the switch between the two reductions
  for (float x = 119.99f; x <= 120.01f; x = nextafterf(x, 1e9f)) { check(x); check(-x); }
  // multiples of pi/2 up to 1e6, +-2 ulp: the largest reduced arguments relative to the result
  for (long k = 1; k <= 636620; ++k) {
    const float m = (float)(k * 1.5707963267948966);
    float lo = m, hi = m;
    for (int j = 0; j < 2; ++j) { lo = nextafterf(lo, 0.f); hi = nextafterf(hi, 1e9f); }
    for (float x = lo; x <= hi; x = nextafterf(x, 1e9f)) { check(x); check(-x); }
  }
  std::printf("%ld %ld %ld\n", n, bad, bad_large);
  return bad ? 1 : 0;
}
'''


def test_sincosf_matches_libm(tmp_path):
    cxx = shutil.which("g++")
    if not cxx:
        pytest.skip("no g++")
    flags = open("/proc/cpuinfo").read()
    if " fma" not in flags or " avx2" not in flags:
        pytest.skip("host CPU without FMA/AVX2: libm does not run the code path the header transcribes")
    src = tmp_path / "t.cpp"
    src.write_text(SRC)
    exe = tmp_path / "t"
    subprocess.run([cxx, "-O2", "-I", os.path.join(ROOT, "hector_slam_b200", "csrc"), str(src), "-o", str(exe), "-lm"],
                   check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    n, bad, bad_large = (int(v) for v in out.stdout.split())
    assert bad == 0 and n > 12000000 + 6000000 + 5 * 636620, f"{n} arguments, {bad} mismatches ({bad_large} at |x| >= 120)"


def _pi_fixed(bits):
    """floor(pi * 2^bits), Machin's formula in integers (20 guard bits)"""
    one = 1 << (bits + 20)

    def arctan_inv(x):
        s = t = one // x
        k, x2, sign = 1, x * x, -1
        while t:
            t //= x2
            s += sign * (t // (2 * k + 1))
            k, sign = k + 1, -sign
        return s

    return (16 * arctan_inv(5) - 4 * arctan_inv(239)) >> 20


def _inv_pio4_words():
    """word i = floor(4/pi * 2^(8i+7)) mod 2^32: overlapping 32-bit windows of 4/pi at 8-bit steps"""
    B = 400
    inv = (4 << (2 * B)) // _pi_fixed(B)   # 4/pi * 2^B, exact in far more bits than the 24 words need
    return [((inv << (8 * i + 7)) >> B) & 0xffffffff for i in range(24)]


def test_inv_pio4_table():
    """the header's 4/pi table is 4/pi's binary expansion, computed here from pi; where the running libm is a glibc
    shared object, the same 96 bytes are in it (its __inv_pio4)"""
    import ctypes.util
    import re
    import struct

    want = _inv_pio4_words()
    assert want[:4] == [0xa2, 0xa2f9, 0xa2f983, 0xa2f9836e]
    text = open(os.path.join(ROOT, "hector_slam_b200", "csrc", "sincosf_glibc.h")).read()
    body = re.search(r"#define HSB_INV_PIO4_TABLE((?:.*\\\n)*.*)", text).group(1)
    got = [int(w, 16) for w in re.findall(r"0x([0-9a-f]{8})u", body)]
    assert got == want
    libm = ctypes.util.find_library("m")
    path = next((os.path.join(d, libm) for d in ("/lib/x86_64-linux-gnu", "/usr/lib/x86_64-linux-gnu", "/lib64", "/usr/lib64")
                 if libm and os.path.exists(os.path.join(d, libm))), None)
    if path is None:
        pytest.skip("no libm shared object found to cross-check against")
    assert struct.pack("<24I", *want) in open(path, "rb").read()


EXP_SRC = r'''
#include <cstdio>
#include <cmath>
#include <cstring>
#include <cstdint>
#include "sincosf_glibc.h"
static bool same(float a, float b) { uint32_t x, y; memcpy(&x, &a, 4); memcpy(&y, &b, 4); return x == y || (a != a && b != b); }
int main() {
  long bad = 0, n = 0; unsigned s = 2463534242u;
  // the log-odds a grid can hold: sums of log(0.4/0.6) and log(0.9/0.1) steps, anything in (-inf, 52.2]; plus the whole
  // float range around the special-case thresholds
  for (long i = 0; i < 16000000; ++i) {
    s = s * 1664525u + 1013904223u;
    float u = (float)(s >> 8) / 16777216.0f * 2.f - 1.f;
    float x = (i % 4 == 0) ? u * 52.2f : (i % 4 == 1) ? u * 110.f : (i % 4 == 2) ? ldexpf(u, -(int)(i % 60)) : -103.f - u;
    ++n;
    if (!same(hsb::expf_glibc(x), expf(x))) ++bad;
  }
  // every float between the underflow thresholds and a little beyond, and the overflow edge
  for (float x = -104.2f; x < -103.0f; x = nextafterf(x, 0.f)) { ++n; if (!same(hsb::expf_glibc(x), expf(x))) ++bad; }
  for (float x = 88.5f; x < 89.0f; x = nextafterf(x, 1e9f)) { ++n; if (!same(hsb::expf_glibc(x), expf(x))) ++bad; }
  const float edge[] = {0.f, -0.f, 1.f, -1.f, 50.f, 52.197224f, -0.4054651f, 2.1972246f, 87.99999f, 88.f, -87.99999f, -88.f,
                        INFINITY, -INFINITY, NAN, 1e-30f, -1e-30f, 3.4e38f, -3.4e38f};
  for (float x : edge) { ++n; if (!same(hsb::expf_glibc(x), expf(x))) ++bad; }
  // cumulative log-odds exactly as a cell accumulates them
  const float lf = logf(0.4f / 0.6f), lo = logf(0.9f / 0.1f);
  for (int occ = 0; occ < 40; ++occ) {
    float l = 0.f;
    for (int k = 0; k < occ; ++k) if (l < 50.f) l += lo;
    for (int k = 0; k < 400; ++k) { l += lf; ++n; if (!same(hsb::expf_glibc(l), expf(l))) ++bad; }
  }
  std::printf("%ld %ld\n", n, bad);
  return bad ? 1 : 0;
}
'''


def test_expf_matches_libm(tmp_path):
    """hsb::expf_glibc (the exp of getGridProbability, GridMapLogOdds.h:165) against the running libm, bit for bit."""
    cxx = shutil.which("g++")
    if not cxx:
        pytest.skip("no g++")
    flags = open("/proc/cpuinfo").read()
    if " fma" not in flags or " avx2" not in flags:
        pytest.skip("host CPU without FMA/AVX2: libm does not run the code path the header transcribes")
    src = tmp_path / "e.cpp"
    src.write_text(EXP_SRC)
    exe = tmp_path / "e"
    subprocess.run([cxx, "-O2", "-I", os.path.join(ROOT, "hector_slam_b200", "csrc"), str(src), "-o", str(exe), "-lm"],
                   check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    n, bad = (int(v) for v in out.stdout.split())
    assert bad == 0 and n > 16000000, out.stdout


# ---- every fp32 argument ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sweep(tmp_path_factory):
    import libm_sweep

    why = libm_sweep.skip_reason()
    if why:
        pytest.skip(why)
    return libm_sweep.build(tmp_path_factory.mktemp("libm_sweep"))


def _exhaustive(run, names):
    import libm_sweep

    total, counts, first_bad, n = None, np.zeros(len(names), np.int64), [[] for _ in names], 0
    for first, size in libm_sweep.chunks(1 << 26):
        c, bad = run(first, size)
        for k in range(len(names)):
            first_bad[k] += bad[k][:max(0, min(int(c[k]), libm_sweep.MAX_BAD) - len(first_bad[k]))].tolist()
        counts += c
        n += size
    bad = np.array([(b + [0] * libm_sweep.MAX_BAD)[:libm_sweep.MAX_BAD] for b in first_bad], np.uint32)
    return n, counts, bad


def test_sincosf_every_argument(sweep):
    """sinf_glibc, cosf_glibc and both outputs of sincosf_glibc (host build) equal libm on all 2^32 arguments"""
    import libm_sweep

    names = ["sinf_glibc", "cosf_glibc", "sincosf_glibc sin", "sincosf_glibc cos"]
    n, counts, bad = _exhaustive(sweep.host_trig, names)
    print(f"sincosf: {n} arguments, mismatches {dict(zip(names, counts.tolist()))}")
    assert n == libm_sweep.ALL and not counts.any(), libm_sweep.report_bad(names, counts, bad)


def test_expf_every_argument(sweep):
    """expf_glibc (host build) equals libm expf on all 2^32 arguments"""
    import libm_sweep

    n, counts, bad = _exhaustive(sweep.host_exp, ["expf_glibc"])
    print(f"expf: {n} arguments, {int(counts[0])} mismatches")
    assert n == libm_sweep.ALL and not counts.any(), libm_sweep.report_bad(["expf_glibc"], counts, bad)
