// libm_sweep.cpp — host side of the exhaustive fp32 sweeps (test infrastructure, compiled at test time by
// tests/libm_sweep.py).
//
// Every function runs over a run of n arguments whose bit patterns are first, first + 1, ... (wrapping at 2^32), split
// over `threads` std::threads, and counts mismatches bit for bit, two NaNs counting as equal.  Each returns the
// mismatch count(s) and writes the lowest mismatching argument bits (up to max_bad per count) to `bad`.
//   lx_check_trig   device sinf / cosf / sincosf outputs against the running libm (+ sincosf against the separate calls)
//   lx_check_exp    device expf output against libm expf
//   lx_compare      two result arrays of the same arguments against each other
//   lx_host_trig    the host build of csrc/sincosf_glibc.h against libm (sinf, cosf, both outputs of sincosf)
//   lx_host_exp     the host build of expf_glibc against libm
//   lx_power        how many arguments have a libm sinf / cosf / expf that is not float64 libm rounded to fp32
//   lx_check_pack   best_pack / best_unpack outputs of a score sweep: round trip, index, no zero, monotone order
//   lx_inverse3_fma counts the cases where cofactors as fmaf(a, b, -c*d) change the port's `H.inverse() * dTr`
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <thread>
#include <vector>

#include "sincosf_glibc.h"

namespace {

inline uint32_t bits(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  return u;
}
inline float from_bits(uint32_t u) {
  float f;
  memcpy(&f, &u, 4);
  return f;
}
inline bool same(float a, float b) { return bits(a) == bits(b) || (a != a && b != b); }

// K mismatch counters, each keeping its lowest max_bad arguments
template <int K>
struct Tally {
  long long n[K] = {};
  std::vector<uint32_t> first[K];
  void add(int k, uint32_t arg, int max_bad) {
    ++n[k];
    if ((int)first[k].size() < max_bad) first[k].push_back(arg);
  }
};

// body(tally, i, arg) over [0, n), split into `threads` contiguous pieces; results merged in piece order, so the
// recorded arguments are the lowest indices
template <int K, class F>
void sweep(long long n, int threads, int max_bad, long long* counts, uint32_t* bad, F body) {
  threads = std::max(1, threads);
  std::vector<Tally<K>> t(threads);
  std::vector<std::thread> th;
  for (int w = 0; w < threads; ++w)
    th.emplace_back([&, w] {
      const long long b = n * w / threads, e = n * (w + 1) / threads;
      for (long long i = b; i < e; ++i) body(t[w], i, max_bad);
    });
  for (auto& x : th) x.join();
  for (int k = 0; k < K; ++k) {
    counts[k] = 0;
    int m = 0;
    for (int w = 0; w < threads; ++w) {
      counts[k] += t[w].n[k];
      for (uint32_t a : t[w].first[k])
        if (m < max_bad) bad[k * max_bad + m++] = a;
    }
    for (; m < max_bad; ++m) bad[k * max_bad + m] = 0;
  }
}

float cof_fma(const float m[9], int i, int j) {
  const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
  return fmaf(m[3 * i1 + j1], m[3 * i2 + j2], -(m[3 * i1 + j2] * m[3 * i2 + j1]));
}

// oracle/hs_oracle.c inverse3_times with every cofactor fused: the variant the power count is about
void inverse3_times_fma(const float m[9], const float v[3], float out[3]) {
  const float c0 = cof_fma(m, 0, 0), c1 = cof_fma(m, 1, 0), c2 = cof_fma(m, 2, 0);
  const float det = c0 * m[0] + (c1 * m[3] + c2 * m[6]);
  const float invdet = 1.0f / det;
  float inv[9];
  inv[0] = c0 * invdet;
  inv[1] = c1 * invdet;
  inv[2] = c2 * invdet;
  inv[3] = cof_fma(m, 0, 1) * invdet;
  inv[4] = cof_fma(m, 1, 1) * invdet;
  inv[5] = cof_fma(m, 2, 1) * invdet;
  inv[6] = cof_fma(m, 0, 2) * invdet;
  inv[7] = cof_fma(m, 1, 2) * invdet;
  inv[8] = cof_fma(m, 2, 2) * invdet;
  for (int r = 0; r < 3; ++r) out[r] = inv[3 * r] * v[0] + (inv[3 * r + 1] * v[1] + inv[3 * r + 2] * v[2]);
}

}  // namespace

extern "C" {

// counts[6] / bad[6 * max_bad]: s vs sinf, c vs cosf, ss vs sinf, sc vs cosf, ss vs s, sc vs c
void lx_check_trig(uint32_t first, long long n, const float* s, const float* c, const float* ss, const float* sc,
                   int threads, int max_bad, long long* counts, uint32_t* bad) {
  sweep<6>(n, threads, max_bad, counts, bad, [&](Tally<6>& t, long long i, int mb) {
    const uint32_t a = first + (uint32_t)i;
    const float x = from_bits(a), ls = sinf(x), lc = cosf(x);
    if (!same(s[i], ls)) t.add(0, a, mb);
    if (!same(c[i], lc)) t.add(1, a, mb);
    if (!same(ss[i], ls)) t.add(2, a, mb);
    if (!same(sc[i], lc)) t.add(3, a, mb);
    if (!same(ss[i], s[i])) t.add(4, a, mb);
    if (!same(sc[i], c[i])) t.add(5, a, mb);
  });
}

void lx_check_exp(uint32_t first, long long n, const float* e, int threads, int max_bad, long long* counts, uint32_t* bad) {
  sweep<1>(n, threads, max_bad, counts, bad, [&](Tally<1>& t, long long i, int mb) {
    const uint32_t a = first + (uint32_t)i;
    if (!same(e[i], expf(from_bits(a)))) t.add(0, a, mb);
  });
}

void lx_compare(uint32_t first, long long n, const float* x, const float* y, int threads, int max_bad, long long* counts,
                uint32_t* bad) {
  sweep<1>(n, threads, max_bad, counts, bad, [&](Tally<1>& t, long long i, int mb) {
    if (!same(x[i], y[i])) t.add(0, first + (uint32_t)i, mb);
  });
}

// counts[4]: sinf_glibc, cosf_glibc, sincosf_glibc's sine, its cosine — each against libm
void lx_host_trig(uint32_t first, long long n, int threads, int max_bad, long long* counts, uint32_t* bad) {
  sweep<4>(n, threads, max_bad, counts, bad, [&](Tally<4>& t, long long i, int mb) {
    const uint32_t a = first + (uint32_t)i;
    const float x = from_bits(a), ls = sinf(x), lc = cosf(x);
    float hs, hc;
    hsb::sincosf_glibc(x, &hs, &hc);
    if (!same(hsb::sinf_glibc(x), ls)) t.add(0, a, mb);
    if (!same(hsb::cosf_glibc(x), lc)) t.add(1, a, mb);
    if (!same(hs, ls)) t.add(2, a, mb);
    if (!same(hc, lc)) t.add(3, a, mb);
  });
}

void lx_host_exp(uint32_t first, long long n, int threads, int max_bad, long long* counts, uint32_t* bad) {
  sweep<1>(n, threads, max_bad, counts, bad, [&](Tally<1>& t, long long i, int mb) {
    const uint32_t a = first + (uint32_t)i;
    const float x = from_bits(a);
    if (!same(hsb::expf_glibc(x), expf(x))) t.add(0, a, mb);
  });
}

// every stride-th argument of the run; counts[2]: sinf or cosf differs from (float)sin/cos((double)x), expf differs
// from (float)exp((double)x)
void lx_power(uint32_t first, long long n, long long stride, int threads, int max_bad, long long* counts, uint32_t* bad) {
  sweep<2>((n + stride - 1) / stride, threads, max_bad, counts, bad, [&](Tally<2>& t, long long j, int mb) {
    const uint32_t a = first + (uint32_t)(j * stride);
    const float x = from_bits(a);
    const double xd = (double)x;
    if (!same(sinf(x), (float)sin(xd)) || !same(cosf(x), (float)cos(xd))) t.add(0, a, mb);
    if (!same(expf(x), (float)exp(xd))) t.add(1, a, mb);
  });
}

// a best_pack sweep over scores first .. first + n - 1 with one finite pose and one index.  prev: the packed value of
// score first - 1 (has_prev 0 when first is 0).  counts[4]:
//   0  best_unpack's score is not the score's bits (NaN: not -1.0f's bits)
//   1  best_unpack's index is not `index`
//   2  the packed value is 0, the empty-accumulator sentinel
//   3  order: over +0 .. +inf (bits 0 .. 0x7f800000) the packed value does not increase strictly with the bits, over
//      -0 .. -inf (0x80000000 .. 0xff800000) it does not decrease strictly
void lx_check_pack(uint32_t first, long long n, const unsigned long long* packed, const float* score,
                   const uint32_t* index_out, uint32_t index, int has_prev, unsigned long long prev, int threads,
                   int max_bad, long long* counts, uint32_t* bad) {
  const float minus_one = -1.0f;
  sweep<4>(n, threads, max_bad, counts, bad, [&](Tally<4>& t, long long i, int mb) {
    const uint32_t a = first + (uint32_t)i;
    const float s = from_bits(a);
    if (bits(score[i]) != bits(s != s ? minus_one : s)) t.add(0, a, mb);
    if (index_out[i] != index) t.add(1, a, mb);
    if (packed[i] == 0ull) t.add(2, a, mb);
    if (i > 0 || has_prev) {
      const uint32_t b = a - 1u;
      const unsigned long long pv = i > 0 ? packed[i - 1] : prev;
      if (a >= 1u && a <= 0x7f800000u && b <= 0x7f800000u && !(packed[i] > pv)) t.add(3, a, mb);
      if (a > 0x80000000u && a <= 0xff800000u && !(packed[i] < pv)) t.add(3, a, mb);
    }
  });
}

// m n x 9, v n x 3, port n x 3 (hso_inverse3_times): how many cases the fused-cofactor variant changes
long long lx_inverse3_fma(const float* m, const float* v, long long n, const float* port, int threads) {
  long long counts[1];
  uint32_t bad[1];
  sweep<1>(n, threads, 1, counts, bad, [&](Tally<1>& t, long long i, int mb) {
    float o[3];
    inverse3_times_fma(m + 9 * i, v + 3 * i, o);
    if (!same(o[0], port[3 * i]) || !same(o[1], port[3 * i + 1]) || !same(o[2], port[3 * i + 2])) t.add(0, (uint32_t)i, mb);
  });
  return counts[0];
}

}  // extern "C"
