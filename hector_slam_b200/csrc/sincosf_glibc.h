// sincosf_glibc.h — sinf / cosf evaluated the way glibc 2.39's x86-64 FMA build does.
//
// Why: the reference calls sinf/cosf on the pose angle (OccGridMapUtil.h:70-71, Rotation2Df at
// :351, OccGridMapBase.h:130-131).  glibc's single-precision sin/cos (Szabolcs Nagy's routines,
// sysdeps/ieee754/flt-32/s_sinf.c, s_cosf.c, sincosf.h) are NOT correctly rounded: they differ
// from the correctly rounded value on 1.3 % of the arguments in [-pi, pi] (measured here).  One
// ulp of cos/sin moves a map coordinate of ~600 cells by ~6e-5 cell, and on a sparsely mapped
// grid that can move the matcher's answer by more than the 1e-4 parity bar (measured: 1.3e-3 on
// one step of the 40 Hz stream test).  So the pose angle's sine and cosine are evaluated with
// glibc's own algorithm: argument reduced with one fused multiply-add against pi/2, degree-7 /
// degree-8 polynomials in DOUBLE with exactly the multiply / fused-multiply-add sequence of the
// FMA-enabled build (transcribed from the disassembly of __sinf_fma / __cosf_fma in
// libm.so.6 2.39-0ubuntu8.5, which every AVX2+FMA host selects through ifunc), constants read
// from that library's __sincosf_table.  tests/test_sincosf_glibc.py checks the host build of
// this header against the running libm bit for bit on every fp32 argument, and
// tests/test_gpu_scalar_functions.py the device build.
//
// Provenance / licence: this header is a restatement of the GNU C Library's single-precision
// sin/cos algorithm (glibc 2.39, sysdeps/ieee754/flt-32/{s_sinf.c,s_cosf.c,sincosf.h,
// sincosf_data.c}; Copyright (C) Free Software Foundation, Inc., contributed by Arm Ltd.,
// licensed LGPL-2.1-or-later).  The polynomial coefficients and the operation order are glibc's
// (they have to be, that is the point); no glibc source text is included.  Treat this file as
// LGPL-2.1-or-later derived material when redistributing.
// Platform note: "as glibc evaluates them" means the x86-64 FMA ifunc variant; on an aarch64 host
// (Grace) glibc's generic build uses the same algorithm with compiler-chosen contraction, so a
// reference running there may differ in the last bit and the table below would need re-pinning.
//
// Arguments with |y| >= 120 take glibc's large-argument reduction (reduce_large): the float's
// 24-bit mantissa times a 96-bit window of 4/pi chosen by the exponent, the quadrant from the top
// two bits and the remainder converted to double and scaled by pi/2^62; then the same
// polynomials.  A correctly rounded sin/cos differs from glibc there on ~1.3 % of the arguments,
// and pose angles reach it unnormalised (the hint of a match's coarsest level, the pose given to
// the map writer, the poses of the likelihood / covariance entry points).  The 4/pi table
// (glibc's __inv_pio4) is overlapping 32-bit windows of 4/pi's binary expansion at 8-bit steps;
// tests/test_sincosf_glibc.py derives it from a computed pi.  +-inf and NaN return NaN.
#ifndef HSB_SINCOSF_GLIBC_H
#define HSB_SINCOSF_GLIBC_H

#include <math.h>
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define HSB_HD __host__ __device__ __forceinline__
#else
#define HSB_HD static inline
#endif

namespace hsb {

#if defined(__CUDA_ARCH__)
#define HSB_DMUL(a, b) __dmul_rn((a), (b))
#define HSB_DFMA(a, b, c) __fma_rn((a), (b), (c))
#else
#define HSB_DMUL(a, b) ((a) * (b))
#define HSB_DFMA(a, b, c) fma((a), (b), (c))
#endif

// __sincosf_table[0]; table[1] has c0..c4 negated
#define HSB_SC_HPI_INV 0x1.45f306dc9c883p+23 /* 2/pi * 2^24 */
#define HSB_SC_HPI 0x1.921fb54442d18p+0      /* pi/2 */
#define HSB_SC_C0 0x1.0000000000000p+0
#define HSB_SC_C1 -0x1.ffffffd0c621cp-2
#define HSB_SC_C2 0x1.55553e1068f19p-5
#define HSB_SC_C3 -0x1.6c087e89a359dp-10
#define HSB_SC_C4 0x1.99343027bf8c3p-16
#define HSB_SC_S1 -0x1.555545995a603p-3
#define HSB_SC_S2 0x1.1107605230bc4p-7
#define HSB_SC_S3 -0x1.994eb3774cf24p-13

HSB_HD uint32_t f32_bits(float f) {
#if defined(__CUDA_ARCH__)
  return __float_as_uint(f);
#else
  uint32_t u;
  memcpy(&u, &f, 4);
  return u;
#endif
}

// sinf_poly with n even: x + x^3*s1 + x^7*(s2 + x^2*s3)
HSB_HD double sc_sin_poly(double xs, double x2) {
  const double s1_ = HSB_DFMA(x2, HSB_SC_S3, HSB_SC_S2);
  const double x3 = HSB_DMUL(x2, xs);
  const double x7 = HSB_DMUL(x2, x3);
  const double s = HSB_DFMA(x3, HSB_SC_S1, xs);
  return HSB_DFMA(s1_, x7, s);
}
// sinf_poly with n odd: (c0 + x^2*c1) + x^4*c2 + x^6*(c3 + x^2*c4); `neg` selects table[1]
HSB_HD double sc_cos_poly(double x2, bool neg) {
  const double sg = neg ? -1.0 : 1.0;  // negating every coefficient negates every partial result exactly
  const double x4 = HSB_DMUL(x2, x2);
  const double c1_ = HSB_DFMA(x2, sg * HSB_SC_C1, sg * HSB_SC_C0);
  const double c2_ = HSB_DFMA(x2, sg * HSB_SC_C4, sg * HSB_SC_C3);
  const double x6 = HSB_DMUL(x2, x4);
  const double c = HSB_DFMA(x4, sg * HSB_SC_C2, c1_);
  return HSB_DFMA(c2_, x6, c);
}

// reduce_fast: n = round(x * 2/pi), xr = x - n*pi/2 (one fused operation)
HSB_HD double sc_reduce(double x, int* np) {
  const double r = HSB_DMUL(x, HSB_SC_HPI_INV);
  const int n = ((int32_t)r + 0x800000) >> 24;  // cvttsd2si, then arithmetic shift
  *np = n;
  return HSB_DFMA(-(double)n, HSB_SC_HPI, x);
}

// __inv_pio4: word i = floor(4/pi * 2^(8i+7)) mod 2^32
#define HSB_INV_PIO4_TABLE \
    0x000000a2u, 0x0000a2f9u, 0x00a2f983u, 0xa2f9836eu, 0xf9836e4eu, 0x836e4e44u, 0x6e4e4415u, 0x4e441529u, \
    0x441529fcu, 0x1529fc27u, 0x29fc2757u, 0xfc2757d1u, 0x2757d1f5u, 0x57d1f534u, 0xd1f534ddu, 0xf534ddc0u, \
    0x34ddc0dbu, 0xddc0db62u, 0xc0db6295u, 0xdb629599u, 0x6295993cu, 0x95993c43u, 0x993c4390u, 0x3c439041u,
static const uint32_t hsb_inv_pio4_host[24] = {HSB_INV_PIO4_TABLE};
#if defined(__CUDACC__)
__device__ const uint32_t hsb_inv_pio4_dev[24] = {HSB_INV_PIO4_TABLE};
#endif

// reduce_large, for 120 <= |y| < inf given the float's bits: returns x - n*pi/2 for the quadrant n (of |y|; the caller
// folds the sign in), from a 96-bit slice of 4/pi selected by the exponent
HSB_HD double sc_reduce_large(uint32_t xi, int* np) {
#if defined(__CUDA_ARCH__)
  const uint32_t* arr = &hsb_inv_pio4_dev[(xi >> 26) & 15];
#else
  const uint32_t* arr = &hsb_inv_pio4_host[(xi >> 26) & 15];
#endif
  const int shift = (xi >> 23) & 7;
  xi = ((xi & 0xffffffu) | 0x800000u) << shift;
  uint64_t res0 = (uint64_t)(uint32_t)(xi * arr[0]);   // a 32-bit product: wraps before it is widened
  const uint64_t res1 = (uint64_t)xi * arr[4];
  const uint64_t res2 = (uint64_t)xi * arr[8];
  res0 = (res2 >> 32) | (res0 << 32);
  res0 += res1;
  const uint64_t n = (res0 + (1ull << 61)) >> 62;
  res0 -= n << 62;
  *np = (int)n;
#if defined(__CUDA_ARCH__)
  return __dmul_rn(__ll2double_rn((long long)res0), 0x1.921FB54442D18p-62);
#else
  return (double)(int64_t)res0 * 0x1.921FB54442D18p-62;
#endif
}

// sin (want_cos false) or cos of 120 <= |y| < inf as glibc: the sign bit joins the quadrant for the sign and table
// choice, the quadrant's parity (flipped for cos) picks the polynomial
HSB_HD float sc_large(float y, bool want_cos) {
  const uint32_t xi = f32_bits(y);
  int n;
  const double xr = sc_reduce_large(xi, &n);
  const int q = (n + (int)(xi >> 31)) & 3;
  const double sign = (q == 1 || q == 2) ? -1.0 : 1.0;
  const double xs = HSB_DMUL(xr, sign), x2 = HSB_DMUL(xr, xr);
  if (((n ^ (want_cos ? 1 : 0)) & 1) == 0) return (float)sc_sin_poly(xs, x2);
  return (float)sc_cos_poly(x2, (q & 2) != 0);
}

HSB_HD float sinf_glibc(float y) {
  const double x = (double)y;
  const uint32_t top = (f32_bits(y) >> 20) & 0x7ffu;
  if (top <= 0x3f3u) {                 // |y| < pi/4
    if (top <= 0x397u) return y;       // |y| < 2^-12
    return (float)sc_sin_poly(x, HSB_DMUL(x, x));
  }
  if (top <= 0x42eu) {                 // |y| < 120
    int n;
    const double xr = sc_reduce(x, &n);
    const double x2 = HSB_DMUL(xr, xr);
    if ((n & 1) == 0) {
      const double sign = ((n & 3) == 1 || (n & 3) == 2) ? -1.0 : 1.0;  // sign[4] = {1,-1,-1,1}
      return (float)sc_sin_poly(HSB_DMUL(xr, sign), x2);
    }
    return (float)sc_cos_poly(x2, (n & 2) != 0);
  }
  if (top < 0x7f8u) return sc_large(y, false);
  return y - y;                        // +-inf, NaN
}

HSB_HD float cosf_glibc(float y) {
  const double x = (double)y;
  const uint32_t top = (f32_bits(y) >> 20) & 0x7ffu;
  if (top <= 0x3f3u) {
    if (top <= 0x397u) return 1.0f;
    return (float)sc_cos_poly(HSB_DMUL(x, x), false);
  }
  if (top <= 0x42eu) {
    int n;
    const double xr = sc_reduce(x, &n);
    const double x2 = HSB_DMUL(xr, xr);
    if ((n & 1) != 0) {
      const double sign = ((n & 3) == 1 || (n & 3) == 2) ? -1.0 : 1.0;
      return (float)sc_sin_poly(HSB_DMUL(xr, sign), x2);
    }
    return (float)sc_cos_poly(x2, (n & 2) != 0);
  }
  if (top < 0x7f8u) return sc_large(y, true);
  return y - y;
}

// sinf_glibc and cosf_glibc of the same argument with ONE argument reduction: the two polynomials are the ones the
// separate functions evaluate (n even: sin from the sine polynomial, cos from the cosine polynomial; n odd: swapped),
// so both results are bit-identical to the separate calls (tests/test_sincosf_glibc.py).
HSB_HD void sincosf_glibc(float y, float* sp, float* cp) {
  const double x = (double)y;
  const uint32_t top = (f32_bits(y) >> 20) & 0x7ffu;
  if (top <= 0x3f3u) {                 // |y| < pi/4
    if (top <= 0x397u) {               // |y| < 2^-12
      *sp = y;
      *cp = 1.0f;
      return;
    }
    const double x2 = HSB_DMUL(x, x);
    *sp = (float)sc_sin_poly(x, x2);
    *cp = (float)sc_cos_poly(x2, false);
    return;
  }
  if (top <= 0x42eu) {                 // |y| < 120
    int n;
    const double xr = sc_reduce(x, &n);
    const double x2 = HSB_DMUL(xr, xr);
    const double sign = ((n & 3) == 1 || (n & 3) == 2) ? -1.0 : 1.0;
    const float a = (float)sc_sin_poly(HSB_DMUL(xr, sign), x2);
    const float b = (float)sc_cos_poly(x2, (n & 2) != 0);
    const bool even = (n & 1) == 0;
    *sp = even ? a : b;
    *cp = even ? b : a;
    return;
  }
  if (top < 0x7f8u) {
    const uint32_t xi = f32_bits(y);
    int n;
    const double xr = sc_reduce_large(xi, &n);
    const int q = (n + (int)(xi >> 31)) & 3;
    const double sign = (q == 1 || q == 2) ? -1.0 : 1.0;
    const double x2 = HSB_DMUL(xr, xr);
    const float a = (float)sc_sin_poly(HSB_DMUL(xr, sign), x2);
    const float b = (float)sc_cos_poly(x2, (q & 2) != 0);
    const bool even = (n & 1) == 0;
    *sp = even ? a : b;
    *cp = even ? b : a;
    return;
  }
  *sp = *cp = y - y;
}

// ---- expf as glibc 2.39's x86-64 FMA build evaluates it (sysdeps/ieee754/flt-32/e_expf.c, exp2f_data.c) -----------------
// Why: the reference turns log-odds into the probability the matcher interpolates with
// `float odds = exp(l); return odds / (odds + 1.0f)` (GridMapLogOdds.h:165-166; exp(float) resolves to expf).  glibc's
// expf is accurate to 0.502 ulp, not correctly rounded: a correctly rounded exp differs from it by one ulp on ~1 % of
// the arguments, i.e. on that share of the cells of a probability plane.  With this restatement the plane is the
// reference's bit for bit.  Operation order transcribed from the disassembly of __expf_fma (libm.so.6 2.39-0ubuntu8.5):
//   kd = fma(InvLn2N, x, SHIFT); ki = bits(kd); kd -= SHIFT; r = fma(InvLn2N, x, -kd);
//   s = asdouble(T[ki % 32] + (ki << 47)); z = fma(r, C0, C1); r2 = r * r; y = fma(r, C2, 1); y = fma(z, r2, y); return (float)(y * s)
// constants and the 2^(i/32) table read from that library's __exp2f_data.  Out-of-range arguments as glibc handles them:
// NaN / +inf -> x + x, x > 0x1.62e42ep6 -> +inf, x < -0x1.9fe368p6 -> +0, x < -0x1.9d1d9ep6 -> 0x1.4p-75f squared (= 2^-149).
// tests/test_sincosf_glibc.py checks the host build against the running libm bit for bit on every fp32 argument,
// tests/test_gpu_scalar_functions.py the device build.
#define HSB_EXPF_SHIFT 0x1.8p+52
#define HSB_EXPF_INVLN2N 0x1.71547652b82fep+5
#define HSB_EXPF_C0 0x1.c6af84b912394p-20
#define HSB_EXPF_C1 0x1.ebfce50fac4f3p-13
#define HSB_EXPF_C2 0x1.62e42ff0c52d6p-6

#define HSB_EXP2F_TABLE \
    0x3ff0000000000000ull, 0x3fefd9b0d3158574ull, 0x3fefb5586cf9890full, 0x3fef9301d0125b51ull, \
    0x3fef72b83c7d517bull, 0x3fef54873168b9aaull, 0x3fef387a6e756238ull, 0x3fef1e9df51fdee1ull, \
    0x3fef06fe0a31b715ull, 0x3feef1a7373aa9cbull, 0x3feedea64c123422ull, 0x3feece086061892dull, \
    0x3feebfdad5362a27ull, 0x3feeb42b569d4f82ull, 0x3feeab07dd485429ull, 0x3feea47eb03a5585ull, \
    0x3feea09e667f3bcdull, 0x3fee9f75e8ec5f74ull, 0x3feea11473eb0187ull, 0x3feea589994cce13ull, \
    0x3feeace5422aa0dbull, 0x3feeb737b0cdc5e5ull, 0x3feec49182a3f090ull, 0x3feed503b23e255dull, \
    0x3feee89f995ad3adull, 0x3feeff76f2fb5e47ull, 0x3fef199bdd85529cull, 0x3fef3720dcef9069ull, \
    0x3fef5818dcfba487ull, 0x3fef7c97337b9b5full, 0x3fefa4afa2a490daull, 0x3fefd0765b6e4540ull,
static const unsigned long long hsb_exp2f_table_host[32] = {HSB_EXP2F_TABLE};
#if defined(__CUDACC__)
// (global, not __constant__ memory: the index differs from lane to lane, and divergent constant-bank reads serialise)
__device__ const unsigned long long hsb_exp2f_table_dev[32] = {HSB_EXP2F_TABLE};
#endif

HSB_HD float expf_glibc(float x) {
  const uint32_t ux = f32_bits(x);
  const uint32_t abstop = (ux >> 20) & 0x7ffu;
  if (abstop > 0x42au) {   // |x| >= 88 or NaN
    if (ux == 0xff800000u) return 0.0f;
    if (abstop >= 0x7f8u) return x + x;
    if (x > 0x1.62e42ep6f) return INFINITY;
    if (x < -0x1.9fe368p6f) return 0.0f;
    if (x < -0x1.9d1d9ep6f) {
#if defined(__CUDA_ARCH__)
      return __uint_as_float(1u);   // 0x1.4p-75f * 0x1.4p-75f rounds to the smallest denormal
#else
      volatile float tiny = 0x1.4p-75f;
      return tiny * tiny;
#endif
    }
  }
  const double xd = (double)x;
  double kd = HSB_DFMA(HSB_EXPF_INVLN2N, xd, HSB_EXPF_SHIFT);
  uint64_t ki;
#if defined(__CUDA_ARCH__)
  ki = (uint64_t)__double_as_longlong(kd);
  kd = __dadd_rn(kd, -HSB_EXPF_SHIFT);
#else
  memcpy(&ki, &kd, 8);
  kd = kd - HSB_EXPF_SHIFT;
#endif
  const double r = HSB_DFMA(HSB_EXPF_INVLN2N, xd, -kd);
#if defined(__CUDA_ARCH__)
  const uint64_t t = (uint64_t)hsb_exp2f_table_dev[ki & 31u] + (ki << 47);
#else
  const uint64_t t = (uint64_t)hsb_exp2f_table_host[ki & 31u] + (ki << 47);
#endif
  double s;
#if defined(__CUDA_ARCH__)
  s = __longlong_as_double((long long)t);
#else
  memcpy(&s, &t, 8);
#endif
  const double z = HSB_DFMA(r, HSB_EXPF_C0, HSB_EXPF_C1);
  const double r2 = HSB_DMUL(r, r);
  double y = HSB_DFMA(r, HSB_EXPF_C2, 1.0);
  y = HSB_DFMA(z, r2, y);
  y = HSB_DMUL(y, s);
  return (float)y;
}

}  // namespace hsb
#endif
