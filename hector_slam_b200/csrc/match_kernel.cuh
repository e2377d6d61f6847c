// match_kernel.cuh — K1: whole multi-level Gauss-Newton scan match on the device (sm_90a).
//
// What it replaces (paths under the reference's hector_mapping/include/hector_slam_lib/):
//   MapRepMultiMap::matchData                 slam_main/MapRepMultiMap.h:116-132  (level schedule)
//   ScanMatcher::matchData                    matcher/ScanMatcher.h:54-190         (GN outer loop)
//   ScanMatcher::estimateTransformationLogLh  matcher/ScanMatcher.h:194-221        (gate, 3x3 solve, clamp)
//   OccGridMapUtil::getCompleteHessianDerivs  map/OccGridMapUtil.h:64-104          (H / dTr accumulation)
//   OccGridMapUtil::interpMapValueWithDerivatives  map/OccGridMapUtil.h:287-347    (bilinear value + gradient)
//
// Shape: a "group" of W warps owns one scan; G groups share a CTA; the grid is persistent and
// strides over the batch.  The scan's endpoints are staged once into shared memory with one TMA
// bulk copy (cp.async.bulk + mbarrier); every Gauss-Newton evaluation then walks the endpoints
// lane-strided, gathers the four probability cells per endpoint (four LDGs on the linear plane or
// one tex2Dgather on the block-linear twin), accumulates the 6+3 sums in registers, reduces them
// with warp shuffles (+ one shared-memory exchange when W > 1) and every thread of the group
// redundantly solves the 3x3 system, so the pose never leaves registers between evaluations and
// levels.  No host round trip, no global-memory traffic besides the gathers and 48 B of result.
#ifndef HSB_MATCH_KERNEL_CUH
#define HSB_MATCH_KERNEL_CUH

#include "hsb_internal.h"
#include "sincosf_glibc.h"

namespace hsb {

// MODE_ANY: the gather path is decided per level descriptor at run time — tex2Dgather where the level has a texture
// twin (tex != 0), four loads otherwise — each branch exactly its own mode's arithmetic.  Only the kernels a
// heterogeneous group holding both modes launches are instantiated with it.
enum { MODE_LDG = 1, MODE_TEX = 2, MODE_ANY = 3 };

struct Acc {
  float h00, h11, h22, h01, h02, h12, d0, d1, d2;
};

__device__ __forceinline__ void acc_zero(Acc& a) { a.h00 = a.h11 = a.h22 = a.h01 = a.h02 = a.h12 = a.d0 = a.d1 = a.d2 = 0.f; }

// out[r] = m[r][0]*vx + (m[r][1]*vy + m[r][2]*1), each operation rounded separately — the order
// the oracle fixes for Transform * vector (oracle/shim/Eigen/Geometry).  Used for the
// world<->map pose conversions (GridMapBase.h:226-239), where we want the oracle's bits.
__device__ __forceinline__ void affine_apply_exact(const float* m, float vx, float vy, float& ox, float& oy) {
  ox = __fadd_rn(__fmul_rn(m[0], vx), __fadd_rn(__fmul_rn(m[1], vy), m[2]));
  oy = __fadd_rn(__fmul_rn(m[3], vx), __fadd_rn(__fmul_rn(m[4], vy), m[5]));
}

// util::normalize_angle, UtilFunctions.h:37-49:  a = fmod(fmod(angle, 2pi) + 2pi, 2pi); if (a > pi) a -= 2pi,
// in double because M_PI is a double, narrowed to float where the reference narrows.  Both fmods are
// exact operations; for |angle| < 2pi the first is the identity and the second is one exact
// subtraction (Sterbenz), so the common case needs no fmod at all — bit-identical either way (on every fp32 argument:
// tests/test_gpu_scalar_functions.py).
__device__ __forceinline__ float normalize_angle(float angle) {
  const double two_pi = 2.0 * 3.14159265358979323846;
  double r = (double)angle;
  if (!(fabs(r) < two_pi)) r = fmod(r, two_pi);
  r += two_pi;                       // in (0, 4pi)
  if (r >= two_pi) r -= two_pi;      // == fmod(r, two_pi), exact
  float a = (float)r;
  if ((double)a > 3.14159265358979323846) a = (float)((double)a - two_pi);
  return a;
}

// util::poseDifferenceLargerThan (util/UtilFunctions.h:73-92): float norm, the angle wrapped with double pi.
__device__ __forceinline__ bool pose_difference_larger_than(const float* p1, const float* p2, float dist_thresh,
                                                            float ang_thresh) {
  const float dx = __fsub_rn(p1[0], p2[0]), dy = __fsub_rn(p1[1], p2[1]);
  if (__fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy))) > dist_thresh) return true;
  float a = __fsub_rn(p1[2], p2[2]);
  const double pi = 3.14159265358979323846, two_pi = pi * 2.0;
  if ((double)a > pi) a = (float)((double)a - two_pi);
  else if ((double)a < -pi) a = (float)((double)a + two_pi);
  return fabsf(a) > ang_thresh;
}

// HectorSlamProcessor::update's gate (slam_main/HectorSlamProcessor.h:83-95) evaluated on the device so that a
// fused step needs no host round trip between match and map write.
//   state: [0..2] lastMapUpdatePose, [3] out: 1.0f if the map is to be written by this step
//   in   : [0] minDist, [1] minAngle, [2] force (map_without_matching)
// pose_out (device) and pose_out_host (mapped host memory, may be null) receive the step's pose (the matched
// pose, or the hint when matching is skipped) and, in [3], a copy of the flag.
__device__ __forceinline__ void slam_gate(float* __restrict__ state, const float* __restrict__ in, float px, float py, float ppsi,
                                          float* pose_out, float* pose_out_host) {
  const float p[3] = {px, py, ppsi};
  const bool upd = pose_difference_larger_than(p, state, in[0], in[1]) || in[2] != 0.0f;
  if (upd) { state[0] = p[0]; state[1] = p[1]; state[2] = p[2]; }
  const float flag = upd ? 1.0f : 0.0f;
  state[3] = flag;
  pose_out[0] = p[0]; pose_out[1] = p[1]; pose_out[2] = p[2];
  pose_out[3] = flag;
  if (pose_out_host) {   // mapped pinned host memory: the result needs no copy operation
    pose_out_host[0] = p[0]; pose_out_host[1] = p[1]; pose_out_host[2] = p[2];
    pose_out_host[3] = flag;
  }
}

// Eigen's fixed-size 3x3 inverse times vector (ScanMatcher.h:205 `H.inverse() * dTr`): cyclic
// cofactors, det from column 0, multiply by 1/det, no pivoting — restated with explicitly rounded
// operations (no FMA contraction) because H is often ill-conditioned and the cancellation in the
// cofactors is where a different rounding would be amplified.  Same order as
// oracle/hs_oracle.c inverse3_times.
__device__ __forceinline__ float cof(float a, float b, float c, float d) { return __fsub_rn(__fmul_rn(a, b), __fmul_rn(c, d)); }

__device__ __forceinline__ void solve3(const Acc& s, float& o0, float& o1, float& o2) {
  // m = [[h00,h01,h02],[h01,h11,h12],[h02,h12,h22]]
  const float m00 = s.h00, m01 = s.h01, m02 = s.h02, m10 = s.h01, m11 = s.h11, m12 = s.h12, m20 = s.h02, m21 = s.h12,
              m22 = s.h22;
  // cof(i,j) = m[i1][j1]*m[i2][j2] - m[i1][j2]*m[i2][j1], i1=(i+1)%3 ...
  const float c00 = cof(m11, m22, m12, m21);
  const float c10 = cof(m21, m02, m22, m01);
  const float c20 = cof(m01, m12, m02, m11);
  const float det = __fadd_rn(__fmul_rn(c00, m00), __fadd_rn(__fmul_rn(c10, m10), __fmul_rn(c20, m20)));
  const float invdet = __fdiv_rn(1.0f, det);
  const float c01 = cof(m12, m20, m10, m22);
  const float c11 = cof(m22, m00, m20, m02);
  const float c21 = cof(m02, m10, m00, m12);
  const float c02 = cof(m10, m21, m11, m20);
  const float c12 = cof(m20, m01, m21, m00);
  const float c22 = cof(m00, m11, m01, m10);
  // inv(i,j) = cof(j,i) * invdet
  const float i00 = __fmul_rn(c00, invdet), i01 = __fmul_rn(c10, invdet), i02 = __fmul_rn(c20, invdet);
  const float i10 = __fmul_rn(c01, invdet), i11 = __fmul_rn(c11, invdet), i12 = __fmul_rn(c21, invdet);
  const float i20 = __fmul_rn(c02, invdet), i21 = __fmul_rn(c12, invdet), i22 = __fmul_rn(c22, invdet);
  o0 = __fadd_rn(__fmul_rn(i00, s.d0), __fadd_rn(__fmul_rn(i01, s.d1), __fmul_rn(i02, s.d2)));
  o1 = __fadd_rn(__fmul_rn(i10, s.d0), __fadd_rn(__fmul_rn(i11, s.d1), __fmul_rn(i12, s.d2)));
  o2 = __fadd_rn(__fmul_rn(i20, s.d0), __fadd_rn(__fmul_rn(i21, s.d1), __fmul_rn(i22, s.d2)));
}

// ---- one batch of U endpoints of one evaluation ------------------------------------------------
// OccGridMapUtil.h:76-98 with interpMapValueWithDerivatives (:287-347) inlined, restructured so
// that the U gathers of a batch are all in flight before the first one is consumed (branch-free
// address phase, predicated accumulate phase).
//
// Rounding.  Measured against the oracle (scripts/parity_probe.py): the summation ORDER
// of H/dTr does not move the result (the Gauss-Newton fixed point is reached bit-identically),
// but the rounding of the map coordinate q = T*p does — q is ~1e3 cells, so one ulp of q is
// ~6e-5 of a cell in the interpolation weights.  q is therefore computed with the oracle's exact
// operation sequence (oracle/hs_oracle.c affine2_apply: m[0]*px + (m[1]*py + m[2]), four products
// shared with rotDeriv), every operation rounded separately.  HSB_FP_VARIANT selects how the rest
// is evaluated: 0 = every operation as the oracle (no contraction anywhere), 1 = the reference's
// formulas with FMA contraction allowed, 2 = algebraically regrouped bilinear form (fewest ops).
#ifndef HSB_FP_VARIANT
#define HSB_FP_VARIANT 2
#endif
#ifndef HSB_UNROLL
#define HSB_UNROLL 4
#endif
// 1: the gather takes the footprint's lower-left cell (ix, iy) as coordinates plus the texel offset (1, 1) carried by
//    the instruction (SASS TLD4.AOFFI, one loop-invariant register) instead of computing (ix + 1, iy + 1) per endpoint.
#ifndef HSB_TLD4_OFFSET
#define HSB_TLD4_OFFSET 1
#endif
// 1: the nine H / dTr accumulations of an endpoint are predicated on "inside the map" (PTX @p fma) instead of sitting in
//    a branch (BSSY / BRA / BSYNC per endpoint): 3 instructions per endpoint fewer, bit-identical — and NOT faster: the kernel is
//    bound by the texture pipe, and the branchy form consumes the gathers one by one as they return (DEPBAR per
//    endpoint) where the predicated form waits for them in pairs.  Off.
// HSB_DIAG: 1 compiles the diagnostics in (tuning keys trace / pace / stagger / prefetch: scripts/k1_probe.py);
// 0 removes them from the kernel (scripts/variant_timing.py measures what carrying them costs).
#ifndef HSB_DIAG
#define HSB_DIAG 1
#endif
#ifndef HSB_PRED_ACC
#define HSB_PRED_ACC 0
#endif

struct PointPre {
  float rx, ry;   // rotated endpoint = d(q)/d(psi) terms: rotDeriv = rx*gy - ry*gx
  float fx, fy;   // interpolation weights
  float cx, cy;   // texture coordinates (MODE_TEX)
  int idx;        // cell index (MODE_LDG)
  bool inside;
};

// The few per-level constants the inner loop touches, copied to registers once per level (indexing
// the __grid_constant__ array with a runtime level inside the loop costs a constant-bank load each).
struct LevelRegs {
  float lim_x, lim_y;
  cudaTextureObject_t tex;
  const float* prob;
  int sx;
};
// A texture instruction wants its (bindless) handle in a UNIFORM register.  The handle of the current level is read
// from the kernel parameters with a run-time level index, which ptxas does not recognise as warp-uniform: it then wraps
// EVERY gather in a "waterfall" loop (R2UR / PLOP3 / BRA.U.ANY — 8 extra instructions per TLD4, ~15 % of the whole
// kernel, measured in the round-1 SASS).  A warp reduction (redux.sync -> REDUX, whose result lands in a uniform
// register) of the — identical — per-lane copies makes the uniformity visible: the TLD4s take the handle from UR
// directly.  Must be called with all 32 lanes converged (every caller does, once per level).
#ifndef HSB_UNIFORM_HANDLE
#define HSB_UNIFORM_HANDLE 1
#endif
__device__ __forceinline__ cudaTextureObject_t uniform_handle(cudaTextureObject_t t) {
#if !HSB_UNIFORM_HANDLE
  return t;
#endif
  const unsigned lo = __reduce_max_sync(0xffffffffu, (unsigned)(t & 0xffffffffull));
  const unsigned hi = __reduce_max_sync(0xffffffffu, (unsigned)(t >> 32));
  return ((cudaTextureObject_t)hi << 32) | (cudaTextureObject_t)lo;
}

__device__ __forceinline__ LevelRegs level_regs(const HsbLevelDev& L) {
  LevelRegs r;
  r.lim_x = L.lim_x;
  r.lim_y = L.lim_y;
  r.tex = uniform_handle(L.tex);
  r.prob = L.prob;
  r.sx = L.sx;
  return r;
}

template <int MODE>
__device__ __forceinline__ void point_address(const LevelRegs& L, float px, float py, bool valid, float cs, float ss,
                                              float x, float y, PointPre& o) {
  // cs, ss carry the level's 2^-k point scale (exact), so cs*px == c*(px*2^-k) bit for bit
  const float m1 = __fmul_rn(cs, px), m2 = __fmul_rn(ss, py), m3 = __fmul_rn(ss, px), m4 = __fmul_rn(cs, py);
  const float qx = __fadd_rn(m1, __fadd_rn(-m2, x));   // OccGridMapUtil.h:80
  const float qy = __fadd_rn(m3, __fadd_rn(m4, y));
  o.rx = __fsub_rn(m1, m2);                            // cosRot*px - sinRot*py   (:87)
  o.ry = __fadd_rn(m3, m4);                            // -( -sinRot*px - cosRot*py )
  // pointOutOfMapBounds, MapDimensionProperties.h:65-68, written so that NaN is OUT (the
  // reference lets NaN through and then indexes memory with it — SURVEY.md Q4)
  o.inside = valid && (qx >= 0.0f) && (qx <= L.lim_x) && (qy >= 0.0f) && (qy <= L.lim_y);
  if (MODE == MODE_TEX) {
    // floor == trunc on the valid domain (:295); one FRND instead of F2I + I2F
    const float flx = truncf(qx), fly = truncf(qy);
    o.fx = __fsub_rn(qx, flx);                         // :298
    o.fy = __fsub_rn(qy, fly);
    // texel centres (ix,iy)..(ix+1,iy+1): a gather at an INTEGER coordinate c selects texels c-1 and c, so the
    // footprint is addressed as (ix + 1, iy + 1) — either added here, or (HSB_TLD4_OFFSET) as the instruction's
    // immediate texel offset (1, 1).  Integers are exact in the unit's fixed-point coordinate conversion, so no
    // neighbouring footprint can be selected; clamp addressing makes any coordinate (also garbage from an outside
    // point) safe.
#if HSB_TLD4_OFFSET
    o.cx = flx;
    o.cy = fly;
#else
    o.cx = flx + 1.0f;
    o.cy = fly + 1.0f;
#endif
  } else {
    const int ix = (int)qx, iy = (int)qy;              // :295 (garbage but harmless when !inside)
    o.fx = __fsub_rn(qx, (float)ix);
    o.fy = __fsub_rn(qy, (float)iy);
    o.idx = o.inside ? iy * L.sx + ix : 0;             // :302
  }
}

template <int MODE>
__device__ __forceinline__ float4 point_fetch(const LevelRegs& L, const PointPre& p) {
  float4 v;  // (i0, i1, i2, i3) = cells (ix,iy) (ix+1,iy) (ix,iy+1) (ix+1,iy+1)
  if (MODE == MODE_TEX) {
#if HSB_TLD4_OFFSET
    float4 g;
    asm("tld4.r.2d.v4.f32.f32 {%0, %1, %2, %3}, [%4, {%5, %6}], {1, 1};"
        : "=f"(g.x), "=f"(g.y), "=f"(g.z), "=f"(g.w)
        : "l"(L.tex), "f"(p.cx), "f"(p.cy));
#else
    const float4 g = tex2Dgather<float4>(L.tex, p.cx, p.cy, 0);
#endif
    v = make_float4(g.w, g.z, g.x, g.y);
  } else {
    const float* c = L.prob + p.idx;
    v = make_float4(__ldg(c), __ldg(c + 1), __ldg(c + L.sx), __ldg(c + L.sx + 1));
  }
  return v;
}

__device__ __forceinline__ void point_accumulate(const PointPre& p, const float4 v, Acc& a) {
  const float i0 = v.x, i1 = v.y, i2 = v.z, i3 = v.w, fx = p.fx, fy = p.fy;
#if HSB_FP_VARIANT == 0
  const float xi = __fsub_rn(1.0f, fx), yi = __fsub_rn(1.0f, fy);
  const float m = __fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(i0, xi), __fmul_rn(i1, fx)), yi),
                            __fmul_rn(__fadd_rn(__fmul_rn(i2, xi), __fmul_rn(i3, fx)), fy));   // :342-343
  const float gx = -__fadd_rn(__fmul_rn(__fsub_rn(i0, i1), xi), __fmul_rn(__fsub_rn(i2, i3), fx));  // :344
  const float gy = -__fadd_rn(__fmul_rn(__fsub_rn(i0, i2), yi), __fmul_rn(__fsub_rn(i1, i3), fy));  // :345
  const float f = __fsub_rn(1.0f, m);                                                          // :82
  const float r = __fadd_rn(__fmul_rn(-p.ry, gx), __fmul_rn(p.rx, gy));                        // :87
  if (p.inside) {
    a.d0 = __fadd_rn(a.d0, __fmul_rn(gx, f));
    a.d1 = __fadd_rn(a.d1, __fmul_rn(gy, f));
    a.d2 = __fadd_rn(a.d2, __fmul_rn(r, f));
    a.h00 = __fadd_rn(a.h00, __fmul_rn(gx, gx));
    a.h11 = __fadd_rn(a.h11, __fmul_rn(gy, gy));
    a.h22 = __fadd_rn(a.h22, __fmul_rn(r, r));
    a.h01 = __fadd_rn(a.h01, __fmul_rn(gx, gy));
    a.h02 = __fadd_rn(a.h02, __fmul_rn(gx, r));
    a.h12 = __fadd_rn(a.h12, __fmul_rn(gy, r));
  }
#else
#if HSB_FP_VARIANT == 1
  const float xi = 1.0f - fx, yi = 1.0f - fy;
  const float m = (i0 * xi + i1 * fx) * yi + (i2 * xi + i3 * fx) * fy;
  const float gx = -((i0 - i1) * xi + (i2 - i3) * fx);
  const float gy = -((i0 - i2) * yi + (i1 - i3) * fy);
#else
  // bilinear form regrouped: d01 = i1-i0, d02 = i2-i0, dd = (i3-i2) - (i1-i0)
  const float d01 = i1 - i0, d02 = i2 - i0, dd = (i3 - i2) - d01;
  const float gx = fmaf(fx, dd, d01);            // = (i1-i0)(1-fx) + (i3-i2)fx
  const float gy = fmaf(fy, dd, d02);            // = (i2-i0)(1-fy) + (i3-i1)fy
  const float m = fmaf(fy, fmaf(fx, dd, d02), fmaf(fx, d01, i0));
#endif
  const float f = 1.0f - m;
  const float r = fmaf(p.rx, gy, -(p.ry * gx));
#if HSB_PRED_ACC
  asm("{\n\t.reg .pred p;\n\t"
      "setp.ne.u32 p, %13, 0;\n\t"
      "@p fma.rn.f32 %0, %9, %12, %0;\n\t"     // d0  += gx * f
      "@p fma.rn.f32 %1, %10, %12, %1;\n\t"    // d1  += gy * f
      "@p fma.rn.f32 %2, %11, %12, %2;\n\t"    // d2  += r  * f
      "@p fma.rn.f32 %3, %9, %9, %3;\n\t"      // h00 += gx * gx
      "@p fma.rn.f32 %4, %10, %10, %4;\n\t"    // h11 += gy * gy
      "@p fma.rn.f32 %5, %11, %11, %5;\n\t"    // h22 += r  * r
      "@p fma.rn.f32 %6, %9, %10, %6;\n\t"     // h01 += gx * gy
      "@p fma.rn.f32 %7, %9, %11, %7;\n\t"     // h02 += gx * r
      "@p fma.rn.f32 %8, %10, %11, %8;\n\t"    // h12 += gy * r
      "}"
      : "+f"(a.d0), "+f"(a.d1), "+f"(a.d2), "+f"(a.h00), "+f"(a.h11), "+f"(a.h22), "+f"(a.h01), "+f"(a.h02), "+f"(a.h12)
      : "f"(gx), "f"(gy), "f"(r), "f"(f), "r"((unsigned)p.inside));
  if (false) {
#else
  if (p.inside) {  // the translation unit is built with -fmad=false: fused operations are explicit
#endif
    a.d0 = fmaf(gx, f, a.d0);
    a.d1 = fmaf(gy, f, a.d1);
    a.d2 = fmaf(r, f, a.d2);
    a.h00 = fmaf(gx, gx, a.h00);
    a.h11 = fmaf(gy, gy, a.h11);
    a.h22 = fmaf(r, r, a.h22);
    a.h01 = fmaf(gx, gy, a.h01);
    a.h02 = fmaf(gx, r, a.h02);
    a.h12 = fmaf(gy, r, a.h12);
  }
#endif
}

// All endpoints i = first, first + stride, ... < n of one evaluation, U at a time: full batches
// without bounds checks, then one guarded batch for the tail.
template <int MODE, int U, typename PtsPtr>
__device__ __forceinline__ void eval_points(const LevelRegs& L, PtsPtr pts, int first, int stride, int n, float cs, float ss,
                                            float x, float y, Acc& a) {
  int base = first;
  const int last_full = n - (U - 1) * stride;  // base < last_full  =>  all U points exist
  for (; base < last_full; base += U * stride) {
    PointPre pre[U];
    float4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const float2 p = pts[base + u * stride];
      point_address<MODE>(L, p.x, p.y, true, cs, ss, x, y, pre[u]);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) v[u] = point_fetch<MODE>(L, pre[u]);
#pragma unroll
    for (int u = 0; u < U; ++u) point_accumulate(pre[u], v[u], a);
  }
  if (base < n) {
    PointPre pre[U];
    float4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = base + u * stride;
      const bool valid = i < n;
      const float2 p = pts[valid ? i : n - 1];
      point_address<MODE>(L, p.x, p.y, valid, cs, ss, x, y, pre[u]);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) v[u] = point_fetch<MODE>(L, pre[u]);
#pragma unroll
    for (int u = 0; u < U; ++u) point_accumulate(pre[u], v[u], a);
  }
}

// eval_points in the level's gather mode: MODE_ANY picks it from the level descriptor (uniform across the group).
template <int MODE, int U, typename PtsPtr>
__device__ __forceinline__ void eval_level(const LevelRegs& L, PtsPtr pts, int first, int stride, int n, float cs, float ss,
                                           float x, float y, Acc& a) {
  if constexpr (MODE == MODE_ANY) {
    if (L.tex) eval_points<MODE_TEX, U>(L, pts, first, stride, n, cs, ss, x, y, a);
    else eval_points<MODE_LDG, U>(L, pts, first, stride, n, cs, ss, x, y, a);
  } else {
    eval_points<MODE, U>(L, pts, first, stride, n, cs, ss, x, y, a);
  }
}

// ---- paired evaluation: two endpoints per lane, tuning key "packed" ------------------------------
// Each lane carries two endpoints side by side (float2 values) through the per-endpoint arithmetic: the
// exact map-coordinate sequence, the interpolation weights, rotDeriv and the nine H / dTr accumulations.
// sm_90 has no packed fp32 instructions, so every pair operation is two scalar operations; each half
// performs exactly the operation sequence of the scalar path, so results per endpoint are bit-identical.
//
// Shared-memory layout for this path ("pairified" in place after staging): slots 2k and 2k+1 are
// stored as (x_2k, x_2k+1, y_2k, y_2k+1), so one LDS.128 delivers the X pair and the Y pair in
// adjacent registers.  Slots that hold no endpoint, and endpoints that are not finite, are set to
// kFar: such a point lies outside every map, its texture coordinates are redirected to (-8,-8) where
// clamp addressing returns four equal texels, hence zero gradient, hence zero contribution —
// no per-endpoint branch and no predication in the accumulation.
constexpr float kFar = 1.0e30f;

// Pair operations, each half rounded on its own (the __f*_rn intrinsics are never contracted).
__device__ __forceinline__ float2 fma2_rn(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 mul2_exact(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 add2_exact(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 sub2_exact(float2 c, float2 a) { return make_float2(__fsub_rn(c.x, a.x), __fsub_rn(c.y, a.y)); }

template <int W>
__device__ __forceinline__ void pairify_in_place(float2* slots, int head, int n, int t) {
  const int nslots = (head + n + 1) & ~1;
  float4* q = reinterpret_cast<float4*>(slots);
  for (int k = t; k < nslots / 2; k += W * 32) {
    float4 v = q[k];  // (x0, y0, x1, y1)
    const int s0 = 2 * k, s1 = 2 * k + 1;
    const bool ok0 = (s0 >= head) && (s0 < head + n) && (fabsf(v.x) < kFar) && (fabsf(v.y) < kFar);
    const bool ok1 = (s1 >= head) && (s1 < head + n) && (fabsf(v.z) < kFar) && (fabsf(v.w) < kFar);
    const float x0 = ok0 ? v.x : kFar, y0 = ok0 ? v.y : kFar;
    const float x1 = ok1 ? v.z : kFar, y1 = ok1 ? v.w : kFar;
    q[k] = make_float4(x0, x1, y0, y1);
  }
}

struct Acc2 {
  float2 h00, h11, h22, h01, h02, h12, d0, d1, d2;
};

template <int UP>
__device__ __forceinline__ void eval_pairs(const LevelRegs& L, const float4* __restrict__ pairs, int first, int stride,
                                           int npairs, float cs, float ss, float x, float y, Acc& out) {
  const float2 cs2 = make_float2(cs, cs), ss2 = make_float2(ss, ss), x2 = make_float2(x, x), y2 = make_float2(y, y);
  const float2 neg1 = make_float2(-1.0f, -1.0f), far4 = make_float2(kFar, kFar);
  const float2 z = make_float2(0.f, 0.f);
  Acc2 a = {z, z, z, z, z, z, z, z, z};
  for (int base = first; base < npairs; base += UP * stride) {
    float2 RX[UP], RY[UP], FX[UP], FY[UP];
    float4 va[UP], vb[UP];
#pragma unroll
    for (int u = 0; u < UP; ++u) {
      const int k = base + u * stride;
      float2 X = far4, Y = far4;
      if (k < npairs) {
        const float4 v = pairs[k];
        X = make_float2(v.x, v.y);
        Y = make_float2(v.z, v.w);
      }
      // q = T * p in the oracle's exact order, pairwise (cs/ss carry the level's 2^-k scale)
      const float2 M1 = mul2_exact(cs2, X), M2 = mul2_exact(ss2, Y), M3 = mul2_exact(ss2, X), M4 = mul2_exact(cs2, Y);
      const float2 QX = add2_exact(M1, sub2_exact(x2, M2));         // m1 + (-m2 + x)     OccGridMapUtil.h:80
      const float2 QY = add2_exact(M3, add2_exact(M4, y2));         // m3 + (m4 + y)
      RX[u] = sub2_exact(M1, M2);                                   // m1 - m2            (:87)
      RY[u] = add2_exact(M3, M4);
      const bool inA = (QX.x >= 0.0f) && (QX.x <= L.lim_x) && (QY.x >= 0.0f) && (QY.x <= L.lim_y);
      const bool inB = (QX.y >= 0.0f) && (QX.y <= L.lim_x) && (QY.y >= 0.0f) && (QY.y <= L.lim_y);
      const float2 FLX = make_float2(truncf(QX.x), truncf(QX.y));   // :295
      const float2 FLY = make_float2(truncf(QY.x), truncf(QY.y));
      FX[u] = sub2_exact(QX, FLX);                                  // q - floor(q)       (:298)
      FY[u] = sub2_exact(QY, FLY);
      // texel centres (ix,iy)..(ix+1,iy+1); outside endpoints look at the clamped corner (4 equal texels)
      const float cxA = inA ? FLX.x + 1.0f : -8.0f, cyA = inA ? FLY.x + 1.0f : -8.0f;
      const float cxB = inB ? FLX.y + 1.0f : -8.0f, cyB = inB ? FLY.y + 1.0f : -8.0f;
      const float4 gA = tex2Dgather<float4>(L.tex, cxA, cyA, 0);
      const float4 gB = tex2Dgather<float4>(L.tex, cxB, cyB, 0);
      va[u] = make_float4(gA.w, gA.z, gA.x, gA.y);                  // (i0, i1, i2, i3)
      vb[u] = make_float4(gB.w, gB.z, gB.x, gB.y);
    }
#pragma unroll
    for (int u = 0; u < UP; ++u) {
      // regrouped bilinear form (HSB_FP_VARIANT 2), per endpoint; results land pairwise
      const float d01a = va[u].y - va[u].x, d02a = va[u].z - va[u].x, dda = (va[u].w - va[u].z) - d01a;
      const float d01b = vb[u].y - vb[u].x, d02b = vb[u].z - vb[u].x, ddb = (vb[u].w - vb[u].z) - d01b;
      const float2 D01 = make_float2(d01a, d01b), D02 = make_float2(d02a, d02b), DD = make_float2(dda, ddb);
      const float2 I0 = make_float2(va[u].x, vb[u].x);
      const float2 GX = fma2_rn(FX[u], DD, D01);                    // :344
      const float2 GY = fma2_rn(FY[u], DD, D02);                    // :345
      const float2 Mv = fma2_rn(FY[u], fma2_rn(FX[u], DD, D02), fma2_rn(FX[u], D01, I0));  // :342-343
      const float2 F = fma2_rn(Mv, neg1, make_float2(1.0f, 1.0f));  // 1 - M            (:82)
      const float2 T = mul2_exact(RY[u], GX);
      const float2 R = fma2_rn(RX[u], GY, make_float2(-T.x, -T.y)); // rx*gy - ry*gx   (:87)
      a.d0 = fma2_rn(GX, F, a.d0);
      a.d1 = fma2_rn(GY, F, a.d1);
      a.d2 = fma2_rn(R, F, a.d2);
      a.h00 = fma2_rn(GX, GX, a.h00);
      a.h11 = fma2_rn(GY, GY, a.h11);
      a.h22 = fma2_rn(R, R, a.h22);
      a.h01 = fma2_rn(GX, GY, a.h01);
      a.h02 = fma2_rn(GX, R, a.h02);
      a.h12 = fma2_rn(GY, R, a.h12);
    }
  }
  out.h00 = a.h00.x + a.h00.y; out.h11 = a.h11.x + a.h11.y; out.h22 = a.h22.x + a.h22.y;
  out.h01 = a.h01.x + a.h01.y; out.h02 = a.h02.x + a.h02.y; out.h12 = a.h12.x + a.h12.y;
  out.d0 = a.d0.x + a.d0.y;    out.d1 = a.d1.x + a.d1.y;    out.d2 = a.d2.x + a.d2.y;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ void warp_reduce(Acc& a) {
  a.h00 = warp_sum(a.h00);
  a.h11 = warp_sum(a.h11);
  a.h22 = warp_sum(a.h22);
  a.h01 = warp_sum(a.h01);
  a.h02 = warp_sum(a.h02);
  a.h12 = warp_sum(a.h12);
  a.d0 = warp_sum(a.d0);
  a.d1 = warp_sum(a.d1);
  a.d2 = warp_sum(a.d2);
}

// ---- mbarrier / bulk-copy helpers (TMA 1-D path) ---------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
// L2 prefetch of [from, to) (rounded inwards to 16-byte units): one instruction for a whole scan.
__device__ __forceinline__ void l2_prefetch(const void* from, const void* to) {
  const uintptr_t a = ((uintptr_t)from + 15) & ~(uintptr_t)15, b = (uintptr_t)to & ~(uintptr_t)15;
  if (b > a) asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(a), "r"((uint32_t)(b - a)) : "memory");
}
__device__ __forceinline__ unsigned long long global_timer_ns() {
  unsigned long long v;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(v));
  return v;
}
__device__ __forceinline__ unsigned warp_id() {
  unsigned v;
  asm volatile("mov.u32 %0, %%warpid;" : "=r"(v));
  return v;
}
__device__ __forceinline__ unsigned sm_id() {
  unsigned v;
  asm volatile("mov.u32 %0, %%smid;" : "=r"(v));
  return v;
}
// Barrier among the W warps of group g.  The id must be an immediate: with a register operand
// ptxas reserves all 16 named barriers for the CTA, and the SM's barrier budget then caps
// residency at 4 CTAs (measured with ncu: launch__occupancy_limit_barriers).
template <int W>
__device__ __forceinline__ void group_sync(int g) {
  if (W == 1) {
    __syncwarp();
    return;
  }
  switch (g) {
    case 0: asm volatile("bar.sync 1, %0;" ::"n"(W * 32) : "memory"); break;
    case 1: asm volatile("bar.sync 2, %0;" ::"n"(W * 32) : "memory"); break;
    case 2: asm volatile("bar.sync 3, %0;" ::"n"(W * 32) : "memory"); break;
    case 3: asm volatile("bar.sync 4, %0;" ::"n"(W * 32) : "memory"); break;
    case 4: asm volatile("bar.sync 5, %0;" ::"n"(W * 32) : "memory"); break;
    case 5: asm volatile("bar.sync 6, %0;" ::"n"(W * 32) : "memory"); break;
    case 6: asm volatile("bar.sync 7, %0;" ::"n"(W * 32) : "memory"); break;
    default: asm volatile("bar.sync 8, %0;" ::"n"(W * 32) : "memory"); break;
  }
}

// ---- N2: sensor_msgs/LaserScan ranges -> DataContainer endpoints, fused into the staging step ----
// Restates HectorMappingRos::rosLaserScanToDataContainer (hector_mapping/src/HectorMappingRos.cpp:
// 483-507): keep returns with range_min < r < range_max - 0.1 (:493,499), dist = r * scaleToMap,
// endpoint = (cos(angle) * dist, sin(angle) * dist) (:501-502); the beam angle is accumulated in
// fp32 on the host (`angle += angle_increment`, :505) and arrives as a (cos, sin) table.  Valid
// endpoints are compacted IN BEAM ORDER into `dst` (the container's order); returns their number.
// Warp w converts the contiguous beam range [w*chunk, (w+1)*chunk).
template <int W>
__device__ __forceinline__ int stage_from_ranges(const float* __restrict__ r_scan, const float2* __restrict__ beam_cs,
                                                 int n_beams, float rmin, float rmaxc, float scale, float2* dst,
                                                 int* warp_cnt, int g, int w, int lane) {
  const int chunk = (n_beams + W - 1) / W;
  const int b0 = w * chunk, b1 = min(n_beams, b0 + chunk);
  int mine = 0;
  if (W > 1) {
    for (int base = b0; base < b1; base += 32) {
      const int i = base + lane;
      const float r = i < b1 ? __ldg(r_scan + i) : 0.0f;
      const bool v = (i < b1) && (r > rmin) && (r < rmaxc);
      mine += __popc(__ballot_sync(0xffffffffu, v));
    }
    if (lane == 0) warp_cnt[w] = mine;
    group_sync<W>(g);
  }
  int off = 0, total = 0;
  if (W > 1) {
#pragma unroll
    for (int k = 0; k < W; ++k) {
      const int c = warp_cnt[k];
      if (k < w) off += c;
      total += c;
    }
  }
  for (int base = b0; base < b1; base += 32) {
    const int i = base + lane;
    const float r = i < b1 ? __ldg(r_scan + i) : 0.0f;
    const bool v = (i < b1) && (r > rmin) && (r < rmaxc);
    const unsigned m = __ballot_sync(0xffffffffu, v);
    if (v) {
      const float dist = __fmul_rn(r, scale);
      const float2 cs = __ldg(beam_cs + i);
      dst[off + __popc(m & ((1u << lane) - 1u))] = make_float2(__fmul_rn(cs.x, dist), __fmul_rn(cs.y, dist));
    }
    off += __popc(m);
  }
  if (W == 1) total = off;
  group_sync<W>(g);  // endpoints visible to the whole group (also protects warp_cnt for the next scan)
  return total;
}

// ---- N2, default path: sensor_msgs/PointCloud (laser frame) -> DataContainer endpoints, fused the same way ----
// Restates HectorMappingRos::rosPointCloudToDataContainer (hector_mapping/src/HectorMappingRos.cpp:509-542), the
// converter a default node uses (use_tf_scan_transformation = true, :82, called at :283): per Point32 (x, y, z):
//   dist_sqr = x*x + y*y in float (:524); keep sqr_min < dist_sqr < sqr_max (:526); drop x < 0 && dist_sqr < 0.5 (:528);
//   p = laserTransform * (x, y, z) in DOUBLE — tf::Transform::operator* = row.dot(v) + origin, dot = r0*x + r1*y + r2*z
//   (tf/LinearMath) (:532); z_laser = float(p.z - laserPos.z) must lie in (z_min, z_max) (:534-536);
//   endpoint = Vector2f(p.x, p.y) * scaleToMap: double -> float, then one float product (:538).
// Every operation is rounded separately (__dmul_rn / __dadd_rn), like the node's x86-64 build.  Kept endpoints are
// compacted in input order.  Warp w converts the contiguous range [w*chunk, (w+1)*chunk) of the cloud.
struct CloudPoint {
  float ex, ey;
  bool keep;
};
__device__ __forceinline__ CloudPoint cloud_point_xyz(float x, float y, float z, const double* T, float min2, float max2,
                                                      float zmin, float zmax, float scale) {
  const float d2 = __fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y));
  CloudPoint o;
  o.keep = (d2 > min2) && (d2 < max2) && !((x < 0.0f) && (d2 < 0.50f));
  const double vx = (double)x, vy = (double)y, vz = (double)z;
  const double bx = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[0], vx), __dmul_rn(T[1], vy)), __dmul_rn(T[2], vz)), T[3]);
  const double by = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[4], vx), __dmul_rn(T[5], vy)), __dmul_rn(T[6], vz)), T[7]);
  const double bz = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T[8], vx), __dmul_rn(T[9], vy)), __dmul_rn(T[10], vz)), T[11]);
  const float zl = (float)__dsub_rn(bz, T[11]);
  o.keep = o.keep && (zl > zmin) && (zl < zmax);
  o.ex = __fmul_rn((float)bx, scale);
  o.ey = __fmul_rn((float)by, scale);
  return o;
}
__device__ __forceinline__ CloudPoint cloud_point(const float* __restrict__ xyz, int i, const double* T, float min2, float max2,
                                                  float zmin, float zmax, float scale) {
  const float x = __ldg(xyz + 3 * (size_t)i), y = __ldg(xyz + 3 * (size_t)i + 1), z = __ldg(xyz + 3 * (size_t)i + 2);
  return cloud_point_xyz(x, y, z, T, min2, max2, zmin, zmax, scale);
}

// ---- N2, default path from the LaserScan itself: laser_geometry's projection, then the cloud rule above ----------
// laser_geometry (ROS1 Melodic/Noetic) LaserProjection::projectLaser_ for the sensor_msgs/PointCloud output, the
// projection the node runs before rosPointCloudToDataContainer (HectorMappingRos.cpp:273, projectLaser(scan, cloud,
// 30.0)): beam i is kept iff (double)range < range_cutoff && range >= range_min (float compare; NaN and +-inf drop out),
// and becomes the Point32 ((float)(range * cos_i), (float)(range * sin_i), 0) with one double product each.  The unit
// vectors (getUnitVectors_: cos / sin of angle_min + i * angle_increment in double) arrive as a table built on the host
// with libm.  The projected point then takes the cloud rule with z = 0 in the full tf dot product.  The two filters
// compose into one over the beams, in beam order.
__device__ __forceinline__ CloudPoint projected_point(const float* __restrict__ r_scan, const double2* __restrict__ unit,
                                                      int i, float rmin, double cutoff, const double* T, float min2,
                                                      float max2, float zmin, float zmax, float scale) {
  const float r = __ldg(r_scan + i);
  const double2 u = __ldg(unit + i);
  const double rd = (double)r;
  CloudPoint o = cloud_point_xyz((float)__dmul_rn(rd, u.x), (float)__dmul_rn(rd, u.y), 0.0f, T, min2, max2, zmin, zmax,
                                 scale);
  o.keep = o.keep && (rd < cutoff) && (r >= rmin);
  return o;
}
// Converts points [0, n_in) with `at(i)` (a CloudPoint) and compacts the kept ones in input order into `dst`; returns
// their number.  Warp w converts the contiguous range [w*chunk, (w+1)*chunk); with W > 1 a first pass counts each warp's
// kept points for the cross-warp prefix.
template <int W, typename PointAt>
__device__ __forceinline__ int stage_compacted(int n_in, PointAt at, float2* dst, int* warp_cnt, int g, int w, int lane) {
  const int chunk = (n_in + W - 1) / W;
  const int b0 = w * chunk, b1 = min(n_in, b0 + chunk);
  int mine = 0;
  if (W > 1) {
    for (int base = b0; base < b1; base += 32) {
      const int i = base + lane;
      const bool v = (i < b1) && at(i).keep;
      mine += __popc(__ballot_sync(0xffffffffu, v));
    }
    if (lane == 0) warp_cnt[w] = mine;
    group_sync<W>(g);
  }
  int off = 0, total = 0;
  if (W > 1) {
#pragma unroll
    for (int k = 0; k < W; ++k) {
      const int c = warp_cnt[k];
      if (k < w) off += c;
      total += c;
    }
  }
  for (int base = b0; base < b1; base += 32) {
    const int i = base + lane;
    CloudPoint p;
    p.keep = false;
    if (i < b1) p = at(i);
    const unsigned m = __ballot_sync(0xffffffffu, p.keep);
    if (p.keep) dst[off + __popc(m & ((1u << lane) - 1u))] = make_float2(p.ex, p.ey);
    off += __popc(m);
  }
  if (W == 1) total = off;
  group_sync<W>(g);
  return total;
}
template <int W>
__device__ __forceinline__ int stage_from_cloud(const float* __restrict__ xyz, int n_in, const double* T, float min2, float max2,
                                                float zmin, float zmax, float scale, float2* dst, int* warp_cnt, int g, int w,
                                                int lane) {
  return stage_compacted<W>(n_in, [&](int i) { return cloud_point(xyz, i, T, min2, max2, zmin, zmax, scale); }, dst,
                            warp_cnt, g, w, lane);
}
template <int W>
__device__ __forceinline__ int stage_from_projected(const float* __restrict__ r_scan, const double2* __restrict__ unit,
                                                    int n_beams, float rmin, double cutoff, const double* T, float min2,
                                                    float max2, float zmin, float zmax, float scale, float2* dst,
                                                    int* warp_cnt, int g, int w, int lane) {
  return stage_compacted<W>(
      n_beams, [&](int i) { return projected_point(r_scan, unit, i, rmin, cutoff, T, min2, max2, zmin, zmax, scale); },
      dst, warp_cnt, g, w, lane);
}

// Shared-memory carve-up for G groups: [G] mbarriers | [G][2][9][32] reduction slots | points
template <int W, int G>
struct MatchSmem {
  static constexpr int kBarBytes = (G * 8 + 15) / 16 * 16;   // mbarriers, padded: the reduction rows are read as float4
  static constexpr int kRedFloats = (W > 1) ? G * 2 * 9 * 32 : 0;
  static constexpr int kCntInts = (W > 1) ? G * 32 : 0;      // per-warp counts of the fused conversions (W > 1 only)
  static constexpr int kProgInts = (G > 1) ? 32 : 0;         // evaluations completed per group (pacing)
  static constexpr int kHeaderBytes = ((kBarBytes + kRedFloats * 4 + kCntInts * 4 + kProgInts * 4) + 15) / 16 * 16;
};

// The scan of a single-scan call can travel INSIDE the kernel launch (kernel parameters, up to 32 KB on sm_70+ since
// CUDA 12.1): [16-float header = hint, gate thresholds | endpoints].  That removes the host-to-device copy operation
// and the copy-engine -> compute dependency from the critical path of hsb_match_data / hsb_slam_update.  Tuning key
// inline_scan: NOT a win in measurement — a launch with 12 KB of parameters and the divergent constant-bank reads of
// the staging loop cost more than the 8.7 KB copy they replace; only the back-to-back rate improves (one stream
// operation fewer per step).  Kept as an opt-in (default off), bit-identical
// (tests/test_gpu_slam_step.py).  InlineScan<false> is empty: the batch kernels' SASS is unchanged.
#define HSB_INLINE_MAX_POINTS 1280
template <bool INL>
struct InlineScan {};
template <>
struct InlineScan<true> {
  float header[16];
  float2 pts[HSB_INLINE_MAX_POINTS];
};

// one-warp scans grouped into CTAs: ask for the registers of 28 warps per SM like the G = 1 shape has.  A one-warp
// MODE_ANY kernel (a heterogeneous group's match) carries both gather paths: at 24 warps per SM its registers hold them
// without spilling.
template <int W, int G, int MODE = MODE_TEX>
struct MatchBounds {
  static constexpr int kMinBlocks = (W == 1 && 28 % G == 0) ? (MODE == MODE_ANY && G == 1 ? 24 : 28 / G) : 1;
};

// Which group a match kernel serves (its GRP template value): none (one handle's map for the whole batch), the group
// SLAM step (one session per scan, hsb_group_slam_update) or the group batch match (one hint per scan,
// hsb_group_match_batch).  A group's scan runs its own member's levels (HsbGroupSessionDev::levels,
// HsbScoreSessionDev::levels), coarsest first; HsbMatchParams::levels is then only the stride of group_lv.
enum { GRP_NONE = 0, GRP_STEP = 1, GRP_MATCH = 2 };
template <int GRP>
constexpr bool kGrpStep = GRP == GRP_STEP;
template <int GRP>
constexpr bool kGrpMatch = GRP == GRP_MATCH;

// The session of hint q of a group batch match or of pose q of a scoring call: the last session whose hints / poses
// start at or before q (empty sessions are passed over), as ray_kernel finds a ray's.
__device__ __forceinline__ int session_of(const int* __restrict__ offsets, int K, int q) {
  int lo = 0, hi = K - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (offsets[mid] <= q) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// Level descriptors of scan `scan`: the kernel parameters' (one map for the whole batch), or — group SLAM step and group
// batch match, every session works on its own member's map — the row of the group's device array that belongs to the
// session's member (`member`: the group batch match's, looked up once per scan).
template <int GRP>
__device__ __forceinline__ const HsbLevelDev& level_desc(const HsbMatchParams& P, int scan, int member, int lvl) {
  if constexpr (kGrpStep<GRP>) return P.group_lv[(size_t)P.group_sess[scan].member * P.levels + lvl];
  else if constexpr (kGrpMatch<GRP>) return P.group_lv[(size_t)member * P.levels + lvl];
  else return P.lv[lvl];
}

// Conversion descriptor of scan `scan`: the kernel parameters' (one handle), or the session's (group SLAM step).
template <int GRP>
__device__ __forceinline__ const HsbConvDev& conv_desc(const HsbMatchParams& P, int scan) {
  if constexpr (kGrpStep<GRP>) return P.group_sess[scan].conv;
  else return P.conv;
}

// Where scan `scan`'s per-evaluation record starts: its row of P.record, or — group SLAM step — the session's own buffer
// (HsbGroupSessionDev::record; its members' records differ in length).  Loaded again at each store (see match_kernel).
template <int GRP>
__device__ __forceinline__ float* record_base(const HsbMatchParams& P, int scan) {
  if constexpr (kGrpStep<GRP>) return P.group_sess[scan].record;
  else return P.record + (size_t)scan * P.record_floats;
}

// GRP: GRP_STEP, the group SLAM step (hsb_group_slam_update), one session per scan — see HsbMatchParams::group_lv;
// GRP_MATCH, the group batch match (hsb_group_match_batch), one hint per scan — see HsbMatchParams::match_sess.
// PROJ: converted input is HSB_IN_PROJECTED (laser_geometry's projection and the cloud rule, stage_from_projected); only
// the instantiations the projected SLAM steps and batch matches launch carry that branch (hsb_api.cu
// launch_match_projected).
template <int W, int G, int MODE, int U, bool PACK, bool INL = false, int GRP = GRP_NONE, bool PROJ = false>
__global__ void __launch_bounds__(W * G * 32, MatchBounds<W, G, MODE>::kMinBlocks)
    match_kernel(const __grid_constant__ HsbMatchParams P, const __grid_constant__ InlineScan<INL> S) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint64_t* mbars = reinterpret_cast<uint64_t*>(smem_raw);
  float* red_all = reinterpret_cast<float*>(smem_raw + MatchSmem<W, G>::kBarBytes);
  int* cnt_all = reinterpret_cast<int*>(smem_raw + MatchSmem<W, G>::kBarBytes + MatchSmem<W, G>::kRedFloats * 4);
  volatile int* prog = reinterpret_cast<volatile int*>(cnt_all + MatchSmem<W, G>::kCntInts);
  float2* spts_all = reinterpret_cast<float2*>(smem_raw + MatchSmem<W, G>::kHeaderBytes);

  constexpr int GT = W * 32;  // threads per group
  const int Gr = blockDim.x / GT;   // groups actually launched per CTA (<= G: the launcher may run a G-group kernel with fewer)
  const int g = threadIdx.x / GT;
  const int t = threadIdx.x - g * GT;
  const int w = t >> 5;
  const int lane = t & 31;
  const int cap = P.pts_cap;
  float2* spts = spts_all + (size_t)g * cap;
  float* red = red_all + g * (2 * 9 * 32);
  uint64_t* mbar = mbars + g;
  int* warp_cnt = cnt_all + g * 32;

  // fused SLAM step: let the map writer's CTAs (launched with programmatic stream serialisation, update_kernel.cuh)
  // become resident on the idle SMs while this single-scan match runs; they wait for this grid's completion
  if (kGrpStep<GRP> || P.gate_state) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  if (t == 0) mbar_init(mbar, 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  // Pacing (G > 1, P.pace_slack > 0).  The per-scan timeline (tuning key trace) shows that the warps of an SM do NOT
  // advance at the same rate — of identical one-warp scans started together the last finishes about half again later
  // than the first — so a one-wave batch ends with a long, thinly occupied tail.  Groups of one CTA
  // therefore publish how many evaluations they have completed and a group that is more than `pace_slack` ahead of
  // the slowest one sleeps: its issue slots and texture bandwidth go to the stragglers and all scans of the CTA end
  // within ~pace_slack evaluations of each other.  No arithmetic is involved: results are unchanged.
  const bool pace = HSB_DIAG && (G > 1) && P.pace_slack > 0;
  const bool fixpoint = P.fixpoint != 0;   // end a level once an evaluation leaves the pose unchanged (see the loop)
  int evals_done = 0;
  if (G > 1) {
    if (threadIdx.x < 32) prog[threadIdx.x] = 0x7fffffff;   // slots of absent / finished groups never hold anyone back
  }
  __syncthreads();
  if (pace && t == 0 && blockIdx.x * Gr + g < P.B) prog[g] = 0;
  if (G > 1) __syncthreads();

  // Staggered start (P.stagger_ns > 0).  In a one-wave batch all scans of an SM start in the same microsecond and —
  // equal work, FIFO texture queue — stay in lock-step: every warp is in its serial section (sincos, reduction, 3x3
  // solve: ~15 % of the instructions, no texture traffic) at the same time, during which the texture pipe, the unit
  // that bounds this kernel, idles.  Many-wave batches do not show this (finished scans are replaced at arbitrary
  // moments: 95 % texture utilisation against ~83 % in one wave).  Starting the warps of an SM a fraction of an
  // evaluation apart de-phases them for the whole launch.
  if (HSB_DIAG && P.stagger_ns > 0) {
    const int rank = (G > 1) ? g : (int)((blockIdx.x / (unsigned)max(P.sm_count, 1)) & 31u);
    if (rank > 0) __nanosleep((unsigned)min(rank * P.stagger_ns, 1000000));
  }
  uint32_t phase = 0;
  int red_flip = 0;
  for (int scan = blockIdx.x * Gr + g; scan < P.B; scan += gridDim.x * Gr) {
    // the scan's input [beg, beg + n): endpoints, or the ranges / cloud points a conversion replaces by the kept endpoints
    size_t beg;
    int n;
    if (P.offsets) {
      beg = P.offsets[scan];
      n = P.offsets[scan + 1] - (int)beg;
    } else {
      n = P.n_shared;
      beg = P.kind == HSB_IN_ENDPOINTS ? 0 : (size_t)scan * n;
    }
    if constexpr (kGrpStep<GRP>) {   // map_without_matching (HectorSlamProcessor.h:80): the hint passes through the gate unmatched
      if (P.kind == HSB_IN_ENDPOINTS && P.gate_in[3 * scan + 2] != 0.0f) n = 0;   // (a conversion runs first, below)
    }
    const float2* __restrict__ gpts = P.pts + beg;
    int member = 0;
    int levels = 0;   // a group's scan: its member's level count (a GRP_NONE scan runs P.levels)
    if constexpr (kGrpMatch<GRP>) {   // group batch match: the scan, its length and the map are the hint's session's
      const HsbScoreSessionDev& s = P.match_sess[session_of(P.match_offsets, P.match_K, scan)];
      gpts = s.pts;
      n = s.n;
      member = s.member;
      levels = s.levels;
    }
    if constexpr (kGrpStep<GRP>) levels = P.group_sess[scan].levels;
    const float2* spts_scan = spts;  // shared-memory copy of the scan's first `ns` points (valid when staged)
    bool staged = false;
    int ns = 0;                      // points [0, ns) are read from shared memory, [ns, n) from global memory
    if (HSB_DIAG && P.trace && t == 0) P.trace[8 * (size_t)scan] = global_timer_ns();
    if constexpr (INL) {
      // the endpoints arrived with the launch: parameter space -> shared memory, and out to device memory for the map
      // writer and the coarse-level containers of later calls (host guarantees cap >= n, n <= HSB_INLINE_MAX_POINTS)
      for (int i = t; i < n; i += GT) {
        const float2 v = S.pts[i];
        spts[i] = v;
        if (P.conv.out_pts) P.conv.out_pts[i] = v;
      }
      group_sync<W>(g);
      ns = n;
      staged = true;
    } else if (!kGrpMatch<GRP> && P.kind != HSB_IN_ENDPOINTS) {
      // a fused conversion: convert + compact straight into shared memory (host guarantees cap >= the input's size)
      const HsbConvDev& C = conv_desc<GRP>(P, scan);
      const double* T = P.cloud_tf ? P.cloud_tf + 12 * (size_t)scan : P.cloud_tf0;
      // cloud and projected: dataContainer.setOrigo(Vector2f(laserPos.x(), laserPos.y()) * scaleToMap)  (:516-517)
      // (called inside both branches: after their join it would cost the unrelated instantiations a register)
      const auto store_origo = [&] {
        if (P.out_origo && t == 0) {
          P.out_origo[2 * (size_t)scan] = __fmul_rn((float)T[3], C.scale_to_map);
          P.out_origo[2 * (size_t)scan + 1] = __fmul_rn((float)T[7], C.scale_to_map);
        }
      };
      if constexpr (PROJ) {   // raw ranges, projected to a cloud in the laser frame and converted by the cloud rule
        n = stage_from_projected<W>(P.conv_in + beg, C.proj_unit, n, C.range_min, C.range_cutoff, T, C.sqr_min_dist,
                                    C.sqr_max_dist, C.z_min, C.z_max, C.scale_to_map, spts, warp_cnt, g, w, lane);
        store_origo();
      } else if (P.kind == HSB_IN_RANGES) {
        n = stage_from_ranges<W>(P.conv_in + beg, C.beam_cs, n, C.range_min, C.range_max_c, C.scale_to_map, spts,
                                 warp_cnt, g, w, lane);
      } else {          // a point cloud
        n = stage_from_cloud<W>(P.conv_in + 3 * beg, n, T, C.sqr_min_dist, C.sqr_max_dist, C.z_min, C.z_max,
                                C.scale_to_map, spts, warp_cnt, g, w, lane);
        store_origo();
      }
      if (C.out_pts) {
        // SLAM step: the endpoints and their number go to the map writer (and, matched, become the last-match
        // container); the count reaches host memory before the step's sequence number (below)
        for (int i = t; i < n; i += GT) C.out_pts[i] = spts[i];
        if (t == 0) {
          *C.out_n = n;
          if (C.out_n_host) *C.out_n_host = n;
        }
      }
      if constexpr (kGrpStep<GRP>) {
        if (P.gate_in[3 * scan + 2] != 0.0f) n = 0;   // map_without_matching: converted for the writer, not matched
      }
      ns = n;
      staged = true;
    } else if (cap > 0 && n > 0 && (n < cap || (!PACK && cap - 2 >= GT))) {
      // Stage the scan — or, when it does not fit the `cap` slots the launcher could afford per group
      // (wave quantisation, hsb_api.cu launch_match_t), a prefix of it whose length is a multiple of the
      // group size, so that every lane keeps its endpoints and visits them in the same order: results
      // do not depend on how much was staged.  Point i goes to spts[i + head] where head = 1 iff the
      // scan starts on an odd point (8- but not 16-byte aligned), so that global and shared
      // addresses share their 16-byte phase and the even-aligned body can move as ONE bulk copy;
      // a misaligned first point / odd last point is carried by plain stores.
      ns = n < cap ? n : ((cap - 2) / GT) * GT;
      const int head = (int)(((uintptr_t)gpts >> 3) & 1);
      const int body = (ns - head) & ~1;
      float2* sdst = spts + head;
      if (t == 0) {
        if (body > 0) {
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
          mbar_expect_tx(mbar, (uint32_t)body * 8u);
          bulk_g2s(sdst + head, gpts + head, (uint32_t)body * 8u, mbar);
        }
        if (head) sdst[0] = gpts[0];
        if (head + body < ns) sdst[ns - 1] = gpts[ns - 1];
      }
      if (HSB_DIAG && P.prefetch && t == 0 && ns < n) l2_prefetch(gpts + ns, gpts + n);
      if (body > 0) {
        mbar_wait(mbar, phase);
        phase ^= 1u;
      }
      group_sync<W>(g);  // head/tail stores visible to the whole group
      spts_scan = sdst;
      staged = true;
    } else if (HSB_DIAG && P.prefetch && t == 0 && n > 0) {
      l2_prefetch(gpts, gpts + n);
    }

    int pack_head = 0;
    if (PACK && staged) {   // (the packed path is only taken with the whole scan staged: ns == n)
      pack_head = (int)(spts_scan - spts);
      pairify_in_place<W>(spts, pack_head, n, t);
      group_sync<W>(g);
    }
    const int npairs = (pack_head + n + 1) >> 1;

    const float* hint;
    if constexpr (INL) hint = S.header;
    else hint = P.hints + 3 * scan;
    float wx = hint[0], wy = hint[1], wpsi = hint[2];
    Acc last;
    acc_zero(last);
    // per-evaluation record (hsb_internal.h HsbMatchParams::record): thread 0 stores what the group holds anyway.  The
    // address is formed from the kernel parameters at each store (level offsets precomputed on the host), so that the
    // evaluation loop carries no extra live register for it.  A group step's session records into its own buffer, set
    // only for a recording member's matched session
    bool recording;
    if constexpr (kGrpStep<GRP>) recording = t == 0 && P.group_sess[scan].record;
    else recording = P.record && t == 0;
    int evals_ran = 0;   // evaluations this scan actually ran (trace slot 5)
    if (n > 0) {
      for (int lvl = (GRP == GRP_NONE ? P.levels : levels) - 1; lvl >= 0; --lvl) {
        const HsbLevelDev& L = level_desc<GRP>(P, scan, member, lvl);
        const LevelRegs LR = level_regs(L);
        float ex, ey, epsi = wpsi;
        if (recording) {
          float* rec = record_base<GRP>(P, scan) + L.rec_off;
          rec[0] = wx; rec[1] = wy; rec[2] = wpsi;
        }
        affine_apply_exact(L.mtw, wx, wy, ex, ey);  // ScanMatcher.h:70 getMapCoordsPose
        int ran = L.evals;                           // evaluations run at this level (fewer at a fixed point, below)
        for (int e = 0; e < L.evals; ++e) {          // ScanMatcher.h:74 + :94-97
          // OccGridMapUtil.h:70-71 and Rotation2Df (:351): sinf/cosf exactly as glibc evaluates them
          float cs, ss;
          if (W > 1) {   // one argument reduction for both (bit-identical to the separate calls)
            sincosf_glibc(epsi, &ss, &cs);
          } else {
            cs = cosf_glibc(epsi);
            ss = sinf_glibc(epsi);
          }
          cs *= L.pt_scale;
          ss *= L.pt_scale;
          Acc a;
          acc_zero(a);
          if (PACK && staged)
            eval_pairs<(U + 1) / 2>(LR, reinterpret_cast<const float4*>(spts), t, GT, npairs, cs, ss, ex, ey, a);
          else if (staged) {
            eval_level<MODE, U>(LR, spts_scan, t, GT, ns, cs, ss, ex, ey, a);
            if (ns < n) eval_level<MODE, U>(LR, gpts, ns + t, GT, n, cs, ss, ex, ey, a);
          } else
            eval_level<MODE, U>(LR, gpts, t, GT, n, cs, ss, ex, ey, a);
          warp_reduce(a);
          if (W > 1) {
            // second stage: the W per-warp sums of each of the 9 values sit transposed in shared
            // memory ([value][warp]); lane l picks warp (l mod WP) and a log2(WP)-step butterfly
            // leaves the group totals in every lane of every warp (same order everywhere).
            // (A reduce-scatter first stage + row sums in the second saves ~100 instructions per
            // evaluation and was tried: on the sparse map of the first scans of a SLAM run, where
            // Gauss-Newton has not reached its fixed point, the different — equally valid — summation
            // order moved one step of the 40 Hz stream test by 1.5e-4 m against the oracle's
            // sequential sum, so the order that is verified against the oracle stays.)
            constexpr int WP = W <= 2 ? 2 : W <= 4 ? 4 : W <= 8 ? 8 : W <= 16 ? 16 : 32;
            float* buf = red + red_flip * (9 * 32);
            if (lane == 0) {
              buf[0 * 32 + w] = a.h00; buf[1 * 32 + w] = a.h11; buf[2 * 32 + w] = a.h22;
              buf[3 * 32 + w] = a.h01; buf[4 * 32 + w] = a.h02; buf[5 * 32 + w] = a.h12;
              buf[6 * 32 + w] = a.d0;  buf[7 * 32 + w] = a.d1;  buf[8 * 32 + w] = a.d2;
            }
            group_sync<W>(g);
            const int src = lane & (WP - 1);
            const bool have = src < W;
            float v[9];
#pragma unroll
            for (int k = 0; k < 9; ++k) v[k] = have ? buf[k * 32 + src] : 0.0f;
#pragma unroll
            for (int o = WP / 2; o > 0; o >>= 1) {
#pragma unroll
              for (int k = 0; k < 9; ++k) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
            }
            a.h00 = v[0]; a.h11 = v[1]; a.h22 = v[2]; a.h01 = v[3]; a.h02 = v[4];
            a.h12 = v[5]; a.d0 = v[6];  a.d1 = v[7];  a.d2 = v[8];
            red_flip ^= 1;
          }
          if (pace) {
            ++evals_done;
            if (t == 0) prog[g] = evals_done;
            for (;;) {
              const int mine = lane < G ? prog[lane] : 0x7fffffff;
              const int slowest = __reduce_min_sync(0xffffffffu, mine);
              if (evals_done <= slowest + P.pace_slack) break;
              __nanosleep(200);
            }
          }
          last = a;
          bool moved = false;
          if (a.h00 != 0.0f && a.h11 != 0.0f) {  // ScanMatcher.h:201
            float d0, d1, d2;
            solve3(a, d0, d1, d2);               // :205
            if (d2 > 0.2f) d2 = 0.2f;            // :209-215
            else if (d2 < -0.2f) d2 = -0.2f;
            const float nx = __fadd_rn(ex, d0);  // :217
            const float ny = __fadd_rn(ey, d1);
            const float npsi = __fadd_rn(epsi, d2);
            moved = (__float_as_uint(nx) != __float_as_uint(ex)) | (__float_as_uint(ny) != __float_as_uint(ey)) |
                    (__float_as_uint(npsi) != __float_as_uint(epsi));
            ex = nx;
            ey = ny;
            epsi = npsi;
          }
          if (recording) {
            float* rec = record_base<GRP>(P, scan) + L.rec_off + 3 + 15 * e;
            rec[0] = a.h00; rec[1] = a.h01; rec[2] = a.h02;
            rec[3] = a.h01; rec[4] = a.h11; rec[5] = a.h12;
            rec[6] = a.h02; rec[7] = a.h12; rec[8] = a.h22;
            rec[9] = a.d0;  rec[10] = a.d1; rec[11] = a.d2;
            rec[12] = ex;   rec[13] = ey;   rec[14] = epsi;
          }
          // Fixed point: the step left the pose bit-for-bit where this evaluation ran it (or the gate made no step).
          // Every later evaluation of the level would run at the same pose on the same map with the same endpoints in
          // the same summation order, i.e. reproduce this one exactly — same sums, same step, same pose — so the level
          // ends here.  The bitwise test counts -0 / +0 as moved (sinf(-0) = -0): conservative.  The pose is the same
          // in every thread of the group, so the exit is uniform.
          if (fixpoint && !moved) {
            ran = e + 1;
            break;
          }
        }
        if (ran < L.evals) {
          // the skipped evaluations: `last` and the pose already are what each of them would leave
          if (recording) {
            for (int e = ran; e < L.evals; ++e) {
              float* rec = record_base<GRP>(P, scan) + L.rec_off + 3 + 15 * e;
              rec[0] = last.h00; rec[1] = last.h01; rec[2] = last.h02;
              rec[3] = last.h01; rec[4] = last.h11; rec[5] = last.h12;
              rec[6] = last.h02; rec[7] = last.h12; rec[8] = last.h22;
              rec[9] = last.d0;  rec[10] = last.d1; rec[11] = last.d2;
              rec[12] = ex;      rec[13] = ey;      rec[14] = epsi;
            }
          }
          if (pace) {   // they count as done: nobody waits for them
            evals_done += L.evals - ran;
            if (t == 0) prog[g] = evals_done;
          }
        }
        evals_ran += ran;
        epsi = normalize_angle(epsi);                 // ScanMatcher.h:170
        affine_apply_exact(L.wtm, ex, ey, wx, wy);    // :186 getWorldCoordsPose
        wpsi = epsi;
        if (HSB_DIAG && P.trace && t == 0) P.trace[8 * (size_t)scan + (P.levels - lvl)] = global_timer_ns();
      }
    } else if (recording) {   // nothing evaluated: every level starts from the hint, the evaluation slots are zero
      // (a group step's session: its member's own levels, in its member's layout; a group match records nothing)
      for (int lvl = (kGrpStep<GRP> ? levels : P.levels) - 1; lvl >= 0; --lvl) {
        const HsbLevelDev& L = kGrpStep<GRP> ? level_desc<GRP>(P, scan, member, lvl) : P.lv[lvl];
        float* rec = record_base<GRP>(P, scan) + L.rec_off;
        rec[0] = wx; rec[1] = wy; rec[2] = wpsi;
        for (int i = 3; i < 3 + 15 * L.evals; ++i) rec[i] = 0.0f;
      }
    }
    if (pace && n <= 0) {   // nothing evaluated: account for the evaluations the others wait for
      for (int lvl = 0; lvl < P.levels; ++lvl) evals_done += P.lv[lvl].evals;
      if (t == 0) prog[g] = evals_done;
    }
    if (HSB_DIAG && P.trace && t == 0) {
      P.trace[8 * (size_t)scan + 1 + P.levels] = global_timer_ns();
      if (P.levels <= 3) P.trace[8 * (size_t)scan + 5] = (unsigned long long)evals_ran;
      P.trace[8 * (size_t)scan + 6] = warp_id();
      P.trace[8 * (size_t)scan + 7] = sm_id();
    }
    if (kGrpStep<GRP> && t == 0) {
      // group SLAM step: the session's gate, against its own handle's state and thresholds
      slam_gate(P.group_sess[scan].gate_state, P.gate_in + 3 * scan, wx, wy, wpsi, P.out_poses + 4 * scan,
                P.gate_out_host + 4 * scan);
    } else if (t == 0 && P.gate_state) {
      // fused SLAM step (one scan): the map-update gate runs in the match kernel's epilogue — no separate launch
      const float* gate_in;
      if constexpr (INL) gate_in = S.header + 3;
      else gate_in = P.gate_in;
      slam_gate(P.gate_state, gate_in, wx, wy, wpsi, P.out_poses, P.gate_out_host);
    } else if (t == 0) {
      P.out_poses[3 * scan + 0] = wx;
      P.out_poses[3 * scan + 1] = wy;
      P.out_poses[3 * scan + 2] = wpsi;
    }
    if (t == 0) {
      if (P.out_cov) {  // covMatrix = H, ScanMatcher.h:184.  An empty scan leaves the caller's matrix
        // untouched in the reference (:68,189): hsb_match_data honours that on the host side, the
        // batch entry points document a zero matrix instead (`last` is still zero then).
        float* c = P.out_cov + 9 * (size_t)scan;
        c[0] = last.h00; c[1] = last.h01; c[2] = last.h02;
        c[3] = last.h01; c[4] = last.h11; c[5] = last.h12;
        c[6] = last.h02; c[7] = last.h12; c[8] = last.h22;
      }
    }
    if (kGrpStep<GRP> && t == 0) {
      // group SLAM step: the LAST session to finish publishes the sequence number — every session's results (each made
      // visible system-wide before its count) are then in host memory
      __threadfence_system();
      if (atomicAdd(P.group_done, 1u) == (unsigned)P.B - 1u) {
        *P.group_done = 0u;   // re-armed for the next step, which is stream-ordered behind this grid
        __threadfence_system();
        *reinterpret_cast<volatile unsigned*>(P.seq_host) = P.seq_value;
      }
    } else if (t == 0 && P.seq_host) {   // fused SLAM step: results are in mapped host memory — tell the polling host
      __threadfence_system();
      *reinterpret_cast<volatile unsigned*>(P.seq_host) = P.seq_value;
    }
    if constexpr (kGrpStep<GRP>) {
      // a matched scan becomes the member's "containers of the last match" (MapRepMultiMap.h:127): the coarse levels of
      // its later map writes without matching read it (after the pose is out: only the map writers wait for this).
      // A converted scan is already there (the conversion's sink, above).
      if (P.kind == HSB_IN_ENDPOINTS) {
        float2* keep = P.group_sess[scan].last_pts;
        for (int i = t; i < n; i += GT) keep[i] = gpts[i];
      }
    }
    if (cap > 0) group_sync<W>(g);  // everyone done with spts before the next bulk copy lands
  }
  if (pace && t == 0) prog[g] = 0x7fffffff;   // this group is done: nobody waits for it any more
}

// The conversion alone, one CTA of 8 warps per scan of the table (table[blockIdx.x]: its input, length, laser transform
// and descriptor) into each scan's sink: the stand-alone conversion calls (a table of one) and the group batch match
// from raw scans (one entry per session).  Each scan's kept count goes to its out_n and, if set, out_n_host.
template <int KIND>
__global__ void __launch_bounds__(256) conv_to_points_kernel(const HsbConvScanDev* __restrict__ table) {
  __shared__ int warp_cnt[32];
  const HsbConvScanDev& S = table[blockIdx.x];
  const HsbConvDev& C = S.conv;
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int n;
  if constexpr (KIND == HSB_IN_RANGES) {
    n = stage_from_ranges<8>(S.in, C.beam_cs, S.n_in, C.range_min, C.range_max_c, C.scale_to_map, C.out_pts, warp_cnt, 0,
                             w, lane);
  } else if constexpr (KIND == HSB_IN_CLOUD) {
    n = stage_from_cloud<8>(S.in, S.n_in, S.T, C.sqr_min_dist, C.sqr_max_dist, C.z_min, C.z_max, C.scale_to_map,
                            C.out_pts, warp_cnt, 0, w, lane);
  } else {
    double Tr[12];   // the transform read once (left to ptxas, the per-point reloads spill at its 32-register choice)
#pragma unroll
    for (int k = 0; k < 12; ++k) Tr[k] = S.T[k];
    n = stage_from_projected<8>(S.in, C.proj_unit, S.n_in, C.range_min, C.range_cutoff, Tr, C.sqr_min_dist,
                                C.sqr_max_dist, C.z_min, C.z_max, C.scale_to_map, C.out_pts, warp_cnt, 0, w, lane);
  }
  if (threadIdx.x == 0) {
    *C.out_n = n;
    if (C.out_n_host) *C.out_n_host = n;
  }
}

// N3: OccGridMapUtil::getLikelihoodForState (OccGridMapUtil.h:189-221) for one state (map coordinates of the level),
// evaluated by one warp; every lane returns the value.  interpMapValue (:233-285) is the value-only bilinear
// interpolation: 0 out of bounds, so such an endpoint contributes funval = 1.
template <int MODE>
__device__ __forceinline__ float warp_likelihood(const LevelRegs& LR, float pt_scale, const float2* __restrict__ pts, int n, float ex,
                                                 float ey, float psi, int lane) {
  if constexpr (MODE == MODE_ANY) {   // the level's own gather path (uniform across the warp)
    return LR.tex ? warp_likelihood<MODE_TEX>(LR, pt_scale, pts, n, ex, ey, psi, lane)
                  : warp_likelihood<MODE_LDG>(LR, pt_scale, pts, n, ex, ey, psi, lane);
  }
  const float cs = cosf_glibc(psi) * pt_scale, ss = sinf_glibc(psi) * pt_scale;
  float residual = 0.0f;
  for (int i = lane; i < n; i += 32) {
    const float2 p = pts[i];
    PointPre pre;
    point_address<MODE>(LR, p.x, p.y, true, cs, ss, ex, ey, pre);
    const float4 v = point_fetch<MODE>(LR, pre);
    const float xi = 1.0f - pre.fx, yi = 1.0f - pre.fy;
    const float m = (v.x * xi + v.y * pre.fx) * yi + (v.z * xi + v.w * pre.fx) * pre.fy;  // :282-284
    residual += pre.inside ? (1.0f - m) : 1.0f;                                         // :216-217
  }
  residual = warp_sum(residual);
  return 1.0f - residual / (float)n;  // getLikelihoodForResidual :203-209
}

// One pose of a likelihood batch, by one warp: the world pose to the level's map coordinates (getMapCoordsPose), then
// warp_likelihood.  Shared by likelihood_kernel (poses and scans on the device) and likelihood_group_kernel (staged from
// host buffers).
template <int MODE>
__device__ __forceinline__ float pose_likelihood(const HsbLevelDev& L, const LevelRegs& LR, const float* __restrict__ pose_world,
                                                 const float2* __restrict__ pts, int n, int lane) {
  float ex, ey;
  affine_apply_exact(L.mtw, pose_world[0], pose_world[1], ex, ey);
  return warp_likelihood<MODE>(LR, L.pt_scale, pts, n, ex, ey, pose_world[2], lane);
}

// arg-max over a batch (relocalisation: the most likely hypothesis): (score, index) packed so that one 64-bit atomicMax
// keeps the highest score and, among equals, the LOWEST index; a non-finite pose scores -1, and so does a NaN
// likelihood (an empty scan: 1 - 0/0), whose bits would otherwise pack above every score.  Every finite pose keeps its
// score, FLT_MAX included (hsb_reset stores FLT_MAX as a pose); only +-inf and NaN are non-finite.
__device__ __forceinline__ unsigned long long best_pack(float lh, const float* __restrict__ pose_world, unsigned index) {
  const float px = pose_world[0], py = pose_world[1], pp = pose_world[2];
  const bool finite = isfinite(px) && isfinite(py) && isfinite(pp);
  const float sc = (finite && lh == lh) ? lh : -1.0f;
  unsigned u = __float_as_uint(sc);
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return ((unsigned long long)u << 32) | (unsigned long long)(0xffffffffu - index);
}
// ... and back: the winner's score and index (v != 0: an accumulator no pose reached stays 0)
__device__ __forceinline__ float best_unpack(unsigned long long v, unsigned& index) {
  unsigned u = (unsigned)(v >> 32);
  u = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
  index = 0xffffffffu - (unsigned)(v & 0xffffffffull);
  return __uint_as_float(u);
}

template <int MODE>
__global__ void __launch_bounds__(128)
    likelihood_kernel(const HsbLevelDev L, int B, const float* __restrict__ poses_world, const float2* __restrict__ pts_all,
                      const int* __restrict__ offsets, int n_shared, float* __restrict__ out,
                      unsigned long long* __restrict__ best = nullptr) {
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const LevelRegs LR = level_regs(L);
  for (int b = warp; b < B; b += nwarps) {
    int beg = 0, n = n_shared;
    if (offsets) {
      beg = offsets[b];
      n = offsets[b + 1] - beg;
    }
    const float lh = pose_likelihood<MODE>(L, LR, poses_world + 3 * b, pts_all + beg, n, lane);
    if (lane == 0) {
      if (out) out[b] = lh;
      if (best) atomicMax(best, best_pack(lh, poses_world + 3 * b, (unsigned)b));
    }
  }
}
// second launch of hsb_best_hypothesis_device: unpack the winner, re-arm the accumulator
__global__ void best_hypothesis_finish_kernel(unsigned long long* __restrict__ best, const float* __restrict__ poses_world,
                                              float* __restrict__ out4) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const unsigned long long v = *best;
  *best = 0ull;
  if (v == 0ull) {   // empty batch
    out4[0] = -1.0f; out4[1] = 0.0f; out4[2] = 0.0f; out4[3] = 0.0f;
    return;
  }
  unsigned b;
  out4[0] = best_unpack(v, b);
  out4[1] = poses_world[3 * b]; out4[2] = poses_world[3 * b + 1]; out4[3] = poses_world[3 * b + 2];
}

// N3 from host buffers (hsb_likelihood_batch, hsb_group_likelihood, hsb_group_best_hypothesis): pose q of the call
// belongs to the session k whose poses are [pose_offsets[k], pose_offsets[k+1]) and is scored against that session's
// scan on its member's map of the level (the descriptor table).  One warp per pose, grid-stride; the value is
// likelihood_kernel's.  With `best`, session k's arg-max goes to best[k], the index being the pose's index in its
// session.
template <int MODE>
__global__ void __launch_bounds__(128) likelihood_group_kernel(const HsbScoreParams P) {
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int q = warp; q < P.Q; q += nwarps) {
    const int k = session_of(P.pose_offsets, P.K, q);
    const HsbScoreSessionDev s = P.sess[k];
    const HsbLevelDev& L = P.lv[(size_t)s.member * P.levels + P.level];
    const LevelRegs LR = level_regs(L);   // (all 32 lanes are here: a warp's lanes share q)
    const float lh = pose_likelihood<MODE>(L, LR, P.poses + 3 * (size_t)q, s.pts, s.n, lane);
    if (lane == 0) {
      if (P.out) P.out[q] = lh;
      if (P.best) atomicMax(P.best + k, best_pack(lh, P.poses + 3 * (size_t)q, (unsigned)(q - P.pose_offsets[k])));
    }
  }
}
// second launch of hsb_group_best_hypothesis: thread k unpacks session k's winner and re-arms its accumulator
__global__ void __launch_bounds__(128) best_group_finish_kernel(const HsbScoreParams P) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= P.K) return;
  const unsigned long long v = P.best[k];
  P.best[k] = 0ull;
  float* out4 = P.out_best4 + 4 * (size_t)k;
  if (v == 0ull) {   // empty session
    out4[0] = -1.0f; out4[1] = 0.0f; out4[2] = 0.0f; out4[3] = 0.0f;
    P.out_best_index[k] = -1;
    return;
  }
  unsigned b;
  out4[0] = best_unpack(v, b);
  const float* pose = P.poses + 3 * ((size_t)P.pose_offsets[k] + b);
  out4[1] = pose[0]; out4[2] = pose[1]; out4[3] = pose[2];
  P.out_best_index[k] = (int)b;
}

// getCovarianceForPose's sigma points (OccGridMapUtil.h:109-135): +-1.5 cells in x and y, +-0.05 rad, the pose itself
constexpr float kSigmaCells = 1.5f, kSigmaAngle = 0.05f;
// sigma point k of the pose (x, y, ang) in map coordinates
__device__ __forceinline__ void sigma_point(int k, float x, float y, float ang, float& sx, float& sy, float& sa) {
  sx = x; sy = y; sa = ang;
  if (k == 0) sx = __fadd_rn(x, kSigmaCells);
  else if (k == 1) sx = __fsub_rn(x, kSigmaCells);
  else if (k == 2) sy = __fadd_rn(y, kSigmaCells);
  else if (k == 3) sy = __fsub_rn(y, kSigmaCells);
  else if (k == 4) sa = __fadd_rn(ang, kSigmaAngle);
  else if (k == 5) sa = __fsub_rn(ang, kSigmaAngle);
}
// The likelihood-weighted mean and covariance of the seven sigma points (:137-154) with the fixed-size Eigen operations
// in the order oracle/shim fixes: likelihoods.sum() by recursive halving, mean += point * lh, mean *= 1/sum,
// cov += (lh * inv) * (d * d^T), every operation rounded separately; then getCovMatrixWorldCoords (:162-187).  One thread;
// the matrices of pose b go to out_map / out_world + 9 b (either may be null).
__device__ __forceinline__ void sigma_covariance(const float* lhs, float x, float y, float ang, float cell_length, int b,
                                                 float* __restrict__ out_map, float* __restrict__ out_world) {
  const float dt = kSigmaCells, da = kSigmaAngle;
  const float sp[7][3] = {{__fadd_rn(x, dt), y, ang}, {__fsub_rn(x, dt), y, ang}, {x, __fadd_rn(y, dt), ang},
                          {x, __fsub_rn(y, dt), ang}, {x, y, __fadd_rn(ang, da)}, {x, y, __fsub_rn(ang, da)}, {x, y, ang}};
  const float sum = __fadd_rn(__fadd_rn(lhs[0], __fadd_rn(lhs[1], lhs[2])),
                              __fadd_rn(__fadd_rn(lhs[3], lhs[4]), __fadd_rn(lhs[5], lhs[6])));
  const float inv = __fdiv_rn(1.0f, sum);                                       // :137
  float mean[3] = {0.f, 0.f, 0.f};
  for (int i = 0; i < 7; ++i)
    for (int c = 0; c < 3; ++c) mean[c] = __fadd_rn(mean[c], __fmul_rn(sp[i][c], lhs[i]));   // :144
  for (int c = 0; c < 3; ++c) mean[c] = __fmul_rn(mean[c], inv);                             // :147
  float cov[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int i = 0; i < 7; ++i) {                                                               // :151-154
    const float d[3] = {__fsub_rn(sp[i][0], mean[0]), __fsub_rn(sp[i][1], mean[1]), __fsub_rn(sp[i][2], mean[2])};
    const float wgt = __fmul_rn(lhs[i], inv);
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) cov[3 * r + c] = __fadd_rn(cov[3 * r + c], __fmul_rn(wgt, __fmul_rn(d[r], d[c])));
  }
  if (out_map)
    for (int c = 0; c < 9; ++c) out_map[9 * (size_t)b + c] = cov[c];
  if (out_world) {                                                                            // :162-187
    float* w = out_world + 9 * (size_t)b;
    const float st = cell_length, st2 = __fmul_rn(st, st);
    w[0] = __fmul_rn(cov[0], st2);
    w[4] = __fmul_rn(cov[4], st2);
    w[3] = __fmul_rn(cov[3], st2);
    w[1] = w[3];
    w[6] = __fmul_rn(cov[6], st);
    w[2] = w[6];
    w[7] = __fmul_rn(cov[7], st);
    w[5] = w[7];
    w[8] = cov[8];
  }
}
// Pose b of a covariance batch, by one CTA of 7 warps: warp k evaluates the likelihood of sigma point k, thread 0 forms
// the matrices.  Ends with a barrier, so the caller may loop.
template <int MODE>
__device__ __forceinline__ void pose_covariance(const HsbLevelDev& L, const LevelRegs& LR, const float* __restrict__ poses_world,
                                                int b, const float2* __restrict__ pts, int n, float cell_length,
                                                float* __restrict__ out_map, float* __restrict__ out_world) {
  __shared__ float lhs[7];
  const int lane = threadIdx.x & 31, k = threadIdx.x >> 5;
  float x, y;
  affine_apply_exact(L.mtw, poses_world[3 * b], poses_world[3 * b + 1], x, y);   // getMapCoordsPose
  const float ang = poses_world[3 * b + 2];
  float sx, sy, sa;
  sigma_point(k, x, y, ang, sx, sy, sa);
  const float lh = warp_likelihood<MODE>(LR, L.pt_scale, pts, n, sx, sy, sa, lane);
  if (lane == 0) lhs[k] = lh;
  __syncthreads();
  if (threadIdx.x == 0) sigma_covariance(lhs, x, y, ang, cell_length, b, out_map, out_world);
  __syncthreads();
}

// N3: OccGridMapUtil::getCovarianceForPose (OccGridMapUtil.h:106-160) + getCovMatrixWorldCoords (:162-187) for
// hsb_covariance_batch and hsb_group_covariance: one CTA of 7 warps per pose (pose_covariance), the pose's session, scan
// and member map found as likelihood_group_kernel finds them; the world matrix takes the session's member's cell length.
template <int MODE>
__global__ void __launch_bounds__(224) covariance_kernel(const HsbScoreParams P) {
  for (int q = blockIdx.x; q < P.Q; q += gridDim.x) {
    const HsbScoreSessionDev s = P.sess[session_of(P.pose_offsets, P.K, q)];
    const HsbLevelDev& L = P.lv[(size_t)s.member * P.levels + P.level];
    const LevelRegs LR = level_regs(L);   // (every warp is whole here: a CTA's threads share q)
    pose_covariance<MODE>(L, LR, P.poses, q, s.pts, s.n, s.cell_length, P.out_map, P.out_world);
  }
}

// Single evaluation (the getCompleteHessianDerivs seam): one CTA of 256 threads.
template <int MODE>
__global__ void __launch_bounds__(256)
    hessian_kernel(const HsbLevelDev L, const float2* __restrict__ pts, int n, float px, float py, float ppsi,
                   float* __restrict__ out12) {
  __shared__ float red[8][12];
  const float cs = cosf_glibc(ppsi), ss = sinf_glibc(ppsi);
  Acc a;
  acc_zero(a);
  eval_points<MODE, HSB_UNROLL>(level_regs(L), pts, threadIdx.x, blockDim.x, n, cs, ss, px, py, a);
  warp_reduce(a);
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
    red[w][0] = a.h00; red[w][1] = a.h11; red[w][2] = a.h22; red[w][3] = a.h01; red[w][4] = a.h02;
    red[w][5] = a.h12; red[w][6] = a.d0;  red[w][7] = a.d1;  red[w][8] = a.d2;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float s[9];
    for (int k = 0; k < 9; ++k) {
      float v = 0.f;
      for (int j = 0; j < 8; ++j) v += red[j][k];
      s[k] = v;
    }
    // H row-major, then dTr
    out12[0] = s[0]; out12[1] = s[3]; out12[2] = s[4];
    out12[3] = s[3]; out12[4] = s[1]; out12[5] = s[5];
    out12[6] = s[4]; out12[7] = s[5]; out12[8] = s[2];
    out12[9] = s[6]; out12[10] = s[7]; out12[11] = s[8];
  }
}

}  // namespace hsb
#endif
