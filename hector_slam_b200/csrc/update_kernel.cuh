// update_kernel.cuh — K2 (Bresenham log-odds map update) and K3 (probability-plane refresh), sm_90a.
//
// What K2 replaces (paths under the reference's hector_mapping/include/hector_slam_lib/):
//   OccGridMapBase::updateByScan          map/OccGridMapBase.h:121-168
//   OccGridMapBase::updateLineBresenhami  map/OccGridMapBase.h:170-214
//   OccGridMapBase::bresenham2D           map/OccGridMapBase.h:243-260
//   bresenhamCellFree / bresenhamCellOcc  map/OccGridMapBase.h:216-241
//   GridMapLogOddsFunctions::updateSetOccupied/SetFree/UnsetFree   map/GridMapLogOdds.h:135-156
// and K3:
//   GridMapLogOddsFunctions::getGridProbability   map/GridMapLogOdds.h:163-166
//   (the reference memoises it per cell in GridMapCacheArray, map/GridMapCacheArray.h:80-102,
//    invalidated by onMapUpdated; here the probability plane is simply kept current)
//
// The reference walks beams one after another and uses per-cell `updateIndex` stamps so that a
// cell is touched once per scan, an end point (occupied) overriding any free marking.  That is
// order-free, so the device does it in two grid-wide phases (cell i of a Bresenham line has a
// closed form, no serial walk):
//   MARK : a team of warps per beam, lanes striding along the line:
//          atomicMax(stamp[cell], base+1) along the line, atomicMax(stamp[end], base+2)
//   APPLY: a coalesced sweep over the bounding box of the scan's beams; every cell whose stamp is
//          base+1 / base+2 gets the log-odds update (free: l += lf ; occupied: if (l < 50) l += lo)
//          and its probability rewritten (and the texture twin through a surface store).
// A cell that the reference first frees and then hits ends as ((l + lf) - lf) + lo there and as
// l + lo here — equal to ~1 ulp (SURVEY.md Q10); tests compare planes with abs tol 1e-5.
#ifndef HSB_UPDATE_KERNEL_CUH
#define HSB_UPDATE_KERNEL_CUH

#include <cfloat>
#include <climits>

#include "hsb_internal.h"
#include "sincosf_glibc.h"

namespace hsb {

// P = e^l / (e^l + 1) in fp32 like the reference (GridMapLogOdds.h:165-166: expf, one addition, one division).  expf is
// glibc's, operation for operation (sincosf_glibc.h: expf_glibc) — a correctly rounded exp differs from it by one ulp on
// ~1 % of the arguments — so the probability plane equals the reference's bit for bit.
__device__ __forceinline__ float prob_from_logodds(float l) {
  const float odds = expf_glibc(l);
  return __fdiv_rn(odds, __fadd_rn(odds, 1.0f));
}

__global__ void refresh_prob_kernel(const float* __restrict__ logodds, float* __restrict__ prob, cudaSurfaceObject_t surf,
                                    int sx, int sy) {
  const size_t n = (size_t)sx * (size_t)sy;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float p = prob_from_logodds(logodds[i]);
    prob[i] = p;
    if (surf) {
      const int y = (int)(i / (size_t)sx), x = (int)(i - (size_t)y * sx);
      surf2Dwrite(p, surf, x * (int)sizeof(float), y);
    }
  }
}

// LogOddsCell::resetGridCell (GridMapBase.h:71-82) of cell i of a level sx cells wide: l = 0, P(0) = 0.5 and the
// texture twin.
__device__ __forceinline__ void clear_cell(float* logodds, float* prob, cudaSurfaceObject_t surf, int sx, size_t i) {
  logodds[i] = 0.0f;
  prob[i] = 0.5f;
  if (surf) {
    const int y = (int)(i / (size_t)sx), x = (int)(i - (size_t)y * sx);
    surf2Dwrite(0.5f, surf, x * (int)sizeof(float), y);
  }
}

// resetGridCell for a whole level, stamps 0 too (hsb_reset, one level per launch).
__global__ void clear_level_kernel(float* __restrict__ logodds, float* __restrict__ prob, uint32_t* __restrict__ stamp,
                                   cudaSurfaceObject_t surf, int sx, int sy) {
  const size_t n = (size_t)sx * (size_t)sy;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    clear_cell(logodds, prob, surf, sx, i);
    stamp[i] = 0u;
  }
}

// N1: nav_msgs/OccupancyGrid values as HectorMappingRos::publishMap derives them
// (hector_mapping/src/HectorMappingRos.cpp:448-468; isFree / isOccupied GridMapLogOdds.h:76-84): 0 where l < 0, 100
// where l > 0, -1 otherwise (+-0 and NaN).  Every occupancy export thresholds with this one expression.
__device__ __forceinline__ int8_t occupancy_value(float l) {
  return l < 0.0f ? (int8_t)0 : (l > 0.0f ? (int8_t)100 : (int8_t)-1);
}

// N1 on a rectangle: the cells of {x0, y0, w, hgt} thresholded into a packed w x hgt buffer (dirty-rectangle publishing,
// and the whole level's export as the rectangle of every cell).
__global__ void occupancy_rect_kernel(const float* __restrict__ logodds, int sx, int x0, int y0, int w, int hgt,
                                      int8_t* __restrict__ out) {
  const size_t n = (size_t)w * hgt;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / (size_t)w), c = (int)(i - (size_t)r * w);
    out[i] = occupancy_value(logodds[(size_t)(y0 + r) * sx + (x0 + c)]);
  }
}

// Group occupancy sync, pass 1: session k's mirror rectangle of `level` (member members[k]'s, found through the group's
// table mirror[member * levels + level]) into rects[4k ..], then, with reset, the rectangle cleared.
__global__ void gather_mirror_rects_kernel(int* const* __restrict__ mirror, int levels, int level,
                                           const int* __restrict__ members, int K, int reset, int4* __restrict__ rects) {
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < K; k += gridDim.x * blockDim.x) {
    int* r = mirror[(size_t)members[k] * levels + level];
    rects[k] = make_int4(r[0], r[1], r[2], r[3]);
    if (reset) {
      r[0] = INT_MAX;
      r[1] = INT_MAX;
      r[2] = -1;
      r[3] = -1;
    }
  }
}

// Group occupancy sync, pass 2: rows [r_begin, r_end) of the call's stacked rectangles (HsbOccRowsDev) thresholded into
// the packed chunk `out`, whose first byte is the call's packed byte `out_base`.  One warp per row, lanes along the row:
// coalesced reads, each cell read once.  n_rows: the entries of `rows` (non-empty rectangles only).
__global__ void occupancy_rows_kernel(const HsbOccRowsDev* __restrict__ rows, int n_rows, int r_begin, int r_end,
                                      size_t out_base, int8_t* __restrict__ out) {
  const int warps = blockDim.x >> 5, lane = threadIdx.x & 31;
  for (int r = r_begin + blockIdx.x * warps + (threadIdx.x >> 5); r < r_end; r += gridDim.x * warps) {
    int lo = 0, hi = n_rows - 1;   // the last rectangle that starts at or before row r
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (rows[mid].row0 <= r) lo = mid;
      else hi = mid - 1;
    }
    const HsbOccRowsDev s = rows[lo];
    const int y = r - s.row0;
    const float* src = s.logodds + (size_t)(s.y0 + y) * s.sx + s.x0;
    int8_t* dst = out + (s.off + (size_t)y * s.w - out_base);
    for (int x = lane; x < s.w; x += 32) dst[x] = occupancy_value(src[x]);
  }
}

// N4: DistanceMeasurementProvider::checkOccupancyBresenhami (HectorMapTools.h:148-214, bresenham2D :216-237), one warp
// per ray.  Same closed-form line as K2; 32 cells are tested per step and the first occupied one wins.
__device__ __forceinline__ float warp_raycast(const float* __restrict__ logodds, int sx, int sy, int2 p0, int2 p1, int lane,
                                              int2& hit) {
  float dist = -1.0f;
  hit = make_int2(-1, -1);
  const bool ok = p0.x >= 0 && p0.x < sx && p0.y >= 0 && p0.y < sy && p1.x >= 0 && p1.x < sx && p1.y >= 0 && p1.y < sy;  // :155-166
  if (ok) {
    const int dx = p1.x - p0.x, dy = p1.y - p0.y;
    const unsigned adx = (unsigned)abs(dx), ady = (unsigned)abs(dy);
    const int off_dx = dx > 0 ? 1 : -1, off_dy = (dy > 0 ? 1 : -1) * sx;   // :174-175
    unsigned ada, adb;
    int off_a, off_b;
    if (adx >= ady) { ada = adx; adb = ady; off_a = off_dx; off_b = off_dy; }   // :182-189
    else            { ada = ady; adb = adx; off_a = off_dy; off_b = off_dx; }
    const unsigned err0 = ada / 2u;
    const unsigned start = (unsigned)p0.y * (unsigned)sx + (unsigned)p0.x;
    const unsigned steps = min(5000u, ada);                                    // :218
    for (unsigned base = 0; base < steps; base += 32u) {
      const unsigned i = base + (unsigned)lane;
      unsigned off = 0;
      bool occ = false;
      if (i < steps) {
        const unsigned carries = (unsigned)(((unsigned long long)err0 + (unsigned long long)i * adb) / ada);
        off = start + (unsigned)((int)i * off_a) + (unsigned)((int)carries * off_b);
        occ = logodds[off] > 0.0f;                                             // data[offset] == 100  (:223)
      }
      const unsigned m = __ballot_sync(0xffffffffu, occ);
      if (m) {
        const int first = __ffs(m) - 1;
        const unsigned hoff = __shfl_sync(0xffffffffu, off, first);
        hit = make_int2((int)(hoff % (unsigned)sx), (int)(hoff / (unsigned)sx));   // :194
        const float fx = (float)(p0.x - hit.x), fy = (float)(p0.y - hit.y);
        dist = (float)(int)__fsqrt_rn(__fadd_rn(__fmul_rn(fx, fx), __fmul_rn(fy, fy)));  // int distMap = norm  (:196)
        break;
      }
    }
  }
  return dist;
}

// N4 (hsb_raycast_batch, hsb_get_dist_batch and their group forms): ray q of the call belongs to the session k whose
// rays are [offsets[k], offsets[k+1]) and is cast on member members[k]'s level, whose plane, size and getDist transform
// are the table entry lv[member * levels + level] (a single handle's call: one session and a one-entry table), so the
// members of a group may differ in map size, resolution and start.  One warp per ray, grid-stride.  kWorld: getDist rays
// (float2 world points); otherwise ray-cast rays (int2 cells).
template <bool kWorld>
__global__ void __launch_bounds__(256) ray_kernel(const HsbRayParams P) {
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int q = warp; q < P.Q; q += nwarps) {
    int lo = 0, hi = P.K - 1;   // the last session whose rays start at or before ray q (empty sessions are passed over)
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (P.offsets[mid] <= q) lo = mid;
      else hi = mid - 1;
    }
    const HsbRayLevelDev R = P.lv[(size_t)P.members[lo] * P.levels + P.level];
    if (kWorld) {
      // DistanceMeasurementProvider::getDist (HectorMapTools.h:133-147): world -> cell with
      // CoordinateTransformer<float>::getC2Coords ((w - origo) * inv_scale, :93-96) truncated by cast<int> (:136-137; a
      // non-finite or absurd coordinate is treated as outside the map), the ray cast, the hit cell back to the world with
      // getC1Coords (origo + cell * scale, :88-91) and the distance scaled by getC1Scale (scale * dist, :98-101; nothing
      // hit: scale * -1 as in the reference, hit_world = (0, 0) and found = 0 where the reference leaves hitCoords
      // undefined).
      const float2 bw = static_cast<const float2*>(P.begin)[q], ew = static_cast<const float2*>(P.end)[q];
      const float bx = __fmul_rn(__fsub_rn(bw.x, R.origo_x), R.inv_scale);
      const float by = __fmul_rn(__fsub_rn(bw.y, R.origo_y), R.inv_scale);
      const float ex = __fmul_rn(__fsub_rn(ew.x, R.origo_x), R.inv_scale);
      const float ey = __fmul_rn(__fsub_rn(ew.y, R.origo_y), R.inv_scale);
      const bool sane = fabsf(bx) < 1.0e9f && fabsf(by) < 1.0e9f && fabsf(ex) < 1.0e9f && fabsf(ey) < 1.0e9f;
      const int2 p0 = sane ? make_int2((int)bx, (int)by) : make_int2(-1, -1);
      const int2 p1 = sane ? make_int2((int)ex, (int)ey) : make_int2(-1, -1);
      int2 hit;
      const float dist = warp_raycast(R.plane, R.sx, R.sy, p0, p1, lane, hit);
      if (lane == 0) {
        P.out_dist[q] = __fmul_rn(R.scale, dist);
        const bool found = dist >= 0.0f;
        if (P.out_found) P.out_found[q] = found ? 1 : 0;
        if (P.out_hit)
          static_cast<float2*>(P.out_hit)[q] =
              found ? make_float2(__fadd_rn(R.origo_x, __fmul_rn((float)hit.x, R.scale)),
                                  __fadd_rn(R.origo_y, __fmul_rn((float)hit.y, R.scale)))
                    : make_float2(0.0f, 0.0f);
      }
    } else {
      int2 hit;
      const float dist = warp_raycast(R.plane, R.sx, R.sy, static_cast<const int2*>(P.begin)[q],
                                      static_cast<const int2*>(P.end)[q], lane, hit);
      if (lane == 0) {
        P.out_dist[q] = dist;
        if (P.out_hit) static_cast<int2*>(P.out_hit)[q] = hit;
      }
    }
  }
}

__device__ __forceinline__ void pdl_launch_dependents_early() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ---- K2 -----------------------------------------------------------------------------------------

// HectorSlamProcessor::update's gate (slam_main/HectorSlamProcessor.h:83-95) evaluated on the device so that a
// fused step needs no host round trip between match and map write.
//   state: [0..2] lastMapUpdatePose, [3] out: 1.0f if the map is to be written by this step
//   in   : [0] minDist, [1] minAngle, [2] force (map_without_matching)
// pose_out (device) and pose_out_host (mapped host memory, may be null) receive the step's pose (the matched
// pose, or the hint when matching is skipped) and, in [3], a copy of the flag.
__global__ void slam_gate_kernel(float* __restrict__ state, const float* __restrict__ in, const float* pose_in,
                                 float* pose_out, float* pose_out_host, unsigned* seq_host, unsigned seq_value) {
  pdl_launch_dependents_early();
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    slam_gate(state, in, pose_in[0], pose_in[1], pose_in[2], pose_out, pose_out_host);
    if (seq_host) {
      __threadfence_system();
      *reinterpret_cast<volatile unsigned*>(seq_host) = seq_value;
    }
  }
}

// map_without_matching step from a point cloud: the kept-endpoint count goes to mapped host memory, then the sequence number
__global__ void publish_int_kernel(const int* __restrict__ value_dev, int* value_host, unsigned* seq_host, unsigned seq_value) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    *value_host = *value_dev;
    if (seq_host) {
      __threadfence_system();
      *reinterpret_cast<volatile unsigned*>(seq_host) = seq_value;
    }
  }
}

// Per-level frame of one updateByScan call: the pose as Translation(x,y)*Rotation(psi) in this level's cells and
// the common start cell of all beams (OccGridMapBase.h:127-137).
struct BeamFrame {
  float c, s, mx, my;
  int x0, y0;
  bool ok;
};
__device__ __forceinline__ BeamFrame beam_frame(const HsbUpdateLevelDev& L, float wx, float wy, float wpsi) {
  BeamFrame f;
  const float* m = L.mtw;
  f.mx = __fadd_rn(__fmul_rn(m[0], wx), __fadd_rn(__fmul_rn(m[1], wy), m[2]));
  f.my = __fadd_rn(__fmul_rn(m[3], wx), __fadd_rn(__fmul_rn(m[4], wy), m[5]));
  f.c = cosf_glibc(wpsi);   // Rotation2Df, as glibc
  f.s = sinf_glibc(wpsi);
  // beam start = (int)(T * origo + 0.5)                                   (:134-137)
  const float ox = L.origo_x * L.pt_scale, oy = L.origo_y * L.pt_scale;
  const float bxf = __fadd_rn(__fmul_rn(f.c, ox), __fadd_rn(__fmul_rn(-f.s, oy), f.mx));
  const float byf = __fadd_rn(__fmul_rn(f.s, ox), __fadd_rn(__fmul_rn(f.c, oy), f.my));
  const float bxh = __fadd_rn(bxf, 0.5f), byh = __fadd_rn(byf, 0.5f);
  f.x0 = 0; f.y0 = 0;
  f.ok = (fabsf(bxh) < 1.0e9f) && (fabsf(byh) < 1.0e9f);   // non-finite / absurd pose: every beam is dropped
  if (f.ok) {
    f.x0 = (int)bxh; f.y0 = (int)byh;
    f.ok = !((f.x0 < 0) || (f.x0 >= L.sx) || (f.y0 < 0) || (f.y0 >= L.sy));   // :176 (same start for all beams)
  }
  return f;
}
// End cell of beam b; false when the reference drops the beam.
__device__ __forceinline__ bool beam_end(const HsbUpdateLevelDev& L, const BeamFrame& f, int b, int& x1, int& y1) {
  const float2 pt = L.pts[b];
  const float px = pt.x * L.pt_scale, py = pt.y * L.pt_scale;   // DataPointContainer.h:46-58 setFrom
  float exf = __fadd_rn(__fmul_rn(f.c, px), __fadd_rn(__fmul_rn(-f.s, py), f.mx));   // :148
  float eyf = __fadd_rn(__fmul_rn(f.s, px), __fadd_rn(__fmul_rn(f.c, py), f.my));
  exf = __fadd_rn(exf, 0.5f);                                                        // :152
  eyf = __fadd_rn(eyf, 0.5f);
  if (!(fabsf(exf) < 1.0e9f) || !(fabsf(eyf) < 1.0e9f)) return false;
  x1 = (int)exf; y1 = (int)eyf;                                                      // :155
  if (x1 == f.x0 && y1 == f.y0) return false;                                        // :158
  if ((x1 < 0) || (x1 >= L.sx) || (y1 < 0) || (y1 >= L.sy)) return false;            // :186
  return true;
}

// MARK: a team of TEAM warps per beam; blockIdx.y = level.  Team lanes stride along the line, four cells per
// lane in flight (the loop is bound by the L2 round trip of the stamp test, not by arithmetic); the stamps are raised
// with result-less atomics (RED.MAX: nothing waits for them).  The bounding box of the start cell and the beams' end
// cells goes to the scan's scratch slot (4 atomics per warp): the apply phase sweeps exactly that box and the dirty
// rectangles are fed from it.  (A variant that also compacted the first-marked cells into a list for the apply phase
// needs the atomics' return values — two more dependent L2 round trips per iteration — and made mark + apply slower;
// at a scan's size the box sweep is launch- and latency-sized, not bandwidth-sized.)
// Programmatic dependent launch (sm_90+): mark and apply are launched with programmatic stream serialisation, i.e.
// their CTAs may become resident while the previous kernel of the stream (the match kernel of a fused SLAM step, or
// mark before apply) is still running; griddepcontrol.wait blocks until that kernel has completed and its writes are
// visible.  Everything a kernel reads from its predecessor (pose, gate flag, stamps, lists) comes after the wait.
// This takes the launch latency of each dependent launch off the critical path of the single-scan step.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// One level of one scan's mark phase (blockIdx.x / gridDim.x stride over the beams); gate_flag / pose_dev as in
// HsbUpdateParams, pose_world the pose when pose_dev is null.
template <int TEAM>
__device__ __forceinline__ void mark_level(const HsbUpdateLevelDev& L, const float* gate_flag, const float* pose_dev,
                                           const float* pose_world) {
  if (!L.active) return;
  // gate flag, pose and beam count in ONE L2 round trip (independent loads, issued before the first dependent branch)
  // (plain loads: every thread reads these words, they have to hit L1)
  const float flag = gate_flag ? *gate_flag : 1.0f;
  const float* pw = pose_dev ? pose_dev : pose_world;
  const float wx = pw[0], wy = pw[1], wpsi = pw[2];
  const int n_dev = L.n_dev ? *L.n_dev : L.n;
  if (flag == 0.0f) return;
  constexpr int TL = 32 * TEAM;   // lanes per team
  constexpr int U = 4;
  const unsigned tlane = threadIdx.x % TL;
  const int team0 = (blockIdx.x * blockDim.x + threadIdx.x) / TL;
  const int team_stride = (gridDim.x * blockDim.x) / TL;
  const BeamFrame f = beam_frame(L, wx, wy, wpsi);
  if (!f.ok) return;
  const unsigned start = (unsigned)f.y0 * (unsigned)L.sx + (unsigned)f.x0;
  const uint32_t free_s = L.stamp_base + 1u, occ_s = L.stamp_base + 2u;
  int* slot = L.scratch + 8 * L.slot;
  int bx0 = INT_MAX, by0 = INT_MAX, bx1 = -1, by1 = -1;

  const int n_beams = min(n_dev, L.n);
  for (int b = team0; b < n_beams; b += team_stride) {
    int x1, y1;
    if (!beam_end(L, f, b, x1, y1)) continue;
    bx0 = min(bx0, x1); by0 = min(by0, y1); bx1 = max(bx1, x1); by1 = max(by1, y1);
    const int dx = x1 - f.x0, dy = y1 - f.y0;
    const unsigned adx = (unsigned)abs(dx), ady = (unsigned)abs(dy);
    const int off_dx = dx > 0 ? 1 : -1;                         // util::sign, UtilFunctions.h:56-59
    const int off_dy = (dy > 0 ? 1 : -1) * L.sx;
    unsigned ada, adb;
    int off_a, off_b;
    if (adx >= ady) { ada = adx; adb = ady; off_a = off_dx; off_b = off_dy; }   // :202-209
    else            { ada = ady; adb = adx; off_a = off_dy; off_b = off_dx; }
    const unsigned err0 = ada / 2u;
    // cell i (0 <= i < ada; start included, end excluded, :245-259): the serial walk adds adb per step and carries when
    // the error reaches ada, so after i steps it has carried q(i) = floor((err0 + i*adb) / ada) times.  A lane visits
    // i = tlane, tlane + TL, ...: q and the remainder r are advanced by the constant step (TL*adb = qT*ada + rT) —
    // two divisions per lane and beam instead of one per cell.
    unsigned q, r, qT, rT;
    if (ada < 32768u) {   // err0 + i*adb and TL*adb fit 32 bits
      const unsigned n0 = err0 + tlane * adb, nT = (unsigned)TL * adb;
      q = n0 / ada; r = n0 - q * ada;
      qT = nT / ada; rT = nT - qT * ada;
    } else {
      const unsigned long long n0 = (unsigned long long)err0 + (unsigned long long)tlane * adb, nT = (unsigned long long)TL * adb;
      q = (unsigned)(n0 / ada); r = (unsigned)(n0 - (unsigned long long)q * ada);
      qT = (unsigned)(nT / ada); rT = (unsigned)(nT - (unsigned long long)qT * ada);
    }
    for (unsigned i0 = tlane; i0 < ada; i0 += U * TL) {
      unsigned off[U];
      uint32_t v[U];
#pragma unroll
      for (int k = 0; k < U; ++k) {
        const unsigned i = i0 + (unsigned)(k * TL);
        v[k] = 0xffffffffu;
        if (i < ada) {
          off[k] = start + (unsigned)((int)i * off_a) + (unsigned)((int)q * off_b);
          v[k] = __ldcg(L.stamp + off[k]);
        }
        q += qT;
        r += rT;
        if (r >= ada) { r -= ada; ++q; }
      }
#pragma unroll
      for (int k = 0; k < U; ++k)
        if (v[k] < free_s) atomicMax(L.stamp + off[k], free_s);   // bresenhamCellFree :216-224
    }
    if (tlane == 0) atomicMax(L.stamp + (unsigned)y1 * (unsigned)L.sx + (unsigned)x1, occ_s);   // bresenhamCellOcc :226-241, :211-212
  }
  // bounding box of this CTA's beams (+ the common start cell) -> scratch slot.  One reduction per CTA and only the
  // atomics that can still enlarge the box: with 4 atomics per WARP (thousands of warps on the same four words) the drain of
  // the same-address atomics dominates the kernel.
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    bx0 = min(bx0, __shfl_xor_sync(0xffffffffu, bx0, o));
    by0 = min(by0, __shfl_xor_sync(0xffffffffu, by0, o));
    bx1 = max(bx1, __shfl_xor_sync(0xffffffffu, bx1, o));
    by1 = max(by1, __shfl_xor_sync(0xffffffffu, by1, o));
  }
  __shared__ int box[4][8];
  const int wi = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { box[0][wi] = bx0; box[1][wi] = by0; box[2][wi] = bx1; box[3][wi] = by1; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < 8; ++k) {
      bx0 = min(bx0, box[0][k]); by0 = min(by0, box[1][k]); bx1 = max(bx1, box[2][k]); by1 = max(by1, box[3][k]);
    }
    if (bx1 >= 0) {
      bx0 = min(bx0, f.x0); by0 = min(by0, f.y0); bx1 = max(bx1, f.x0); by1 = max(by1, f.y0);
      // the four current bounds in ONE L2 round trip (a stale value only costs an atomic that changes nothing; read one
      // by one through a volatile pointer they were four dependent round trips at the end of every CTA)
      const int c1 = __ldcg(slot + 1), c2 = __ldcg(slot + 2), c3 = __ldcg(slot + 3), c4 = __ldcg(slot + 4);
      if (bx0 < c1) atomicMin(slot + 1, bx0);
      if (by0 < c2) atomicMin(slot + 2, by0);
      if (bx1 > c3) atomicMax(slot + 3, bx1);
      if (by1 > c4) atomicMax(slot + 4, by1);
    }
  }
}

template <int TEAM>
__global__ void __launch_bounds__(256) update_mark_kernel(const __grid_constant__ HsbUpdateParams P) {
  pdl_launch_dependents();   // the apply kernel's CTAs may take the free slots now; they wait for this grid to finish
  pdl_wait();
  mark_level<TEAM>(P.lv[blockIdx.y], P.gate_flag, P.pose_dev, P.pose_world);
}

// Group SLAM step: the mark phase of every session's every level in one launch (blockIdx.z = session, blockIdx.y =
// level); each session's pose and write flag come from the group match kernel's gate.
template <int TEAM>
__global__ void __launch_bounds__(256) update_mark_group_kernel(const __grid_constant__ HsbGroupUpdateParams P) {
  pdl_launch_dependents();
  pdl_wait();
  const float* res = P.res + 4 * blockIdx.z;
  mark_level<TEAM>(P.lv[(size_t)blockIdx.z * P.levels + blockIdx.y], res + 3, res, res);
}

// APPLY: every marked cell lies in the bounding box of the start cell and the end cells, which the mark phase left in
// the scan's scratch slot, so the apply phase is a coalesced sweep of that box over the stamp plane (uint4 loads, four
// in flight per thread; a scalar variant for levels whose rows are not 16-byte multiples): stamp == base+1 -> l += lf,
// base+2 -> if (l < 50) l += lo, then P and the texture twin are rewritten.  One owner per cell by construction — no
// atomics, deterministic.
__device__ __forceinline__ void apply_cell(const HsbUpdateLevelDev& L, unsigned off, uint32_t v, float lf, float lo) {
  const uint32_t d = v - (L.stamp_base + 1u);
  if (d < 2u) {
    float l = L.logodds[off];
    if (d == 0u) {
      l = __fadd_rn(l, lf);                       // updateSetFree, GridMapLogOdds.h:146-151
    } else if (l < 50.0f) {
      l = __fadd_rn(l, lo);                       // updateSetOccupied, GridMapLogOdds.h:135-140
    }
    L.logodds[off] = l;
    const float p = prob_from_logodds(l);
    L.prob[off] = p;
    if (L.surf) {
      const int y = (int)(off / (unsigned)L.sx), x = (int)(off - (unsigned)y * (unsigned)L.sx);
      surf2Dwrite(p, L.surf, x * (int)sizeof(float), y);
    }
  }
}

// One level of one scan's apply phase (blockIdx.x / gridDim.x sweep the box); lf / lo the log-odds increments.
__device__ __forceinline__ void apply_level(const HsbUpdateLevelDev& L, const float* gate_flag, float lf, float lo) {
  if (!L.active) return;
  const int* cur = L.scratch + 8 * L.slot;
  if (blockIdx.x == 0 && threadIdx.x == 0) {   // the other slot is the next scan's: clear it (nobody reads it now)
    int* nxt = L.scratch + 8 * (L.slot ^ 1);
    nxt[0] = 0;
    nxt[1] = INT_MAX; nxt[2] = INT_MAX; nxt[3] = -1; nxt[4] = -1;
  }
  // gate flag and box in ONE round trip (independent loads, issued before the first dependent branch; plain loads:
  // every thread of the grid reads these words, they have to hit L1 — ld.cg here hot-spots one L2 sector)
  const float flag = gate_flag ? *gate_flag : 1.0f;
  const int bx0 = cur[1], by0 = cur[2], bx1 = cur[3], by1 = cur[4];
  if (flag == 0.0f) return;
  if (bx1 < bx0) return;                       // nothing was marked (pose outside the map, every beam dropped)
  if (blockIdx.x == 0 && threadIdx.x == 0 && L.dirty) {   // both rectangles: replication [0..3] and host mirror [4..7]
    atomicMin(L.dirty + 0, bx0); atomicMin(L.dirty + 4, bx0);
    atomicMin(L.dirty + 1, by0); atomicMin(L.dirty + 5, by0);
    atomicMax(L.dirty + 2, bx1); atomicMax(L.dirty + 6, bx1);
    atomicMax(L.dirty + 3, by1); atomicMax(L.dirty + 7, by1);
  }
  const unsigned nthreads = gridDim.x * blockDim.x, tid = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned rows = (unsigned)(by1 - by0 + 1);
  constexpr int U = 4;
  if ((L.sx & 3) == 0) {   // rows are 16-byte aligned: four cells per load
    const unsigned xa = (unsigned)bx0 & ~3u;
    const unsigned w4 = (((unsigned)bx1 - xa) >> 2) + 1u;
    const unsigned total = w4 * rows;
    for (unsigned base = tid; base < total; base += U * nthreads) {
      unsigned off[U];
      uint4 v[U];
#pragma unroll
      for (int k = 0; k < U; ++k) {
        const unsigned idx = base + (unsigned)k * nthreads;
        v[k] = make_uint4(L.stamp_base, L.stamp_base, L.stamp_base, L.stamp_base);
        if (idx < total) {
          const unsigned r = idx / w4, c = idx - r * w4;
          off[k] = ((unsigned)by0 + r) * (unsigned)L.sx + xa + 4u * c;
          v[k] = __ldcg(reinterpret_cast<const uint4*>(L.stamp + off[k]));
        }
      }
#pragma unroll
      for (int k = 0; k < U; ++k) {
        apply_cell(L, off[k] + 0u, v[k].x, lf, lo);
        apply_cell(L, off[k] + 1u, v[k].y, lf, lo);
        apply_cell(L, off[k] + 2u, v[k].z, lf, lo);
        apply_cell(L, off[k] + 3u, v[k].w, lf, lo);
      }
    }
  } else {
    const unsigned wd = (unsigned)(bx1 - bx0 + 1);
    const unsigned total = wd * rows;
    for (unsigned idx = tid; idx < total; idx += nthreads) {
      const unsigned rr = idx / wd, c = idx - rr * wd;
      const unsigned off = ((unsigned)by0 + rr) * (unsigned)L.sx + (unsigned)bx0 + c;
      apply_cell(L, off, __ldcg(L.stamp + off), lf, lo);
    }
  }
}

__global__ void __launch_bounds__(256) update_apply_kernel(const __grid_constant__ HsbUpdateParams P) {
  pdl_wait();
  apply_level(P.lv[blockIdx.y], P.gate_flag, P.log_odds_free, P.log_odds_occ);
}

// Group SLAM step: every session's every level (blockIdx.z = session, blockIdx.y = level) with that member's
// increments; one owner per cell as above (a session writes only its own member's planes).
__global__ void __launch_bounds__(256) update_apply_group_kernel(const __grid_constant__ HsbGroupUpdateParams P) {
  pdl_wait();
  const float2 lo = P.log_odds[blockIdx.z];
  apply_level(P.lv[(size_t)blockIdx.z * P.levels + blockIdx.y], P.res + 4 * blockIdx.z + 3, lo.x, lo.y);
}

// Dirty-rectangle transport: pack the log-odds of rect = {x0, y0, x1, y1} (inclusive) row by row
// into a contiguous buffer / write such a buffer back and refresh P (and the texture twin) there.
__global__ void pack_rect_kernel(const float* __restrict__ logodds, int sx, int x0, int y0, int w, int hgt,
                                 float* __restrict__ buf) {
  const size_t n = (size_t)w * hgt;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / (size_t)w), c = (int)(i - (size_t)r * w);
    buf[i] = logodds[(size_t)(y0 + r) * sx + (x0 + c)];
  }
}
// (a replica's host mirror has to follow too: the rectangle is folded into the level's mirror rectangle)
__global__ void unpack_rect_kernel(float* __restrict__ logodds, float* __restrict__ prob, cudaSurfaceObject_t surf, int sx,
                                   int x0, int y0, int w, int hgt, const float* __restrict__ buf, int* mirror_dirty) {
  const size_t n = (size_t)w * hgt;
  if (mirror_dirty && blockIdx.x == 0 && threadIdx.x == 0) {
    atomicMin(mirror_dirty + 0, x0);
    atomicMin(mirror_dirty + 1, y0);
    atomicMax(mirror_dirty + 2, x0 + w - 1);
    atomicMax(mirror_dirty + 3, y0 + hgt - 1);
  }
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / (size_t)w), c = (int)(i - (size_t)r * w);
    const size_t off = (size_t)(y0 + r) * sx + (x0 + c);
    const float l = buf[i];
    logodds[off] = l;
    const float p = prob_from_logodds(l);
    prob[off] = p;
    if (surf) surf2Dwrite(p, surf, (x0 + c) * (int)sizeof(float), y0 + r);
  }
}


// ---- one-shot tile transport: everything the host-synchronous protocol asked the host for stays on the device ----
// The owner's pack kernel reads the dirty rectangles of all levels from device memory, writes them into the buffer's
// header and the rectangles' log-odds rows behind it; the replicas' unpack kernel reads the header from the buffer the
// collective delivered.  No size ever travels through a host, so the whole replication step is stream-ordered: pack ->
// ONE fixed-size ncclBroadcast -> unpack (DESIGN.md §6).
//
// One body serves a single handle and a group (hsb_group_pack_dirty_device / hsb_group_unpack_dirty_device).  It walks
// a table of blocks, one per session: the block's member, its level descriptors (P.table's member-major row, or the
// single handle's P.lv) and the word where the block starts.  A single handle's buffer is one block at word 0 and no
// group header.  Sessions are laid out kTileChunk at a time in shared memory (every CTA lays out every chunk: the
// layout of a block depends on all blocks before it), then the chunk's rows go one warp per row over the grid.

constexpr int kTileChunk = 128;   // sessions laid out per pass (threads 0 .. kTileChunk-1 of the 256-thread CTA)

struct TileChunk {
  int4 rect[kTileChunk][HSB_MAX_LEVELS];   // the block's rectangles {x0, y0, x1, y1} (x1 < x0: clean)
  unsigned long long start[kTileChunk];    // the block's first word in the buffer (its HSB_TILE_* header)
  unsigned long long cells[kTileChunk];    // the block's row words (cells of all its rectangles)
  unsigned row0[kTileChunk + 1];           // shipped rows of the chunk before the block's; row0[n]: all of them
  int member[kTileChunk];
  int ship[kTileChunk];                    // 1: rows shipped, 0: deferred
  unsigned cleared[kTileChunk];            // the block's clear record (HSB_TILE_CLEARED_WORD; unpack: shipped blocks only)
};

__device__ __forceinline__ bool tile_dirty(int4 r) { return r.z >= r.x && r.w >= r.y; }
// a rectangle's width / height as 64-bit counts (a foreign buffer's rectangles may be anything)
__device__ __forceinline__ long long tile_w(int4 r) { return tile_dirty(r) ? (long long)r.z - r.x + 1 : 0; }
__device__ __forceinline__ long long tile_h(int4 r) { return tile_dirty(r) ? (long long)r.w - r.y + 1 : 0; }

__device__ __forceinline__ const HsbTileLevelDev* tile_levels(const HsbTileParams& P, int member) {
  return P.table ? P.table + (size_t)member * P.levels : P.lv;
}
// How many levels a block's member has: the launch's (P.levels: a single handle), or — a group, whose members may each
// have their own — its entry of hsb_group::d_member_levels.  A member's rows of the group's table past its own levels
// are never read.
struct TileLevelsSingle {};
struct TileLevelsMember {
  const int* n;
};
// member m's level count; `single` is the launch's (P.levels, or a copy of it the body already holds)
__device__ __forceinline__ int tile_member_levels(TileLevelsSingle, int single, int) { return single; }
__device__ __forceinline__ int tile_member_levels(const TileLevelsMember& LV, int, int m) { return LV.n[m]; }
// whether level l lies past member m's levels (never, for a single handle)
__device__ __forceinline__ bool tile_level_past(TileLevelsSingle, int, int) { return false; }
__device__ __forceinline__ bool tile_level_past(const TileLevelsMember& LV, int m, int l) { return l >= LV.n[m]; }

// where a block's deferral is counted: its member's overflow counter (a single handle: its own)
__device__ __forceinline__ int* tile_counter(const HsbTileParams& P, int member) {
  return P.table ? P.counters[member] : P.error_count;
}

// Warp 0: row0[1 .. n] hold each block's row count; turned into the exclusive prefix row0[0 .. n].
__device__ __forceinline__ void tile_row_prefix(TileChunk& c, int n) {
  const int lane = threadIdx.x;
  unsigned carry = 0;
  for (int b = 0; b < n; b += 32) {
    unsigned v = b + lane < n ? c.row0[b + lane + 1] : 0u;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned y = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += y;
    }
    if (b + lane < n) c.row0[b + lane + 1] = carry + v;
    carry += __shfl_sync(0xffffffffu, v, 31);
  }
  if (lane == 0) c.row0[0] = 0u;
}

// The chunk's rows, one warp per row: row r belongs to the block whose rows [row0[j], row0[j+1]) hold it (blocks
// without rows are passed over), then to the first of its dirty levels that still has rows left.  kPack: plane -> buffer;
// otherwise buffer -> plane, probability and texture twin, with the per-cell bounds guard (a foreign geometry must not
// write out of bounds).
template <bool kPack>
__device__ __forceinline__ void tile_rows(const HsbTileParams& P, const TileChunk& c, int n) {
  const int lane = threadIdx.x & 31;
  const unsigned total = c.row0[n];
  const unsigned nwarps = (gridDim.x * blockDim.x) >> 5;
  for (unsigned r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < total; r += nwarps) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (c.row0[mid] <= r) lo = mid;
      else hi = mid - 1;
    }
    unsigned long long off = c.start[lo] + HSB_TILE_HEADER_WORDS;
    long long rr = r - c.row0[lo];
    int l = 0;
    int4 q = c.rect[lo][0];
    for (;; ++l) {
      q = c.rect[lo][l];
      const long long h = tile_h(q);
      if (rr < h) break;
      rr -= h;
      off += (unsigned long long)(tile_w(q) * h);
    }
    const long long w = tile_w(q);
    off += (unsigned long long)(rr * w);
    const HsbTileLevelDev L = tile_levels(P, c.member[lo])[l];
    const int y = q.y + (int)rr;
    if (kPack) {
      const float* src = L.logodds + (size_t)y * L.sx + q.x;
      for (int x = lane; x < w; x += 32) P.buf[off + x] = src[x];
    } else {
      if (y < 0 || y >= L.sy) continue;
      for (int x = lane; x < w; x += 32) {
        const int cx = q.x + x;
        if (cx < 0 || cx >= L.sx) continue;
        const size_t o = (size_t)y * L.sx + cx;
        const float v = P.buf[off + x];
        L.logodds[o] = v;
        const float p = prob_from_logodds(v);
        L.prob[o] = p;
        if (L.surf) surf2Dwrite(p, L.surf, cx * (int)sizeof(float), y);
      }
    }
  }
}

// The sessions of a pack: a single handle (one block, member 0), every member of a group in order, or a subset listed
// in the launch's parameters (N sessions at most).
struct TileSingle {
  __device__ int member(int) const { return 0; }
};
struct TileAll {
  __device__ int member(int k) const { return k; }
};
template <int N>
struct TileMembers {
  int idx[N];
  __device__ int member(int k) const { return idx[k]; }
};

// Pack: each session's block header, first-fit placement of its rows in session order (a block whose rows do not fit
// behind those already placed is deferred: overflow = 1, no rows), the rows, and for a group the group header.
template <class Sessions, class Levels>
__device__ __forceinline__ void pack_dirty_body(const HsbTileParams& P, const Sessions& S, const Levels& LV) {
  __shared__ TileChunk c;
  __shared__ unsigned long long s_used;   // row words placed before the current chunk
  __shared__ int s_deferred;
  const int K = P.K, levels = P.levels;
  const bool group = P.table != nullptr;
  const unsigned long long G = group ? hsb_tile_group_header_words(K) : 0ull;
  const unsigned long long room = P.capacity_words - G - (unsigned long long)HSB_TILE_HEADER_WORDS * K;
  if (threadIdx.x == 0) { s_used = 0ull; s_deferred = 0; }
  for (int k0 = 0; k0 < K; k0 += kTileChunk) {
    const int n = min(kTileChunk, K - k0);
    const int j = threadIdx.x;
    if (j < n) {
      const int m = S.member(k0 + j);
      const HsbTileLevelDev* lv = tile_levels(P, m);
      unsigned long long cells = 0;
      unsigned rows = 0, cleared = 0;
      const int nl = tile_member_levels(LV, levels, m);
      for (int l = 0; l < nl; ++l) {
        const int* d = lv[l].dirty;
        const int4 q = make_int4(d[0], d[1], d[2], d[3]);
        c.rect[j][l] = q;
        cells += (unsigned long long)(tile_w(q) * tile_h(q));
        rows += (unsigned)tile_h(q);
        if (d[HSB_DIRTY_CLEARED]) cleared |= 1u << l;
      }
      c.member[j] = m;
      c.cleared[j] = cleared;
      c.cells[j] = cells;
      c.row0[j + 1] = rows;
    }
    __syncthreads();
    if (threadIdx.x < 32) {   // first fit, 32 sessions at a time: ship the run of blocks that fits, defer the first that
      const int lane = threadIdx.x;   // does not, repeat with the rest
      unsigned long long used = s_used;
      int deferred = 0;
      for (int b = 0; b < n; b += 32) {
        const int jj = b + lane;
        const unsigned long long cj = jj < n ? c.cells[jj] : 0ull;
        const unsigned long long base = G + (unsigned long long)HSB_TILE_HEADER_WORDS * (k0 + jj);
        unsigned pending = __ballot_sync(0xffffffffu, jj < n);
        while (pending) {
          const bool mine = (pending >> lane) & 1u;
          unsigned long long x = mine ? cj : 0ull;
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
          }
          const unsigned over = __ballot_sync(0xffffffffu, mine && used + x > room);
          const unsigned ship = pending & (over ? (over & (0u - over)) - 1u : 0xffffffffu);
          if ((ship >> lane) & 1u) { c.start[jj] = base + used + x - cj; c.ship[jj] = 1; }
          const unsigned long long placed = ship ? __shfl_sync(0xffffffffu, x, 31 - __clz(ship)) : 0ull;
          pending &= ~ship;
          if (over) {
            const int f = __ffs(over) - 1;
            if (lane == f) { c.start[jj] = base + used + placed; c.ship[jj] = 0; c.row0[jj + 1] = 0u; }
            pending &= ~(1u << f);
            ++deferred;
          }
          used += placed;
        }
      }
      __syncwarp();
      tile_row_prefix(c, n);
      if (lane == 0) { s_used = used; s_deferred += deferred; }
    }
    __syncthreads();
    if (blockIdx.x == 0 && j < n) {   // the block's header, exactly hsb_pack_dirty_device's for this member alone
      int* hdr = reinterpret_cast<int*>(P.buf + c.start[j]);
      const int nl = tile_member_levels(LV, levels, c.member[j]);
      hdr[0] = HSB_TILE_MAGIC; hdr[1] = nl; hdr[2] = c.ship[j] ? 0 : 1; hdr[3] = (int)c.cells[j];
      for (int l = 0; l < nl; ++l) {
        const int4 q = c.rect[j][l];
        hdr[4 + 4 * l] = q.x; hdr[5 + 4 * l] = q.y; hdr[6 + 4 * l] = q.z; hdr[7 + 4 * l] = q.w;
      }
      hdr[HSB_TILE_CLEARED_WORD] = (int)c.cleared[j];
      if (group) {
        int* gh = reinterpret_cast<int*>(P.buf);
        gh[HSB_TILE_GROUP_FIXED_WORDS + 2 * (k0 + j)] = c.member[j];
        gh[HSB_TILE_GROUP_FIXED_WORDS + 2 * (k0 + j) + 1] = (int)(unsigned)c.start[j];
      }
    }
    tile_rows<true>(P, c, n);
    __syncthreads();   // the next chunk reuses c
  }
  if (group && blockIdx.x == 0 && threadIdx.x == 0) {
    int* gh = reinterpret_cast<int*>(P.buf);
    gh[0] = HSB_TILE_GROUP_MAGIC; gh[1] = K; gh[2] = levels; gh[3] = s_deferred;
    gh[4] = (int)(unsigned)(G + (unsigned long long)HSB_TILE_HEADER_WORDS * K + s_used);
    for (unsigned long long w = HSB_TILE_GROUP_FIXED_WORDS + 2ull * K; w < G; ++w) gh[w] = 0;
  }
}

__global__ void __launch_bounds__(256) pack_dirty_kernel(const __grid_constant__ HsbTileParams P) {
  pack_dirty_body(P, TileSingle(), TileLevelsSingle());
}
// a group: every block carries its member's own levels (header word 1, exactly hsb_pack_dirty_device's block), the
// group header the group's largest count (P.levels)
__global__ void __launch_bounds__(256) pack_dirty_group_kernel(const __grid_constant__ HsbTileParams P,
                                                               const int* __restrict__ member_levels) {
  pack_dirty_body(P, TileAll(), TileLevelsMember{member_levels});
}
template <int N>
__global__ void __launch_bounds__(256) pack_dirty_subset_kernel(const __grid_constant__ HsbTileParams P,
                                                                const __grid_constant__ TileMembers<N> S,
                                                                const int* __restrict__ member_levels) {
  pack_dirty_body(P, S, TileLevelsMember{member_levels});
}

// after pack (stream order): the shipped blocks' rectangles and cleared flags are forgotten, a deferred block's are kept.
// One thread per (block, level, coordinate); the block's member and start come from the group header (a single handle:
// member 0, 0).
template <class Levels>
__device__ __forceinline__ void reset_dirty_body(const HsbTileParams& P, const Levels& LV) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int per = 4 * P.levels, k = i / per;
  if (k >= P.K) return;
  const int* gh = reinterpret_cast<const int*>(P.buf);
  const int member = P.table ? gh[HSB_TILE_GROUP_FIXED_WORDS + 2 * k] : 0;
  const unsigned long long start = P.table ? (unsigned)gh[HSB_TILE_GROUP_FIXED_WORDS + 2 * k + 1] : 0u;
  if (reinterpret_cast<const int*>(P.buf + start)[2] != 0) return;
  const int l = (i - k * per) >> 2, q = i & 3;
  if (tile_level_past(LV, member, l)) return;   // (a level past the member's own: nothing there)
  int* d = tile_levels(P, member)[l].dirty;
  d[q] = (q < 2) ? INT_MAX : -1;
  if (q == 0) d[HSB_DIRTY_CLEARED] = 0;
}
__global__ void reset_dirty_kernel(const __grid_constant__ HsbTileParams P) {
  reset_dirty_body(P, TileLevelsSingle());
}
__global__ void reset_dirty_group_kernel(const __grid_constant__ HsbTileParams P, const int* __restrict__ member_levels) {
  reset_dirty_body(P, TileLevelsMember{member_levels});
}

// hsb_group_reset: hsb_reset's end state for every level of K members in one launch — log-odds 0, P 0.5, texture twin
// 0.5 and stamps 0 over every plane (blockIdx.y = session; blockIdx.x strides over each of the member's levels in turn,
// so every CTA of the launch clears the same share of a member and none idles while a level-0 plane finishes), then, by
// thread l of the session's first CTA, level l's mirror rectangle := the whole level, its replication rectangle clean and
// its cleared flag set (the next pack ships the clear record instead of the whole level), and by thread 0 the gate
// state := lastMapUpdatePose FLT_MAX^3, write flag 0 (HectorSlamProcessor.h:117).
template <class Sessions, class Levels>
__device__ __forceinline__ void group_reset_body(const HsbResetParams& P, const Sessions& S, const Levels& LV) {
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, nthreads = (size_t)gridDim.x * blockDim.x;
  for (int k = blockIdx.y; k < P.K; k += gridDim.y) {
    const int m = S.member(k);
    const HsbTileLevelDev* lv = P.table + (size_t)m * P.levels;
    for (int l = 0; l < tile_member_levels(LV, P.levels, m); ++l) {
      const HsbTileLevelDev L = lv[l];
      uint32_t* stamp = P.mem[m].stamp[l];
      const size_t n = (size_t)L.sx * (size_t)L.sy;
      for (size_t i = tid; i < n; i += nthreads) {
        clear_cell(L.logodds, L.prob, L.surf, L.sx, i);
        stamp[i] = 0u;
      }
    }
    if (blockIdx.x == 0 && threadIdx.x < tile_member_levels(LV, P.levels, m)) {
      const HsbTileLevelDev L = lv[threadIdx.x];
      int* d = L.dirty;
      d[0] = INT_MAX; d[1] = INT_MAX; d[2] = -1; d[3] = -1;
      d[4] = 0; d[5] = 0; d[6] = L.sx - 1; d[7] = L.sy - 1;
      d[HSB_DIRTY_CLEARED] = 1;
      if (threadIdx.x == 0) {
        float* g = P.mem[m].gate;
        g[0] = FLT_MAX; g[1] = FLT_MAX; g[2] = FLT_MAX; g[3] = 0.0f;
      }
    }
  }
}
// each member's own levels only
__global__ void __launch_bounds__(256) group_reset_kernel(const __grid_constant__ HsbResetParams P,
                                                          const int* __restrict__ member_levels) {
  group_reset_body(P, TileAll(), TileLevelsMember{member_levels});
}
template <int N>
__global__ void __launch_bounds__(256) group_reset_subset_kernel(const __grid_constant__ HsbResetParams P,
                                                                 const __grid_constant__ TileMembers<N> S,
                                                                 const int* __restrict__ member_levels) {
  group_reset_body(P, S, TileLevelsMember{member_levels});
}

// Unpack, pass 1: the buffer fits the replica (group header and every block's header inside the capacity, every shipped
// block's rows too, and every shipped rectangle inside its level of the member it lands on), evaluated identically by
// every CTA.  Reads block j of the chunk into c (rectangles, start, member, ship, cells).  A deferred block carries no
// rows: its rectangles may be larger than the whole buffer (that is why it was deferred) and are not checked.  The
// level-size check keeps a block packed on a member of another size (an owner group listing its handles in another
// order than a mixed replica group) from growing a mirror rectangle past the plane it lands on.
template <class Levels>
__device__ __forceinline__ bool tile_read_block(const HsbTileParams& P, const Levels& LV, TileChunk& c, int k, int j) {
  const int* gh = reinterpret_cast<const int*>(P.buf);
  int member = 0;
  unsigned long long start = 0;
  if (P.table) {
    member = gh[HSB_TILE_GROUP_FIXED_WORDS + 2 * k];
    start = (unsigned)gh[HSB_TILE_GROUP_FIXED_WORDS + 2 * k + 1];
    if (member < 0 || member >= P.M) return false;
  }
  if (start + HSB_TILE_HEADER_WORDS > P.capacity_words) return false;
  const int* hdr = reinterpret_cast<const int*>(P.buf + start);
  if (hdr[0] != HSB_TILE_MAGIC || hdr[1] != tile_member_levels(LV, P.levels, member)) return false;
  const bool ship = hdr[2] == 0;
  const unsigned cleared = (unsigned)hdr[HSB_TILE_CLEARED_WORD];
  if (cleared >> tile_member_levels(LV, P.levels, member)) return false;   // a cleared level the replica does not have
  const HsbTileLevelDev* lv = tile_levels(P, member);
  unsigned long long cells = 0;
  unsigned rows = 0;
  for (int l = 0; l < tile_member_levels(LV, P.levels, member); ++l) {
    const int4 q = make_int4(hdr[4 + 4 * l], hdr[5 + 4 * l], hdr[6 + 4 * l], hdr[7 + 4 * l]);
    c.rect[j][l] = q;
    if (!ship) continue;
    if (tile_dirty(q) && (q.x < 0 || q.y < 0 || q.z >= lv[l].sx || q.w >= lv[l].sy)) return false;
    const long long w = tile_w(q), h = tile_h(q);
    if (w > P.capacity_words || h > P.capacity_words) return false;   // (keeps w * h and the sums below in 64 bits)
    cells += (unsigned long long)(w * h);
    rows += (unsigned)h;
  }
  if (ship && start + HSB_TILE_HEADER_WORDS + cells > P.capacity_words) return false;
  c.start[j] = start;
  c.cells[j] = cells;
  c.member[j] = member;
  c.ship[j] = ship ? 1 : 0;
  c.cleared[j] = ship ? cleared : 0u;
  c.row0[j + 1] = ship ? rows : 0u;
  return true;
}

// Unpack's clear record: every cell of a cleared level outside the block's shipped rectangle is reset (log-odds 0, P
// 0.5, texture twin 0.5), grid-stride over the plane.  Disjoint from the cells tile_rows writes, so both run in the one
// unpack launch in any order.
__device__ __forceinline__ void tile_clear(const HsbTileParams& P, const TileChunk& c, int n) {
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, nthreads = (size_t)gridDim.x * blockDim.x;
  for (int j = 0; j < n; ++j) {
    const unsigned cleared = c.cleared[j];
    if (!cleared) continue;
    const HsbTileLevelDev* lv = tile_levels(P, c.member[j]);
    for (int l = 0; l < P.levels; ++l) {
      if (!((cleared >> l) & 1u)) continue;
      const HsbTileLevelDev L = lv[l];
      const int4 q = c.rect[j][l];
      const bool inside_any = tile_dirty(q);
      const size_t cells = (size_t)L.sx * (size_t)L.sy;
      for (size_t i = tid; i < cells; i += nthreads) {
        const int y = (int)(i / (size_t)L.sx), x = (int)(i - (size_t)y * L.sx);
        if (inside_any && x >= q.x && x <= q.z && y >= q.y && y <= q.w) continue;
        clear_cell(L.logodds, L.prob, L.surf, L.sx, i);
      }
    }
  }
}

template <class Levels>
__device__ __forceinline__ void unpack_dirty_body(const HsbTileParams& P, const Levels& LV) {
  __shared__ TileChunk c;
  const int* gh = reinterpret_cast<const int*>(P.buf);
  int K = 1;
  bool fits = true;
  if (P.table) {
    fits = P.capacity_words >= HSB_TILE_GROUP_FIXED_WORDS && gh[0] == HSB_TILE_GROUP_MAGIC && gh[2] == P.levels &&
           gh[1] >= 0 && gh[1] <= P.M;
    if (fits) {
      K = gh[1];
      fits = hsb_tile_group_header_words(K) <= P.capacity_words;
    }
  }
  for (int k0 = 0; fits && k0 < K; k0 += kTileChunk) {
    const int j = threadIdx.x, n = min(kTileChunk, K - k0);
    const bool ok = j >= n || tile_read_block(P, LV, c, k0 + j, j);
    fits = __syncthreads_and(ok);
  }
  if (!fits) {   // nothing from a buffer that does not fit is applied; counted once on handles[0]
    if (blockIdx.x == 0 && threadIdx.x == 0 && P.error_count) atomicAdd(P.error_count, 1);
    return;
  }
  for (int k0 = 0; k0 < K; k0 += kTileChunk) {
    const int j = threadIdx.x, n = min(kTileChunk, K - k0);
    if (j < n) tile_read_block(P, LV, c, k0 + j, j);
    const bool any_cleared = __syncthreads_or(j < n && c.cleared[j] != 0u);
    if (threadIdx.x < 32) tile_row_prefix(c, n);
    if (blockIdx.x == 0 && j < n) {
      const int m = c.member[j];
      if (!c.ship[j]) {   // a deferred block: counted once on its member's counter
        int* cnt = tile_counter(P, m);
        if (cnt) atomicAdd(cnt, 1);
      } else {            // the replica's host mirror has to follow (a cleared level: all of it)
        const HsbTileLevelDev* lv = tile_levels(P, m);
        for (int l = 0; l < tile_member_levels(LV, P.levels, m); ++l) {
          const int4 q = (c.cleared[j] >> l) & 1u ? make_int4(0, 0, lv[l].sx - 1, lv[l].sy - 1) : c.rect[j][l];
          if (!tile_dirty(q)) continue;
          int* md = lv[l].dirty + 4;
          atomicMin(md + 0, q.x); atomicMin(md + 1, q.y);
          atomicMax(md + 2, q.z); atomicMax(md + 3, q.w);
        }
      }
    }
    __syncthreads();
    tile_rows<false>(P, c, n);
    if (any_cleared) tile_clear(P, c, n);
    __syncthreads();
  }
}

__global__ void __launch_bounds__(256) unpack_dirty_kernel(const __grid_constant__ HsbTileParams P) {
  unpack_dirty_body(P, TileLevelsSingle());
}
// a group: a block must carry exactly its member's level count; a block whose count differs does not fit, like a
// rectangle outside its level
__global__ void __launch_bounds__(256) unpack_dirty_group_kernel(const __grid_constant__ HsbTileParams P,
                                                                 const int* __restrict__ member_levels) {
  unpack_dirty_body(P, TileLevelsMember{member_levels});
}

}  // namespace hsb
#endif
