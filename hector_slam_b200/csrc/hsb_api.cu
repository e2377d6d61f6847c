// hsb_api.cu — implementation of the C-ABI in include/hector_slam_b200.h on top of the sm_90a
// kernels in match_kernel.cuh / update_kernel.cuh.  No torch types, no CPU fallback: every entry
// point that computes something launches a CUDA kernel or fails with an error code.
#include <algorithm>
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "hsb_internal.h"
#include "match_kernel.cuh"
#include "update_kernel.cuh"

namespace {

struct Level {
  int sx = 0, sy = 0;
  float cell_length = 0.f, scale = 0.f;
  float mtw[6] = {0}, wtm[6] = {0};
  float* logodds = nullptr;
  float* prob = nullptr;
  uint32_t* stamp = nullptr;
  uint32_t stamp_base = 0;
  int* scratch = nullptr;      // two slots of 8 ints for the two-phase writer (see HsbUpdateLevelDev)
  int parity = 0;              // slot the NEXT map write of this level uses
  cudaArray_t arr = nullptr;
  cudaTextureObject_t tex = 0;
  cudaSurfaceObject_t surf = 0;
  int evals = 0;
  int* dirty = nullptr;  // device: two rectangles {xmin, ymin, xmax, ymax} of cells written since their last reset —
                         // [0..3] for replication (hsb_get_dirty_rect), [4..7] for host mirrors (hsb_get_mirror_dirty_rect);
                         // points into hsb_handle::d_dirty_all
};

struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
};

struct BatchSet {
  DevBuf hints, in, offsets, poses, cov, origo, tf;
  cudaEvent_t chunk_ready[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  cudaEvent_t done[2] = {nullptr, nullptr};
  bool busy = false;
};

}  // namespace

struct hsb_handle {
  hsb_config cfg;
  int device = 0;
  int sm_count = 132;
  int levels = 0;
  Level lv[HSB_MAX_LEVELS];
  float log_odds_free = 0.f, log_odds_occ = 0.f;
  int gather_mode = HSB_GATHER_LDG;
  cudaStream_t stream = nullptr;      // main stream
  cudaStream_t copy_stream[2] = {nullptr, nullptr};
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  // device staging for the host-buffer entry points
  DevBuf d_hints, d_pts, d_offsets, d_poses, d_cov, d_scratch;
  // "containers of the last match" (MapRepMultiMap::dataContainers) and the update scan
  DevBuf d_last_pts, d_upd_pts;   // single-scan buffers: 16 floats of header (hint, gate inputs), then the points
  float* h_stage = nullptr;       // pinned staging for the single-scan calls (header + points, one H2D per call)
  size_t h_stage_bytes = 0;
  // raw-range input (N2)
  DevBuf d_beam_cs, d_ranges, d_occ;
  hsb_scan_format fmt = hsb_scan_format();
  bool fmt_set = false;
  hsb_cloud_format cfmt = hsb_cloud_format();
  bool cfmt_set = false;
  DevBuf d_cloud, d_cloud_off, d_cloud_tf, d_origo, d_cloud1;
  int last_n = 0;
  float last_origo[2] = {0.f, 0.f};
  // pinned host scratch
  float* h_pin = nullptr;  // 64 floats, mapped: kernels of the single-scan calls write their results here
  float* h_pin_dev = nullptr;    // device alias of h_pin
  int shape_batch = 0;           // > 0: pick the launch shape for this batch size instead of the launch's own (pipelined host calls)
  int tune_host_out = 1;         // single-scan calls: kernels write results into mapped host memory (no D2H copy)
  int tune_inline_scan = 0;      // 1: single-scan calls send the scan in the kernel parameters (no H2D copy operation) — measured slower, see match_kernel.cuh
  hsb::InlineScan<true> inline_scan;   // host image of those parameters
  cudaEvent_t ev_time[2] = {nullptr, nullptr};   // timing events around K2 (tuning "time_update")
  int tune_time_update = 0;
  BatchSet bset[2];             // device staging of the host-buffer batch calls, alternating between calls
  int next_set = 0;
  int* d_dirty_all = nullptr;   // HSB_MAX_LEVELS x 8 ints, see Level::dirty
  uint64_t d2h_bytes = 0;       // bytes the plane / rectangle download entry points copied to the host (diagnostic)
  cudaEvent_t ev_sync[4] = {nullptr, nullptr, nullptr, nullptr};   // ordering of caller streams against the handle's own
  DevBuf d_gate;           // fused SLAM step: lastMapUpdatePose[3], write-the-map flag
  float min_dist = 0.4f, min_angle = 0.13f;   // HectorSlamProcessor.h:62-63 defaults
  // tuning
  int tune_warps_per_scan = 0, tune_scans_per_block = 0, tune_stage_smem = 1, tune_chunk = 0, tune_unroll = 0, tune_packed = 0, tune_seq = 0, tune_partial = 1, tune_prefetch = 0, tune_trace = 0, tune_pace = 0, tune_pdl = 1, tune_auto_group = 1, tune_stagger = 0;
  DevBuf d_trace;
  DevBuf d_best;   // arg-max accumulator of hsb_best_hypothesis_device
  DevBuf d_record; // per-evaluation record of hsb_match_data_record
  bool map_write_pending = false;   // a nowait SLAM step's map write may still be running on `stream`
  unsigned step_seq = 0;   // sequence number of the fused SLAM steps (host polling, hsb_slam_update_nowait)
  int trace_scans = 0;
  int last_shape[6] = {0, 0, 0, 0, 0, 0};  // W, G, U, staged points per scan (0 = none), grid, resident CTAs / SM
  uint64_t launches = 0;
  std::string err;
};

namespace {

int fail(hsb_handle* h, int code, const char* fmt, ...) {
  if (h) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    h->err = buf;
  }
  return code;
}

#define HSB_CUDA(h, expr)                                                                          \
  do {                                                                                             \
    cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess) {                                                                       \
      return fail((h), _e == cudaErrorMemoryAllocation ? HSB_ERR_OUT_OF_MEMORY : HSB_ERR_CUDA,     \
                  "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__);     \
    }                                                                                              \
  } while (0)

struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    cudaGetDevice(&prev);
    if (prev != dev) cudaSetDevice(dev);
    else prev = -1;
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

int ensure(hsb_handle* h, DevBuf& b, size_t bytes) {
  if (bytes <= b.cap) return HSB_OK;
  if (b.p) HSB_CUDA(h, cudaFree(b.p));
  b.p = nullptr;
  b.cap = 0;
  size_t want = bytes + bytes / 4 + 256;
  HSB_CUDA(h, cudaMalloc(&b.p, want));
  b.cap = want;
  return HSB_OK;
}

// GridMapLogOdds.h:197-201 probToLogOdds (fp32 division, logf)
float prob_to_log_odds(float prob) {
  float odds = prob / (1.0f - prob);
  return logf(odds);
}

// Affine-mode inverse of the 2x3 map_T_world — the arithmetic the reference's
// `worldTmap = mapTworld.inverse()` performs (GridMapBase.h:279; order as oracle/hs_oracle.c
// affine2_inverse).  Host code is compiled without FMA contraction (x86-64 baseline).
void affine_inverse(const float a[6], float r[6]) {
  volatile float det = a[0] * a[4] - a[3] * a[1];
  float invdet = 1.0f / det;
  float l00 = a[4] * invdet;
  float l10 = -a[3] * invdet;
  float l01 = -a[1] * invdet;
  float l11 = a[0] * invdet;
  r[0] = l00;
  r[1] = l01;
  r[3] = l10;
  r[4] = l11;
  volatile float p0 = (-l00) * a[2], p1 = (-l01) * a[5];
  volatile float q0 = (-l10) * a[2], q1 = (-l11) * a[5];
  r[2] = p0 + p1;
  r[5] = q0 + q1;
}

void affine_apply_host(const float m[6], float vx, float vy, float* ox, float* oy) {
  volatile float p0 = m[0] * vx, p1 = m[1] * vy, p2 = m[2] * 1.0f;
  volatile float q0 = m[3] * vx, q1 = m[4] * vy, q2 = m[5] * 1.0f;
  volatile float s1 = p1 + p2, t1 = q1 + q2;
  *ox = p0 + s1;
  *oy = q0 + t1;
}

int refresh_level(hsb_handle* h, int level, cudaStream_t st) {
  Level& L = h->lv[level];
  size_t n = (size_t)L.sx * L.sy;
  int blocks = (int)std::min<size_t>((n + 255) / 256, (size_t)h->sm_count * 16);
  hsb::refresh_prob_kernel<<<blocks, 256, 0, st>>>(L.logodds, L.prob, L.surf, L.sx, L.sy);
  h->launches++;
  HSB_CUDA(h, cudaGetLastError());
  return HSB_OK;
}

int check_rect(hsb_handle* h, const Level& L, const int rect[4]) {
  if (rect[0] < 0 || rect[1] < 0 || rect[2] >= L.sx || rect[3] >= L.sy || rect[2] < rect[0] || rect[3] < rect[1])
    return fail(h, HSB_ERR_INVALID_ARG, "rectangle outside the level or empty");
  return HSB_OK;
}

// both dirty rectangles of a level := the whole level (after a reset or an upload every cell may differ)
int mark_level_dirty(hsb_handle* h, int level, cudaStream_t st) {
  Level& L = h->lv[level];
  if (!L.dirty) return HSB_OK;
  const int full[8] = {0, 0, L.sx - 1, L.sy - 1, 0, 0, L.sx - 1, L.sy - 1};
  HSB_CUDA(h, cudaMemcpyAsync(L.dirty, full, sizeof(full), cudaMemcpyHostToDevice, st));
  return HSB_OK;
}

int clear_level(hsb_handle* h, int level, cudaStream_t st) {
  Level& L = h->lv[level];
  size_t n = (size_t)L.sx * L.sy;
  int blocks = (int)std::min<size_t>((n + 255) / 256, (size_t)h->sm_count * 16);
  hsb::clear_level_kernel<<<blocks, 256, 0, st>>>(L.logodds, L.prob, L.stamp, L.surf, L.sx, L.sy);
  h->launches++;
  HSB_CUDA(h, cudaGetLastError());
  L.stamp_base = 0;
  return mark_level_dirty(h, level, st);   // every cell changed: replicas / mirrors must see the whole level
}

void fill_level_dev(const hsb_handle* h, int l, HsbLevelDev& d) {
  const Level& L = h->lv[l];
  d.prob = L.prob;
  d.tex = L.tex;
  d.sx = L.sx;
  d.sy = L.sy;
  d.lim_x = (float)L.sx - 2.0f;  // MapDimensionProperties.h:73
  d.lim_y = (float)L.sy - 2.0f;
  memcpy(d.mtw, L.mtw, sizeof(d.mtw));
  memcpy(d.wtm, L.wtm, sizeof(d.wtm));
  d.evals = L.evals;
  d.pt_scale = (float)(1.0 / pow(2.0, (double)l));  // MapRepMultiMap.h:127
}

// ---- match launch -----------------------------------------------------------------------------
template <int W, int G, int MODE, int U, bool PACK, bool INL = false>
int launch_match_t(hsb_handle* h, HsbMatchParams& P, int max_n, cudaStream_t st, int Gr,
                   const hsb::InlineScan<INL>& S = hsb::InlineScan<INL>()) {
  if (Gr <= 0 || Gr > G) Gr = G;   // groups per CTA actually launched (a G-group kernel runs with fewer: see launch_match)
  const size_t header = hsb::MatchSmem<W, G>::kHeaderBytes;
  auto kern = hsb::match_kernel<W, G, MODE, U, PACK, INL>;
  constexpr size_t kMaxDyn = 232448;   // dynamic shared memory one CTA may ask for (227 KB)
  constexpr int gt = W * 32;           // threads per scan
  int cap = 0;
  const bool fused = P.ranges || P.cloud || INL;   // conversion / inline scan: the whole scan must be staged
  if (h->tune_stage_smem || fused) cap = ((max_n + 1) + 1) & ~1;  // n + head padding, even
  // resident CTAs per SM for a given dynamic shared-memory size: block, thread, register and
  // shared-memory limits (1 KB per CTA is reserved by the driver)
  static int regs = 0;
  if (!regs) {
    cudaFuncAttributes fa;
    HSB_CUDA(h, cudaFuncGetAttributes(&fa, kern));
    regs = fa.numRegs > 0 ? fa.numRegs : 32;
  }
  const int threads = W * Gr * 32;
  auto resident = [&](size_t smem_bytes) {
    int blocks = std::min(32, 2048 / threads);
    blocks = std::min(blocks, 65536 / (((regs + 7) / 8 * 8) * threads));
    blocks = std::min<long>(blocks, (long)(kMaxDyn / (smem_bytes + 1024)));
    return std::max(blocks, 1);
  };
  // slots (a multiple of the group size, + 2 for the alignment head) that fit when `ctas` CTAs share an SM
  auto cap_for = [&](long ctas) {
    const long budget = std::min<long>((long)kMaxDyn, (long)kMaxDyn / ctas - 1024) - (long)header;
    int pts = (int)(budget / 8 / Gr);
    pts = (pts - 2) / gt * gt;
    return pts >= 4 * gt ? pts + 2 : 0;
  };
  const bool may_split = h->tune_partial && !PACK && !fused;   // a staged PREFIX is allowed
  if (cap > 0 && header + (size_t)Gr * cap * 8 > kMaxDyn) {        // the CTA's scans do not fit whole
    if (fused) return fail(h, HSB_ERR_UNSUPPORTED, "scan too long for the fused conversion (%d points)", max_n);
    cap = may_split ? cap_for(1) : 0;
  }
  if (cap > 0 && !fused && h->tune_stage_smem == 1) {
    // Wave quantisation: staging costs ~9 KB of shared memory
    // per scan, i.e. fewer resident groups.  If the batch does not fit the resident groups WITH the
    // scans staged but does fit WITHOUT (one wave instead of one and a bit), stage only the prefix
    // of each scan that the shared memory of a one-wave residency affords and read the rest through
    // L1 (tuning "partial" = 0: stage nothing in that case).
    const long groups = ((long)P.B + Gr - 1) / Gr;
    const long slots_staged = (long)resident(header + (size_t)Gr * cap * 8) * h->sm_count;
    const long slots_plain = (long)resident(header) * h->sm_count;
    if (groups > slots_staged && groups <= slots_plain)
      cap = may_split ? cap_for((groups + h->sm_count - 1) / h->sm_count) : 0;
  }
  P.stagger_ns = h->tune_stagger;
  P.sm_count = h->sm_count;
  P.prefetch = h->tune_prefetch;
  P.pace_slack = h->tune_pace;
  P.pts_cap = cap;
  size_t smem = header + (size_t)Gr * cap * 8;
  if (smem > 48 * 1024) {
    HSB_CUDA(h, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  }
  {
    // Shared-memory carve-out: left alone the driver picks a small one for kernels that ask for a
    // few hundred bytes, which then caps resident CTAs (measured: 7 CTAs/SM for 64-thread blocks).
    // Ask for what full occupancy of this launch shape needs, no more (the rest stays L1).
    size_t need = (size_t)resident(smem) * (smem + 1024);
    int pct = (int)((need * 100 + 233471) / 233472);
    pct = std::min(100, std::max(pct, 4));
    // (function attributes are per device: set on every launch rather than cached per process)
    HSB_CUDA(h, cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, pct));
  }
  P.trace = nullptr;
  if (h->tune_trace) {
    int s = ensure(h, h->d_trace, (size_t)P.B * 64);
    if (s != HSB_OK) return s;
    P.trace = static_cast<unsigned long long*>(h->d_trace.p);
    h->trace_scans = P.B;
  }
  const int seq = h->tune_seq > 0 ? h->tune_seq : 1;  // scans each group handles one after the other
  int grid = (P.B + Gr * seq - 1) / (Gr * seq);
  kern<<<grid, W * Gr * 32, smem, st>>>(P, S);
  h->launches++;
  {
    const int shape[6] = {W, Gr, U, cap > 0 ? (cap > max_n ? max_n : ((cap - 2) / (W * 32)) * (W * 32)) : 0, grid, resident(smem)};
    memcpy(h->last_shape, shape, sizeof(shape));
  }
  HSB_CUDA(h, cudaGetLastError());
  return HSB_OK;
}

template <int MODE>
int launch_match_mode(hsb_handle* h, HsbMatchParams& P, int max_n, cudaStream_t st, int W, int G, int U, int Gr) {
#define HSB_CASE(w, g, u)                                                                          \
  if (W == w && G == g && U == u) {                                                                \
    if (MODE == hsb::MODE_TEX && h->tune_packed) return launch_match_t<w, g, hsb::MODE_TEX, u, true>(h, P, max_n, st, Gr); \
    return launch_match_t<w, g, MODE, u, false>(h, P, max_n, st, Gr);                              \
  }
  // launch shapes kept after launch-shape sweeps (groups per CTA > 1 and more than 16 warps per scan
  // never won anywhere and were dropped)
  HSB_CASE(1, 1, 4);
  HSB_CASE(1, 2, 4);
  HSB_CASE(2, 1, 4);
  HSB_CASE(2, 2, 4);
  HSB_CASE(4, 1, 4);
  HSB_CASE(8, 1, 4);
  HSB_CASE(16, 1, 4);
  // many one-warp scans per CTA, paced (see match_kernel): 4 / 2 / 1 CTAs per SM; 32 = a whole SM's warps in one CTA
  HSB_CASE(1, 7, 4);
  HSB_CASE(1, 14, 4);
  HSB_CASE(1, 28, 4);
  HSB_CASE(1, 32, 4);
  // deeper gather batches: the whole per-lane share of a 1081-point scan in flight at once
  HSB_CASE(1, 1, 8);
  HSB_CASE(2, 1, 8);
  HSB_CASE(8, 1, 5);
  HSB_CASE(16, 1, 3);
#undef HSB_CASE
  return fail(h, HSB_ERR_INVALID_ARG, "unsupported tuning warps_per_scan=%d scans_per_block=%d unroll=%d", W, G, U);
}

int launch_match(hsb_handle* h, HsbMatchParams& P, int max_n, cudaStream_t st) {
  if (h->map_write_pending && st != h->stream) {
    // hsb_slam_update_nowait left a map write running on the handle's stream: a match on another stream waits for it
    HSB_CUDA(h, cudaEventRecord(h->ev_sync[0], h->stream));
    HSB_CUDA(h, cudaStreamWaitEvent(st, h->ev_sync[0], 0));
  }
  int W = h->tune_warps_per_scan, G = h->tune_scans_per_block;
  if (W <= 0) {
    // One warp per scan as soon as the batch fills the chip, more warps per scan for small batches,
    // never more than 8 (the per-evaluation reduction / barrier cost grows with the group size).
    // (a pipelined host-batch call passes ONE size for all its chunks: a scan's result must not depend on the
    // chunk it happens to travel in — the reduction order follows the shape — so that results are invariant
    // under a permutation of the batch, as the reference's are)
    const long Bs = h->shape_batch > 0 ? h->shape_batch : P.B;
    long want = ((long)h->sm_count * 24) / (Bs > 0 ? Bs : 1);
    W = 1;
    while (W * 2 <= want && W < 8) W *= 2;
  }
  int Gr = 0;   // 0: as many groups per CTA as the instantiation has
  if (G <= 0) {
    G = 1;
    // One-wave batches of one-warp scans (tuning "auto_group", on by default): ONE CTA per SM holding ceil(B / SMs) <= 32
    // scans instead of one-warp CTAs.  One CTA pays the 1 KB per-CTA shared-memory reservation once, so more of each
    // scan can be staged at full residency, and its warps start and end together.  Up to 28 scans per SM the 28-group
    // kernel runs (72 registers, the one-warp kernel's budget); up to 32 the 32-group kernel (1024 threads, 64 registers),
    // which keeps the benchmark's 4096 scans in one wave on a 132-SM H100 where 28 per SM would leave a second wave.
    // Larger batches keep one scan per CTA: finished warps are replaced at once there, which a CTA-wide drain would
    // prevent.  With one warp per scan the reduction order does not depend on the CTA shape: results are the same bits.
    const long Bs = h->shape_batch > 0 ? h->shape_batch : P.B;
    if (h->tune_auto_group && W == 1 && !P.ranges && !P.cloud && std::max<long>(Bs, P.B) <= (long)h->sm_count * 32 &&
        (h->tune_unroll == 0 || h->tune_unroll == 4)) {
      Gr = (int)((Bs + h->sm_count - 1) / h->sm_count);
      G = Gr <= 28 ? 28 : 32;
    }
  }
  int U = h->tune_unroll > 0 ? h->tune_unroll : 4;
  if (h->gather_mode == HSB_GATHER_TEX) return launch_match_mode<hsb::MODE_TEX>(h, P, max_n, st, W, G, U, Gr);
  return launch_match_mode<hsb::MODE_LDG>(h, P, max_n, st, W, G, U, Gr);
}

// Single-scan launch with the scan INSIDE the kernel parameters (hsb_match_data, hsb_slam_update; match_kernel.cuh
// InlineScan): the shape a single scan always takes (8 warps, 4 gathers in flight), so results equal the copy path's.
bool inline_scan_applies(const hsb_handle* h, int n) {
  return h->tune_inline_scan && n <= HSB_INLINE_MAX_POINTS && (h->tune_warps_per_scan == 0 || h->tune_warps_per_scan == 8) &&
         h->tune_scans_per_block <= 1 && (h->tune_unroll == 0 || h->tune_unroll == 4) && !h->tune_packed && h->tune_seq <= 1;
}
int launch_match_inline(hsb_handle* h, HsbMatchParams& P, const float* header, int nh, const float* pts, int n, float* d_pts_out,
                        cudaStream_t st) {
  hsb::InlineScan<true>& S = h->inline_scan;
  memset(S.header, 0, sizeof(S.header));
  if (nh > 0) memcpy(S.header, header, (size_t)nh * sizeof(float));
  if (n > 0) memcpy(S.pts, pts, (size_t)n * 8);
  P.B = 1;
  P.hints = nullptr;
  P.pts = nullptr;
  P.offsets = nullptr;
  P.n_shared = n;
  P.out_pts = reinterpret_cast<float2*>(d_pts_out);
  if (h->map_write_pending && st != h->stream) {
    HSB_CUDA(h, cudaEventRecord(h->ev_sync[0], h->stream));
    HSB_CUDA(h, cudaStreamWaitEvent(st, h->ev_sync[0], 0));
  }
  if (h->gather_mode == HSB_GATHER_TEX) return launch_match_t<8, 1, hsb::MODE_TEX, 4, false, true>(h, P, n, st, 1, S);
  return launch_match_t<8, 1, hsb::MODE_LDG, 4, false, true>(h, P, n, st, 1, S);
}

// Copy/compute pipeline of the host-buffer batch calls.  A call of >= 2048 scans travels in TWO halves: the second
// half's host->device copy overlaps the first half's kernel, and — with the submit / wait form — the next call's copies
// overlap this call's second kernel, so a stream of batches is bound by the PCIe copy of its inputs.  (More, smaller
// chunks do not shorten a call: every chunk kernel costs at least one scan latency whatever its size, so several small
// launches take longer than one large one.)
// Both halves use ONE launch shape, that of a B/2-scan batch (ShapeScope): a scan's result must not depend on the half
// it travels in, so that results are invariant under a permutation of the batch, as the reference's are.
struct ShapeScope {
  hsb_handle* h;
  ShapeScope(hsb_handle* hh, int B, size_t nchunks) : h(hh) { h->shape_batch = nchunks > 1 ? std::max(1, B / (int)nchunks) : 0; }
  ~ShapeScope() { h->shape_batch = 0; }
};
std::vector<int> pipeline_bounds(int B, int fixed_chunk) {
  std::vector<int> b;
  b.push_back(0);
  if (fixed_chunk > 0) {
    for (int x = fixed_chunk; x < B; x += fixed_chunk) b.push_back(x);
  } else if (B >= 2048) {
    b.push_back(B / 2);
  }
  b.push_back(B);
  return b;
}

void fill_match_params(const hsb_handle* h, HsbMatchParams& P) {
  memset(&P, 0, sizeof(P));
  P.levels = h->levels;
  for (int l = 0; l < h->levels; ++l) fill_level_dev(h, l, P.lv[l]);
  int off = 0;   // the record holds the levels coarsest first
  for (int l = h->levels - 1; l >= 0; --l) {
    P.lv[l].rec_off = off;
    off += 3 + 15 * P.lv[l].evals;
  }
}

int destroy_level(hsb_handle* h, Level& L) {
  if (L.tex) cudaDestroyTextureObject(L.tex);
  if (L.surf) cudaDestroySurfaceObject(L.surf);
  if (L.arr) cudaFreeArray(L.arr);
  if (L.logodds) cudaFree(L.logodds);
  if (L.prob) cudaFree(L.prob);
  if (L.stamp) cudaFree(L.stamp);
  if (L.scratch) cudaFree(L.scratch);
  L = Level();
  (void)h;
  return HSB_OK;
}

}  // namespace

extern "C" {

const char* hsb_version(void) { return "hector_slam_b200 0.1 (sm_90a)"; }

const char* hsb_status_string(int status) {
  switch (status) {
    case HSB_OK: return "ok";
    case HSB_ERR_INVALID_ARG: return "invalid argument";
    case HSB_ERR_CUDA: return "CUDA error";
    case HSB_ERR_OUT_OF_MEMORY: return "out of device memory";
    case HSB_ERR_NO_DEVICE: return "no CUDA device";
    case HSB_ERR_UNSUPPORTED: return "unsupported";
    default: return "unknown status";
  }
}

static std::string g_create_error;

const char* hsb_last_error(const hsb_handle* h) { return h ? h->err.c_str() : g_create_error.c_str(); }

uint64_t hsb_get_launch_count(const hsb_handle* h) { return h ? h->launches : 0; }

int hsb_get_last_launch_shape(const hsb_handle* h, int out[6]) {
  if (!h || !out) return HSB_ERR_INVALID_ARG;
  memcpy(out, h->last_shape, sizeof(h->last_shape));
  return HSB_OK;
}

int hsb_get_last_update_device_ms(hsb_handle* h, float* ms) {
  if (!h || !ms) return HSB_ERR_INVALID_ARG;
  DeviceGuard guard(h->device);
  HSB_CUDA(h, cudaEventSynchronize(h->ev_time[1]));
  HSB_CUDA(h, cudaEventElapsedTime(ms, h->ev_time[0], h->ev_time[1]));
  return HSB_OK;
}

int hsb_read_trace(hsb_handle* h, uint64_t* out, int max_scans) {
  if (!h || !out || max_scans < 0) return HSB_ERR_INVALID_ARG;
  DeviceGuard guard(h->device);
  const int n = std::min(max_scans, h->trace_scans);
  if (n > 0) HSB_CUDA(h, cudaMemcpy(out, h->d_trace.p, (size_t)n * 64, cudaMemcpyDeviceToHost));
  return n;
}
int hsb_get_gather_mode(const hsb_handle* h) { return h ? h->gather_mode : 0; }

int hsb_create(const hsb_config* cfg, hsb_handle** out) {
  if (!cfg || !out) return HSB_ERR_INVALID_ARG;
  *out = nullptr;
  if (cfg->levels < 1 || cfg->levels > HSB_MAX_LEVELS || cfg->map_size_x < 4 || cfg->map_size_y < 4 ||
      !(cfg->map_resolution > 0.f)) {
    g_create_error = "hsb_create: bad config (levels 1..8, sizes >= 4, resolution > 0)";
    return HSB_ERR_INVALID_ARG;
  }
  if ((cfg->map_size_x >> (cfg->levels - 1)) < 4 || (cfg->map_size_y >> (cfg->levels - 1)) < 4) {
    g_create_error = "hsb_create: coarsest level would be smaller than 4 cells";
    return HSB_ERR_INVALID_ARG;
  }
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    g_create_error = std::string("hsb_create: no CUDA device (") + cudaGetErrorString(e) + ")";
    return HSB_ERR_NO_DEVICE;
  }
  if (cfg->device < 0 || cfg->device >= ndev) {
    g_create_error = "hsb_create: device ordinal out of range";
    return HSB_ERR_INVALID_ARG;
  }
  hsb_handle* h = new (std::nothrow) hsb_handle();
  if (!h) return HSB_ERR_OUT_OF_MEMORY;
  h->cfg = *cfg;
  h->device = cfg->device;
  h->levels = cfg->levels;
  DeviceGuard guard(h->device);
  int status = HSB_OK;
  auto bail = [&](int code) {
    g_create_error = h->err;
    hsb_destroy(h);
    return code;
  };
#define HSB_TRY(expr)            \
  status = (expr);               \
  if (status != HSB_OK) return bail(status)
#define HSB_CUDA_C(expr)                                                                     \
  do {                                                                                       \
    cudaError_t _e = (expr);                                                                 \
    if (_e != cudaSuccess) {                                                                 \
      fail(h, HSB_ERR_CUDA, "%s failed: %s", #expr, cudaGetErrorString(_e));                 \
      return bail(_e == cudaErrorMemoryAllocation ? HSB_ERR_OUT_OF_MEMORY : HSB_ERR_CUDA);   \
    }                                                                                        \
  } while (0)

  cudaDeviceProp prop;
  HSB_CUDA_C(cudaGetDeviceProperties(&prop, h->device));
  h->sm_count = prop.multiProcessorCount;
  HSB_CUDA_C(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
  for (int i = 0; i < 2; ++i) HSB_CUDA_C(cudaStreamCreateWithFlags(&h->copy_stream[i], cudaStreamNonBlocking));
  for (int i = 0; i < 4; ++i) HSB_CUDA_C(cudaEventCreateWithFlags(&h->ev[i], cudaEventDisableTiming));
  for (int i = 0; i < 4; ++i) HSB_CUDA_C(cudaEventCreateWithFlags(&h->ev_sync[i], cudaEventDisableTiming));
  for (int k = 0; k < 2; ++k) {
    for (int i = 0; i < 2; ++i) HSB_CUDA_C(cudaEventCreateWithFlags(&h->bset[k].done[i], cudaEventDisableTiming));
    for (int i = 0; i < 8; ++i) HSB_CUDA_C(cudaEventCreateWithFlags(&h->bset[k].chunk_ready[i], cudaEventDisableTiming));
  }
  for (int i = 0; i < 2; ++i) HSB_CUDA_C(cudaEventCreate(&h->ev_time[i]));
  HSB_CUDA_C(cudaMalloc(&h->d_dirty_all, (HSB_MAX_LEVELS * 8 + 4) * sizeof(int)));   // + the replication error counter
  HSB_CUDA_C(cudaMemset(h->d_dirty_all, 0, (HSB_MAX_LEVELS * 8 + 4) * sizeof(int)));
  HSB_CUDA_C(cudaHostAlloc(&h->h_pin, 64 * sizeof(float), cudaHostAllocMapped));
  HSB_CUDA_C(cudaHostGetDevicePointer(&h->h_pin_dev, h->h_pin, 0));

  h->gather_mode = cfg->gather_mode == HSB_GATHER_LDG ? HSB_GATHER_LDG : HSB_GATHER_TEX;  // AUTO -> TEX (measured faster)
  // The texture twin is a CUDA array with texture gather, whose extent the device limits (maxTexture2DGather, 32768 x
  // 32768 on sm_90).  Level 0 is the largest level.  A wider map takes the linear-plane gathers in AUTO mode (the
  // reference accepts any size); an explicit TEX request for it is refused.
  if (h->gather_mode == HSB_GATHER_TEX &&
      (cfg->map_size_x > prop.maxTexture2DGather[0] || cfg->map_size_y > prop.maxTexture2DGather[1])) {
    if (cfg->gather_mode == HSB_GATHER_TEX) {
      fail(h, HSB_ERR_UNSUPPORTED, "hsb_create: map %d x %d exceeds the device's texture gather limit %d x %d; use LDG or AUTO",
           cfg->map_size_x, cfg->map_size_y, prop.maxTexture2DGather[0], prop.maxTexture2DGather[1]);
      return bail(HSB_ERR_UNSUPPORTED);
    }
    h->gather_mode = HSB_GATHER_LDG;
  }
  float ffree = cfg->update_factor_free > 0.f ? cfg->update_factor_free : 0.4f;      // GridMapLogOdds.h:117
  float focc = cfg->update_factor_occupied > 0.f ? cfg->update_factor_occupied : 0.6f;  // :118
  h->log_odds_free = prob_to_log_odds(ffree);
  h->log_odds_occ = prob_to_log_odds(focc);

  // MapRepMultiMap.h:48-72
  volatile float total_x = cfg->map_resolution * (float)cfg->map_size_x;
  volatile float mid_x = total_x * cfg->start_x;
  volatile float total_y = cfg->map_resolution * (float)cfg->map_size_y;
  volatile float mid_y = total_y * cfg->start_y;
  float res = cfg->map_resolution;
  int dx = cfg->map_size_x, dy = cfg->map_size_y;
  for (int l = 0; l < h->levels; ++l) {
    Level& L = h->lv[l];
    L.sx = dx;
    L.sy = dy;
    L.cell_length = res;
    L.scale = 1.0f / res;  // GridMapBase.h:270
    // AlignedScaling2f(s,s) * Translation2f(off): GridMapBase.h:272
    L.mtw[0] = L.scale;
    L.mtw[1] = 0.f;
    L.mtw[3] = 0.f;
    L.mtw[4] = L.scale;
    volatile float tx = L.scale * mid_x, ty = L.scale * mid_y;
    L.mtw[2] = tx;
    L.mtw[5] = ty;
    affine_inverse(L.mtw, L.wtm);  // GridMapBase.h:279
    int mi = cfg->max_iterations[l];
    if (mi == 0) mi = (l == 0) ? 5 : 3;  // MapRepMultiMap.h:125,128
    if (mi < 0) mi = 0;
    L.evals = mi + 1;  // ScanMatcher.h:74 + :94
    size_t n = (size_t)dx * dy;
    HSB_CUDA_C(cudaMalloc(&L.logodds, n * sizeof(float)));
    HSB_CUDA_C(cudaMalloc(&L.prob, n * sizeof(float)));
    HSB_CUDA_C(cudaMalloc(&L.stamp, n * sizeof(uint32_t)));
    L.dirty = h->d_dirty_all + 8 * l;
    HSB_CUDA_C(cudaMalloc(&L.scratch, 16 * sizeof(int)));
    {
      const int clean[16] = {0, INT_MAX, INT_MAX, -1, -1, 0, 0, 0, 0, INT_MAX, INT_MAX, -1, -1, 0, 0, 0};
      HSB_CUDA_C(cudaMemcpy(L.scratch, clean, sizeof(clean), cudaMemcpyHostToDevice));
    }
    if (h->gather_mode == HSB_GATHER_TEX) {
      cudaChannelFormatDesc desc = cudaCreateChannelDesc<float>();
      HSB_CUDA_C(cudaMallocArray(&L.arr, &desc, dx, dy, cudaArrayTextureGather | cudaArraySurfaceLoadStore));
      cudaResourceDesc rd;
      memset(&rd, 0, sizeof(rd));
      rd.resType = cudaResourceTypeArray;
      rd.res.array.array = L.arr;
      cudaTextureDesc td;
      memset(&td, 0, sizeof(td));
      td.addressMode[0] = cudaAddressModeClamp;
      td.addressMode[1] = cudaAddressModeClamp;
      td.filterMode = cudaFilterModePoint;
      td.readMode = cudaReadModeElementType;
      td.normalizedCoords = 0;
      HSB_CUDA_C(cudaCreateTextureObject(&L.tex, &rd, &td, nullptr));
      HSB_CUDA_C(cudaCreateSurfaceObject(&L.surf, &rd));
    }
    HSB_TRY(clear_level(h, l, h->stream));
    dx /= 2;      // MapRepMultiMap.h:67
    dy /= 2;
    res *= 2.0f;  // :68
  }
  {
    int clean[HSB_MAX_LEVELS * 8];
    for (int i = 0; i < HSB_MAX_LEVELS * 8; ++i) clean[i] = (i & 2) ? -1 : INT_MAX;
    HSB_CUDA_C(cudaMemcpyAsync(h->d_dirty_all, clean, sizeof(clean), cudaMemcpyHostToDevice, h->stream));
  }
  HSB_CUDA_C(cudaStreamSynchronize(h->stream));
#undef HSB_TRY
#undef HSB_CUDA_C
  *out = h;
  return HSB_OK;
}

int hsb_destroy(hsb_handle* h) {
  if (!h) return HSB_OK;
  DeviceGuard guard(h->device);
  cudaDeviceSynchronize();
  for (int l = 0; l < HSB_MAX_LEVELS; ++l) destroy_level(h, h->lv[l]);
  DevBuf* bufs[] = {&h->d_hints, &h->d_pts, &h->d_offsets, &h->d_poses, &h->d_cov, &h->d_scratch, &h->d_gate, &h->d_last_pts, &h->d_upd_pts,
                    &h->d_beam_cs, &h->d_ranges, &h->d_occ, &h->d_trace, &h->d_best, &h->d_record,
                    &h->d_cloud, &h->d_cloud_off, &h->d_cloud_tf, &h->d_origo, &h->d_cloud1};
  for (DevBuf* b : bufs)
    if (b->p) cudaFree(b->p);
  for (int k = 0; k < 2; ++k) {
    BatchSet& S = h->bset[k];
    DevBuf* sb[] = {&S.hints, &S.in, &S.offsets, &S.poses, &S.cov, &S.origo, &S.tf};
    for (DevBuf* b : sb)
      if (b->p) cudaFree(b->p);
    for (int i = 0; i < 2; ++i)
      if (S.done[i]) cudaEventDestroy(S.done[i]);
    for (int i = 0; i < 8; ++i)
      if (S.chunk_ready[i]) cudaEventDestroy(S.chunk_ready[i]);
  }
  if (h->d_dirty_all) cudaFree(h->d_dirty_all);
  for (int i = 0; i < 2; ++i)
    if (h->ev_time[i]) cudaEventDestroy(h->ev_time[i]);
  for (int i = 0; i < 4; ++i)
    if (h->ev_sync[i]) cudaEventDestroy(h->ev_sync[i]);
  if (h->h_pin) cudaFreeHost(h->h_pin);
  if (h->h_stage) cudaFreeHost(h->h_stage);
  for (int i = 0; i < 4; ++i)
    if (h->ev[i]) cudaEventDestroy(h->ev[i]);
  for (int i = 0; i < 2; ++i)
    if (h->copy_stream[i]) cudaStreamDestroy(h->copy_stream[i]);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
  return HSB_OK;
}

// Single-scan buffers carry a 16-float header in front of the points so that one copy moves both.
static const size_t kScanHeaderFloats = 16;
static inline float* scan_header(DevBuf& b) { return static_cast<float*>(b.p); }
static inline float* scan_points(DevBuf& b) { return static_cast<float*>(b.p) + kScanHeaderFloats; }
static int ensure_scan_buf(hsb_handle* h, DevBuf& b, int n) {
  return ensure(h, b, kScanHeaderFloats * sizeof(float) + (size_t)(n > 0 ? n : 1) * 8 + 16);
}
// header (nh floats) + points -> pinned staging -> ONE host-to-device copy on `st`
static int upload_scan(hsb_handle* h, DevBuf& b, const float* header, int nh, const float* pts, int n, cudaStream_t st) {
  int s = ensure_scan_buf(h, b, n);
  if (s != HSB_OK) return s;
  const size_t bytes = kScanHeaderFloats * sizeof(float) + (size_t)n * 8;
  if (bytes > h->h_stage_bytes) {
    if (h->h_stage) cudaFreeHost(h->h_stage);
    h->h_stage = nullptr;
    h->h_stage_bytes = 0;
    size_t cap = bytes < (64u << 10) ? (64u << 10) : bytes * 2;
    HSB_CUDA(h, cudaMallocHost(&h->h_stage, cap));
    h->h_stage_bytes = cap;
  }
  memset(h->h_stage, 0, kScanHeaderFloats * sizeof(float));
  if (nh > 0) memcpy(h->h_stage, header, (size_t)nh * sizeof(float));
  if (n > 0) memcpy(h->h_stage + kScanHeaderFloats, pts, (size_t)n * 8);
  HSB_CUDA(h, cudaMemcpyAsync(b.p, h->h_stage, bytes, cudaMemcpyHostToDevice, st));
  return HSB_OK;
}

// lastMapUpdatePose = FLT_MAX^3 (HectorSlamProcessor.h:117) for the fused step
static int reset_gate(hsb_handle* h) {
  int s = ensure(h, h->d_gate, 4 * sizeof(float));
  if (s != HSB_OK) return s;
  const float init[4] = {FLT_MAX, FLT_MAX, FLT_MAX, 0.f};
  memcpy(h->h_pin + 56, init, sizeof(init));
  HSB_CUDA(h, cudaMemcpyAsync(h->d_gate.p, h->h_pin + 56, sizeof(init), cudaMemcpyHostToDevice, h->stream));
  return HSB_OK;
}

int hsb_reset(hsb_handle* h) {
  if (!h) return HSB_ERR_INVALID_ARG;
  DeviceGuard guard(h->device);
  for (int l = 0; l < h->levels; ++l) {
    int s = clear_level(h, l, h->stream);
    if (s != HSB_OK) return s;
  }
  int s = reset_gate(h);
  if (s != HSB_OK) return s;
  HSB_CUDA(h, cudaStreamSynchronize(h->stream));
  return HSB_OK;
}

int hsb_set_update_factor_free(hsb_handle* h, float factor) {
  if (!h) return HSB_ERR_INVALID_ARG;
  h->log_odds_free = prob_to_log_odds(factor);
  return HSB_OK;
}
int hsb_set_update_factor_occupied(hsb_handle* h, float factor) {
  if (!h) return HSB_ERR_INVALID_ARG;
  h->log_odds_occ = prob_to_log_odds(factor);
  return HSB_OK;
}
int hsb_get_logodds_increments(hsb_handle* h, float out[2]) {
  if (!h || !out) return HSB_ERR_INVALID_ARG;
  out[0] = h->log_odds_free;
  out[1] = h->log_odds_occ;
  return HSB_OK;
}

int hsb_set_tuning(hsb_handle* h, const char* key, int value) {
  if (!h || !key) return HSB_ERR_INVALID_ARG;
  if (!strcmp(key, "warps_per_scan")) h->tune_warps_per_scan = value;
  else if (!strcmp(key, "scans_per_block")) h->tune_scans_per_block = value;
  else if (!strcmp(key, "stage_smem")) h->tune_stage_smem = value;
  else if (!strcmp(key, "chunk")) h->tune_chunk = value;
  else if (!strcmp(key, "unroll")) h->tune_unroll = value;
  else if (!strcmp(key, "packed")) h->tune_packed = value;
  else if (!strcmp(key, "seq")) h->tune_seq = value;
  else if (!strcmp(key, "host_out")) h->tune_host_out = value;
  else if (!strcmp(key, "inline_scan")) h->tune_inline_scan = value;
  else if (!strcmp(key, "partial")) h->tune_partial = value;
  else if (!strcmp(key, "prefetch")) h->tune_prefetch = value;
  else if (!strcmp(key, "trace")) h->tune_trace = value;
  else if (!strcmp(key, "pace")) h->tune_pace = value;
  else if (!strcmp(key, "time_update")) h->tune_time_update = value;
  else if (!strcmp(key, "pdl")) h->tune_pdl = value;
  else if (!strcmp(key, "auto_group")) h->tune_auto_group = value;
  else if (!strcmp(key, "stagger")) h->tune_stagger = value;
  else return fail(h, HSB_ERR_INVALID_ARG, "hsb_set_tuning: unknown key '%s'", key);
  return HSB_OK;
}

float hsb_get_scale_to_map(const hsb_handle* h) { return h ? h->lv[0].scale : 0.f; }
int hsb_get_map_levels(const hsb_handle* h) { return h ? h->levels : 0; }

int hsb_get_level_info(const hsb_handle* h, int level, int* size_x, int* size_y, float* cell_length) {
  if (!h || level < 0 || level >= h->levels) return HSB_ERR_INVALID_ARG;
  if (size_x) *size_x = h->lv[level].sx;
  if (size_y) *size_y = h->lv[level].sy;
  if (cell_length) *cell_length = h->lv[level].cell_length;
  return HSB_OK;
}

int hsb_map_coords_pose(const hsb_handle* h, int level, const float world[3], float out[3]) {
  if (!h || level < 0 || level >= h->levels || !world || !out) return HSB_ERR_INVALID_ARG;
  affine_apply_host(h->lv[level].mtw, world[0], world[1], &out[0], &out[1]);
  out[2] = world[2];
  return HSB_OK;
}
int hsb_world_coords_pose(const hsb_handle* h, int level, const float map[3], float out[3]) {
  if (!h || level < 0 || level >= h->levels || !map || !out) return HSB_ERR_INVALID_ARG;
  affine_apply_host(h->lv[level].wtm, map[0], map[1], &out[0], &out[1]);
  out[2] = map[2];
  return HSB_OK;
}

// ---- matching ----------------------------------------------------------------------------------

// R of HsbMatchParams::record: floats of one scan's per-evaluation record
static int record_floats(const hsb_handle* h) {
  int r = 0;
  for (int l = 0; l < h->levels; ++l) r += 3 + 15 * h->lv[l].evals;
  return r;
}

int hsb_get_match_record_floats(const hsb_handle* h) { return h ? record_floats(h) : HSB_ERR_INVALID_ARG; }

static int match_device(hsb_handle* h, int B, const float* d_hints, const float* d_pts, const int* d_offsets, int n_shared,
                        int max_points_per_scan, float* d_out_poses, float* d_out_cov, float* gate_state, const float* gate_in,
                        float* gate_out_host, cudaStream_t stream, unsigned* seq_host = nullptr, unsigned seq_value = 0,
                        float* d_record = nullptr) {
  if (!h || B < 0 || !d_hints || !d_out_poses) return HSB_ERR_INVALID_ARG;
  if (B == 0) return HSB_OK;
  if (!d_offsets && n_shared < 0) return fail(h, HSB_ERR_INVALID_ARG, "shared-scan mode needs n_shared >= 0");
  if (!d_pts && (d_offsets || n_shared > 0)) return fail(h, HSB_ERR_INVALID_ARG, "points pointer is NULL");
  DeviceGuard guard(h->device);
  HsbMatchParams P;
  fill_match_params(h, P);
  P.B = B;
  P.hints = d_hints;
  P.pts = reinterpret_cast<const float2*>(d_pts);
  P.offsets = d_offsets;
  P.n_shared = d_offsets ? 0 : n_shared;
  P.out_poses = d_out_poses;
  P.out_cov = d_out_cov;
  P.gate_state = gate_state;   // fused SLAM step only (B == 1)
  P.gate_in = gate_in;
  P.gate_out_host = gate_out_host;
  P.seq_host = seq_host;
  P.seq_value = seq_value;
  P.record = d_record;
  P.record_floats = record_floats(h);
  int max_n = d_offsets ? max_points_per_scan : n_shared;
  if (max_n < 0) max_n = 0;
  return launch_match(h, P, max_n, stream);
}

int hsb_match_batch_device(hsb_handle* h, int B, const float* d_hints, const float* d_pts, const int* d_offsets,
                           int n_shared, int max_points_per_scan, float* d_out_poses, float* d_out_cov, void* stream) {
  return match_device(h, B, d_hints, d_pts, d_offsets, n_shared, max_points_per_scan, d_out_poses, d_out_cov, nullptr, nullptr,
                      nullptr, (cudaStream_t)stream);
}

int hsb_match_batch_record_device(hsb_handle* h, int B, const float* d_hints, const float* d_pts, const int* d_offsets,
                                  int n_shared, int max_points_per_scan, float* d_out_poses, float* d_out_cov, float* d_record,
                                  void* stream) {
  if (!d_record) return HSB_ERR_INVALID_ARG;
  return match_device(h, B, d_hints, d_pts, d_offsets, n_shared, max_points_per_scan, d_out_poses, d_out_cov, nullptr, nullptr,
                      nullptr, (cudaStream_t)stream, nullptr, 0, d_record);
}

static int match_data_impl(hsb_handle* h, const float hint[3], const float* pts, int n, const float origo[2], float out_pose[3],
                           float cov_inout[9], float* record_out) {
  if (!h || !hint || !out_pose || n < 0 || (n > 0 && !pts)) return HSB_ERR_INVALID_ARG;
  DeviceGuard guard(h->device);
  // MapRepMultiMap::matchData fills dataContainers[] from this scan (MapRepMultiMap.h:127) whenever
  // there is a coarse level; hsb_update_by_scan reuses it for the coarse levels (:143).
  int s = ensure(h, h->d_scratch, 64 * sizeof(float));
  if (s != HSB_OK) return s;
  float* d_s = static_cast<float*>(h->d_scratch.p);  // [4..6] pose, [8..16] cov
  cudaStream_t st = h->stream;
  h->last_n = n;
  h->last_origo[0] = origo ? origo[0] : 0.f;
  h->last_origo[1] = origo ? origo[1] : 0.f;
  // the kernel writes pose + Hessian straight into mapped host memory: no device-to-host copy operation on the
  // critical path (reading the scan from host memory the same way was slower than copying it)
  const bool host_out = h->tune_host_out != 0;
  float* o_pose = host_out ? h->h_pin_dev + 4 : d_s + 4;
  float* o_cov = host_out ? h->h_pin_dev + 8 : d_s + 8;
  const int R = record_floats(h);
  float* d_rec = nullptr;
  if (record_out) {
    if ((s = ensure(h, h->d_record, (size_t)R * sizeof(float))) != HSB_OK) return s;
    d_rec = static_cast<float*>(h->d_record.p);
  }
  if (inline_scan_applies(h, n)) {
    // ... and the scan goes in with the launch itself: no host-to-device copy operation either; the kernel leaves
    // the endpoints in d_last_pts for hsb_update_by_scan's coarse levels
    if ((s = ensure_scan_buf(h, h->d_last_pts, n)) != HSB_OK) return s;
    HsbMatchParams P;
    fill_match_params(h, P);
    P.out_poses = o_pose;
    P.out_cov = o_cov;
    P.record = d_rec;
    P.record_floats = R;
    s = launch_match_inline(h, P, hint, 3, pts, n, scan_points(h->d_last_pts), st);
  } else {
    if ((s = upload_scan(h, h->d_last_pts, hint, 3, pts, n, st)) != HSB_OK) return s;   // header [0..2] = hint
    s = match_device(h, 1, scan_header(h->d_last_pts), scan_points(h->d_last_pts), nullptr, n, n, o_pose, o_cov, nullptr,
                     nullptr, nullptr, st, nullptr, 0, d_rec);
  }
  if (s != HSB_OK) return s;
  if (!host_out) HSB_CUDA(h, cudaMemcpyAsync(h->h_pin + 4, d_s + 4, 13 * sizeof(float), cudaMemcpyDeviceToHost, st));
  if (record_out) HSB_CUDA(h, cudaMemcpyAsync(record_out, d_rec, (size_t)R * sizeof(float), cudaMemcpyDeviceToHost, st));
  HSB_CUDA(h, cudaStreamSynchronize(st));
  memcpy(out_pose, h->h_pin + 4, 3 * sizeof(float));
  if (cov_inout && n > 0) memcpy(cov_inout, h->h_pin + 8, 9 * sizeof(float));
  return HSB_OK;
}

int hsb_match_data(hsb_handle* h, const float hint[3], const float* pts, int n, const float origo[2], float out_pose[3],
                   float cov_inout[9]) {
  return match_data_impl(h, hint, pts, n, origo, out_pose, cov_inout, nullptr);
}

int hsb_match_data_record(hsb_handle* h, const float hint[3], const float* pts, int n, const float origo[2],
                          float out_pose[3], float cov_inout[9], float* record_out) {
  if (!record_out) return HSB_ERR_INVALID_ARG;
  return match_data_impl(h, hint, pts, n, origo, out_pose, cov_inout, record_out);
}

int hsb_hessian_derivs(hsb_handle* h, int level, const float pose_map[3], const float* pts, int n, float H_out[9],
                       float dTr_out[3]) {
  if (!h || level < 0 || level >= h->levels || !pose_map || n < 0 || (n > 0 && !pts) || !H_out || !dTr_out)
    return HSB_ERR_INVALID_ARG;
  DeviceGuard guard(h->device);
  int s;
  if ((s = ensure(h, h->d_pts, (size_t)(n > 0 ? n : 1) * 8 + 16)) != HSB_OK) return s;
  if ((s = ensure(h, h->d_scratch, 64 * sizeof(float))) != HSB_OK) return s;
  cudaStream_t st = h->stream;
  if (n > 0) HSB_CUDA(h, cudaMemcpyAsync(h->d_pts.p, pts, (size_t)n * 8, cudaMemcpyHostToDevice, st));
  HsbLevelDev L;
  fill_level_dev(h, level, L);
  float* d_out = static_cast<float*>(h->d_scratch.p) + 32;
  if (h->gather_mode == HSB_GATHER_TEX)
    hsb::hessian_kernel<hsb::MODE_TEX><<<1, 256, 0, st>>>(L, static_cast<const float2*>(h->d_pts.p), n, pose_map[0],
                                                          pose_map[1], pose_map[2], d_out);
  else
    hsb::hessian_kernel<hsb::MODE_LDG><<<1, 256, 0, st>>>(L, static_cast<const float2*>(h->d_pts.p), n, pose_map[0],
                                                          pose_map[1], pose_map[2], d_out);
  h->launches++;
  HSB_CUDA(h, cudaGetLastError());
  HSB_CUDA(h, cudaMemcpyAsync(h->h_pin + 32, d_out, 12 * sizeof(float), cudaMemcpyDeviceToHost, st));
  HSB_CUDA(h, cudaStreamSynchronize(st));
  memcpy(H_out, h->h_pin + 32, 9 * sizeof(float));
  memcpy(dTr_out, h->h_pin + 41, 3 * sizeof(float));
  return HSB_OK;
}

// ---- raw ranges (N2) ---------------------------------------------------------------------------

int hsb_set_scan_format(hsb_handle* h, const hsb_scan_format* fmt) {
  if (!h || !fmt || fmt->n_beams < 1 || fmt->n_beams > (1 << 20)) return HSB_ERR_INVALID_ARG;
  DeviceGuard guard(h->device);
  int s = ensure(h, h->d_beam_cs, (size_t)fmt->n_beams * 8);
  if (s != HSB_OK) return s;
  std::vector<float> tab((size_t)fmt->n_beams * 2);
  float angle = fmt->angle_min;  // HectorMappingRos.cpp:487
  for (int i = 0; i < fmt->n_beams; ++i) {
    tab[2 * (size_t)i] = cosf(angle);      // :501 cos(angle) on a float
    tab[2 * (size_t)i + 1] = sinf(angle);  // :502
    volatile float next = angle + fmt->angle_increment;  // :505, fp32 accumulation
    angle = next;
  }
  HSB_CUDA(h, cudaMemcpy(h->d_beam_cs.p, tab.data(), tab.size() * sizeof(float), cudaMemcpyHostToDevice));
  h->fmt = *fmt;
  h->fmt_set = true;
  return HSB_OK;
}

static void fill_range_params(const hsb_handle* h, HsbMatchParams& P, const float* d_ranges) {
  P.ranges = d_ranges;
  P.beam_cs = static_cast<const float2*>(h->d_beam_cs.p);
  P.n_beams = h->fmt.n_beams;
  P.range_min = h->fmt.range_min;
  volatile float mx = h->fmt.range_max - 0.1f;  // :493 maxRangeForContainer
  P.range_max_c = mx;
  P.scale_to_map = h->lv[0].scale;
}

int hsb_scan_to_points(hsb_handle* h, const float* ranges, float* out_xy, int* out_n) {
  if (!h || !ranges || !out_xy || !out_n) return HSB_ERR_INVALID_ARG;
  if (!h->fmt_set) return fail(h, HSB_ERR_INVALID_ARG, "hsb_set_scan_format has not been called");
  DeviceGuard guard(h->device);
  const int nb = h->fmt.n_beams;
  int s;
  if ((s = ensure(h, h->d_ranges, (size_t)nb * 4)) != HSB_OK) return s;
  if ((s = ensure(h, h->d_pts, (size_t)nb * 8 + 16)) != HSB_OK) return s;
  if ((s = ensure(h, h->d_scratch, 64 * sizeof(float))) != HSB_OK) return s;
  cudaStream_t st = h->stream;
  HSB_CUDA(h, cudaMemcpyAsync(h->d_ranges.p, ranges, (size_t)nb * 4, cudaMemcpyHostToDevice, st));
  HsbMatchParams P;
  memset(&P, 0, sizeof(P));
  fill_range_params(h, P, static_cast<const float*>(h->d_ranges.p));
  int* d_n = reinterpret_cast<int*>(static_cast<float*>(h->d_scratch.p) + 48);
  hsb::scan_to_points_kernel<<<1, 256, 0, st>>>(P.ranges, P.beam_cs, nb, P.range_min, P.range_max_c, P.scale_to_map,
                                                static_cast<float2*>(h->d_pts.p), d_n);
  h->launches++;
  HSB_CUDA(h, cudaGetLastError());
  HSB_CUDA(h, cudaMemcpyAsync(h->h_pin + 48, d_n, sizeof(int), cudaMemcpyDeviceToHost, st));
  HSB_CUDA(h, cudaStreamSynchronize(st));
  int n = *reinterpret_cast<int*>(h->h_pin + 48);
  if (n > 0) HSB_CUDA(h, cudaMemcpy(out_xy, h->d_pts.p, (size_t)n * 8, cudaMemcpyDeviceToHost));
  *out_n = n;
  return HSB_OK;
}

int hsb_match_batch_ranges_device(hsb_handle* h, int B, const float* d_hints, const float* d_ranges, float* d_out_poses,
                                  float* d_out_cov, void* stream) {
  if (!h || B < 0 || !d_hints || !d_ranges || !d_out_poses) return HSB_ERR_INVALID_ARG;
  if (!h->fmt_set) return fail(h, HSB_ERR_INVALID_ARG, "hsb_set_scan_format has not been called");
  if (B == 0) return HSB_OK;
  DeviceGuard guard(h->device);
  HsbMatchParams P;
  fill_match_params(h, P);
  P.B = B;
  P.hints = d_hints;
  P.out_poses = d_out_poses;
  P.out_cov = d_out_cov;
  fill_range_params(h, P, d_ranges);
  return launch_match(h, P, h->fmt.n_beams, (cudaStream_t)stream);
}

// ---- point clouds (N2, the node's default input) ------------------------------------------------

int hsb_set_cloud_format(hsb_handle* h, const hsb_cloud_format* fmt) {
  if (!h || !fmt) return HSB_ERR_INVALID_ARG;
  for (int i = 0; i < 12; ++i)
    if (!std::isfinite(fmt->laser_transform[i])) return fail(h, HSB_ERR_INVALID_ARG, "laser_transform is not finite");
  h->cfmt = *fmt;
  h->cfmt_set = true;
  return HSB_OK;
}

static void fill_cloud_params(const hsb_handle* h, HsbMatchParams& P, const float* d_cloud, const int* d_offsets,
                              const double* d_transforms, float* d_origo) {
  P.cloud = d_cloud;
  P.cloud_offsets = d_offsets;
  P.cloud_tf = d_transforms;
  memcpy(P.cloud_tf0, h->cfmt.laser_transform, sizeof(P.cloud_tf0));
  P.sqr_min_dist = h->cfmt.sqr_laser_min_dist;
  P.sqr_max_dist = h->cfmt.sqr_laser_max_dist;
  P.z_min = h->cfmt.laser_z_min_value;
  P.z_max = h->cfmt.laser_z_max_value;
  P.scale_to_map = h->lv[0].scale;
  P.out_origo = d_origo;
}

int hsb_cloud_to_points(hsb_handle* h, const float* points_xyz, int n, float* out_xy, int* out_n, float out_origo[2]) {
  if (!h || n < 0 || (n > 0 && !points_xyz) || !out_xy || !out_n) return HSB_ERR_INVALID_ARG;
  if (!h->cfmt_set) return fail(h, HSB_ERR_INVALID_ARG, "hsb_set_cloud_format has not been called");
  DeviceGuard guard(h->device);
  int s;
  if ((s = ensure(h, h->d_cloud, (size_t)(n > 0 ? n : 1) * 12)) != HSB_OK) return s;
  if ((s = ensure(h, h->d_pts, (size_t)(n > 0 ? n : 1) * 8 + 16)) != HSB_OK) return s;
  if ((s = ensure(h, h->d_cloud_tf, 12 * sizeof(double))) != HSB_OK) return s;
  if ((s = ensure(h, h->d_scratch, 64 * sizeof(float))) != HSB_OK) return s;
  cudaStream_t st = h->stream;
  if (n > 0) HSB_CUDA(h, cudaMemcpyAsync(h->d_cloud.p, points_xyz, (size_t)n * 12, cudaMemcpyHostToDevice, st));
  HSB_CUDA(h, cudaMemcpyAsync(h->d_cloud_tf.p, h->cfmt.laser_transform, 12 * sizeof(double), cudaMemcpyHostToDevice, st));
  int* d_n = reinterpret_cast<int*>(static_cast<float*>(h->d_scratch.p) + 48);
  hsb::cloud_to_points_kernel<<<1, 256, 0, st>>>(static_cast<const float*>(h->d_cloud.p), n, static_cast<const double*>(h->d_cloud_tf.p),
                                                 h->cfmt.sqr_laser_min_dist, h->cfmt.sqr_laser_max_dist, h->cfmt.laser_z_min_value,
                                                 h->cfmt.laser_z_max_value, h->lv[0].scale, static_cast<float2*>(h->d_pts.p), d_n);
  h->launches++;
  HSB_CUDA(h, cudaGetLastError());
  HSB_CUDA(h, cudaMemcpyAsync(h->h_pin + 48, d_n, sizeof(int), cudaMemcpyDeviceToHost, st));
  HSB_CUDA(h, cudaStreamSynchronize(st));
  const int kept = *reinterpret_cast<int*>(h->h_pin + 48);
  if (kept > 0) HSB_CUDA(h, cudaMemcpy(out_xy, h->d_pts.p, (size_t)kept * 8, cudaMemcpyDeviceToHost));
  *out_n = kept;
  if (out_origo) {   // HectorMappingRos.cpp:516-517: Vector2f(laserPos.x(), laserPos.y()) * scaleToMap (host fp32, no contraction)
    volatile float ox = (float)h->cfmt.laser_transform[3], oy = (float)h->cfmt.laser_transform[7];
    volatile float sx = ox * h->lv[0].scale, sy = oy * h->lv[0].scale;
    out_origo[0] = sx;
    out_origo[1] = sy;
  }
  return HSB_OK;
}

int hsb_match_batch_cloud_device(hsb_handle* h, int B, const float* d_hints, const float* d_points_xyz, const int* d_offsets,
                                 int max_points_per_scan, const double* d_transforms, float* d_out_poses, float* d_out_cov,
                                 float* d_out_origo, void* stream) {
  if (!h || B < 0 || !d_hints || !d_offsets || !d_out_poses || max_points_per_scan < 0) return HSB_ERR_INVALID_ARG;
  if (!h->cfmt_set) return fail(h, HSB_ERR_INVALID_ARG, "hsb_set_cloud_format has not been called");
  if (B == 0) return HSB_OK;
  if (!d_points_xyz && max_points_per_scan > 0) return fail(h, HSB_ERR_INVALID_ARG, "points pointer is NULL");
  DeviceGuard guard(h->device);
  HsbMatchParams P;
  fill_match_params(h, P);
  P.B = B;
  P.hints = d_hints;
  P.out_poses = d_out_poses;
  P.out_cov = d_out_cov;
  fill_cloud_params(h, P, d_points_xyz, d_offsets, d_transforms, d_out_origo);
  return launch_match(h, P, max_points_per_scan, (cudaStream_t)stream);
}

}  // extern "C"

// ---- host-buffer batch calls: one pipelined implementation for the three input formats -----------
// A call is cut into chunks (pipeline_bounds); chunk c's host->device copy runs on copy stream c%2 while chunk
// c-1 is being matched, results stream back behind each kernel.  Two staging SETS of device buffers alternate
// between calls, so that — with the submit / wait form — call k+1's first copies already travel while call k's
// last chunk is still being matched: the steady state of a stream of batches is bound by the PCIe copy of the
// inputs, not by copy + the exposed tail kernel.  The blocking entry points are submit + wait.
namespace {

enum { IN_ENDPOINTS = 0, IN_RANGES = 1, IN_CLOUD = 2 };
struct HostBatch {
  int kind = IN_ENDPOINTS;
  int B = 0;
  const float* hints = nullptr;
  const float* in = nullptr;        // endpoints xy | ranges | cloud xyz
  const int* offsets = nullptr;     // endpoints (NULL = shared scan) | cloud
  int n_shared = 0;
  const double* transforms = nullptr;
  float* out_poses = nullptr;
  float* out_cov = nullptr;
  float* out_origo = nullptr;
};

int wait_set(hsb_handle* h, int s) {
  BatchSet& S = h->bset[s];
  if (!S.busy) return HSB_OK;
  HSB_CUDA(h, cudaEventSynchronize(S.done[0]));
  HSB_CUDA(h, cudaEventSynchronize(S.done[1]));
  S.busy = false;
  return HSB_OK;
}

int submit_host_batch(hsb_handle* h, const HostBatch& hb, int* ticket) {
  const int B = hb.B;
  const int si = h->next_set;
  BatchSet& S = h->bset[si];
  int s;
  if ((s = wait_set(h, si)) != HSB_OK) return s;   // the set is reused: its previous call must have delivered
  int max_n = 0;
  size_t in_bytes = 0, unit = 8;
  if (hb.kind == IN_RANGES) {
    max_n = h->fmt.n_beams;
    in_bytes = (size_t)B * (size_t)h->fmt.n_beams * 4;
  } else {
    unit = hb.kind == IN_CLOUD ? 12 : 8;
    if (hb.offsets) {
      for (int b = 0; b < B; ++b) {
        const int n = hb.offsets[b + 1] - hb.offsets[b];
        if (n < 0) return fail(h, HSB_ERR_INVALID_ARG, "offsets must be non-decreasing");
        max_n = std::max(max_n, n);
      }
      in_bytes = (size_t)hb.offsets[B] * unit;
    } else {
      max_n = hb.n_shared > 0 ? hb.n_shared : 0;
      in_bytes = (size_t)max_n * unit;
    }
    if (in_bytes > 0 && !hb.in) return fail(h, HSB_ERR_INVALID_ARG, "points pointer is NULL");
  }
  if ((s = ensure(h, S.hints, (size_t)B * 12)) != HSB_OK) return s;
  if ((s = ensure(h, S.in, in_bytes + 16)) != HSB_OK) return s;
  if ((s = ensure(h, S.offsets, (size_t)(B + 1) * 4)) != HSB_OK) return s;
  if ((s = ensure(h, S.poses, (size_t)B * 12)) != HSB_OK) return s;
  if (hb.out_cov && (s = ensure(h, S.cov, (size_t)B * 36)) != HSB_OK) return s;
  if (hb.out_origo && (s = ensure(h, S.origo, (size_t)B * 8)) != HSB_OK) return s;
  if (hb.transforms && (s = ensure(h, S.tf, (size_t)B * 12 * sizeof(double))) != HSB_OK) return s;
  float* d_hints = static_cast<float*>(S.hints.p);
  char* d_in = static_cast<char*>(S.in.p);
  int* d_off = static_cast<int*>(S.offsets.p);
  float* d_poses = static_cast<float*>(S.poses.p);
  float* d_cov = hb.out_cov ? static_cast<float*>(S.cov.p) : nullptr;
  float* d_origo = hb.out_origo ? static_cast<float*>(S.origo.p) : nullptr;
  double* d_tf = hb.transforms ? static_cast<double*>(S.tf.p) : nullptr;

  std::vector<int> bounds = pipeline_bounds(B, h->tune_chunk);
  const bool shared = hb.kind == IN_ENDPOINTS && !hb.offsets;
  if (shared) bounds = std::vector<int>{0, B};   // one shared scan: nothing big to overlap
  ShapeScope shape_scope(h, B, bounds.size() - 1);
  // Stream roles: copy_stream[0] carries ALL host->device copies of all calls back to back, copy_stream[1] the kernels
  // and the result copies; a chunk's kernel waits for its copy through an event, so the copy engine never queues behind
  // a kernel.
  cudaStream_t s0 = h->copy_stream[0], s1 = h->copy_stream[1];
  if (hb.offsets) HSB_CUDA(h, cudaMemcpyAsync(d_off, hb.offsets, (size_t)(B + 1) * 4, cudaMemcpyHostToDevice, s0));
  if (shared && in_bytes > 0) HSB_CUDA(h, cudaMemcpyAsync(d_in, hb.in, in_bytes, cudaMemcpyHostToDevice, s0));
  HSB_CUDA(h, cudaMemcpyAsync(d_hints, hb.hints, (size_t)B * 12, cudaMemcpyHostToDevice, s0));
  if (d_tf) HSB_CUDA(h, cudaMemcpyAsync(d_tf, hb.transforms, (size_t)B * 12 * sizeof(double), cudaMemcpyHostToDevice, s0));
  for (size_t ci = 0; ci + 1 < bounds.size(); ++ci) {
    const int b0 = bounds[ci], b1 = bounds[ci + 1];
    cudaStream_t st = s1;
    if (!shared) {
      size_t p0, p1;
      if (hb.kind == IN_RANGES) {
        p0 = (size_t)b0 * h->fmt.n_beams * 4;
        p1 = (size_t)b1 * h->fmt.n_beams * 4;
      } else {
        p0 = (size_t)hb.offsets[b0] * unit;
        p1 = (size_t)hb.offsets[b1] * unit;
      }
      if (p1 > p0)
        HSB_CUDA(h, cudaMemcpyAsync(d_in + p0, reinterpret_cast<const char*>(hb.in) + p0, p1 - p0, cudaMemcpyHostToDevice, s0));
    }
    cudaEvent_t ready = S.chunk_ready[ci < 8 ? ci : 7];
    HSB_CUDA(h, cudaEventRecord(ready, s0));           // hints / offsets / this chunk's input are on the device
    HSB_CUDA(h, cudaStreamWaitEvent(s1, ready, 0));
    float* o_pose = d_poses + 3 * (size_t)b0;
    float* o_cov = d_cov ? d_cov + 9 * (size_t)b0 : nullptr;
    if (hb.kind == IN_RANGES)
      s = hsb_match_batch_ranges_device(h, b1 - b0, d_hints + 3 * (size_t)b0,
                                        reinterpret_cast<const float*>(d_in) + (size_t)b0 * h->fmt.n_beams, o_pose, o_cov, st);
    else if (hb.kind == IN_CLOUD)
      s = hsb_match_batch_cloud_device(h, b1 - b0, d_hints + 3 * (size_t)b0, reinterpret_cast<const float*>(d_in), d_off + b0, max_n,
                                       d_tf ? d_tf + 12 * (size_t)b0 : nullptr, o_pose, o_cov,
                                       d_origo ? d_origo + 2 * (size_t)b0 : nullptr, st);
    else
      s = hsb_match_batch_device(h, b1 - b0, d_hints + 3 * (size_t)b0, reinterpret_cast<const float*>(d_in),
                                 hb.offsets ? d_off + b0 : nullptr, hb.n_shared, max_n, o_pose, o_cov, st);
    if (s != HSB_OK) return s;
    HSB_CUDA(h, cudaMemcpyAsync(hb.out_poses + 3 * (size_t)b0, o_pose, (size_t)(b1 - b0) * 12, cudaMemcpyDeviceToHost, st));
    if (hb.out_cov)
      HSB_CUDA(h, cudaMemcpyAsync(hb.out_cov + 9 * (size_t)b0, o_cov, (size_t)(b1 - b0) * 36, cudaMemcpyDeviceToHost, st));
    if (hb.out_origo)
      HSB_CUDA(h, cudaMemcpyAsync(hb.out_origo + 2 * (size_t)b0, d_origo + 2 * (size_t)b0, (size_t)(b1 - b0) * 8,
                                  cudaMemcpyDeviceToHost, st));
  }
  HSB_CUDA(h, cudaEventRecord(S.done[0], h->copy_stream[0]));
  HSB_CUDA(h, cudaEventRecord(S.done[1], h->copy_stream[1]));
  S.busy = true;
  h->next_set = si ^ 1;
  if (ticket) *ticket = si;
  return HSB_OK;
}

int run_host_batch(hsb_handle* h, const HostBatch& hb, int* ticket) {
  int t = 0;
  int s = submit_host_batch(h, hb, &t);
  if (s != HSB_OK) return s;
  if (ticket) {
    *ticket = t;
    return HSB_OK;
  }
  return wait_set(h, t);
}

int check_batch_args(hsb_handle* h, int B, const float* hints, float* out_poses) {
  if (!h || B < 0 || !hints || !out_poses) return HSB_ERR_INVALID_ARG;
  return HSB_OK;
}

}  // namespace

extern "C" {

int hsb_match_batch_submit(hsb_handle* h, int B, const float* hints, const float* pts, const int* offsets, int n_shared,
                           float* out_poses, float* out_cov, int* ticket) {
  int s = check_batch_args(h, B, hints, out_poses);
  if (s != HSB_OK) return s;
  if (B == 0) {
    if (ticket) *ticket = -1;
    return HSB_OK;
  }
  DeviceGuard guard(h->device);
  HostBatch hb;
  hb.kind = IN_ENDPOINTS;
  hb.B = B;
  hb.hints = hints;
  hb.in = pts;
  hb.offsets = offsets;
  hb.n_shared = n_shared;
  hb.out_poses = out_poses;
  hb.out_cov = out_cov;
  return run_host_batch(h, hb, ticket);
}
int hsb_match_batch(hsb_handle* h, int B, const float* hints, const float* pts, const int* offsets, int n_shared,
                    float* out_poses, float* out_cov) {
  return hsb_match_batch_submit(h, B, hints, pts, offsets, n_shared, out_poses, out_cov, nullptr);
}

int hsb_match_batch_ranges_submit(hsb_handle* h, int B, const float* hints, const float* ranges, float* out_poses,
                                  float* out_cov, int* ticket) {
  int s = check_batch_args(h, B, hints, out_poses);
  if (s != HSB_OK) return s;
  if (!ranges) return HSB_ERR_INVALID_ARG;
  if (!h->fmt_set) return fail(h, HSB_ERR_INVALID_ARG, "hsb_set_scan_format has not been called");
  if (B == 0) {
    if (ticket) *ticket = -1;
    return HSB_OK;
  }
  DeviceGuard guard(h->device);
  HostBatch hb;
  hb.kind = IN_RANGES;
  hb.B = B;
  hb.hints = hints;
  hb.in = ranges;
  hb.out_poses = out_poses;
  hb.out_cov = out_cov;
  return run_host_batch(h, hb, ticket);
}
int hsb_match_batch_ranges(hsb_handle* h, int B, const float* hints, const float* ranges, float* out_poses, float* out_cov) {
  return hsb_match_batch_ranges_submit(h, B, hints, ranges, out_poses, out_cov, nullptr);
}

int hsb_match_batch_cloud_submit(hsb_handle* h, int B, const float* hints, const float* points_xyz, const int* offsets,
                                 const double* transforms, float* out_poses, float* out_cov, float* out_origo, int* ticket) {
  int s = check_batch_args(h, B, hints, out_poses);
  if (s != HSB_OK) return s;
  if (!offsets) return HSB_ERR_INVALID_ARG;
  if (!h->cfmt_set) return fail(h, HSB_ERR_INVALID_ARG, "hsb_set_cloud_format has not been called");
  if (B == 0) {
    if (ticket) *ticket = -1;
    return HSB_OK;
  }
  DeviceGuard guard(h->device);
  HostBatch hb;
  hb.kind = IN_CLOUD;
  hb.B = B;
  hb.hints = hints;
  hb.in = points_xyz;
  hb.offsets = offsets;
  hb.transforms = transforms;
  hb.out_poses = out_poses;
  hb.out_cov = out_cov;
  hb.out_origo = out_origo;
  return run_host_batch(h, hb, ticket);
}
int hsb_match_batch_cloud(hsb_handle* h, int B, const float* hints, const float* points_xyz, const int* offsets,
                          const double* transforms, float* out_poses, float* out_cov, float* out_origo) {
  return hsb_match_batch_cloud_submit(h, B, hints, points_xyz, offsets, transforms, out_poses, out_cov, out_origo, nullptr);
}

int hsb_match_batch_wait(hsb_handle* h, int ticket) {
  if (!h || ticket < -1 || ticket > 1) return HSB_ERR_INVALID_ARG;
  if (ticket < 0) return HSB_OK;
  DeviceGuard guard(h->device);
  return wait_set(h, ticket);
}

int hsb_measure_h2d_gbs(hsb_handle* h, const void* host, size_t bytes, int reps, float* out_gbs) {
  if (!h || !host || !bytes || reps < 1 || !out_gbs) return HSB_ERR_INVALID_ARG;
  DeviceGuard guard(h->device);
  int s = ensure(h, h->d_occ, bytes);
  if (s != HSB_OK) return s;
  cudaStream_t st = h->stream;
  HSB_CUDA(h, cudaMemcpyAsync(h->d_occ.p, host, bytes, cudaMemcpyHostToDevice, st));
  HSB_CUDA(h, cudaEventRecord(h->ev_time[0], st));
  for (int i = 0; i < reps; ++i) HSB_CUDA(h, cudaMemcpyAsync(h->d_occ.p, host, bytes, cudaMemcpyHostToDevice, st));
  HSB_CUDA(h, cudaEventRecord(h->ev_time[1], st));
  HSB_CUDA(h, cudaEventSynchronize(h->ev_time[1]));
  float ms = 0.f;
  HSB_CUDA(h, cudaEventElapsedTime(&ms, h->ev_time[0], h->ev_time[1]));
  *out_gbs = (float)((double)bytes * reps / (ms * 1e-3) / 1e9);
  return HSB_OK;
}

void* hsb_alloc_pinned(size_t bytes) {
  void* p = nullptr;
  if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  return p;
}
int hsb_free_pinned(void* p) {
  if (p && cudaFreeHost(p) != cudaSuccess) {
    cudaGetLastError();
    return HSB_ERR_CUDA;
  }
  return HSB_OK;
}

}  // extern "C"

extern "C" {

// ---- map writing -------------------------------------------------------------------------------

static int run_update(hsb_handle* h, HsbUpdateParams& P, int max_n) {
  if (max_n <= 0) return HSB_OK;
  cudaStream_t st = h->stream;
  // mark: two warps per beam, four beams per CTA; apply: a fixed one-wave grid sweeping each level's box
  constexpr int TEAM = 2;
  int blocks = (max_n * TEAM + 7) / 8;
  int cap = (h->sm_count * 6) / (P.levels > 0 ? P.levels : 1);   // all levels' CTAs resident at once (6 per SM: its launch bounds)
  if (cap < 1) cap = 1;
  if (blocks > cap) blocks = cap;
  if (h->tune_time_update) HSB_CUDA(h, cudaEventRecord(h->ev_time[0], st));
  // (as many CTAs as are resident at once — the register count decides, asked from the occupancy API — so that the
  // sweep is ONE wave)
  static int apply_ctas_per_sm = 0;
  if (!apply_ctas_per_sm) {
    int nb = 0;
    HSB_CUDA(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, hsb::update_apply_kernel, 256, 0));
    apply_ctas_per_sm = nb > 0 ? nb : 4;
  }
  int sweep = (h->sm_count * apply_ctas_per_sm) / (P.levels > 0 ? P.levels : 1);
  if (sweep < 1) sweep = 1;
  if (h->tune_pdl) {
    // programmatic dependent launch: see pdl_wait() in update_kernel.cuh
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t cfg = {};
    cfg.blockDim = dim3(256);
    cfg.dynamicSmemBytes = 0;
    cfg.stream = st;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    cfg.gridDim = dim3(blocks, P.levels);
    HSB_CUDA(h, cudaLaunchKernelEx(&cfg, hsb::update_mark_kernel<TEAM>, P));
    cfg.gridDim = dim3(sweep, P.levels);
    HSB_CUDA(h, cudaLaunchKernelEx(&cfg, hsb::update_apply_kernel, P));
  } else {
    hsb::update_mark_kernel<TEAM><<<dim3(blocks, P.levels), 256, 0, st>>>(P);
    hsb::update_apply_kernel<<<dim3(sweep, P.levels), 256, 0, st>>>(P);
  }
  if (h->tune_time_update) HSB_CUDA(h, cudaEventRecord(h->ev_time[1], st));
  h->launches += 2;
  HSB_CUDA(h, cudaGetLastError());
  return HSB_OK;
}

static int next_stamp_base(hsb_handle* h, int level, uint32_t* base) {
  Level& L = h->lv[level];
  if (L.stamp_base > 0xfffffff0u - 8u) {  // wrap guard: forget old stamps
    HSB_CUDA(h, cudaMemsetAsync(L.stamp, 0, (size_t)L.sx * L.sy * sizeof(uint32_t), h->stream));
    L.stamp_base = 0;
  }
  *base = L.stamp_base;
  L.stamp_base += 4;
  L.parity ^= 1;   // this write uses the slot fill_update_level just handed out; the next one the other
  return HSB_OK;
}

static void fill_update_level(hsb_handle* h, int l, HsbUpdateLevelDev& d) {
  const Level& L = h->lv[l];
  memset(&d, 0, sizeof(d));
  d.logodds = L.logodds;
  d.prob = L.prob;
  d.stamp = L.stamp;
  d.surf = L.surf;
  d.sx = L.sx;
  d.sy = L.sy;
  memcpy(d.mtw, L.mtw, sizeof(d.mtw));
  d.dirty = L.dirty;
  d.scratch = L.scratch;
  d.slot = L.parity;
}

// MapRepMultiMap::updateByScan (MapRepMultiMap.h:134-147) as launches on h->stream; level 0 reads `d_pts0`,
// the coarse levels the container the last matchData left behind (:143).  pose_dev / gate_flag: see HsbUpdateParams.
static int enqueue_update_by_scan(hsb_handle* h, const float2* d_pts0, int n, const float origo[2], const float pose[3],
                                  const float* pose_dev, const float* gate_flag, const int* n_dev = nullptr) {
  HsbUpdateParams P;
  memset(&P, 0, sizeof(P));
  P.levels = h->levels;
  if (pose) memcpy(P.pose_world, pose, 3 * sizeof(float));
  P.pose_dev = pose_dev;
  P.gate_flag = gate_flag;
  P.log_odds_free = h->log_odds_free;
  P.log_odds_occ = h->log_odds_occ;
  int max_n = 0, s;
  for (int l = 0; l < h->levels; ++l) {
    HsbUpdateLevelDev& d = P.lv[l];
    fill_update_level(h, l, d);
    d.pt_scale = (float)(1.0 / pow(2.0, (double)l));
    if (l == 0) {  // MapRepMultiMap.h:140-141
      d.pts = d_pts0;
      d.n = n;
      d.n_dev = n_dev;   // fused point-cloud step: `n` is the cloud's size, the kept endpoints are counted on the device
      d.origo_x = origo ? origo[0] : 0.f;
      d.origo_y = origo ? origo[1] : 0.f;
    } else {  // :143 — the container left behind by the last matchData
      d.pts = reinterpret_cast<const float2*>(scan_points(h->d_last_pts));
      d.n = h->last_n;
      d.n_dev = (n_dev && d.pts == d_pts0) ? n_dev : nullptr;   // ... which is this very scan when the step matched it
      d.origo_x = h->last_origo[0];
      d.origo_y = h->last_origo[1];
    }
    // an empty container still advances the stamps in the reference (OccGridMapBase.h:164-167); no-op here
    d.active = d.n > 0;
    if (d.active) {
      if ((s = next_stamp_base(h, l, &d.stamp_base)) != HSB_OK) return s;
      if (d.n > max_n) max_n = d.n;
    }
  }
  return run_update(h, P, max_n);
}

int hsb_update_by_scan(hsb_handle* h, const float* pts, int n, const float origo[2], const float pose[3]) {
  if (!h || !pose || n < 0 || (n > 0 && !pts)) return HSB_ERR_INVALID_ARG;
  DeviceGuard guard(h->device);
  int s;
  cudaStream_t st = h->stream;
  if ((s = upload_scan(h, h->d_upd_pts, nullptr, 0, pts, n, st)) != HSB_OK) return s;
  if ((s = enqueue_update_by_scan(h, reinterpret_cast<const float2*>(scan_points(h->d_upd_pts)), n, origo, pose, nullptr, nullptr)) != HSB_OK)
    return s;
  HSB_CUDA(h, cudaStreamSynchronize(st));
  return HSB_OK;
}

int hsb_set_map_update_min_dist_diff(hsb_handle* h, float min_dist) {
  if (!h) return HSB_ERR_INVALID_ARG;
  h->min_dist = min_dist;
  return HSB_OK;
}
int hsb_set_map_update_min_angle_diff(hsb_handle* h, float min_angle) {
  if (!h) return HSB_ERR_INVALID_ARG;
  h->min_angle = min_angle;
  return HSB_OK;
}

static int slam_update_impl(hsb_handle* h, const float hint[3], const float* pts, int n, const float origo[2],
                            int map_without_matching, float out_pose[3], float cov_inout[9], int* map_updated, bool wait_map) {
  if (!h || !hint || !out_pose || n < 0 || (n > 0 && !pts)) return HSB_ERR_INVALID_ARG;
  DeviceGuard guard(h->device);
  int s;
  if ((s = ensure(h, h->d_scratch, 64 * sizeof(float))) != HSB_OK) return s;
  if (!h->d_gate.p && (s = reset_gate(h)) != HSB_OK) return s;
  // scan header: [0..2] hint, [3..5] minDist / minAngle / force; scratch: [8..10] pose, [11] flag, [12..20] cov
  float* d_s = static_cast<float*>(h->d_scratch.p);
  float* d_gate = static_cast<float*>(h->d_gate.p);
  cudaStream_t st = h->stream;
  // without matching the reference leaves the coarse containers alone (HectorSlamProcessor.h:77-81,
  // MapRepMultiMap.h:143): only level 0 sees this scan
  DevBuf& pbuf = map_without_matching ? h->d_upd_pts : h->d_last_pts;
  const float header[6] = {hint[0], hint[1], hint[2], h->min_dist, h->min_angle, map_without_matching ? 1.f : 0.f};
  // results (pose, flag, Hessian) are written into mapped host memory by the kernels themselves: the step is one
  // host-to-device copy and three launches (match with the gate in its epilogue, mark, apply — the latter two with
  // programmatic dependent launch)
  const bool host_out = h->tune_host_out != 0;
  const bool poll = host_out && !wait_map;   // return when the pose has arrived; the map write continues on the stream
  volatile unsigned* seq = reinterpret_cast<volatile unsigned*>(h->h_pin + 22);
  unsigned* seq_dev = reinterpret_cast<unsigned*>(h->h_pin_dev + 22);
  const unsigned seq_value = ++h->step_seq;
  const bool inl = !map_without_matching && inline_scan_applies(h, n);   // header + scan travel in the match launch
  if (inl) s = ensure_scan_buf(h, pbuf, n);
  else s = upload_scan(h, pbuf, header, 6, pts, n, st);
  if (s != HSB_OK) return s;
  const float* d_hdr = scan_header(pbuf);
  const float* d_pose_in = d_hdr;  // the hint, unless matched below
  if (!map_without_matching) {
    h->last_n = n;
    h->last_origo[0] = origo ? origo[0] : 0.f;
    h->last_origo[1] = origo ? origo[1] : 0.f;
    // :78 match, and :83-89 the gate in the same kernel's epilogue (an empty scan still passes through it: pose = hint)
    if (inl) {
      HsbMatchParams P;
      fill_match_params(h, P);
      P.out_poses = d_s + 8;
      P.out_cov = host_out ? h->h_pin_dev + 12 : d_s + 12;
      P.gate_state = d_gate;
      P.gate_out_host = host_out ? h->h_pin_dev + 8 : nullptr;
      P.seq_host = poll ? seq_dev : nullptr;
      P.seq_value = seq_value;
      s = launch_match_inline(h, P, header, 6, pts, n, scan_points(pbuf), st);
    } else {
      s = match_device(h, 1, d_hdr, scan_points(pbuf), nullptr, n, n, d_s + 8, host_out ? h->h_pin_dev + 12 : d_s + 12, d_gate,
                       d_hdr + 3, host_out ? h->h_pin_dev + 8 : nullptr, st, poll ? seq_dev : nullptr, seq_value);
    }
    if (s != HSB_OK) return s;
  } else {
    hsb::slam_gate_kernel<<<1, 32, 0, st>>>(d_gate, d_hdr + 3, d_pose_in, d_s + 8, host_out ? h->h_pin_dev + 8 : nullptr,
                                            poll ? seq_dev : nullptr, seq_value);  // :80, :89
    h->launches += 1;
    HSB_CUDA(h, cudaGetLastError());
  }
  if ((s = enqueue_update_by_scan(h, reinterpret_cast<const float2*>(scan_points(pbuf)), n, origo, nullptr, d_s + 8, d_gate + 3)) != HSB_OK)  // :91
    return s;
  if (poll) {
    // the pose is all the caller needs now; every later call on this handle is stream-ordered behind the map write
    unsigned spins = 0;
    while (*seq != seq_value) {
      if ((++spins & 0xfffu) == 0) {   // every 4096 polls make sure the stream has not died underneath us
        cudaError_t e = cudaStreamQuery(st);
        if (e != cudaSuccess && e != cudaErrorNotReady) return fail(h, HSB_ERR_CUDA, "stream failed: %s", cudaGetErrorString(e));
        if (e == cudaSuccess && *seq != seq_value) return fail(h, HSB_ERR_CUDA, "fused step finished without publishing its pose");
      }
    }
    __sync_synchronize();
    h->map_write_pending = true;
  } else {
    if (!host_out) HSB_CUDA(h, cudaMemcpyAsync(h->h_pin + 8, d_s + 8, 13 * sizeof(float), cudaMemcpyDeviceToHost, st));
    HSB_CUDA(h, cudaStreamSynchronize(st));  // :93 onMapUpdated — the probability plane is current
    h->map_write_pending = false;
  }
  memcpy(out_pose, h->h_pin + 8, 3 * sizeof(float));
  if (map_updated) *map_updated = h->h_pin[11] != 0.f;
  if (cov_inout && n > 0 && !map_without_matching) memcpy(cov_inout, h->h_pin + 12, 9 * sizeof(float));
  return HSB_OK;
}

int hsb_slam_update(hsb_handle* h, const float hint[3], const float* pts, int n, const float origo[2],
                    int map_without_matching, float out_pose[3], float cov_inout[9], int* map_updated) {
  return slam_update_impl(h, hint, pts, n, origo, map_without_matching, out_pose, cov_inout, map_updated, true);
}

int hsb_slam_update_nowait(hsb_handle* h, const float hint[3], const float* pts, int n, const float origo[2],
                           int map_without_matching, float out_pose[3], float cov_inout[9], int* map_updated) {
  return slam_update_impl(h, hint, pts, n, origo, map_without_matching, out_pose, cov_inout, map_updated, false);
}

// HectorMappingRos::scanCallback's default branch in one call: rosPointCloudToDataContainer (HectorMappingRos.cpp:283,
// 509-542) + HectorSlamProcessor::update (:297 / HectorSlamProcessor.h:71-113).  The cloud is converted by the match
// kernel's staging step; the converted endpoints, which the map writer needs too, are written out by the same kernel and
// their number stays on the device (the writer reads it there), so no host round trip appears between conversion, match,
// gate and map write.
int hsb_slam_update_cloud(hsb_handle* h, const float hint[3], const float* points_xyz, int n, const double* transform,
                          int map_without_matching, int nowait, float out_pose[3], float cov_inout[9], int* map_updated,
                          int* out_kept) {
  if (!h || !hint || !out_pose || n < 0 || (n > 0 && !points_xyz)) return HSB_ERR_INVALID_ARG;
  if (!h->cfmt_set) return fail(h, HSB_ERR_INVALID_ARG, "hsb_set_cloud_format has not been called");
  DeviceGuard guard(h->device);
  int s;
  if ((s = ensure(h, h->d_scratch, 64 * sizeof(float))) != HSB_OK) return s;
  if (!h->d_gate.p && (s = reset_gate(h)) != HSB_OK) return s;
  const double* T = transform ? transform : h->cfmt.laser_transform;
  // staging layout (floats): [0..15] header: hint, thresholds, force, [8] = 0, [9] = n (cloud offsets, as ints);
  // [16..39] the laser transform (12 doubles); [40..] the cloud
  const size_t kHdr = 16, kTf = 24;
  const size_t bytes = (kHdr + kTf + (size_t)n * 3) * sizeof(float);
  if ((s = ensure(h, h->d_cloud1, bytes + 16)) != HSB_OK) return s;
  if (bytes > h->h_stage_bytes) {
    if (h->h_stage) cudaFreeHost(h->h_stage);
    h->h_stage = nullptr;
    h->h_stage_bytes = 0;
    size_t cap = bytes < (64u << 10) ? (64u << 10) : bytes * 2;
    HSB_CUDA(h, cudaMallocHost(&h->h_stage, cap));
    h->h_stage_bytes = cap;
  }
  float* hs = h->h_stage;
  memset(hs, 0, kHdr * sizeof(float));
  hs[0] = hint[0]; hs[1] = hint[1]; hs[2] = hint[2];
  hs[3] = h->min_dist; hs[4] = h->min_angle; hs[5] = map_without_matching ? 1.f : 0.f;
  reinterpret_cast<int*>(hs)[8] = 0;
  reinterpret_cast<int*>(hs)[9] = n;
  memcpy(hs + kHdr, T, 12 * sizeof(double));
  if (n > 0) memcpy(hs + kHdr + kTf, points_xyz, (size_t)n * 12);
  cudaStream_t st = h->stream;
  HSB_CUDA(h, cudaMemcpyAsync(h->d_cloud1.p, hs, bytes, cudaMemcpyHostToDevice, st));
  float* d_c = static_cast<float*>(h->d_cloud1.p);
  const float* d_hdr = d_c;
  const int* d_offs = reinterpret_cast<const int*>(d_c) + 8;
  const double* d_tf = reinterpret_cast<const double*>(d_c + kHdr);
  const float* d_xyz = d_c + kHdr + kTf;
  float* d_s = static_cast<float*>(h->d_scratch.p);
  float* d_gate = static_cast<float*>(h->d_gate.p);
  int* d_n = reinterpret_cast<int*>(d_s + 40);
  // the container's origo (HectorMappingRos.cpp:516-517) is known on the host: Vector2f(laserPos) * scaleToMap in fp32
  volatile float ox = (float)T[3], oy = (float)T[7];
  volatile float sx = ox * h->lv[0].scale, sy = oy * h->lv[0].scale;
  const float origo[2] = {sx, sy};
  const bool host_out = true;   // results always travel through mapped host memory here
  const bool poll = nowait != 0;
  volatile unsigned* seq = reinterpret_cast<volatile unsigned*>(h->h_pin + 22);
  unsigned* seq_dev = reinterpret_cast<unsigned*>(h->h_pin_dev + 22);
  const unsigned seq_value = ++h->step_seq;
  int* kept_host = reinterpret_cast<int*>(h->h_pin + 24);
  int* kept_dev = reinterpret_cast<int*>(h->h_pin_dev + 24);
  DevBuf& pbuf = map_without_matching ? h->d_upd_pts : h->d_last_pts;
  if ((s = ensure_scan_buf(h, pbuf, n)) != HSB_OK) return s;
  float2* d_pts_out = reinterpret_cast<float2*>(scan_points(pbuf));
  (void)host_out;
  if (!map_without_matching) {
    HsbMatchParams P;
    fill_match_params(h, P);
    P.B = 1;
    P.hints = d_hdr;
    P.out_poses = d_s + 8;
    P.out_cov = h->h_pin_dev + 12;
    fill_cloud_params(h, P, d_xyz, d_offs, d_tf, nullptr);
    P.out_pts = d_pts_out;
    P.out_n = d_n;
    P.out_n_host = kept_dev;
    P.gate_state = d_gate;
    P.gate_in = d_hdr + 3;
    P.gate_out_host = h->h_pin_dev + 8;
    P.seq_host = poll ? seq_dev : nullptr;
    P.seq_value = seq_value;
    if ((s = launch_match(h, P, n, st)) != HSB_OK) return s;
    h->last_n = n;   // upper bound until the kept count arrives (the writer reads the exact one on the device)
    h->last_origo[0] = origo[0];
    h->last_origo[1] = origo[1];
  } else {
    hsb::cloud_to_points_kernel<<<1, 256, 0, st>>>(d_xyz, n, d_tf, h->cfmt.sqr_laser_min_dist, h->cfmt.sqr_laser_max_dist,
                                                   h->cfmt.laser_z_min_value, h->cfmt.laser_z_max_value, h->lv[0].scale, d_pts_out, d_n);
    hsb::slam_gate_kernel<<<1, 32, 0, st>>>(d_gate, d_hdr + 3, d_hdr, d_s + 8, h->h_pin_dev + 8, nullptr, 0);
    hsb::publish_int_kernel<<<1, 32, 0, st>>>(d_n, kept_dev, poll ? seq_dev : nullptr, seq_value);
    h->launches += 3;
    HSB_CUDA(h, cudaGetLastError());
  }
  if ((s = enqueue_update_by_scan(h, d_pts_out, n, origo, nullptr, d_s + 8, d_gate + 3, d_n)) != HSB_OK) return s;
  if (poll) {
    unsigned spins = 0;
    while (*seq != seq_value) {
      if ((++spins & 0xfffu) == 0) {
        cudaError_t e = cudaStreamQuery(st);
        if (e != cudaSuccess && e != cudaErrorNotReady) return fail(h, HSB_ERR_CUDA, "stream failed: %s", cudaGetErrorString(e));
        if (e == cudaSuccess && *seq != seq_value) return fail(h, HSB_ERR_CUDA, "fused step finished without publishing its pose");
      }
    }
    __sync_synchronize();
    h->map_write_pending = true;
  } else {
    HSB_CUDA(h, cudaStreamSynchronize(st));
    h->map_write_pending = false;
  }
  const int kept = *kept_host;
  if (!map_without_matching) h->last_n = kept;
  memcpy(out_pose, h->h_pin + 8, 3 * sizeof(float));
  if (map_updated) *map_updated = h->h_pin[11] != 0.f;
  if (cov_inout && kept > 0 && !map_without_matching) memcpy(cov_inout, h->h_pin + 12, 9 * sizeof(float));
  if (out_kept) *out_kept = kept;
  return HSB_OK;
}

int hsb_set_last_map_update_pose(hsb_handle* h, const float pose[3]) {
  if (!h || !pose) return HSB_ERR_INVALID_ARG;
  DeviceGuard guard(h->device);
  int s = ensure(h, h->d_gate, 4 * sizeof(float));
  if (s != HSB_OK) return s;
  memcpy(h->h_pin + 56, pose, 3 * sizeof(float));
  HSB_CUDA(h, cudaMemcpyAsync(h->d_gate.p, h->h_pin + 56, 3 * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  HSB_CUDA(h, cudaStreamSynchronize(h->stream));
  return HSB_OK;
}

int hsb_get_last_map_update_pose(hsb_handle* h, float out[3]) {
  if (!h || !out) return HSB_ERR_INVALID_ARG;
  DeviceGuard guard(h->device);
  if (!h->d_gate.p) {
    int s = reset_gate(h);
    if (s != HSB_OK) return s;
  }
  HSB_CUDA(h, cudaMemcpyAsync(h->h_pin + 56, h->d_gate.p, 3 * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  HSB_CUDA(h, cudaStreamSynchronize(h->stream));
  memcpy(out, h->h_pin + 56, 3 * sizeof(float));
  return HSB_OK;
}

int hsb_update_level_by_scan(hsb_handle* h, int level, const float* pts, int n, const float origo[2], const float pose[3]) {
  if (!h || level < 0 || level >= h->levels || !pose || n < 0 || (n > 0 && !pts)) return HSB_ERR_INVALID_ARG;
  DeviceGuard guard(h->device);
  int s;
  cudaStream_t st = h->stream;
  if ((s = upload_scan(h, h->d_upd_pts, nullptr, 0, pts, n, st)) != HSB_OK) return s;
  HsbUpdateParams P;
  memset(&P, 0, sizeof(P));
  P.levels = 1;
  memcpy(P.pose_world, pose, 3 * sizeof(float));
  P.log_odds_free = h->log_odds_free;
  P.log_odds_occ = h->log_odds_occ;
  HsbUpdateLevelDev& d = P.lv[0];
  fill_update_level(h, level, d);
  d.pt_scale = 1.0f;
  d.pts = reinterpret_cast<const float2*>(scan_points(h->d_upd_pts));
  d.n = n;
  d.origo_x = origo ? origo[0] : 0.f;
  d.origo_y = origo ? origo[1] : 0.f;
  d.active = n > 0;
  if (d.active && (s = next_stamp_base(h, level, &d.stamp_base)) != HSB_OK) return s;
  if ((s = run_update(h, P, n)) != HSB_OK) return s;
  HSB_CUDA(h, cudaStreamSynchronize(st));
  return HSB_OK;
}

int hsb_on_map_updated(hsb_handle* h) {
  if (!h) return HSB_ERR_INVALID_ARG;
  DeviceGuard guard(h->device);
  HSB_CUDA(h, cudaStreamSynchronize(h->stream));
  h->map_write_pending = false;
  return HSB_OK;
}

// ---- planes ------------------------------------------------------------------------------------

int hsb_upload_level(hsb_handle* h, int level, const float* logodds_host) {
  if (!h || level < 0 || level >= h->levels || !logodds_host) return HSB_ERR_INVALID_ARG;
  DeviceGuard guard(h->device);
  Level& L = h->lv[level];
  HSB_CUDA(h, cudaMemcpyAsync(L.logodds, logodds_host, (size_t)L.sx * L.sy * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  int s = refresh_level(h, level, h->stream);
  if (s != HSB_OK) return s;
  if ((s = mark_level_dirty(h, level, h->stream)) != HSB_OK) return s;
  HSB_CUDA(h, cudaStreamSynchronize(h->stream));
  return HSB_OK;
}

int hsb_download_level(hsb_handle* h, int level, float* out) {
  if (!h || level < 0 || level >= h->levels || !out) return HSB_ERR_INVALID_ARG;
  DeviceGuard guard(h->device);
  Level& L = h->lv[level];
  HSB_CUDA(h, cudaMemcpyAsync(out, L.logodds, (size_t)L.sx * L.sy * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  HSB_CUDA(h, cudaStreamSynchronize(h->stream));
  h->d2h_bytes += (size_t)L.sx * L.sy * sizeof(float);
  return HSB_OK;
}

int hsb_download_level_rect(hsb_handle* h, int level, const int rect[4], float* out) {
  if (!h || level < 0 || level >= h->levels || !rect || !out) return HSB_ERR_INVALID_ARG;
  DeviceGuard guard(h->device);
  Level& L = h->lv[level];
  int s = check_rect(h, L, rect);
  if (s != HSB_OK) return s;
  const size_t w = (size_t)(rect[2] - rect[0] + 1), hgt = (size_t)(rect[3] - rect[1] + 1);
  HSB_CUDA(h, cudaMemcpy2DAsync(out, w * sizeof(float), L.logodds + (size_t)rect[1] * L.sx + rect[0], (size_t)L.sx * sizeof(float),
                                w * sizeof(float), hgt, cudaMemcpyDeviceToHost, h->stream));
  HSB_CUDA(h, cudaStreamSynchronize(h->stream));
  h->d2h_bytes += w * hgt * sizeof(float);
  return HSB_OK;
}

int hsb_download_occupancy_rect(hsb_handle* h, int level, const int rect[4], int8_t* out) {
  if (!h || level < 0 || level >= h->levels || !rect || !out) return HSB_ERR_INVALID_ARG;
  DeviceGuard guard(h->device);
  Level& L = h->lv[level];
  int s = check_rect(h, L, rect);
  if (s != HSB_OK) return s;
  const int w = rect[2] - rect[0] + 1, hgt = rect[3] - rect[1] + 1;
  const size_t n = (size_t)w * hgt;
  if ((s = ensure(h, h->d_occ, n)) != HSB_OK) return s;
  int blocks = (int)std::min<size_t>((n + 255) / 256, (size_t)h->sm_count * 16);
  hsb::occupancy_rect_kernel<<<blocks, 256, 0, h->stream>>>(L.logodds, L.sx, rect[0], rect[1], w, hgt, static_cast<int8_t*>(h->d_occ.p));
  h->launches++;
  HSB_CUDA(h, cudaGetLastError());
  HSB_CUDA(h, cudaMemcpyAsync(out, h->d_occ.p, n, cudaMemcpyDeviceToHost, h->stream));
  HSB_CUDA(h, cudaStreamSynchronize(h->stream));
  h->d2h_bytes += n;
  return HSB_OK;
}

uint64_t hsb_get_d2h_bytes(const hsb_handle* h) { return h ? h->d2h_bytes : 0; }

int hsb_download_prob(hsb_handle* h, int level, float* out) {
  if (!h || level < 0 || level >= h->levels || !out) return HSB_ERR_INVALID_ARG;
  DeviceGuard guard(h->device);
  Level& L = h->lv[level];
  if (L.arr) {  // read what the texture path sees
    HSB_CUDA(h, cudaMemcpy2DFromArrayAsync(out, (size_t)L.sx * sizeof(float), L.arr, 0, 0, (size_t)L.sx * sizeof(float), L.sy,
                                           cudaMemcpyDeviceToHost, h->stream));
  } else {
    HSB_CUDA(h, cudaMemcpyAsync(out, L.prob, (size_t)L.sx * L.sy * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  }
  HSB_CUDA(h, cudaStreamSynchronize(h->stream));
  return HSB_OK;
}

int hsb_download_occupancy(hsb_handle* h, int level, int8_t* out) {
  if (!h || level < 0 || level >= h->levels || !out) return HSB_ERR_INVALID_ARG;
  DeviceGuard guard(h->device);
  Level& L = h->lv[level];
  const size_t n = (size_t)L.sx * L.sy;
  int s = ensure(h, h->d_occ, n);
  if (s != HSB_OK) return s;
  int blocks = (int)std::min<size_t>((n + 255) / 256, (size_t)h->sm_count * 16);
  hsb::occupancy_kernel<<<blocks, 256, 0, h->stream>>>(L.logodds, static_cast<int8_t*>(h->d_occ.p), n);
  h->launches++;
  HSB_CUDA(h, cudaGetLastError());
  HSB_CUDA(h, cudaMemcpyAsync(out, h->d_occ.p, n, cudaMemcpyDeviceToHost, h->stream));
  HSB_CUDA(h, cudaStreamSynchronize(h->stream));
  h->d2h_bytes += n;
  return HSB_OK;
}

// the likelihood launch on device pointers; `st` may be a caller's stream (ordered behind a pending map write)
static int likelihood_device(hsb_handle* h, int level, int B, const float* d_poses, const float2* d_pts, const int* d_off,
                             int n_shared, float* d_out, cudaStream_t st, unsigned long long* d_best = nullptr) {
  if (h->map_write_pending && st != h->stream) {
    HSB_CUDA(h, cudaEventRecord(h->ev_sync[0], h->stream));
    HSB_CUDA(h, cudaStreamWaitEvent(st, h->ev_sync[0], 0));
  }
  HsbLevelDev L;
  fill_level_dev(h, level, L);
  int blocks = std::min((B + 3) / 4, h->sm_count * 16);
  if (h->gather_mode == HSB_GATHER_TEX)
    hsb::likelihood_kernel<hsb::MODE_TEX><<<blocks, 128, 0, st>>>(L, B, d_poses, d_pts, d_off, d_off ? 0 : n_shared, d_out, d_best);
  else
    hsb::likelihood_kernel<hsb::MODE_LDG><<<blocks, 128, 0, st>>>(L, B, d_poses, d_pts, d_off, d_off ? 0 : n_shared, d_out, d_best);
  h->launches++;
  HSB_CUDA(h, cudaGetLastError());
  return HSB_OK;
}

int hsb_likelihood_batch_device(hsb_handle* h, int level, int B, const float* d_poses_world, const float* d_points_xy,
                                const int* d_offsets, int n_shared, float* d_out_likelihood, void* stream) {
  if (!h || level < 0 || level >= h->levels || B < 0 || !d_poses_world || !d_out_likelihood) return HSB_ERR_INVALID_ARG;
  if (!d_offsets && n_shared < 0) return HSB_ERR_INVALID_ARG;
  if (B == 0) return HSB_OK;
  if (!d_points_xy && (d_offsets || n_shared > 0)) return fail(h, HSB_ERR_INVALID_ARG, "points pointer is NULL");
  DeviceGuard guard(h->device);
  return likelihood_device(h, level, B, d_poses_world, reinterpret_cast<const float2*>(d_points_xy), d_offsets, n_shared,
                           d_out_likelihood, (cudaStream_t)stream);
}

int hsb_best_hypothesis_device(hsb_handle* h, int level, int B, const float* d_poses_world, const float* d_points_xy,
                               const int* d_offsets, int n_shared, float* d_out_likelihood, float* d_best4, void* stream) {
  if (!h || level < 0 || level >= h->levels || B < 0 || !d_best4 || (B > 0 && !d_poses_world)) return HSB_ERR_INVALID_ARG;
  if (!d_offsets && n_shared < 0) return HSB_ERR_INVALID_ARG;
  if (B > 0 && !d_points_xy && (d_offsets || n_shared > 0)) return fail(h, HSB_ERR_INVALID_ARG, "points pointer is NULL");
  DeviceGuard guard(h->device);
  int s;
  if (!h->d_best.p) {
    if ((s = ensure(h, h->d_best, sizeof(unsigned long long))) != HSB_OK) return s;
    HSB_CUDA(h, cudaMemsetAsync(h->d_best.p, 0, sizeof(unsigned long long), (cudaStream_t)stream));
  }
  unsigned long long* d_best = static_cast<unsigned long long*>(h->d_best.p);
  if (B > 0 && (s = likelihood_device(h, level, B, d_poses_world, reinterpret_cast<const float2*>(d_points_xy), d_offsets, n_shared,
                                      d_out_likelihood, (cudaStream_t)stream, d_best)) != HSB_OK)
    return s;
  hsb::best_hypothesis_finish_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(d_best, d_poses_world, d_best4);
  h->launches++;
  HSB_CUDA(h, cudaGetLastError());
  return HSB_OK;
}

int hsb_likelihood_batch(hsb_handle* h, int level, int B, const float* poses, const float* pts, const int* offsets,
                         int n_shared, float* out) {
  if (!h || level < 0 || level >= h->levels || B < 0 || !poses || !out) return HSB_ERR_INVALID_ARG;
  if (B == 0) return HSB_OK;
  DeviceGuard guard(h->device);
  size_t total = offsets ? (size_t)offsets[B] : (size_t)(n_shared > 0 ? n_shared : 0);
  if (total > 0 && !pts) return fail(h, HSB_ERR_INVALID_ARG, "points pointer is NULL");
  int s;
  if ((s = ensure(h, h->d_hints, (size_t)B * 12)) != HSB_OK) return s;
  if ((s = ensure(h, h->d_pts, total * 8 + 16)) != HSB_OK) return s;
  if ((s = ensure(h, h->d_offsets, (size_t)(B + 1) * 4)) != HSB_OK) return s;
  if ((s = ensure(h, h->d_poses, (size_t)B * 12)) != HSB_OK) return s;
  cudaStream_t st = h->stream;
  HSB_CUDA(h, cudaMemcpyAsync(h->d_hints.p, poses, (size_t)B * 12, cudaMemcpyHostToDevice, st));
  if (total > 0) HSB_CUDA(h, cudaMemcpyAsync(h->d_pts.p, pts, total * 8, cudaMemcpyHostToDevice, st));
  if (offsets) HSB_CUDA(h, cudaMemcpyAsync(h->d_offsets.p, offsets, (size_t)(B + 1) * 4, cudaMemcpyHostToDevice, st));
  float* d_out = static_cast<float*>(h->d_poses.p);
  s = likelihood_device(h, level, B, static_cast<const float*>(h->d_hints.p), static_cast<const float2*>(h->d_pts.p),
                        offsets ? static_cast<const int*>(h->d_offsets.p) : nullptr, offsets ? 0 : (n_shared > 0 ? n_shared : 0),
                        d_out, st);
  if (s != HSB_OK) return s;
  HSB_CUDA(h, cudaMemcpyAsync(out, d_out, (size_t)B * 4, cudaMemcpyDeviceToHost, st));
  HSB_CUDA(h, cudaStreamSynchronize(st));
  return HSB_OK;
}

int hsb_covariance_batch(hsb_handle* h, int level, int B, const float* poses, const float* pts, const int* offsets, int n_shared,
                         float* out_cov_map, float* out_cov_world) {
  if (!h || level < 0 || level >= h->levels || B < 0 || !poses || (!out_cov_map && !out_cov_world)) return HSB_ERR_INVALID_ARG;
  if (B == 0) return HSB_OK;
  DeviceGuard guard(h->device);
  size_t total = offsets ? (size_t)offsets[B] : (size_t)(n_shared > 0 ? n_shared : 0);
  if (total > 0 && !pts) return fail(h, HSB_ERR_INVALID_ARG, "points pointer is NULL");
  int s;
  if ((s = ensure(h, h->d_hints, (size_t)B * 12)) != HSB_OK) return s;
  if ((s = ensure(h, h->d_pts, total * 8 + 16)) != HSB_OK) return s;
  if ((s = ensure(h, h->d_offsets, (size_t)(B + 1) * 4)) != HSB_OK) return s;
  if ((s = ensure(h, h->d_cov, (size_t)B * 72)) != HSB_OK) return s;
  cudaStream_t st = h->stream;
  HSB_CUDA(h, cudaMemcpyAsync(h->d_hints.p, poses, (size_t)B * 12, cudaMemcpyHostToDevice, st));
  if (total > 0) HSB_CUDA(h, cudaMemcpyAsync(h->d_pts.p, pts, total * 8, cudaMemcpyHostToDevice, st));
  if (offsets) HSB_CUDA(h, cudaMemcpyAsync(h->d_offsets.p, offsets, (size_t)(B + 1) * 4, cudaMemcpyHostToDevice, st));
  HsbLevelDev L;
  fill_level_dev(h, level, L);
  const int blocks = std::min(B, h->sm_count * 8);
  const int* d_off = offsets ? static_cast<const int*>(h->d_offsets.p) : nullptr;
  float* d_map = static_cast<float*>(h->d_cov.p);
  float* d_world = d_map + 9 * (size_t)B;
  if (h->gather_mode == HSB_GATHER_TEX)
    hsb::covariance_kernel<hsb::MODE_TEX><<<blocks, 224, 0, st>>>(L, B, static_cast<const float*>(h->d_hints.p),
                                                                  static_cast<const float2*>(h->d_pts.p), d_off,
                                                                  offsets ? 0 : n_shared, h->lv[level].cell_length, d_map, d_world);
  else
    hsb::covariance_kernel<hsb::MODE_LDG><<<blocks, 224, 0, st>>>(L, B, static_cast<const float*>(h->d_hints.p),
                                                                  static_cast<const float2*>(h->d_pts.p), d_off,
                                                                  offsets ? 0 : n_shared, h->lv[level].cell_length, d_map, d_world);
  h->launches++;
  HSB_CUDA(h, cudaGetLastError());
  if (out_cov_map) HSB_CUDA(h, cudaMemcpyAsync(out_cov_map, d_map, (size_t)B * 36, cudaMemcpyDeviceToHost, st));
  if (out_cov_world) HSB_CUDA(h, cudaMemcpyAsync(out_cov_world, d_world, (size_t)B * 36, cudaMemcpyDeviceToHost, st));
  HSB_CUDA(h, cudaStreamSynchronize(st));
  return HSB_OK;
}

static int get_dirty(hsb_handle* h, int level, int which, int rect[4], int reset) {
  if (!h || level < 0 || level >= h->levels || !rect) return HSB_ERR_INVALID_ARG;
  DeviceGuard guard(h->device);
  Level& L = h->lv[level];
  int* src = L.dirty + 4 * which;
  int* pin = reinterpret_cast<int*>(h->h_pin + 60);
  HSB_CUDA(h, cudaMemcpyAsync(pin, src, 4 * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  if (reset) {
    static const int clean[4] = {INT_MAX, INT_MAX, -1, -1};
    HSB_CUDA(h, cudaMemcpyAsync(src, clean, sizeof(clean), cudaMemcpyHostToDevice, h->stream));
  }
  HSB_CUDA(h, cudaStreamSynchronize(h->stream));
  memcpy(rect, pin, 4 * sizeof(int));
  return HSB_OK;
}
int hsb_get_dirty_rect(hsb_handle* h, int level, int rect[4], int reset) { return get_dirty(h, level, 0, rect, reset); }
int hsb_get_mirror_dirty_rect(hsb_handle* h, int level, int rect[4], int reset) { return get_dirty(h, level, 1, rect, reset); }

// All levels' replication rectangles with one copy and one synchronize (levels x 4 ints).
int hsb_get_dirty_rects(hsb_handle* h, int* rects, int reset) {
  if (!h || !rects) return HSB_ERR_INVALID_ARG;
  DeviceGuard guard(h->device);
  int all[HSB_MAX_LEVELS * 8];
  HSB_CUDA(h, cudaMemcpyAsync(all, h->d_dirty_all, sizeof(all), cudaMemcpyDeviceToHost, h->stream));
  HSB_CUDA(h, cudaStreamSynchronize(h->stream));
  for (int l = 0; l < h->levels; ++l) memcpy(rects + 4 * l, all + 8 * l, 4 * sizeof(int));
  if (reset) {
    for (int l = 0; l < h->levels; ++l) {
      all[8 * l + 0] = all[8 * l + 1] = INT_MAX;
      all[8 * l + 2] = all[8 * l + 3] = -1;
    }
    HSB_CUDA(h, cudaMemcpyAsync(h->d_dirty_all, all, sizeof(all), cudaMemcpyHostToDevice, h->stream));
    HSB_CUDA(h, cudaStreamSynchronize(h->stream));
  }
  return HSB_OK;
}

// Stream ordering of the rectangle transport (ADVICE r01): the handle's own work runs on private non-blocking
// streams (h->stream for map writes and single-scan calls, copy_stream[] for the host-buffer batch calls), the
// caller's `stream` is a different one.  pack: reads the log-odds after everything queued on h->stream, and the next
// map write waits for the read.  unpack: writes log-odds / probabilities / texture twin after everything queued on
// the handle's streams (earlier matches may still be reading them), and whatever the handle queues next waits for it.
static int order_before(hsb_handle* h, cudaStream_t user, bool all_streams) {
  HSB_CUDA(h, cudaEventRecord(h->ev_sync[0], h->stream));
  HSB_CUDA(h, cudaStreamWaitEvent(user, h->ev_sync[0], 0));
  if (all_streams)
    for (int i = 0; i < 2; ++i) {
      HSB_CUDA(h, cudaEventRecord(h->ev_sync[1 + i], h->copy_stream[i]));
      HSB_CUDA(h, cudaStreamWaitEvent(user, h->ev_sync[1 + i], 0));
    }
  return HSB_OK;
}
static int order_after(hsb_handle* h, cudaStream_t user, bool all_streams) {
  HSB_CUDA(h, cudaEventRecord(h->ev_sync[3], user));
  HSB_CUDA(h, cudaStreamWaitEvent(h->stream, h->ev_sync[3], 0));
  if (all_streams)
    for (int i = 0; i < 2; ++i) HSB_CUDA(h, cudaStreamWaitEvent(h->copy_stream[i], h->ev_sync[3], 0));
  return HSB_OK;
}

int hsb_pack_rect_device(hsb_handle* h, int level, const int rect[4], float* d_buf, void* stream) {
  if (!h || level < 0 || level >= h->levels || !rect || !d_buf) return HSB_ERR_INVALID_ARG;
  DeviceGuard guard(h->device);
  Level& L = h->lv[level];
  int s = check_rect(h, L, rect);
  if (s != HSB_OK) return s;
  const int w = rect[2] - rect[0] + 1, hgt = rect[3] - rect[1] + 1;
  const size_t n = (size_t)w * hgt;
  int blocks = (int)std::min<size_t>((n + 255) / 256, (size_t)h->sm_count * 16);
  if ((s = order_before(h, (cudaStream_t)stream, false)) != HSB_OK) return s;
  hsb::pack_rect_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(L.logodds, L.sx, rect[0], rect[1], w, hgt, d_buf);
  h->launches++;
  HSB_CUDA(h, cudaGetLastError());
  return order_after(h, (cudaStream_t)stream, false);
}

int hsb_unpack_rect_device(hsb_handle* h, int level, const int rect[4], const float* d_buf, void* stream) {
  if (!h || level < 0 || level >= h->levels || !rect || !d_buf) return HSB_ERR_INVALID_ARG;
  DeviceGuard guard(h->device);
  Level& L = h->lv[level];
  int s = check_rect(h, L, rect);
  if (s != HSB_OK) return s;
  const int w = rect[2] - rect[0] + 1, hgt = rect[3] - rect[1] + 1;
  const size_t n = (size_t)w * hgt;
  int blocks = (int)std::min<size_t>((n + 255) / 256, (size_t)h->sm_count * 16);
  if ((s = order_before(h, (cudaStream_t)stream, true)) != HSB_OK) return s;
  hsb::unpack_rect_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(L.logodds, L.prob, L.surf, L.sx, rect[0], rect[1], w, hgt,
                                                                    d_buf, L.dirty + 4);
  h->launches++;
  HSB_CUDA(h, cudaGetLastError());
  return order_after(h, (cudaStream_t)stream, true);
}

static void fill_tile_params(hsb_handle* h, HsbTileParams& T, float* d_buf, size_t capacity_bytes) {
  memset(&T, 0, sizeof(T));
  T.levels = h->levels;
  for (int l = 0; l < h->levels; ++l) {
    Level& L = h->lv[l];
    T.lv[l].logodds = L.logodds;
    T.lv[l].prob = L.prob;
    T.lv[l].surf = L.surf;
    T.lv[l].sx = L.sx;
    T.lv[l].sy = L.sy;
    T.lv[l].dirty = L.dirty;
  }
  T.buf = d_buf;
  T.capacity_words = (unsigned)std::min<size_t>(capacity_bytes / 4, 0xffffffffu);
  T.error_count = h->d_dirty_all + HSB_MAX_LEVELS * 8;
}

int hsb_pack_dirty_device(hsb_handle* h, float* d_buf, size_t capacity_bytes, int reset, void* stream) {
  if (!h || !d_buf || capacity_bytes < HSB_TILE_HEADER_WORDS * 4) return HSB_ERR_INVALID_ARG;
  DeviceGuard guard(h->device);
  HsbTileParams T;
  fill_tile_params(h, T, d_buf, capacity_bytes);
  T.reset = reset;
  int s;
  if ((s = order_before(h, (cudaStream_t)stream, false)) != HSB_OK) return s;
  hsb::pack_dirty_kernel<<<h->sm_count * 4, 256, 0, (cudaStream_t)stream>>>(T);
  if (reset) hsb::reset_dirty_kernel<<<1, 4 * HSB_MAX_LEVELS, 0, (cudaStream_t)stream>>>(T);
  h->launches += reset ? 2 : 1;
  HSB_CUDA(h, cudaGetLastError());
  return order_after(h, (cudaStream_t)stream, false);
}

int hsb_unpack_dirty_device(hsb_handle* h, const float* d_buf, size_t capacity_bytes, void* stream) {
  if (!h || !d_buf || capacity_bytes < HSB_TILE_HEADER_WORDS * 4) return HSB_ERR_INVALID_ARG;
  DeviceGuard guard(h->device);
  HsbTileParams T;
  fill_tile_params(h, T, const_cast<float*>(d_buf), capacity_bytes);
  int s;
  if ((s = order_before(h, (cudaStream_t)stream, true)) != HSB_OK) return s;
  hsb::unpack_dirty_kernel<<<h->sm_count * 4, 256, 0, (cudaStream_t)stream>>>(T);
  h->launches++;
  HSB_CUDA(h, cudaGetLastError());
  return order_after(h, (cudaStream_t)stream, true);
}

int hsb_get_replication_overflows(hsb_handle* h, int* count, int reset) {
  if (!h || !count) return HSB_ERR_INVALID_ARG;
  DeviceGuard guard(h->device);
  int* d = h->d_dirty_all + HSB_MAX_LEVELS * 8;
  HSB_CUDA(h, cudaDeviceSynchronize());
  HSB_CUDA(h, cudaMemcpy(count, d, sizeof(int), cudaMemcpyDeviceToHost));
  if (reset) HSB_CUDA(h, cudaMemset(d, 0, sizeof(int)));
  return HSB_OK;
}

int hsb_raycast_batch(hsb_handle* h, int level, int B, const int* begin_cells, const int* end_cells, float* out_dist,
                      int* out_hit) {
  if (!h || level < 0 || level >= h->levels || B < 0 || !begin_cells || !end_cells || !out_dist) return HSB_ERR_INVALID_ARG;
  if (B == 0) return HSB_OK;
  DeviceGuard guard(h->device);
  Level& L = h->lv[level];
  int s;
  if ((s = ensure(h, h->d_pts, (size_t)B * 16 + 16)) != HSB_OK) return s;      // begin | end
  if ((s = ensure(h, h->d_poses, (size_t)B * 12 + 16)) != HSB_OK) return s;    // dist | hit
  cudaStream_t st = h->stream;
  int2* d_begin = static_cast<int2*>(h->d_pts.p);
  int2* d_end = d_begin + B;
  float* d_dist = static_cast<float*>(h->d_poses.p);
  int2* d_hit = reinterpret_cast<int2*>(d_dist + ((B + 1) & ~1));
  HSB_CUDA(h, cudaMemcpyAsync(d_begin, begin_cells, (size_t)B * 8, cudaMemcpyHostToDevice, st));
  HSB_CUDA(h, cudaMemcpyAsync(d_end, end_cells, (size_t)B * 8, cudaMemcpyHostToDevice, st));
  int blocks = std::min((B + 7) / 8, h->sm_count * 8);
  hsb::raycast_kernel<<<blocks, 256, 0, st>>>(L.logodds, L.sx, L.sy, B, d_begin, d_end, d_dist, out_hit ? d_hit : nullptr);
  h->launches++;
  HSB_CUDA(h, cudaGetLastError());
  HSB_CUDA(h, cudaMemcpyAsync(out_dist, d_dist, (size_t)B * 4, cudaMemcpyDeviceToHost, st));
  if (out_hit) HSB_CUDA(h, cudaMemcpyAsync(out_hit, d_hit, (size_t)B * 8, cudaMemcpyDeviceToHost, st));
  HSB_CUDA(h, cudaStreamSynchronize(st));
  return HSB_OK;
}

int hsb_get_map_origin(const hsb_handle* h, int level, float out[2]) {
  if (!h || level < 0 || level >= h->levels || !out) return HSB_ERR_INVALID_ARG;
  // HectorMappingRos::setServiceGetMapData (HectorMappingRos.cpp:546-550): getWorldCoords(0, 0) - cellLength * 0.5f
  float wx, wy;
  affine_apply_host(h->lv[level].wtm, 0.0f, 0.0f, &wx, &wy);
  volatile float half = h->lv[level].cell_length * 0.5f;
  volatile float ox = wx - half, oy = wy - half;
  out[0] = ox;
  out[1] = oy;
  return HSB_OK;
}

int hsb_get_dist_batch(hsb_handle* h, int level, int B, const float* begin_world, const float* end_world, float* out_dist,
                       float* out_hit_world, int* out_found) {
  if (!h || level < 0 || level >= h->levels || B < 0 || !begin_world || !end_world || !out_dist) return HSB_ERR_INVALID_ARG;
  if (B == 0) return HSB_OK;
  DeviceGuard guard(h->device);
  Level& L = h->lv[level];
  int s;
  if ((s = ensure(h, h->d_pts, (size_t)B * 16 + 16)) != HSB_OK) return s;      // begin | end
  if ((s = ensure(h, h->d_poses, (size_t)B * 16 + 16)) != HSB_OK) return s;    // dist | hit (2) | found
  cudaStream_t st = h->stream;
  float2* d_begin = static_cast<float2*>(h->d_pts.p);
  float2* d_end = d_begin + B;
  float2* d_hit = static_cast<float2*>(h->d_poses.p);
  float* d_dist = reinterpret_cast<float*>(d_hit + B);
  int* d_found = reinterpret_cast<int*>(d_dist + B);
  HSB_CUDA(h, cudaMemcpyAsync(d_begin, begin_world, (size_t)B * 8, cudaMemcpyHostToDevice, st));
  HSB_CUDA(h, cudaMemcpyAsync(d_end, end_world, (size_t)B * 8, cudaMemcpyHostToDevice, st));
  float origo[2];
  hsb_get_map_origin(h, level, origo);
  volatile float inv_scale = 1.0f / L.cell_length;   // CoordinateTransformer::setTransforms, HectorMapTools.h:64
  int blocks = std::min((B + 7) / 8, h->sm_count * 8);
  hsb::getdist_kernel<<<blocks, 256, 0, st>>>(L.logodds, L.sx, L.sy, B, origo[0], origo[1], L.cell_length, inv_scale, d_begin, d_end,
                                              d_dist, out_hit_world ? d_hit : nullptr, out_found ? d_found : nullptr);
  h->launches++;
  HSB_CUDA(h, cudaGetLastError());
  HSB_CUDA(h, cudaMemcpyAsync(out_dist, d_dist, (size_t)B * 4, cudaMemcpyDeviceToHost, st));
  if (out_hit_world) HSB_CUDA(h, cudaMemcpyAsync(out_hit_world, d_hit, (size_t)B * 8, cudaMemcpyDeviceToHost, st));
  if (out_found) HSB_CUDA(h, cudaMemcpyAsync(out_found, d_found, (size_t)B * 4, cudaMemcpyDeviceToHost, st));
  HSB_CUDA(h, cudaStreamSynchronize(st));
  return HSB_OK;
}

void* hsb_level_logodds_device_ptr(hsb_handle* h, int level) {
  if (!h || level < 0 || level >= h->levels) return nullptr;
  return h->lv[level].logodds;
}

int hsb_refresh_level(hsb_handle* h, int level, void* stream) {
  if (!h || level < 0 || level >= h->levels) return HSB_ERR_INVALID_ARG;
  DeviceGuard guard(h->device);
  return refresh_level(h, level, (cudaStream_t)stream);
}

}  // extern "C"
