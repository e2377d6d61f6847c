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
#include <memory>
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
                         // [0..3] for replication (hsb_get_dirty_rect), [4..7] for host mirrors (hsb_get_mirror_dirty_rect)
                         // — and the cleared flag [8] (HSB_DIRTY_WORDS); points into hsb_handle::d_dirty_all
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

// Pose, write-the-map flag and covariance of a single-scan match or SLAM step, in the order one copy moves them
struct PoseResult {
  float pose[3];
  float flag;     // the step's gate decision (unused by hsb_match_data)
  float cov[9];
};

// The single-scan calls' mapped pinned block (hsb_handle::h_pin): what their kernels write, or their copies bring, for
// the host.  Every slot is written and read by calls on the handle's stream.
struct PinnedSlots {
  PoseResult match;    // hsb_match_data
  PoseResult step;     // the SLAM steps
  unsigned step_seq;   // a nowait step's sequence number, published once `step` and step_kept are in place
  int step_kept;       // a converted step's kept-endpoint count
  int conv_kept;       // the stand-alone conversions' kept-endpoint count
  float hessian[12];   // hsb_hessian_derivs: H row-major, then dTr
  float gate[4];       // the gate state on its way to or from the device: lastMapUpdatePose, write flag
  int dirty[HSB_DIRTY_WORDS];   // a level's rectangles and cleared flag on their way to the host
};

// The single-scan calls' device block (hsb_handle::d_scratch)
struct DeviceSlots {
  PoseResult match;    // hsb_match_data with tuning host_out = 0
  PoseResult step;     // a SLAM step's pose and flag, which its map write reads (with host_out = 0 also its covariance)
  int step_kept;       // a converted step's kept-endpoint count, which its map write reads
  int conv_kept;       // the stand-alone conversions' kept-endpoint count
  float hessian[12];   // hsb_hessian_derivs
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
  DevBuf d_pts;
  DeviceSlots* d_scratch = nullptr;
  // "containers of the last match" (MapRepMultiMap::dataContainers) and the update scan
  DevBuf d_last_pts, d_upd_pts;   // single-scan buffers: 16 floats of header (hint, gate inputs), then the points
  float* h_stage = nullptr;       // pinned staging for the single-scan calls (header + points, one H2D per call)
  size_t h_stage_bytes = 0;
  // raw-range input (N2)
  DevBuf d_beam_cs, d_occ;
  hsb_scan_format fmt = hsb_scan_format();
  bool fmt_set = false;
  hsb_cloud_format cfmt = hsb_cloud_format();
  bool cfmt_set = false;
  DevBuf d_conv_in, d_cloud_tf;   // the stand-alone conversions' input (ranges or cloud) and laser transform
  DevBuf d_proj_unit;   // laser_geometry's unit vectors, n_beams x double (cos, sin)
  hsb_laser_projection proj = hsb_laser_projection();
  bool proj_set = false;
  DevBuf d_fused_in;   // the fused single SLAM steps' upload: header, (laser transform,) cloud or ranges
  int last_n = 0;
  float last_origo[2] = {0.f, 0.f};
  // pinned host scratch
  PinnedSlots* h_pin = nullptr;       // mapped: kernels of the single-scan calls write their results here
  PinnedSlots* h_pin_dev = nullptr;   // device alias of h_pin
  int shape_batch = 0;           // > 0: pick the launch shape for this batch size instead of the launch's own (pipelined host calls)
  int tune_host_out = 1;         // single-scan calls: kernels write results into mapped host memory (no D2H copy)
  int tune_inline_scan = 0;      // 1: single-scan calls send the scan in the kernel parameters (no H2D copy operation) — measured slower, see match_kernel.cuh
  hsb::InlineScan<true> inline_scan;   // host image of those parameters
  cudaEvent_t ev_time[2] = {nullptr, nullptr};   // timing events around K2 (tuning "time_update")
  int tune_time_update = 0;
  BatchSet bset[2];             // device staging of the host-buffer batch calls, alternating between calls
  int next_set = 0;
  int* d_dirty_all = nullptr;   // HSB_MAX_LEVELS x HSB_DIRTY_WORDS ints (see Level::dirty), then kOverflowWord's 4
  uint64_t d2h_bytes = 0;       // bytes the plane / rectangle download entry points copied to the host (diagnostic)
  cudaEvent_t ev_sync[4] = {nullptr, nullptr, nullptr, nullptr};   // ordering of caller streams against the handle's own
  float* d_gate = nullptr;   // SLAM steps: lastMapUpdatePose[3], write-the-map flag
  float min_dist = 0.4f, min_angle = 0.13f;   // HectorSlamProcessor.h:62-63 defaults
  // tuning
  int tune_warps_per_scan = 0, tune_scans_per_block = 0, tune_stage_smem = 1, tune_chunk = 0, tune_unroll = 0, tune_packed = 0, tune_seq = 0, tune_partial = 1, tune_prefetch = 0, tune_trace = 0, tune_pace = 0, tune_pdl = 1, tune_auto_group = 1, tune_stagger = 0, tune_fixpoint = 1;
  int tune_occ_chunk = 0;   // > 0: staging bytes per chunk of a group occupancy sync whose handles[0] this is
  DevBuf d_trace;
  DevBuf d_best;   // arg-max accumulator of hsb_best_hypothesis_device
  DevBuf d_record; // per-evaluation record of hsb_match_data_record
  bool map_write_pending = false;   // a nowait SLAM step's map write may still be running on `stream`
  // group steps (hsb_group_slam_update) run on the group's stream: the event of the last nowait step this handle took
  // part in, which the handle's stream waits on before its next own operation (HandleScope) ...
  cudaEvent_t group_ev = nullptr;
  // ... and whether the handle may have queued work of its own since its last group step, which that step then waits for
  bool queued = false;
  unsigned step_seq = 0;   // sequence number of the fused SLAM steps (host polling, hsb_slam_update_nowait)
  int trace_scans = 0;
  // step record (hsb_set_step_record): R floats of mapped pinned memory the match of every fused step writes the
  // record into while the switch is on, published with the step's pose.  step_rec_matched: the last fused step ran a
  // match with the switch on (its record is in h_step_rec); stepped: a fused step has run on the handle
  float* h_step_rec = nullptr;
  float* h_step_rec_dev = nullptr;   // device alias of h_step_rec
  bool step_rec_on = false, step_rec_matched = false, stepped = false;
  bool have_last_match = false;   // the last-match container holds a scan (hsb_get_last_match_scan)
  int last_shape[6] = {0, 0, 0, 0, 0, 0};  // W, G, U, staged points per scan (0 = none), grid, resident CTAs / SM
  uint64_t launches = 0;
  std::string err;
};

namespace {

// hsb_handle::d_dirty_all: the replication overflow counter (hsb_get_replication_overflows) behind the levels' words
constexpr int kOverflowWord = HSB_MAX_LEVELS * HSB_DIRTY_WORDS;

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

// Every entry point that works on a handle's streams opens one of these: it selects the handle's device and orders the
// handle's stream behind the last nowait group step the handle took part in.  A group step records ONE event instead of
// making each member's streams wait on it; a member waits here, lazily, before its next own operation (and a member that
// takes only group steps never waits).  It also notes that the handle may now have work of its own queued, which its
// next group step orders itself behind.
struct HandleScope {
  DeviceGuard dev;
  explicit HandleScope(hsb_handle* h) : dev(h->device) {
    if (h->group_ev) {
      // (a failure here is the context's: the next CUDA call of the entry point reports it)
      cudaStreamWaitEvent(h->stream, h->group_ev, 0);
      h->group_ev = nullptr;
    }
    h->queued = true;
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

// Pinned host staging `p` of `cap` bytes grown to hold `bytes` (the contents are not kept).
template <typename T>
int ensure_pinned(hsb_handle* h, T*& p, size_t& cap, size_t bytes) {
  if (bytes <= cap) return HSB_OK;
  if (p) cudaFreeHost(p);
  p = nullptr;
  cap = 0;
  const size_t want = bytes < (64u << 10) ? (64u << 10) : bytes * 2;
  HSB_CUDA(h, cudaMallocHost(reinterpret_cast<void**>(&p), want));
  cap = want;
  return HSB_OK;
}

// A nowait step's return: spin until the device has published `value` in the mapped word `seq` (the step's results are
// in host memory then), checking every 4096 polls that `st` has neither failed nor finished without publishing.
int wait_published(hsb_handle* h, volatile unsigned* seq, unsigned value, cudaStream_t st, const char* unpublished) {
  unsigned spins = 0;
  while (*seq != value) {
    if ((++spins & 0xfffu) == 0) {
      cudaError_t e = cudaStreamQuery(st);
      if (e != cudaSuccess && e != cudaErrorNotReady) return fail(h, HSB_ERR_CUDA, "stream failed: %s", cudaGetErrorString(e));
      if (e == cudaSuccess && *seq != value) return fail(h, HSB_ERR_CUDA, "%s", unpublished);
    }
  }
  __sync_synchronize();
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

// both dirty rectangles of a level := the whole level (after a reset or an upload every cell may differ), cleared flag 0:
// the next pack ships the whole level's rows
int mark_level_dirty(hsb_handle* h, int level, cudaStream_t st) {
  Level& L = h->lv[level];
  if (!L.dirty) return HSB_OK;
  const int full[HSB_DIRTY_WORDS] = {0, 0, L.sx - 1, L.sy - 1, 0, 0, L.sx - 1, L.sy - 1, 0};
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
  d.rec_off = 0;   // the record holds the levels coarsest first
  for (int k = h->levels - 1; k > l; --k) d.rec_off += 3 + 15 * h->lv[k].evals;
}

// ---- match launch -----------------------------------------------------------------------------
constexpr size_t kMaxDynSmem = 232448;   // dynamic shared memory one CTA may ask for (227 KB)

// shared-memory slots that stage a whole scan of n points: n + head padding, even
inline int whole_scan_slots(int n) { return ((n + 1) + 1) & ~1; }

// whether Gr groups of the <W, G> match kernel can each stage `cap` slots in one CTA
template <int W, int G>
bool staging_fits(int cap, int Gr) {
  return hsb::MatchSmem<W, G>::kHeaderBytes + (size_t)Gr * cap * 8 <= kMaxDynSmem;
}

int fail_fused_too_long(hsb_handle* h, int max_n) {
  return fail(h, HSB_ERR_UNSUPPORTED, "scan too long for the fused conversion (%d points)", max_n);
}

template <int W, int G, int MODE, int U, bool PACK, bool INL = false, int GRP = hsb::GRP_NONE, bool PROJ = false>
int launch_match_t(hsb_handle* h, HsbMatchParams& P, int max_n, cudaStream_t st, int Gr,
                   const hsb::InlineScan<INL>& S = hsb::InlineScan<INL>()) {
  // launch_match's one-wave path passes its group count to a G > 1 kernel: one CTA per SM, one warp per scan
  const bool one_wave_groups = G > 1 && Gr > 0;
  if (Gr <= 0 || Gr > G) Gr = G;   // groups per CTA actually launched (a G-group kernel runs with fewer: see launch_match)
  const size_t header = hsb::MatchSmem<W, G>::kHeaderBytes;
  auto kern = hsb::match_kernel<W, G, MODE, U, PACK, INL, GRP, PROJ>;
  constexpr size_t kMaxDyn = kMaxDynSmem;
  constexpr int gt = W * 32;           // threads per scan
  int cap = 0;
  const bool fused = P.kind != HSB_IN_ENDPOINTS || INL;   // conversion / inline scan: the whole scan must be staged
  if (h->tune_stage_smem || fused) cap = whole_scan_slots(max_n);
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
  // A staged PREFIX is allowed — except on the one-wave path: there the CTA's scans, when they do not fit whole, are not
  // staged at all.  A prefix of each of ~32 scans fills the SM's shared memory and leaves L1 about 28 KB for the map
  // gathers of all of them; unstaged, L1 keeps nearly all 256 KB, and the gathers that miss it and the endpoints read
  // through it cost less than the prefix saves (DESIGN.md §4, scan staging).
  const bool may_split = h->tune_partial && !PACK && !fused && !one_wave_groups;
  if (cap > 0 && !staging_fits<W, G>(cap, Gr)) {        // the CTA's scans do not fit whole
    if (fused) return fail_fused_too_long(h, max_n);
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
  P.fixpoint = h->tune_fixpoint;
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
  // (hsb_set_tuning refuses the key above HSB_TRACE_MAX_LEVELS; a launch with more levels, whichever handle's tuning
  // it runs under, gets no trace pointer, so the kernel's stores cannot leave a scan's 8 slots)
  if (h->tune_trace && P.levels <= HSB_TRACE_MAX_LEVELS) {
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

// Projected input (HSB_IN_PROJECTED): whether the match kernel is compiled with the projection (match_kernel PROJ) for
// the launch shape W warps per scan, G scans per CTA, U gathers in flight.  The shapes are the ones launch_match selects
// for a converted batch under the default tuning — W in {1, 2, 4, 8}, one scan per CTA (a converted batch never takes
// the auto-group path), 4 gathers in flight, unpacked — so a projected batch matches in the shape a cloud batch of the
// same size takes.
bool has_projected_kernel(const hsb_handle* h, int W, int G, int U) {
  return (W == 1 || W == 2 || W == 4 || W == 8) && G == 1 && U == 4 && !(h->gather_mode == HSB_GATHER_TEX && h->tune_packed);
}

// The entry points reject a tuning without a projected kernel before they queue anything (check_projected_tuning);
// this is the launcher's own guard.
int launch_match_projected(hsb_handle* h, HsbMatchParams& P, int max_n, cudaStream_t st, int W, int G, int U) {
  if (has_projected_kernel(h, W, G, U)) {
    const bool tex = h->gather_mode == HSB_GATHER_TEX;
#define HSB_PROJ_CASE(w)                                                                                     \
  if (W == w)                                                                                                \
    return tex ? launch_match_t<w, 1, hsb::MODE_TEX, 4, false, false, hsb::GRP_NONE, true>(h, P, max_n, st, 1) \
               : launch_match_t<w, 1, hsb::MODE_LDG, 4, false, false, hsb::GRP_NONE, true>(h, P, max_n, st, 1);
    HSB_PROJ_CASE(1);
    HSB_PROJ_CASE(2);
    HSB_PROJ_CASE(4);
    HSB_PROJ_CASE(8);
#undef HSB_PROJ_CASE
  }
  return fail(h, HSB_ERR_UNSUPPORTED, "no projected-scan kernel for tuning warps_per_scan=%d scans_per_block=%d unroll=%d",
              W, G, U);
}

// Warps per scan of a batch of B scans under the default tuning: one warp per scan as soon as the batch fills the chip,
// more warps per scan for small batches, never more than 8 (the per-evaluation reduction / barrier cost grows with the
// group size).
int auto_warps_per_scan(const hsb_handle* h, long B) {
  const long want = ((long)h->sm_count * 24) / (B > 0 ? B : 1);
  int W = 1;
  while (W * 2 <= want && W < 8) W *= 2;
  return W;
}

int launch_match(hsb_handle* h, HsbMatchParams& P, int max_n, cudaStream_t st) {
  if (h->map_write_pending && st != h->stream) {
    // hsb_slam_update_nowait left a map write running on the handle's stream: a match on another stream waits for it
    HSB_CUDA(h, cudaEventRecord(h->ev_sync[0], h->stream));
    HSB_CUDA(h, cudaStreamWaitEvent(st, h->ev_sync[0], 0));
  }
  int W = h->tune_warps_per_scan, G = h->tune_scans_per_block;
  if (W <= 0) {
    // (a pipelined host-batch call passes ONE size for all its chunks: a scan's result must not depend on the
    // chunk it happens to travel in — the reduction order follows the shape — so that results are invariant
    // under a permutation of the batch, as the reference's are)
    W = auto_warps_per_scan(h, h->shape_batch > 0 ? h->shape_batch : P.B);
  }
  int Gr = 0;   // 0: as many groups per CTA as the instantiation has
  if (G <= 0) {
    G = 1;
    // One-wave batches of one-warp scans (tuning "auto_group", on by default): ONE CTA per SM holding ceil(B / SMs) <= 32
    // scans instead of one-warp CTAs.  One CTA pays the 1 KB per-CTA shared-memory reservation once, so up to 26 scans
    // per SM can be staged whole at full residency (more are not staged: launch_match_t), and its warps start and end
    // together.  Up to 28 scans per SM the 28-group
    // kernel runs (72 registers, the one-warp kernel's budget); up to 32 the 32-group kernel (1024 threads, 64 registers),
    // which keeps the benchmark's 4096 scans in one wave on a 132-SM H100 where 28 per SM would leave a second wave.
    // Larger batches keep one scan per CTA: finished warps are replaced at once there, which a CTA-wide drain would
    // prevent.  With one warp per scan the reduction order does not depend on the CTA shape: results are the same bits.
    const long Bs = h->shape_batch > 0 ? h->shape_batch : P.B;
    if (h->tune_auto_group && W == 1 && P.kind == HSB_IN_ENDPOINTS && std::max<long>(Bs, P.B) <= (long)h->sm_count * 32 &&
        (h->tune_unroll == 0 || h->tune_unroll == 4)) {
      Gr = (int)((Bs + h->sm_count - 1) / h->sm_count);
      G = Gr <= 28 ? 28 : 32;
    }
  }
  int U = h->tune_unroll > 0 ? h->tune_unroll : 4;
  if (P.kind == HSB_IN_PROJECTED) return launch_match_projected(h, P, max_n, st, W, G, U);
  if (h->gather_mode == HSB_GATHER_TEX) return launch_match_mode<hsb::MODE_TEX>(h, P, max_n, st, W, G, U, Gr);
  return launch_match_mode<hsb::MODE_LDG>(h, P, max_n, st, W, G, U, Gr);
}

// Whether a single scan of n endpoints (hsb_match_data, hsb_slam_update) travels INSIDE the kernel parameters
// (match_kernel.cuh InlineScan): tuning "inline_scan", and a tuning that leaves the single scan its usual shape.
bool inline_scan_applies(const hsb_handle* h, int n) {
  return h->tune_inline_scan && n <= HSB_INLINE_MAX_POINTS && (h->tune_warps_per_scan == 0 || h->tune_warps_per_scan == 8) &&
         h->tune_scans_per_block <= 1 && (h->tune_unroll == 0 || h->tune_unroll == 4) && !h->tune_packed && h->tune_seq <= 1;
}

// The single-scan match of hsb_match_data and the SLAM steps on the handle's stream: P describes one scan of P.n_shared
// inputs staged on the device.  With `inl` (inline_scan_applies) the host's header (nh floats) and endpoints are sent in
// the kernel parameters instead, in the shape a single scan always takes (8 warps, 4 gathers in flight), so results
// equal the staged path's; the kernel writes the endpoints to P.pts, where the map writer reads them.
int launch_match_single(hsb_handle* h, HsbMatchParams& P, bool inl, const float* header, int nh, const float* pts) {
  const int n = P.n_shared;
  if (!inl) return launch_match(h, P, n, h->stream);
  hsb::InlineScan<true>& S = h->inline_scan;
  memset(S.header, 0, sizeof(S.header));
  if (nh > 0) memcpy(S.header, header, (size_t)nh * sizeof(float));
  if (n > 0) memcpy(S.pts, pts, (size_t)n * 8);
  P.conv.out_pts = const_cast<float2*>(P.pts);
  P.hints = nullptr;
  P.pts = nullptr;
  if (h->gather_mode == HSB_GATHER_TEX) return launch_match_t<8, 1, hsb::MODE_TEX, 4, false, true>(h, P, n, h->stream, 1, S);
  return launch_match_t<8, 1, hsb::MODE_LDG, 4, false, true>(h, P, n, h->stream, 1, S);
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

// lastMapUpdatePose = FLT_MAX^3 (HectorSlamProcessor.h:117), write flag 0
int reset_gate(hsb_handle* h) {
  const float init[4] = {FLT_MAX, FLT_MAX, FLT_MAX, 0.f};
  memcpy(h->h_pin->gate, init, sizeof(init));
  HSB_CUDA(h, cudaMemcpyAsync(h->d_gate, h->h_pin->gate, sizeof(init), cudaMemcpyHostToDevice, h->stream));
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
  HandleScope guard(h);
  HSB_CUDA(h, cudaEventSynchronize(h->ev_time[1]));
  HSB_CUDA(h, cudaEventElapsedTime(ms, h->ev_time[0], h->ev_time[1]));
  return HSB_OK;
}

int hsb_read_trace(hsb_handle* h, uint64_t* out, int max_scans) {
  if (!h || !out || max_scans < 0) return HSB_ERR_INVALID_ARG;
  HandleScope guard(h);
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
  HandleScope guard(h);
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
  HSB_CUDA_C(cudaMalloc(&h->d_dirty_all, (kOverflowWord + 4) * sizeof(int)));
  HSB_CUDA_C(cudaMemset(h->d_dirty_all, 0, (kOverflowWord + 4) * sizeof(int)));
  HSB_CUDA_C(cudaHostAlloc(&h->h_pin, sizeof(PinnedSlots), cudaHostAllocMapped));
  HSB_CUDA_C(cudaHostGetDevicePointer(&h->h_pin_dev, h->h_pin, 0));
  // pinned memory comes back from earlier allocations with their contents: a nowait step polls step_seq for its
  // sequence number (1, 2, ...), which must not be there before the step publishes it
  memset(h->h_pin, 0, sizeof(PinnedSlots));
  HSB_CUDA_C(cudaMalloc(&h->d_scratch, sizeof(DeviceSlots)));
  HSB_CUDA_C(cudaMalloc(&h->d_gate, 4 * sizeof(float)));

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
    L.dirty = h->d_dirty_all + HSB_DIRTY_WORDS * l;
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
    int clean[kOverflowWord];
    for (int i = 0; i < kOverflowWord; ++i) {
      const int w = i % HSB_DIRTY_WORDS;
      clean[i] = w == HSB_DIRTY_CLEARED ? 0 : (w & 2) ? -1 : INT_MAX;
    }
    HSB_CUDA_C(cudaMemcpyAsync(h->d_dirty_all, clean, sizeof(clean), cudaMemcpyHostToDevice, h->stream));
  }
  HSB_TRY(reset_gate(h));
  HSB_CUDA_C(cudaStreamSynchronize(h->stream));
#undef HSB_TRY
#undef HSB_CUDA_C
  *out = h;
  return HSB_OK;
}

int hsb_destroy(hsb_handle* h) {
  if (!h) return HSB_OK;
  HandleScope guard(h);
  cudaDeviceSynchronize();
  for (int l = 0; l < HSB_MAX_LEVELS; ++l) destroy_level(h, h->lv[l]);
  DevBuf* bufs[] = {&h->d_pts, &h->d_last_pts, &h->d_upd_pts,
                    &h->d_beam_cs, &h->d_occ, &h->d_trace, &h->d_best, &h->d_record,
                    &h->d_conv_in, &h->d_cloud_tf, &h->d_fused_in, &h->d_proj_unit};
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
  if (h->d_scratch) cudaFree(h->d_scratch);
  if (h->d_gate) cudaFree(h->d_gate);
  for (int i = 0; i < 2; ++i)
    if (h->ev_time[i]) cudaEventDestroy(h->ev_time[i]);
  for (int i = 0; i < 4; ++i)
    if (h->ev_sync[i]) cudaEventDestroy(h->ev_sync[i]);
  if (h->h_pin) cudaFreeHost(h->h_pin);
  if (h->h_step_rec) cudaFreeHost(h->h_step_rec);
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
  if ((s = ensure_pinned(h, h->h_stage, h->h_stage_bytes, bytes)) != HSB_OK) return s;
  memset(h->h_stage, 0, kScanHeaderFloats * sizeof(float));
  if (nh > 0) memcpy(h->h_stage, header, (size_t)nh * sizeof(float));
  if (n > 0) memcpy(h->h_stage + kScanHeaderFloats, pts, (size_t)n * 8);
  HSB_CUDA(h, cudaMemcpyAsync(b.p, h->h_stage, bytes, cudaMemcpyHostToDevice, st));
  return HSB_OK;
}

int hsb_reset(hsb_handle* h) {
  if (!h) return HSB_ERR_INVALID_ARG;
  HandleScope guard(h);
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
  else if (!strcmp(key, "trace")) {
    // a scan's 8-slot record holds the start, one time per level and the end only up to HSB_TRACE_MAX_LEVELS levels
    if (value && h->levels > HSB_TRACE_MAX_LEVELS)
      return fail(h, HSB_ERR_UNSUPPORTED, "hsb_set_tuning: trace records at most %d levels, the handle has %d",
                  HSB_TRACE_MAX_LEVELS, h->levels);
    h->tune_trace = value;
  }
  else if (!strcmp(key, "pace")) h->tune_pace = value;
  else if (!strcmp(key, "time_update")) h->tune_time_update = value;
  else if (!strcmp(key, "pdl")) h->tune_pdl = value;
  else if (!strcmp(key, "auto_group")) h->tune_auto_group = value;
  else if (!strcmp(key, "stagger")) h->tune_stagger = value;
  else if (!strcmp(key, "fixpoint")) h->tune_fixpoint = value;
  else if (!strcmp(key, "occupancy_chunk")) h->tune_occ_chunk = value;
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

}  // extern "C"

// ---- matching ----------------------------------------------------------------------------------

namespace {

// :493 maxRangeForContainer = range_max - 0.1, host fp32
float range_max_c(const hsb_scan_format& f) {
  volatile float mx = f.range_max - 0.1f;
  return mx;
}

// projectLaser: a negative cutoff means the scan's range_max
double projection_cutoff(const hsb_laser_projection& p) { return p.range_cutoff < 0.0 ? (double)p.range_max : p.range_cutoff; }

// The container's origo of a cloud with laser transform T (HectorMappingRos.cpp:516-517):
// Vector2f(laserPos.x(), laserPos.y()) * scaleToMap, host fp32 without contraction
void cloud_origo(const hsb_handle* h, const double* T, float out[2]) {
  volatile float ox = (float)T[3], oy = (float)T[7];
  volatile float sx = ox * h->lv[0].scale, sy = oy * h->lv[0].scale;
  out[0] = sx;
  out[1] = sy;
}

// How h converts a scan of `kind` (not endpoints) at call time; the sink is left null.
void fill_conv(const hsb_handle* h, HsbInputKind kind, HsbConvDev& c) {
  memset(&c, 0, sizeof(c));
  c.scale_to_map = h->lv[0].scale;
  if (kind == HSB_IN_RANGES) {
    c.beam_cs = static_cast<const float2*>(h->d_beam_cs.p);
    c.range_min = h->fmt.range_min;
    c.range_max_c = range_max_c(h->fmt);
    return;
  }
  c.sqr_min_dist = h->cfmt.sqr_laser_min_dist;
  c.sqr_max_dist = h->cfmt.sqr_laser_max_dist;
  c.z_min = h->cfmt.laser_z_min_value;
  c.z_max = h->cfmt.laser_z_max_value;
  if (kind == HSB_IN_PROJECTED) {
    c.proj_unit = static_cast<const double2*>(h->d_proj_unit.p);
    c.range_min = h->proj.range_min;
    c.range_cutoff = projection_cutoff(h->proj);
  }
}

// The scan of n endpoints (converted input: an upper bound until the kept count is known) with container origo `origo`
// (NULL = 0, 0) is the last match's container now (MapRepMultiMap::matchData, MapRepMultiMap.h:127): a later
// updateByScan draws the coarse levels from it (:143).
void record_match(hsb_handle* h, int n, const float origo[2]) {
  h->have_last_match = true;
  h->last_n = n;
  h->last_origo[0] = origo ? origo[0] : 0.f;
  h->last_origo[1] = origo ? origo[1] : 0.f;
}

// One scan of a SLAM step (HectorSlamProcessor::update), as the single and the group steps take it.
struct StepSession {
  float origo[2];     // the container origo
  float gate_in[3];   // minDist, minAngle, map_without_matching
  // where the scan's endpoints go: the last match's container when the scan is matched; without matching the
  // reference leaves that container alone (HectorSlamProcessor.h:77-81, MapRepMultiMap.h:143) and they go to the
  // update-scan buffer
  DevBuf* sink;
  HsbConvDev conv;    // converted input: h's conversion into the sink; zero for endpoints
};

// The session of a step of h on a scan of `kind` with n inputs (converted: an upper bound of the endpoints kept), laser
// transform T (cloud and projected) or caller origo (endpoints; NULL = 0, 0), matched or map_without_matching.  The
// sink is grown to n endpoints; a converted scan's kept count goes to n_dev (device) and, if set, n_host (mapped host).
int step_session(hsb_handle* h, HsbInputKind kind, int n, const double* T, const float origo[2], bool matched, int* n_dev,
                 int* n_host, StepSession& ss) {
  ss.origo[0] = ss.origo[1] = 0.f;
  if (T) cloud_origo(h, T, ss.origo);   // (a LaserScan's origo is zero, HectorMappingRos.cpp:491)
  else if (origo) memcpy(ss.origo, origo, sizeof(ss.origo));
  ss.gate_in[0] = h->min_dist;
  ss.gate_in[1] = h->min_angle;
  ss.gate_in[2] = matched ? 0.f : 1.f;
  ss.sink = matched ? &h->d_last_pts : &h->d_upd_pts;
  const int s = ensure_scan_buf(h, *ss.sink, n);
  if (s != HSB_OK) return s;
  memset(&ss.conv, 0, sizeof(ss.conv));
  if (kind != HSB_IN_ENDPOINTS) {
    fill_conv(h, kind, ss.conv);
    ss.conv.out_pts = reinterpret_cast<float2*>(scan_points(*ss.sink));
    ss.conv.out_n = n_dev;
    ss.conv.out_n_host = n_host;
  }
  return HSB_OK;
}

// A finished session's results: pose and write flag from res (4 floats), the covariance from cov when the session
// matched and had endpoints (`kept`: counted on the device for converted input), and the kept count.  A matched
// scan's container holds exactly the kept endpoints.
void step_results(hsb_handle* h, bool matched, int kept, const float* res, const float* cov, float* out_pose,
                  int* map_updated, float* cov_inout, int* out_kept) {
  memcpy(out_pose, res, 3 * sizeof(float));
  if (map_updated) *map_updated = res[3] != 0.f;
  if (cov_inout && matched && kept > 0) memcpy(cov_inout, cov, 9 * sizeof(float));
  if (out_kept) *out_kept = kept;
  if (matched) h->last_n = kept;
}

// A scan, or a batch of scans, of one input kind.
struct ScanIn {
  HsbInputKind kind;
  const float* in;        // endpoints: xy pairs; cloud: xyz triples; ranges / projected: one range per beam
  const int* offsets;     // B + 1 bounds of the scans in `in`, in points (NULL: every scan has n_shared inputs)
  int n_shared;
  int max_n;              // the longest scan
  const double* tf;       // cloud / projected: B x 12 laser transforms (NULL: the cloud format's)
};

// The match kernel's description of `sc` (device memory): the input, its layout and h's conversion of it.
void fill_scan(const hsb_handle* h, const ScanIn& sc, HsbMatchParams& P) {
  P.kind = sc.kind;
  P.offsets = sc.offsets;
  P.n_shared = sc.offsets ? 0 : sc.n_shared;
  if (sc.kind == HSB_IN_ENDPOINTS) {
    P.pts = reinterpret_cast<const float2*>(sc.in);
    return;
  }
  P.conv_in = sc.in;
  P.cloud_tf = sc.tf;
  memcpy(P.cloud_tf0, h->cfmt.laser_transform, sizeof(P.cloud_tf0));
  fill_conv(h, sc.kind, P.conv);
}

// R of HsbMatchParams::record: floats of one scan's per-evaluation record
int record_floats(const hsb_handle* h) {
  int r = 0;
  for (int l = 0; l < h->levels; ++l) r += 3 + 15 * h->lv[l].evals;
  return r;
}

// The batch match of every input kind on device buffers (the hsb_match_batch*_device calls, and each chunk of the
// host-buffer calls): B scans `sc` with their hints; poses B x 3, covariances B x 9 (or NULL), origo B x 2 (cloud and
// projected, or NULL), per-evaluation records B x R (or NULL).  The caller has checked the arguments.
int match_batch(hsb_handle* h, int B, const float* hints, const ScanIn& sc, float* out_poses, float* out_cov,
                float* out_origo, float* record, cudaStream_t st) {
  HsbMatchParams P;
  fill_match_params(h, P);
  P.B = B;
  P.hints = hints;
  fill_scan(h, sc, P);
  P.out_poses = out_poses;
  P.out_cov = out_cov;
  P.out_origo = out_origo;
  P.record = record;
  P.record_floats = record_floats(h);
  return launch_match(h, P, std::max(sc.max_n, 0), st);
}

int match_endpoints_device(hsb_handle* h, int B, const float* d_hints, const float* d_pts, const int* d_offsets, int n_shared,
                           int max_points_per_scan, float* d_out_poses, float* d_out_cov, float* d_record, void* stream) {
  if (!h || B < 0 || !d_hints || !d_out_poses) return HSB_ERR_INVALID_ARG;
  if (B == 0) return HSB_OK;
  if (!d_offsets && n_shared < 0) return fail(h, HSB_ERR_INVALID_ARG, "shared-scan mode needs n_shared >= 0");
  if (!d_pts && (d_offsets || n_shared > 0)) return fail(h, HSB_ERR_INVALID_ARG, "points pointer is NULL");
  HandleScope guard(h);
  const ScanIn sc = {HSB_IN_ENDPOINTS, d_pts, d_offsets, n_shared, d_offsets ? max_points_per_scan : n_shared, nullptr};
  return match_batch(h, B, d_hints, sc, d_out_poses, d_out_cov, nullptr, d_record, (cudaStream_t)stream);
}

}  // namespace

extern "C" {

int hsb_get_match_record_floats(const hsb_handle* h) { return h ? record_floats(h) : HSB_ERR_INVALID_ARG; }

int hsb_match_batch_device(hsb_handle* h, int B, const float* d_hints, const float* d_pts, const int* d_offsets,
                           int n_shared, int max_points_per_scan, float* d_out_poses, float* d_out_cov, void* stream) {
  return match_endpoints_device(h, B, d_hints, d_pts, d_offsets, n_shared, max_points_per_scan, d_out_poses, d_out_cov,
                                nullptr, stream);
}

int hsb_match_batch_record_device(hsb_handle* h, int B, const float* d_hints, const float* d_pts, const int* d_offsets,
                                  int n_shared, int max_points_per_scan, float* d_out_poses, float* d_out_cov, float* d_record,
                                  void* stream) {
  if (!d_record) return HSB_ERR_INVALID_ARG;
  return match_endpoints_device(h, B, d_hints, d_pts, d_offsets, n_shared, max_points_per_scan, d_out_poses, d_out_cov,
                                d_record, stream);
}

static int match_data_impl(hsb_handle* h, const float hint[3], const float* pts, int n, const float origo[2], float out_pose[3],
                           float cov_inout[9], float* record_out) {
  if (!h || !hint || !out_pose || n < 0 || (n > 0 && !pts)) return HSB_ERR_INVALID_ARG;
  HandleScope guard(h);
  cudaStream_t st = h->stream;
  record_match(h, n, origo);
  // the kernel writes pose + Hessian straight into mapped host memory: no device-to-host copy operation on the
  // critical path (reading the scan from host memory the same way was slower than copying it)
  const bool host_out = h->tune_host_out != 0;
  PoseResult* res = host_out ? &h->h_pin_dev->match : &h->d_scratch->match;
  const int R = record_floats(h);
  float* d_rec = nullptr;
  int s;
  if (record_out) {
    if ((s = ensure(h, h->d_record, (size_t)R * sizeof(float))) != HSB_OK) return s;
    d_rec = static_cast<float*>(h->d_record.p);
  }
  // the scan goes into the container of the last match (header [0..2] = hint) — or in with the launch itself
  // (inline_scan): no host-to-device copy operation either
  const bool inl = inline_scan_applies(h, n);
  if ((s = inl ? ensure_scan_buf(h, h->d_last_pts, n) : upload_scan(h, h->d_last_pts, hint, 3, pts, n, st)) != HSB_OK) return s;
  HsbMatchParams P;
  fill_match_params(h, P);
  P.B = 1;
  P.hints = scan_header(h->d_last_pts);
  fill_scan(h, {HSB_IN_ENDPOINTS, scan_points(h->d_last_pts), nullptr, n, n, nullptr}, P);
  P.out_poses = res->pose;
  P.out_cov = res->cov;
  P.record = d_rec;
  P.record_floats = R;
  if ((s = launch_match_single(h, P, inl, hint, 3, pts)) != HSB_OK) return s;
  if (!host_out) HSB_CUDA(h, cudaMemcpyAsync(&h->h_pin->match, res, sizeof(PoseResult), cudaMemcpyDeviceToHost, st));
  if (record_out) HSB_CUDA(h, cudaMemcpyAsync(record_out, d_rec, (size_t)R * sizeof(float), cudaMemcpyDeviceToHost, st));
  HSB_CUDA(h, cudaStreamSynchronize(st));
  memcpy(out_pose, h->h_pin->match.pose, 3 * sizeof(float));
  if (cov_inout && n > 0) memcpy(cov_inout, h->h_pin->match.cov, 9 * sizeof(float));
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

int hsb_get_level_evals(const hsb_handle* h, int level) {
  if (!h || level < 0 || level >= h->levels) return HSB_ERR_INVALID_ARG;
  return h->lv[level].evals;
}

int hsb_set_step_record(hsb_handle* h, int on) {
  if (!h) return HSB_ERR_INVALID_ARG;
  if (on && !h->h_step_rec) {
    DeviceGuard dev(h->device);
    const size_t bytes = (size_t)record_floats(h) * sizeof(float);
    HSB_CUDA(h, cudaHostAlloc(reinterpret_cast<void**>(&h->h_step_rec), bytes, cudaHostAllocMapped));
    memset(h->h_step_rec, 0, bytes);
    HSB_CUDA(h, cudaHostGetDevicePointer(reinterpret_cast<void**>(&h->h_step_rec_dev), h->h_step_rec, 0));
  }
  if (on && !h->step_rec_on) h->step_rec_matched = false;   // no step since the switch was turned on
  h->step_rec_on = on != 0;
  return HSB_OK;
}

int hsb_get_step_record(hsb_handle* h, float* record_out, int* matched) {
  if (!h) return HSB_ERR_INVALID_ARG;
  if (!record_out || !matched)
    return fail(h, HSB_ERR_INVALID_ARG, "hsb_get_step_record: %s is NULL", record_out ? "matched" : "record_out");
  if (!h->stepped) return fail(h, HSB_ERR_INVALID_ARG, "hsb_get_step_record: the handle has taken no fused SLAM step");
  *matched = h->step_rec_matched ? 1 : 0;
  // (every step returns after its match has finished: a nowait step's record is published with its pose)
  if (h->step_rec_matched) memcpy(record_out, h->h_step_rec, (size_t)record_floats(h) * sizeof(float));
  return HSB_OK;
}

int hsb_get_last_match_scan(hsb_handle* h, float* points_xy_out, int capacity, int* n_out, float origo_out[2]) {
  if (!h) return HSB_ERR_INVALID_ARG;
  if (!n_out || !origo_out)
    return fail(h, HSB_ERR_INVALID_ARG, "hsb_get_last_match_scan: %s is NULL", n_out ? "origo_out" : "n_out");
  if (!h->have_last_match) return fail(h, HSB_ERR_INVALID_ARG, "hsb_get_last_match_scan: the handle has matched no scan");
  const int n = h->last_n;
  *n_out = n;
  if (capacity < n)
    return fail(h, HSB_ERR_INVALID_ARG, "hsb_get_last_match_scan: capacity %d is below the container's %d endpoints",
                capacity, n);
  if (n > 0 && !points_xy_out) return fail(h, HSB_ERR_INVALID_ARG, "hsb_get_last_match_scan: points_xy_out is NULL");
  origo_out[0] = h->last_origo[0];
  origo_out[1] = h->last_origo[1];
  if (n == 0) return HSB_OK;
  HandleScope guard(h);   // behind the step that filled the container (a group step runs on its group's stream)
  HSB_CUDA(h, cudaMemcpyAsync(points_xy_out, scan_points(h->d_last_pts), (size_t)n * 8, cudaMemcpyDeviceToHost, h->stream));
  HSB_CUDA(h, cudaStreamSynchronize(h->stream));
  return HSB_OK;
}

int hsb_hessian_derivs(hsb_handle* h, int level, const float pose_map[3], const float* pts, int n, float H_out[9],
                       float dTr_out[3]) {
  if (!h || level < 0 || level >= h->levels || !pose_map || n < 0 || (n > 0 && !pts) || !H_out || !dTr_out)
    return HSB_ERR_INVALID_ARG;
  HandleScope guard(h);
  int s;
  if ((s = ensure(h, h->d_pts, (size_t)(n > 0 ? n : 1) * 8 + 16)) != HSB_OK) return s;
  cudaStream_t st = h->stream;
  if (n > 0) HSB_CUDA(h, cudaMemcpyAsync(h->d_pts.p, pts, (size_t)n * 8, cudaMemcpyHostToDevice, st));
  HsbLevelDev L;
  fill_level_dev(h, level, L);
  float* d_out = h->d_scratch->hessian;
  if (h->gather_mode == HSB_GATHER_TEX)
    hsb::hessian_kernel<hsb::MODE_TEX><<<1, 256, 0, st>>>(L, static_cast<const float2*>(h->d_pts.p), n, pose_map[0],
                                                          pose_map[1], pose_map[2], d_out);
  else
    hsb::hessian_kernel<hsb::MODE_LDG><<<1, 256, 0, st>>>(L, static_cast<const float2*>(h->d_pts.p), n, pose_map[0],
                                                          pose_map[1], pose_map[2], d_out);
  h->launches++;
  HSB_CUDA(h, cudaGetLastError());
  HSB_CUDA(h, cudaMemcpyAsync(h->h_pin->hessian, d_out, 12 * sizeof(float), cudaMemcpyDeviceToHost, st));
  HSB_CUDA(h, cudaStreamSynchronize(st));
  memcpy(H_out, h->h_pin->hessian, 9 * sizeof(float));
  memcpy(dTr_out, h->h_pin->hessian + 9, 3 * sizeof(float));
  return HSB_OK;
}

// ---- converted input (N2): the node's conversions of a LaserScan or point cloud to endpoints -------

int hsb_set_scan_format(hsb_handle* h, const hsb_scan_format* fmt) {
  if (!h || !fmt || fmt->n_beams < 1 || fmt->n_beams > (1 << 20)) return HSB_ERR_INVALID_ARG;
  HandleScope guard(h);
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

int hsb_set_cloud_format(hsb_handle* h, const hsb_cloud_format* fmt) {
  if (!h || !fmt) return HSB_ERR_INVALID_ARG;
  for (int i = 0; i < 12; ++i)
    if (!std::isfinite(fmt->laser_transform[i])) return fail(h, HSB_ERR_INVALID_ARG, "laser_transform is not finite");
  h->cfmt = *fmt;
  h->cfmt_set = true;
  return HSB_OK;
}

int hsb_set_laser_projection(hsb_handle* h, const hsb_laser_projection* proj) {
  if (!h || !proj) return HSB_ERR_INVALID_ARG;
  if (proj->n_beams < 1 || proj->n_beams > (1 << 20))
    return fail(h, HSB_ERR_INVALID_ARG, "hsb_set_laser_projection: n_beams is %d, must lie in [1, 2^20]", proj->n_beams);
  if (!std::isfinite(proj->angle_min) || !std::isfinite(proj->angle_increment) || !std::isfinite(proj->range_min))
    return fail(h, HSB_ERR_INVALID_ARG, "hsb_set_laser_projection: angle_min, angle_increment and range_min must be finite");
  if (std::isnan(proj->range_cutoff)) return fail(h, HSB_ERR_INVALID_ARG, "hsb_set_laser_projection: range_cutoff is NaN");
  if (proj->range_cutoff < 0.0 && std::isnan(proj->range_max))   // the cutoff is range_max then
    return fail(h, HSB_ERR_INVALID_ARG, "hsb_set_laser_projection: range_cutoff < 0 selects range_max, which is NaN");
  HandleScope guard(h);
  // getUnitVectors_: cos / sin of angle_min + index * angle_increment, all double, libm
  std::vector<double> tab((size_t)proj->n_beams * 2);
  for (int i = 0; i < proj->n_beams; ++i) {
    const double a = (double)proj->angle_min + (double)i * (double)proj->angle_increment;
    tab[2 * (size_t)i] = cos(a);
    tab[2 * (size_t)i + 1] = sin(a);
  }
  // a step still queued on the handle's stream may read the old table
  HSB_CUDA(h, cudaStreamSynchronize(h->stream));
  int s = ensure(h, h->d_proj_unit, tab.size() * sizeof(double));
  if (s != HSB_OK) return s;
  HSB_CUDA(h, cudaMemcpy(h->d_proj_unit.p, tab.data(), tab.size() * sizeof(double), cudaMemcpyHostToDevice));
  h->proj = *proj;
  h->proj_set = true;
  return HSB_OK;
}

}  // extern "C"

namespace {

// Whether h can convert a scan of `kind` with n inputs: the formats the kind needs are set, a scan of ranges has the
// format's beam count (n < 0: not checked) and, if `whole`, the scan fits the shared memory of the single step's match
// shape.  The error goes to `err` and names the entry point `fn` and, if session >= 0, the group session.
int check_input(const hsb_handle* h, hsb_handle* err, HsbInputKind kind, const char* fn, int session, int n, bool whole) {
  char who[160];
  if (session < 0) snprintf(who, sizeof(who), "%s", fn);
  else snprintf(who, sizeof(who), "%s: session %d", fn, session);
  const char* on = session < 0 ? "" : " on its handle";
  if (kind == HSB_IN_PROJECTED && !h->proj_set)
    return fail(err, HSB_ERR_INVALID_ARG, "%s: hsb_set_laser_projection has not been called%s", who, on);
  if ((kind == HSB_IN_CLOUD || kind == HSB_IN_PROJECTED) && !h->cfmt_set)
    return fail(err, HSB_ERR_INVALID_ARG, "%s: hsb_set_cloud_format has not been called%s", who, on);
  if (kind == HSB_IN_RANGES && !h->fmt_set)
    return fail(err, HSB_ERR_INVALID_ARG, "%s: hsb_set_scan_format has not been called%s", who, on);
  if (n >= 0 && (kind == HSB_IN_RANGES || kind == HSB_IN_PROJECTED)) {
    const int nb = kind == HSB_IN_RANGES ? h->fmt.n_beams : h->proj.n_beams;
    const char* format = kind == HSB_IN_RANGES ? "scan format" : "laser projection";
    if (n != nb && session < 0) return fail(err, HSB_ERR_INVALID_ARG, "%s: n is %d, the %s has %d beams", who, n, format, nb);
    if (n != nb) return fail(err, HSB_ERR_INVALID_ARG, "%s has %d ranges, its %s has %d beams", who, n, format, nb);
  }
  if (whole && !staging_fits<8, 1>(whole_scan_slots(n), 1)) return fail_fused_too_long(err, n);
  return HSB_OK;
}

// Whether h's tuning selects a match shape compiled with the projection (has_projected_kernel), with 8 warps per scan
// for the single step (`single`).  HSB_ERR_UNSUPPORTED naming the entry point `fn` otherwise.
int check_projected_tuning(hsb_handle* h, const char* fn, bool single) {
  // the shape launch_match picks: warps_per_scan = 0 picks 8 for a single scan and one of 1, 2, 4, 8 for a batch
  const int W = h->tune_warps_per_scan == 0 ? 8 : h->tune_warps_per_scan;
  const int G = h->tune_scans_per_block <= 1 ? 1 : h->tune_scans_per_block;
  const int U = h->tune_unroll == 0 ? 4 : h->tune_unroll;
  if (has_projected_kernel(h, W, G, U) && (!single || W == 8)) return HSB_OK;
  return fail(h, HSB_ERR_UNSUPPORTED,
              "%s: no projected-scan kernel for tuning warps_per_scan=%d scans_per_block=%d unroll=%d packed=%d", fn,
              h->tune_warps_per_scan, h->tune_scans_per_block, h->tune_unroll, h->tune_packed);
}

// Everything a batch call of `kind` checks on the handle before it queues anything: the formats the kind needs and,
// for projected input, the scan length and the tuning.
int check_batch_input(hsb_handle* h, HsbInputKind kind, const char* fn) {
  if (kind == HSB_IN_ENDPOINTS) return HSB_OK;
  const bool proj = kind == HSB_IN_PROJECTED;
  int s = check_input(h, h, kind, fn, -1, proj ? h->proj.n_beams : -1, proj);
  if (s != HSB_OK || !proj) return s;
  return check_projected_tuning(h, fn, false);
}

// The beam count of a fixed-length kind (ranges: the scan format's, projected: the laser projection's), 0 for the kinds
// whose scans have their own lengths (endpoints, cloud).
int fixed_beams(const hsb_handle* h, HsbInputKind kind) {
  if (kind == HSB_IN_RANGES) return h->fmt.n_beams;
  if (kind == HSB_IN_PROJECTED) return h->proj.n_beams;
  return 0;
}

// The stand-alone conversion of n_in inputs of `kind` at d_in (laser transform d_T) into c's sink.
int launch_conversion(hsb_handle* h, HsbInputKind kind, const float* d_in, int n_in, const double* d_T, const HsbConvDev& c,
                      cudaStream_t st) {
  if (kind == HSB_IN_RANGES) hsb::conv_to_points_kernel<HSB_IN_RANGES><<<1, 256, 0, st>>>(d_in, n_in, d_T, c);
  else if (kind == HSB_IN_CLOUD) hsb::conv_to_points_kernel<HSB_IN_CLOUD><<<1, 256, 0, st>>>(d_in, n_in, d_T, c);
  else hsb::conv_to_points_kernel<HSB_IN_PROJECTED><<<1, 256, 0, st>>>(d_in, n_in, d_T, c);
  h->launches++;
  HSB_CUDA(h, cudaGetLastError());
  return HSB_OK;
}

// hsb_scan_to_points / hsb_cloud_to_points / hsb_projected_scan_to_points: n inputs of `kind` (host) with laser
// transform T (host, null for ranges) -> the kept endpoints and, for a cloud, the container's origo (host)
int to_points(hsb_handle* h, HsbInputKind kind, const float* in, int n, const double* T, float* out_xy, int* out_n,
              float out_origo[2]) {
  HandleScope guard(h);
  const size_t in_bytes = (size_t)n * (kind == HSB_IN_CLOUD ? 12 : 4);
  int s;
  if ((s = ensure(h, h->d_conv_in, in_bytes > 0 ? in_bytes : 12)) != HSB_OK) return s;
  if ((s = ensure(h, h->d_pts, (size_t)(n > 0 ? n : 1) * 8 + 16)) != HSB_OK) return s;
  if (T && (s = ensure(h, h->d_cloud_tf, 12 * sizeof(double))) != HSB_OK) return s;
  cudaStream_t st = h->stream;
  if (n > 0) HSB_CUDA(h, cudaMemcpyAsync(h->d_conv_in.p, in, in_bytes, cudaMemcpyHostToDevice, st));
  if (T) HSB_CUDA(h, cudaMemcpyAsync(h->d_cloud_tf.p, T, 12 * sizeof(double), cudaMemcpyHostToDevice, st));
  HsbConvDev c;
  fill_conv(h, kind, c);
  c.out_pts = static_cast<float2*>(h->d_pts.p);
  c.out_n = &h->d_scratch->conv_kept;
  if ((s = launch_conversion(h, kind, static_cast<const float*>(h->d_conv_in.p), n,
                             T ? static_cast<const double*>(h->d_cloud_tf.p) : nullptr, c, st)) != HSB_OK)
    return s;
  HSB_CUDA(h, cudaMemcpyAsync(&h->h_pin->conv_kept, c.out_n, sizeof(int), cudaMemcpyDeviceToHost, st));
  HSB_CUDA(h, cudaStreamSynchronize(st));
  const int kept = h->h_pin->conv_kept;
  if (kept > 0) HSB_CUDA(h, cudaMemcpy(out_xy, h->d_pts.p, (size_t)kept * 8, cudaMemcpyDeviceToHost));
  *out_n = kept;
  if (T && out_origo) cloud_origo(h, T, out_origo);
  return HSB_OK;
}

}  // namespace

extern "C" {

int hsb_scan_to_points(hsb_handle* h, const float* ranges, float* out_xy, int* out_n) {
  if (!h || !ranges || !out_xy || !out_n) return HSB_ERR_INVALID_ARG;
  int s = check_input(h, h, HSB_IN_RANGES, "hsb_scan_to_points", -1, -1, false);
  if (s != HSB_OK) return s;
  return to_points(h, HSB_IN_RANGES, ranges, h->fmt.n_beams, nullptr, out_xy, out_n, nullptr);
}

int hsb_cloud_to_points(hsb_handle* h, const float* points_xyz, int n, float* out_xy, int* out_n, float out_origo[2]) {
  if (!h || n < 0 || (n > 0 && !points_xyz) || !out_xy || !out_n) return HSB_ERR_INVALID_ARG;
  int s = check_input(h, h, HSB_IN_CLOUD, "hsb_cloud_to_points", -1, -1, false);
  if (s != HSB_OK) return s;
  return to_points(h, HSB_IN_CLOUD, points_xyz, n, h->cfmt.laser_transform, out_xy, out_n, out_origo);
}

int hsb_projected_scan_to_points(hsb_handle* h, const float* ranges, int n, const double* transform, float* out_xy,
                                 int* out_n, float out_origo[2]) {
  if (!h || !ranges || !out_xy || !out_n) return HSB_ERR_INVALID_ARG;
  int s = check_input(h, h, HSB_IN_PROJECTED, "hsb_projected_scan_to_points", -1, n, true);
  if (s != HSB_OK) return s;
  return to_points(h, HSB_IN_PROJECTED, ranges, n, transform ? transform : h->cfmt.laser_transform, out_xy, out_n,
                   out_origo);
}

int hsb_match_batch_ranges_device(hsb_handle* h, int B, const float* d_hints, const float* d_ranges, float* d_out_poses,
                                  float* d_out_cov, void* stream) {
  if (!h || B < 0 || !d_hints || !d_ranges || !d_out_poses) return HSB_ERR_INVALID_ARG;
  int s = check_batch_input(h, HSB_IN_RANGES, "hsb_match_batch_ranges_device");
  if (s != HSB_OK) return s;
  if (B == 0) return HSB_OK;
  HandleScope guard(h);
  const int nb = h->fmt.n_beams;   // scan b is d_ranges[b * n_beams ..]
  return match_batch(h, B, d_hints, {HSB_IN_RANGES, d_ranges, nullptr, nb, nb, nullptr}, d_out_poses, d_out_cov, nullptr,
                     nullptr, (cudaStream_t)stream);
}

int hsb_match_batch_cloud_device(hsb_handle* h, int B, const float* d_hints, const float* d_points_xyz, const int* d_offsets,
                                 int max_points_per_scan, const double* d_transforms, float* d_out_poses, float* d_out_cov,
                                 float* d_out_origo, void* stream) {
  if (!h || B < 0 || !d_hints || !d_offsets || !d_out_poses || max_points_per_scan < 0) return HSB_ERR_INVALID_ARG;
  int s = check_batch_input(h, HSB_IN_CLOUD, "hsb_match_batch_cloud_device");
  if (s != HSB_OK) return s;
  if (B == 0) return HSB_OK;
  if (!d_points_xyz && max_points_per_scan > 0) return fail(h, HSB_ERR_INVALID_ARG, "points pointer is NULL");
  HandleScope guard(h);
  return match_batch(h, B, d_hints, {HSB_IN_CLOUD, d_points_xyz, d_offsets, 0, max_points_per_scan, d_transforms},
                     d_out_poses, d_out_cov, d_out_origo, nullptr, (cudaStream_t)stream);
}

int hsb_match_batch_projected_device(hsb_handle* h, int B, const float* d_hints, const float* d_ranges,
                                     const double* d_transforms, float* d_out_poses, float* d_out_cov, float* d_out_origo,
                                     void* stream) {
  if (!h || B < 0 || !d_hints || !d_ranges || !d_out_poses) return HSB_ERR_INVALID_ARG;
  int s = check_batch_input(h, HSB_IN_PROJECTED, "hsb_match_batch_projected_device");
  if (s != HSB_OK) return s;
  if (B == 0) return HSB_OK;
  HandleScope guard(h);
  const int nb = h->proj.n_beams;   // scan b is d_ranges[b * n_beams ..]
  return match_batch(h, B, d_hints, {HSB_IN_PROJECTED, d_ranges, nullptr, nb, nb, d_transforms}, d_out_poses, d_out_cov,
                     d_out_origo, nullptr, (cudaStream_t)stream);
}

}  // extern "C"

// ---- host-buffer batch calls: one pipelined implementation for the four input formats ------------
// A call is cut into chunks (pipeline_bounds); chunk c's host->device copy runs on copy stream c%2 while chunk
// c-1 is being matched, results stream back behind each kernel.  Two staging SETS of device buffers alternate
// between calls, so that — with the submit / wait form — call k+1's first copies already travel while call k's
// last chunk is still being matched: the steady state of a stream of batches is bound by the PCIe copy of the
// inputs, not by copy + the exposed tail kernel.  The blocking entry points are submit + wait.
namespace {

int wait_set(hsb_handle* h, int s) {
  BatchSet& S = h->bset[s];
  if (!S.busy) return HSB_OK;
  HSB_CUDA(h, cudaEventSynchronize(S.done[0]));
  HSB_CUDA(h, cudaEventSynchronize(S.done[1]));
  S.busy = false;
  return HSB_OK;
}

// The host-buffer batch call `fn` of every input kind: B scans `sc` (host memory; the longest is found here) with their
// hints, results into host memory.  Everything that can reject the call is checked before anything is queued, and
// B == 0 returns after the checks.  With a ticket the call returns once everything is queued (hsb_match_batch_wait),
// without one it waits.
int submit_batch(hsb_handle* h, const char* fn, int B, const float* hints, const ScanIn& sc, float* out_poses,
                 float* out_cov, float* out_origo, int* ticket) {
  if (!h || B < 0 || !hints || !out_poses) return HSB_ERR_INVALID_ARG;
  // what a converted kind cannot do without: a cloud's offsets, the ranges
  if (sc.kind != HSB_IN_ENDPOINTS && (sc.kind == HSB_IN_CLOUD ? !sc.offsets : !sc.in)) return HSB_ERR_INVALID_ARG;
  int s = check_batch_input(h, sc.kind, fn);
  if (s != HSB_OK) return s;
  if (B == 0) {
    if (ticket) *ticket = -1;
    return HSB_OK;
  }
  if (!sc.offsets && sc.n_shared < 0) return fail(h, HSB_ERR_INVALID_ARG, "%s: shared-scan mode needs n_shared >= 0", fn);
  HandleScope guard(h);
  const int si = h->next_set;
  BatchSet& S = h->bset[si];
  if ((s = wait_set(h, si)) != HSB_OK) return s;   // the set is reused: its previous call must have delivered
  int max_n = 0;
  size_t in_bytes = 0, unit = 8;
  const int nb = fixed_beams(h, sc.kind);   // ranges / projected: scan b is in[b * nb .. (b + 1) * nb)
  if (nb > 0) {
    max_n = nb;
    unit = 4;
    in_bytes = (size_t)B * (size_t)nb * unit;
  } else {
    unit = sc.kind == HSB_IN_CLOUD ? 12 : 8;
    if (sc.offsets) {
      for (int b = 0; b < B; ++b) {
        const int n = sc.offsets[b + 1] - sc.offsets[b];
        if (n < 0) return fail(h, HSB_ERR_INVALID_ARG, "offsets must be non-decreasing");
        max_n = std::max(max_n, n);
      }
      in_bytes = (size_t)sc.offsets[B] * unit;
    } else {
      max_n = sc.n_shared > 0 ? sc.n_shared : 0;
      in_bytes = (size_t)max_n * unit;
    }
    if (in_bytes > 0 && !sc.in) return fail(h, HSB_ERR_INVALID_ARG, "points pointer is NULL");
  }
  if ((s = ensure(h, S.hints, (size_t)B * 12)) != HSB_OK) return s;
  if ((s = ensure(h, S.in, in_bytes + 16)) != HSB_OK) return s;
  if ((s = ensure(h, S.offsets, (size_t)(B + 1) * 4)) != HSB_OK) return s;
  if ((s = ensure(h, S.poses, (size_t)B * 12)) != HSB_OK) return s;
  if (out_cov && (s = ensure(h, S.cov, (size_t)B * 36)) != HSB_OK) return s;
  if (out_origo && (s = ensure(h, S.origo, (size_t)B * 8)) != HSB_OK) return s;
  if (sc.tf && (s = ensure(h, S.tf, (size_t)B * 12 * sizeof(double))) != HSB_OK) return s;
  float* d_hints = static_cast<float*>(S.hints.p);
  char* d_in = static_cast<char*>(S.in.p);
  int* d_off = static_cast<int*>(S.offsets.p);
  float* d_poses = static_cast<float*>(S.poses.p);
  float* d_cov = out_cov ? static_cast<float*>(S.cov.p) : nullptr;
  float* d_origo = out_origo ? static_cast<float*>(S.origo.p) : nullptr;
  double* d_tf = sc.tf ? static_cast<double*>(S.tf.p) : nullptr;

  std::vector<int> bounds = pipeline_bounds(B, h->tune_chunk);
  const bool shared = sc.kind == HSB_IN_ENDPOINTS && !sc.offsets;
  if (shared) bounds = std::vector<int>{0, B};   // one shared scan: nothing big to overlap
  ShapeScope shape_scope(h, B, bounds.size() - 1);
  // Stream roles: copy_stream[0] carries ALL host->device copies of all calls back to back, copy_stream[1] the kernels
  // and the result copies; a chunk's kernel waits for its copy through an event, so the copy engine never queues behind
  // a kernel.
  cudaStream_t s0 = h->copy_stream[0], s1 = h->copy_stream[1];
  if (sc.offsets) HSB_CUDA(h, cudaMemcpyAsync(d_off, sc.offsets, (size_t)(B + 1) * 4, cudaMemcpyHostToDevice, s0));
  if (shared && in_bytes > 0) HSB_CUDA(h, cudaMemcpyAsync(d_in, sc.in, in_bytes, cudaMemcpyHostToDevice, s0));
  HSB_CUDA(h, cudaMemcpyAsync(d_hints, hints, (size_t)B * 12, cudaMemcpyHostToDevice, s0));
  if (d_tf) HSB_CUDA(h, cudaMemcpyAsync(d_tf, sc.tf, (size_t)B * 12 * sizeof(double), cudaMemcpyHostToDevice, s0));
  for (size_t ci = 0; ci + 1 < bounds.size(); ++ci) {
    const int b0 = bounds[ci], b1 = bounds[ci + 1];
    if (!shared) {
      const size_t p0 = (nb > 0 ? (size_t)b0 * nb : (size_t)sc.offsets[b0]) * unit;
      const size_t p1 = (nb > 0 ? (size_t)b1 * nb : (size_t)sc.offsets[b1]) * unit;
      if (p1 > p0)
        HSB_CUDA(h, cudaMemcpyAsync(d_in + p0, reinterpret_cast<const char*>(sc.in) + p0, p1 - p0, cudaMemcpyHostToDevice, s0));
    }
    cudaEvent_t ready = S.chunk_ready[ci < 8 ? ci : 7];
    HSB_CUDA(h, cudaEventRecord(ready, s0));           // hints / offsets / this chunk's input are on the device
    HSB_CUDA(h, cudaStreamWaitEvent(s1, ready, 0));
    // the chunk's scans on the device (offsets index the whole input, fixed-length scans start at the chunk's first)
    const ScanIn chunk = {sc.kind, reinterpret_cast<const float*>(d_in) + (size_t)b0 * nb, sc.offsets ? d_off + b0 : nullptr,
                          nb > 0 ? nb : sc.n_shared, max_n, d_tf ? d_tf + 12 * (size_t)b0 : nullptr};
    float* o_pose = d_poses + 3 * (size_t)b0;
    float* o_cov = d_cov ? d_cov + 9 * (size_t)b0 : nullptr;
    float* o_origo = d_origo ? d_origo + 2 * (size_t)b0 : nullptr;
    if ((s = match_batch(h, b1 - b0, d_hints + 3 * (size_t)b0, chunk, o_pose, o_cov, o_origo, nullptr, s1)) != HSB_OK) return s;
    HSB_CUDA(h, cudaMemcpyAsync(out_poses + 3 * (size_t)b0, o_pose, (size_t)(b1 - b0) * 12, cudaMemcpyDeviceToHost, s1));
    if (out_cov)
      HSB_CUDA(h, cudaMemcpyAsync(out_cov + 9 * (size_t)b0, o_cov, (size_t)(b1 - b0) * 36, cudaMemcpyDeviceToHost, s1));
    if (out_origo)
      HSB_CUDA(h, cudaMemcpyAsync(out_origo + 2 * (size_t)b0, o_origo, (size_t)(b1 - b0) * 8, cudaMemcpyDeviceToHost, s1));
  }
  HSB_CUDA(h, cudaEventRecord(S.done[0], h->copy_stream[0]));
  HSB_CUDA(h, cudaEventRecord(S.done[1], h->copy_stream[1]));
  S.busy = true;
  h->next_set = si ^ 1;
  if (!ticket) return wait_set(h, si);
  *ticket = si;
  return HSB_OK;
}

}  // namespace

extern "C" {

int hsb_match_batch_submit(hsb_handle* h, int B, const float* hints, const float* pts, const int* offsets, int n_shared,
                           float* out_poses, float* out_cov, int* ticket) {
  return submit_batch(h, "hsb_match_batch", B, hints, {HSB_IN_ENDPOINTS, pts, offsets, n_shared, 0, nullptr}, out_poses,
                      out_cov, nullptr, ticket);
}
int hsb_match_batch(hsb_handle* h, int B, const float* hints, const float* pts, const int* offsets, int n_shared,
                    float* out_poses, float* out_cov) {
  return hsb_match_batch_submit(h, B, hints, pts, offsets, n_shared, out_poses, out_cov, nullptr);
}

int hsb_match_batch_ranges_submit(hsb_handle* h, int B, const float* hints, const float* ranges, float* out_poses,
                                  float* out_cov, int* ticket) {
  return submit_batch(h, "hsb_match_batch_ranges", B, hints, {HSB_IN_RANGES, ranges, nullptr, 0, 0, nullptr}, out_poses,
                      out_cov, nullptr, ticket);
}
int hsb_match_batch_ranges(hsb_handle* h, int B, const float* hints, const float* ranges, float* out_poses, float* out_cov) {
  return hsb_match_batch_ranges_submit(h, B, hints, ranges, out_poses, out_cov, nullptr);
}

int hsb_match_batch_cloud_submit(hsb_handle* h, int B, const float* hints, const float* points_xyz, const int* offsets,
                                 const double* transforms, float* out_poses, float* out_cov, float* out_origo, int* ticket) {
  return submit_batch(h, "hsb_match_batch_cloud", B, hints, {HSB_IN_CLOUD, points_xyz, offsets, 0, 0, transforms},
                      out_poses, out_cov, out_origo, ticket);
}
int hsb_match_batch_cloud(hsb_handle* h, int B, const float* hints, const float* points_xyz, const int* offsets,
                          const double* transforms, float* out_poses, float* out_cov, float* out_origo) {
  return hsb_match_batch_cloud_submit(h, B, hints, points_xyz, offsets, transforms, out_poses, out_cov, out_origo, nullptr);
}

int hsb_match_batch_projected_submit(hsb_handle* h, int B, const float* hints, const float* ranges,
                                     const double* transforms, float* out_poses, float* out_cov, float* out_origo,
                                     int* ticket) {
  return submit_batch(h, "hsb_match_batch_projected", B, hints, {HSB_IN_PROJECTED, ranges, nullptr, 0, 0, transforms},
                      out_poses, out_cov, out_origo, ticket);
}
int hsb_match_batch_projected(hsb_handle* h, int B, const float* hints, const float* ranges, const double* transforms,
                              float* out_poses, float* out_cov, float* out_origo) {
  return hsb_match_batch_projected_submit(h, B, hints, ranges, transforms, out_poses, out_cov, out_origo, nullptr);
}

int hsb_match_batch_wait(hsb_handle* h, int ticket) {
  if (!h || ticket < -1 || ticket > 1) return HSB_ERR_INVALID_ARG;
  if (ticket < 0) return HSB_OK;
  HandleScope guard(h);
  return wait_set(h, ticket);
}

int hsb_measure_h2d_gbs(hsb_handle* h, const void* host, size_t bytes, int reps, float* out_gbs) {
  if (!h || !host || !bytes || reps < 1 || !out_gbs) return HSB_ERR_INVALID_ARG;
  HandleScope guard(h);
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

// ---- map writing -------------------------------------------------------------------------------

namespace {

constexpr int kMarkTeam = 2;   // warps per beam of the mark phase

// The map writer's two launches on st, Mark then Apply, over `levels` levels of `sessions` scans whose longest has
// max_n endpoints (grid y = level, z = session).  Mark: kMarkTeam warps per beam, four beams per CTA, at most as many
// CTAs as are resident at once (six per SM: its launch bounds), shared out among the (session, level) slots.  Apply: a
// one-wave sweep of each level's box, its CTAs per SM asked once from the occupancy API (the register count decides).
// Mark is order-free and apply has one owner per cell (update_kernel.cuh), so the bits do not depend on the grids.
// pdl: programmatic dependent launch (pdl_wait() in update_kernel.cuh).
template <auto Mark, auto Apply, typename Params>
int launch_map_write(hsb_handle* h, cudaStream_t st, const Params& P, int levels, int sessions, int max_n, bool pdl) {
  static int apply_ctas_per_sm = 0;
  if (!apply_ctas_per_sm) {
    int nb = 0;
    HSB_CUDA(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, Apply, 256, 0));
    apply_ctas_per_sm = nb > 0 ? nb : 4;
  }
  const int slots = levels * sessions;
  const int blocks = std::max(1, std::min((max_n * kMarkTeam + 7) / 8, (h->sm_count * 6 + slots - 1) / slots));
  const int sweep = std::max(1, (h->sm_count * apply_ctas_per_sm + slots - 1) / slots);
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.blockDim = dim3(256);
  cfg.stream = st;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  cfg.gridDim = dim3(blocks, levels, sessions);
  HSB_CUDA(h, cudaLaunchKernelEx(&cfg, Mark, P));
  cfg.gridDim = dim3(sweep, levels, sessions);
  HSB_CUDA(h, cudaLaunchKernelEx(&cfg, Apply, P));
  h->launches += 2;
  HSB_CUDA(h, cudaGetLastError());
  return HSB_OK;
}

}  // namespace

extern "C" {

static int run_update(hsb_handle* h, const HsbUpdateParams& P, int max_n) {
  if (max_n <= 0) return HSB_OK;
  cudaStream_t st = h->stream;
  if (h->tune_time_update) HSB_CUDA(h, cudaEventRecord(h->ev_time[0], st));
  const int s = launch_map_write<hsb::update_mark_kernel<kMarkTeam>, hsb::update_apply_kernel>(h, st, P, P.levels, 1,
                                                                                             max_n, h->tune_pdl != 0);
  if (s != HSB_OK) return s;
  if (h->tune_time_update) HSB_CUDA(h, cudaEventRecord(h->ev_time[1], st));
  return HSB_OK;
}

// `st`: the stream the map write goes to (the handle's, or a group's)
static int next_stamp_base(hsb_handle* h, int level, uint32_t* base, cudaStream_t st) {
  Level& L = h->lv[level];
  if (L.stamp_base > 0xfffffff0u - 8u) {  // wrap guard: forget old stamps
    HSB_CUDA(h, cudaMemsetAsync(L.stamp, 0, (size_t)L.sx * L.sy * sizeof(uint32_t), st));
    L.stamp_base = 0;
  }
  *base = L.stamp_base;
  L.stamp_base += 4;
  L.parity ^= 1;   // this write uses the slot fill_update_level just handed out; the next one the other
  return HSB_OK;
}

// Level l's map-writer descriptor d for a write of the scan `pts` (n endpoints; with n_dev the count the device holds
// there, n an upper bound) from origo (NULL = 0, 0), both scaled by pt_scale.  A level with endpoints advances its stamp
// base (a wrap clears the stamps on `st`) and writer slot, and raises *max_n to n.
static int fill_update_level(hsb_handle* h, int l, float pt_scale, const float2* pts, int n, const int* n_dev,
                             const float origo[2], cudaStream_t st, HsbUpdateLevelDev& d, int* max_n) {
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
  d.pt_scale = pt_scale;
  d.pts = pts;
  d.n = n;
  d.n_dev = n_dev;
  d.origo_x = origo ? origo[0] : 0.f;
  d.origo_y = origo ? origo[1] : 0.f;
  // an empty container still advances the stamps in the reference (OccGridMapBase.h:164-167); no-op here
  d.active = n > 0;
  if (!d.active) return HSB_OK;
  *max_n = std::max(*max_n, n);
  return next_stamp_base(h, l, &d.stamp_base, st);
}

// MapRepMultiMap::updateByScan (MapRepMultiMap.h:134-147) for one scan of h: its map-writer level descriptors
// d[0 .. levels).  Level 0 reads this scan (`pts`, n, n_dev as fill_update_level takes them); the coarse levels read it
// too if it has just become the last match's container (`matched`), and otherwise the container the last matchData
// left behind (:143).
static int fill_update_levels(hsb_handle* h, HsbUpdateLevelDev* d, const float2* pts, int n, const int* n_dev,
                              const float origo[2], bool matched, cudaStream_t st, int* max_n) {
  const float2* last = h->d_last_pts.p ? reinterpret_cast<const float2*>(scan_points(h->d_last_pts)) : nullptr;
  for (int l = 0; l < h->levels; ++l) {
    const float pt_scale = (float)(1.0 / pow(2.0, (double)l));
    const int s = l == 0 || matched
                      ? fill_update_level(h, l, pt_scale, pts, n, n_dev, origo, st, d[l], max_n)
                      : fill_update_level(h, l, pt_scale, last, h->last_n, nullptr, h->last_origo, st, d[l], max_n);
    if (s != HSB_OK) return s;
  }
  return HSB_OK;
}

// The map write of hsb_update_by_scan and the single SLAM steps (fill_update_levels) as launches on h->stream.
// pose_dev / gate_flag: see HsbUpdateParams.
static int enqueue_update_by_scan(hsb_handle* h, const float2* pts, int n, const int* n_dev, const float origo[2],
                                  bool matched, const float pose[3], const float* pose_dev, const float* gate_flag) {
  HsbUpdateParams P;
  memset(&P, 0, sizeof(P));
  P.levels = h->levels;
  if (pose) memcpy(P.pose_world, pose, 3 * sizeof(float));
  P.pose_dev = pose_dev;
  P.gate_flag = gate_flag;
  P.log_odds_free = h->log_odds_free;
  P.log_odds_occ = h->log_odds_occ;
  int max_n = 0;
  const int s = fill_update_levels(h, P.lv, pts, n, n_dev, origo, matched, h->stream, &max_n);
  if (s != HSB_OK) return s;
  return run_update(h, P, max_n);
}

int hsb_update_by_scan(hsb_handle* h, const float* pts, int n, const float origo[2], const float pose[3]) {
  if (!h || !pose || n < 0 || (n > 0 && !pts)) return HSB_ERR_INVALID_ARG;
  HandleScope guard(h);
  int s;
  cudaStream_t st = h->stream;
  if ((s = upload_scan(h, h->d_upd_pts, nullptr, 0, pts, n, st)) != HSB_OK) return s;
  if ((s = enqueue_update_by_scan(h, reinterpret_cast<const float2*>(scan_points(h->d_upd_pts)), n, nullptr, origo, false,
                                  pose, nullptr, nullptr)) != HSB_OK)
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

// HectorSlamProcessor::update (HectorSlamProcessor.h:71-113) for one scan `in` (host memory, n_shared inputs) of any
// kind, after the node's conversion for converted input (HectorMappingRos::scanCallback :297): match with the gate in
// its epilogue, then the map write, behind ONE host-to-device copy.  Converted input is converted by the match kernel's
// staging step, which also writes the endpoints out for the map writer and leaves their number on the device (the
// writer reads it there), so no host round trip appears between conversion, match, gate and map write.  origo: the
// endpoints' container origo (NULL = 0, 0); a converted scan's follows from its laser transform.  nowait: return when
// the pose has arrived, the map write continues on the handle's stream.
static int slam_step(hsb_handle* h, const float hint[3], const ScanIn& in, const float origo_in[2], int map_without_matching,
                     bool nowait, float out_pose[3], float cov_inout[9], int* map_updated, int* out_kept) {
  HandleScope guard(h);
  int s;
  const int n = in.n_shared;   // converted: a cloud's points or a scan's beams, an upper bound of the endpoints kept
  const bool conv = in.kind != HSB_IN_ENDPOINTS;
  const bool matched = !map_without_matching;
  PoseResult* d_res = &h->d_scratch->step;
  int* n_dev = conv ? &h->d_scratch->step_kept : nullptr;
  cudaStream_t st = h->stream;
  // results (pose, flag, Hessian, kept count) are written into mapped host memory by the kernels themselves: the step
  // is one host-to-device copy and three launches (match with the gate in its epilogue, mark, apply — the latter two
  // with programmatic dependent launch).  Endpoint steps only: tuning host_out = 0 copies them back instead.
  const bool host_out = conv || h->tune_host_out != 0;
  const bool poll = host_out && nowait;   // return when the pose has arrived; the map write continues on the stream
  PoseResult* h_res = &h->h_pin_dev->step;
  unsigned* seq_dev = &h->h_pin_dev->step_seq;
  const unsigned seq_value = ++h->step_seq;
  int* kept_dev = &h->h_pin_dev->step_kept;
  // the match kernel publishes a converted scan's kept count itself; without matching publish_int_kernel does
  StepSession ss;
  if ((s = step_session(h, in.kind, n, in.tf, origo_in, matched, n_dev, matched ? kept_dev : nullptr, ss)) != HSB_OK) return s;
  const float header[6] = {hint[0], hint[1], hint[2], ss.gate_in[0], ss.gate_in[1], ss.gate_in[2]};
  const bool inl = !conv && matched && inline_scan_applies(h, n);   // header + scan travel in the match launch
  const float* d_hdr;   // the header on the device: [0..2] hint, [3..5] minDist / minAngle / force
  ScanIn dev;           // the scan on the device
  if (!conv) {
    // staging, endpoints: header + points straight into the container the map writer reads
    if (!inl && (s = upload_scan(h, *ss.sink, header, 6, in.in, n, st)) != HSB_OK) return s;
    d_hdr = scan_header(*ss.sink);
    dev = {HSB_IN_ENDPOINTS, scan_points(*ss.sink), nullptr, n, n, nullptr};
  } else {
    // staging, converted input (floats): [0..15] header; cloud / projected: [16..39] the laser transform (12 doubles),
    // [40..] the cloud or the ranges; ranges: [16..] the ranges.  The conversion writes the endpoints into the sink.
    const size_t kHdr = 16, kTf = in.tf ? 24 : 0, per_pt = in.kind == HSB_IN_CLOUD ? 3 : 1;
    const size_t bytes = (kHdr + kTf + (size_t)n * per_pt) * sizeof(float);
    if ((s = ensure(h, h->d_fused_in, bytes + 16)) != HSB_OK) return s;
    if ((s = ensure_pinned(h, h->h_stage, h->h_stage_bytes, bytes)) != HSB_OK) return s;
    float* hs = h->h_stage;
    memset(hs, 0, kHdr * sizeof(float));
    memcpy(hs, header, sizeof(header));
    if (in.tf) memcpy(hs + kHdr, in.tf, 12 * sizeof(double));
    if (n > 0) memcpy(hs + kHdr + kTf, in.in, (size_t)n * per_pt * sizeof(float));
    HSB_CUDA(h, cudaMemcpyAsync(h->d_fused_in.p, hs, bytes, cudaMemcpyHostToDevice, st));
    const float* d_c = static_cast<const float*>(h->d_fused_in.p);
    d_hdr = d_c;
    dev = {in.kind, d_c + kHdr + kTf, nullptr, n, n, in.tf ? reinterpret_cast<const double*>(d_c + kHdr) : nullptr};
  }
  float2* d_pts = reinterpret_cast<float2*>(scan_points(*ss.sink));
  h->stepped = true;
  h->step_rec_matched = h->step_rec_on && matched;
  if (matched) {
    // :78 match, and :83-89 the gate in the same kernel's epilogue (an empty scan still passes through it: pose = hint)
    HsbMatchParams P;
    fill_match_params(h, P);
    P.B = 1;
    P.hints = d_hdr;
    fill_scan(h, dev, P);
    P.conv = ss.conv;
    P.out_poses = d_res->pose;
    P.out_cov = host_out ? h_res->cov : d_res->cov;
    P.gate_state = h->d_gate;
    P.gate_in = d_hdr + 3;
    P.gate_out_host = host_out ? h_res->pose : nullptr;
    P.seq_host = poll ? seq_dev : nullptr;
    P.seq_value = seq_value;
    // the step record: stored by the match before the sequence number (or the synchronise) releases the pose
    P.record = h->step_rec_on ? h->h_step_rec_dev : nullptr;
    P.record_floats = record_floats(h);
    // (a projected step takes the single step's default shape: hsb_slam_update_projected checked the tuning)
    s = launch_match_single(h, P, inl, header, 6, in.in);
    // (endpoints: the scan is in the container since the staging copy, whether or not the match launched)
    if (s == HSB_OK || !conv) record_match(h, n, ss.origo);
    if (s != HSB_OK) return s;
  } else if (!conv) {
    // without matching, endpoints: the gate alone (:80, :89)
    hsb::slam_gate_kernel<<<1, 32, 0, st>>>(h->d_gate, d_hdr + 3, d_hdr, d_res->pose, host_out ? h_res->pose : nullptr,
                                            poll ? seq_dev : nullptr, seq_value);
    h->launches += 1;
    HSB_CUDA(h, cudaGetLastError());
  } else {
    // without matching, converted input: the stand-alone conversion kernel, the gate, then the kept count's publication
    if ((s = launch_conversion(h, in.kind, dev.in, n, dev.tf, ss.conv, st)) != HSB_OK) return s;
    hsb::slam_gate_kernel<<<1, 32, 0, st>>>(h->d_gate, d_hdr + 3, d_hdr, d_res->pose, h_res->pose, nullptr, 0);
    hsb::publish_int_kernel<<<1, 32, 0, st>>>(n_dev, kept_dev, poll ? seq_dev : nullptr, seq_value);
    h->launches += 2;
    HSB_CUDA(h, cudaGetLastError());
  }
  if ((s = enqueue_update_by_scan(h, d_pts, n, n_dev, ss.origo, matched, nullptr, d_res->pose, h->d_gate + 3)) != HSB_OK)
    return s;   // :91
  if (poll) {
    // the pose is all the caller needs now; every later call on this handle is stream-ordered behind the map write
    s = wait_published(h, &h->h_pin->step_seq, seq_value, st, "fused step finished without publishing its pose");
    if (s != HSB_OK) return s;
    h->map_write_pending = true;
  } else {
    if (!host_out) HSB_CUDA(h, cudaMemcpyAsync(&h->h_pin->step, d_res, sizeof(PoseResult), cudaMemcpyDeviceToHost, st));
    HSB_CUDA(h, cudaStreamSynchronize(st));  // :93 onMapUpdated — the probability plane is current
    h->map_write_pending = false;
  }
  // the endpoints the step had: known on the host for endpoints, counted on the device for converted input
  const PoseResult& r = h->h_pin->step;
  step_results(h, matched, conv ? h->h_pin->step_kept : n, r.pose, r.cov, out_pose, map_updated, cov_inout, out_kept);
  return HSB_OK;
}

int hsb_slam_update(hsb_handle* h, const float hint[3], const float* pts, int n, const float origo[2],
                    int map_without_matching, float out_pose[3], float cov_inout[9], int* map_updated) {
  if (!h || !hint || !out_pose || n < 0 || (n > 0 && !pts)) return HSB_ERR_INVALID_ARG;
  return slam_step(h, hint, {HSB_IN_ENDPOINTS, pts, nullptr, n, n, nullptr}, origo, map_without_matching, false, out_pose,
                   cov_inout, map_updated, nullptr);
}

int hsb_slam_update_nowait(hsb_handle* h, const float hint[3], const float* pts, int n, const float origo[2],
                           int map_without_matching, float out_pose[3], float cov_inout[9], int* map_updated) {
  if (!h || !hint || !out_pose || n < 0 || (n > 0 && !pts)) return HSB_ERR_INVALID_ARG;
  return slam_step(h, hint, {HSB_IN_ENDPOINTS, pts, nullptr, n, n, nullptr}, origo, map_without_matching, true, out_pose,
                   cov_inout, map_updated, nullptr);
}

// HectorMappingRos::scanCallback's default branch in one call: rosPointCloudToDataContainer (HectorMappingRos.cpp:283,
// 509-542) + HectorSlamProcessor::update (:297)
int hsb_slam_update_cloud(hsb_handle* h, const float hint[3], const float* points_xyz, int n, const double* transform,
                          int map_without_matching, int nowait, float out_pose[3], float cov_inout[9], int* map_updated,
                          int* out_kept) {
  if (!h || !hint || !out_pose || n < 0 || (n > 0 && !points_xyz)) return HSB_ERR_INVALID_ARG;
  int s = check_input(h, h, HSB_IN_CLOUD, "hsb_slam_update_cloud", -1, -1, false);
  if (s != HSB_OK) return s;
  const ScanIn in = {HSB_IN_CLOUD, points_xyz, nullptr, n, n, transform ? transform : h->cfmt.laser_transform};
  return slam_step(h, hint, in, nullptr, map_without_matching, nowait != 0, out_pose, cov_inout, map_updated, out_kept);
}

// ... and its branch without the laser tf (use_tf_scan_transformation = false, :248-254): rosLaserScanToDataContainer
// (:483-507) + HectorSlamProcessor::update with the last match as the start estimate
int hsb_slam_update_ranges(hsb_handle* h, const float hint[3], const float* ranges, int n, int map_without_matching,
                           int nowait, float out_pose[3], float cov_inout[9], int* map_updated, int* out_kept) {
  if (!h || !hint || !out_pose || !ranges) return HSB_ERR_INVALID_ARG;
  int s = check_input(h, h, HSB_IN_RANGES, "hsb_slam_update_ranges", -1, n, false);
  if (s != HSB_OK) return s;
  return slam_step(h, hint, {HSB_IN_RANGES, ranges, nullptr, n, n, nullptr}, nullptr, map_without_matching, nowait != 0,
                   out_pose, cov_inout, map_updated, out_kept);
}

// ... and the default branch from the LaserScan itself (:258-297): laser_geometry's projection (:273), then
// rosPointCloudToDataContainer (:283) + HectorSlamProcessor::update (:297)
int hsb_slam_update_projected(hsb_handle* h, const float hint[3], const float* ranges, int n, const double* transform,
                              int map_without_matching, int nowait, float out_pose[3], float cov_inout[9],
                              int* map_updated, int* out_kept) {
  if (!h || !hint || !out_pose || !ranges) return HSB_ERR_INVALID_ARG;
  int s = check_input(h, h, HSB_IN_PROJECTED, "hsb_slam_update_projected", -1, n, true);
  if (s != HSB_OK) return s;
  if ((s = check_projected_tuning(h, "hsb_slam_update_projected", true)) != HSB_OK) return s;
  const ScanIn in = {HSB_IN_PROJECTED, ranges, nullptr, n, n, transform ? transform : h->cfmt.laser_transform};
  return slam_step(h, hint, in, nullptr, map_without_matching, nowait != 0, out_pose, cov_inout, map_updated, out_kept);
}

int hsb_set_last_map_update_pose(hsb_handle* h, const float pose[3]) {
  if (!h || !pose) return HSB_ERR_INVALID_ARG;
  HandleScope guard(h);
  memcpy(h->h_pin->gate, pose, 3 * sizeof(float));
  HSB_CUDA(h, cudaMemcpyAsync(h->d_gate, h->h_pin->gate, 3 * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  HSB_CUDA(h, cudaStreamSynchronize(h->stream));
  return HSB_OK;
}

int hsb_get_last_map_update_pose(hsb_handle* h, float out[3]) {
  if (!h || !out) return HSB_ERR_INVALID_ARG;
  HandleScope guard(h);
  HSB_CUDA(h, cudaMemcpyAsync(h->h_pin->gate, h->d_gate, 3 * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  HSB_CUDA(h, cudaStreamSynchronize(h->stream));
  memcpy(out, h->h_pin->gate, 3 * sizeof(float));
  return HSB_OK;
}

int hsb_update_level_by_scan(hsb_handle* h, int level, const float* pts, int n, const float origo[2], const float pose[3]) {
  if (!h || level < 0 || level >= h->levels || !pose || n < 0 || (n > 0 && !pts)) return HSB_ERR_INVALID_ARG;
  HandleScope guard(h);
  int s;
  cudaStream_t st = h->stream;
  if ((s = upload_scan(h, h->d_upd_pts, nullptr, 0, pts, n, st)) != HSB_OK) return s;
  HsbUpdateParams P;
  memset(&P, 0, sizeof(P));
  P.levels = 1;
  memcpy(P.pose_world, pose, 3 * sizeof(float));
  P.log_odds_free = h->log_odds_free;
  P.log_odds_occ = h->log_odds_occ;
  int max_n = 0;
  if ((s = fill_update_level(h, level, 1.0f, reinterpret_cast<const float2*>(scan_points(h->d_upd_pts)), n, nullptr, origo,
                             st, P.lv[0], &max_n)) != HSB_OK)
    return s;
  if ((s = run_update(h, P, max_n)) != HSB_OK) return s;
  HSB_CUDA(h, cudaStreamSynchronize(st));
  return HSB_OK;
}

int hsb_on_map_updated(hsb_handle* h) {
  if (!h) return HSB_ERR_INVALID_ARG;
  HandleScope guard(h);
  HSB_CUDA(h, cudaStreamSynchronize(h->stream));
  h->map_write_pending = false;
  return HSB_OK;
}

// ---- planes ------------------------------------------------------------------------------------

int hsb_upload_level(hsb_handle* h, int level, const float* logodds_host) {
  if (!h || level < 0 || level >= h->levels || !logodds_host) return HSB_ERR_INVALID_ARG;
  HandleScope guard(h);
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
  HandleScope guard(h);
  Level& L = h->lv[level];
  HSB_CUDA(h, cudaMemcpyAsync(out, L.logodds, (size_t)L.sx * L.sy * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
  HSB_CUDA(h, cudaStreamSynchronize(h->stream));
  h->d2h_bytes += (size_t)L.sx * L.sy * sizeof(float);
  return HSB_OK;
}

int hsb_download_level_rect(hsb_handle* h, int level, const int rect[4], float* out) {
  if (!h || level < 0 || level >= h->levels || !rect || !out) return HSB_ERR_INVALID_ARG;
  HandleScope guard(h);
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
  HandleScope guard(h);
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
  HandleScope guard(h);
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
  const int rect[4] = {0, 0, h->lv[level].sx - 1, h->lv[level].sy - 1};
  return hsb_download_occupancy_rect(h, level, rect, out);
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
  HandleScope guard(h);
  return likelihood_device(h, level, B, d_poses_world, reinterpret_cast<const float2*>(d_points_xy), d_offsets, n_shared,
                           d_out_likelihood, (cudaStream_t)stream);
}

int hsb_best_hypothesis_device(hsb_handle* h, int level, int B, const float* d_poses_world, const float* d_points_xy,
                               const int* d_offsets, int n_shared, float* d_out_likelihood, float* d_best4, void* stream) {
  if (!h || level < 0 || level >= h->levels || B < 0 || !d_best4 || (B > 0 && !d_poses_world)) return HSB_ERR_INVALID_ARG;
  if (!d_offsets && n_shared < 0) return HSB_ERR_INVALID_ARG;
  if (B > 0 && !d_points_xy && (d_offsets || n_shared > 0)) return fail(h, HSB_ERR_INVALID_ARG, "points pointer is NULL");
  HandleScope guard(h);
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

}  // extern "C"

namespace {

// What a pose query computes for every pose (likelihood, covariance, the group match's pose and Hessian from a hint) or
// session (best hypothesis).
enum ScoreKind { SCORE_LIKELIHOOD, SCORE_COVARIANCE, SCORE_BEST, SCORE_MATCH };
constexpr size_t kScoreChunk = 1 << 20;   // most bytes of points score_query stages in its pinned copy

// The group match's part of a score_query (SCORE_MATCH): the launch shape group_match chose, W warps per scan and
// max_n, the longest scan of a session with hints (launch_match_t sizes its staging by it), and where the results go.
struct MatchQuery {
  int W, max_n;
  float* out_poses;   // Q x 3
  float* out_cov;     // Q x 9 Hessians, or NULL
};

// Every host-buffer pose-query body (hsb_likelihood_batch, hsb_covariance_batch, the group scoring calls and the group
// match): Q poses of K sessions, session k's poses [pose_offsets[k], pose_offsets[k+1]) scored on member
// sess[k].member's map of `level`, whose descriptor is lv[member * levels + level] — or, with lv NULL, h's own level,
// staged with the poses as a one-entry table.  For SCORE_MATCH the poses are hints, each matched over every level of
// its member's row of lv.  sessions(sess, pose_offsets, staged) writes the K session descriptors and K + 1 pose
// offsets into the staging; `staged` is where the n_pts points of `pts` will lie on the device, so a session's scan is
// a slice of them or any other device scan the caller knows of.  One host-to-device copy from the pinned staging hs
// (points past kScoreChunk bytes: a second one from `pts`), one launch on `st` (two for the best hypothesis, whose K
// arg-max accumulators are `best`; the match's in match->W), one device-to-host copy of the asked-for results and one
// synchronise.  The launches, the match's launch shape and any error are counted on h.  sessions() also gives each
// session its member's cell length of `level` (the covariance's world matrix) and its level count.  A heterogeneous
// group's call passes `ragged` (its members differ in level count: the match runs each hint over its member's own
// levels, GRP_MATCH_HET) and `any_mode` (they differ in gather mode: every kernel takes each level's own path,
// MODE_ANY); otherwise h's gather mode is every session's, and a ragged group's match runs in it.
// The group match's launch at W warps per scan: GRP_MATCH when the members share their level count and gather mode,
// GRP_MATCH_HET otherwise (het), in the members' one gather mode (MODE_TEX / MODE_LDG) or, when they hold both,
// MODE_ANY.
template <int W>
int launch_group_match(hsb_handle* h, HsbMatchParams& M, int max_n, cudaStream_t st, bool het, int mode) {
  if (!het)
    return mode == hsb::MODE_TEX ? launch_match_t<W, 1, hsb::MODE_TEX, 4, false, false, hsb::GRP_MATCH>(h, M, max_n, st, 1)
                                 : launch_match_t<W, 1, hsb::MODE_LDG, 4, false, false, hsb::GRP_MATCH>(h, M, max_n, st, 1);
  if (mode == hsb::MODE_ANY)
    return launch_match_t<W, 1, hsb::MODE_ANY, 4, false, false, hsb::GRP_MATCH_HET>(h, M, max_n, st, 1);
  return mode == hsb::MODE_TEX ? launch_match_t<W, 1, hsb::MODE_TEX, 4, false, false, hsb::GRP_MATCH_HET>(h, M, max_n, st, 1)
                               : launch_match_t<W, 1, hsb::MODE_LDG, 4, false, false, hsb::GRP_MATCH_HET>(h, M, max_n, st, 1);
}

template <typename Sessions>
int score_query(hsb_handle* h, cudaStream_t st, float*& hs_buf, size_t& hs_bytes, DevBuf& d_stage, const HsbLevelDev* lv,
                int levels, int level, ScoreKind kind, int K, int Q, const float* poses, const float* pts, size_t n_pts,
                const Sessions& sessions, unsigned long long* best, float* out_lh, float* out_map, float* out_world,
                float* out_best4, int* out_best_index, const MatchQuery* match = nullptr, bool ragged = false,
                bool any_mode = false) {
  // staging: sessions | pose offsets | (level descriptor) | poses | scans, then the results: likelihoods | best4 | best
  // index, or covariance (map) | covariance (world), or poses | Hessians, each only if asked for
  auto al = [](size_t x) { return (x + 15) & ~(size_t)15; };
  const size_t o_off = (size_t)K * sizeof(HsbScoreSessionDev), o_lv = al(o_off + (size_t)(K + 1) * 4);
  const size_t o_poses = lv ? o_lv : al(o_lv + sizeof(HsbLevelDev));
  const size_t o_pts = al(o_poses + (size_t)Q * 12), in_end = o_pts + n_pts * 8, o_out = al(in_end);
  size_t o_lh = o_out, o_best4 = o_out, o_index = o_out, o_map = o_out, o_world = o_out, o_cov = o_out, out_end = o_out;
  if (kind == SCORE_MATCH) {
    o_cov = o_out + (size_t)Q * 12;
    out_end = o_cov + (match->out_cov ? (size_t)Q * 36 : 0);
  } else if (kind == SCORE_COVARIANCE) {
    o_world = o_map + (out_map ? (size_t)Q * 36 : 0);
    out_end = o_world + (out_world ? (size_t)Q * 36 : 0);
  } else {
    o_best4 = al(o_lh + (size_t)Q * 4);
    o_index = o_best4 + (kind == SCORE_BEST ? (size_t)K * 16 : 0);
    out_end = kind == SCORE_BEST ? o_index + (size_t)K * 4 : o_lh + (size_t)Q * 4;
  }
  int s;
  if ((s = ensure_pinned(h, hs_buf, hs_bytes, out_end)) != HSB_OK) return s;
  if ((s = ensure(h, d_stage, out_end)) != HSB_OK) return s;
  char* hs = reinterpret_cast<char*>(hs_buf);
  char* ds = static_cast<char*>(d_stage.p);
  sessions(reinterpret_cast<HsbScoreSessionDev*>(hs), reinterpret_cast<int*>(hs + o_off),
           reinterpret_cast<const float2*>(ds + o_pts));
  if (!lv) {
    HsbLevelDev L = {};
    fill_level_dev(h, level, L);
    memcpy(hs + o_lv, &L, sizeof(L));
  }
  memcpy(hs + o_poses, poses, (size_t)Q * 12);
  // More points than kScoreChunk bytes go straight from the caller's memory: the driver overlaps its host staging of a
  // pageable copy with the transfer, where staging megabytes here first would serialise the two.
  const bool inline_pts = n_pts * 8 <= kScoreChunk;
  if (inline_pts && n_pts > 0) memcpy(hs + o_pts, pts, n_pts * 8);
  HSB_CUDA(h, cudaMemcpyAsync(ds, hs, inline_pts ? in_end : o_pts, cudaMemcpyHostToDevice, st));
  if (!inline_pts) HSB_CUDA(h, cudaMemcpyAsync(ds + o_pts, pts, n_pts * 8, cudaMemcpyHostToDevice, st));

  HsbScoreParams P;
  memset(&P, 0, sizeof(P));
  P.lv = lv ? lv : reinterpret_cast<const HsbLevelDev*>(ds + o_lv);
  P.sess = reinterpret_cast<const HsbScoreSessionDev*>(ds);
  P.pose_offsets = reinterpret_cast<const int*>(ds + o_off);
  P.poses = reinterpret_cast<const float*>(ds + o_poses);
  P.levels = lv ? levels : 1;
  P.level = lv ? level : 0;
  P.K = K;
  P.Q = Q;
  const bool tex = h->gather_mode == HSB_GATHER_TEX;
  if (kind == SCORE_MATCH) {
    HsbMatchParams M;
    fill_match_params(h, M);   // (lv[] is unused: every hint reads its member's row of the group's table)
    M.levels = levels;         // (the table's stride)
    M.B = Q;
    M.hints = P.poses;
    M.kind = HSB_IN_ENDPOINTS;
    M.out_poses = reinterpret_cast<float*>(ds + o_out);
    M.out_cov = match->out_cov ? reinterpret_cast<float*>(ds + o_cov) : nullptr;
    M.group_lv = lv;
    M.match_sess = P.sess;
    M.match_offsets = P.pose_offsets;
    M.match_K = K;
    s = HSB_ERR_UNSUPPORTED;
    const int mode = any_mode ? hsb::MODE_ANY : tex ? hsb::MODE_TEX : hsb::MODE_LDG;
#define HSB_GM_CASE(w) \
  if (match->W == w) s = launch_group_match<w>(h, M, match->max_n, st, ragged || any_mode, mode);
    HSB_GM_CASE(1);
    HSB_GM_CASE(2);
    HSB_GM_CASE(4);
    HSB_GM_CASE(8);
#undef HSB_GM_CASE
    if (s != HSB_OK) return s;
  } else if (kind == SCORE_COVARIANCE) {
    P.out_map = out_map ? reinterpret_cast<float*>(ds + o_map) : nullptr;
    P.out_world = out_world ? reinterpret_cast<float*>(ds + o_world) : nullptr;
    const int blocks = std::min(Q, h->sm_count * 8);
    if (any_mode) hsb::covariance_kernel<hsb::MODE_ANY><<<blocks, 224, 0, st>>>(P);
    else if (tex) hsb::covariance_kernel<hsb::MODE_TEX><<<blocks, 224, 0, st>>>(P);
    else hsb::covariance_kernel<hsb::MODE_LDG><<<blocks, 224, 0, st>>>(P);
    h->launches++;
  } else {
    P.out = reinterpret_cast<float*>(ds + o_lh);
    if (kind == SCORE_BEST) {
      P.best = best;
      P.out_best4 = reinterpret_cast<float*>(ds + o_best4);
      P.out_best_index = reinterpret_cast<int*>(ds + o_index);
    }
    const int blocks = std::min((Q + 3) / 4, h->sm_count * 16);
    if (any_mode) hsb::likelihood_group_kernel<hsb::MODE_ANY><<<blocks, 128, 0, st>>>(P);
    else if (tex) hsb::likelihood_group_kernel<hsb::MODE_TEX><<<blocks, 128, 0, st>>>(P);
    else hsb::likelihood_group_kernel<hsb::MODE_LDG><<<blocks, 128, 0, st>>>(P);
    h->launches++;
    if (kind == SCORE_BEST) {
      HSB_CUDA(h, cudaGetLastError());
      hsb::best_group_finish_kernel<<<(K + 127) / 128, 128, 0, st>>>(P);
      h->launches++;
    }
  }
  HSB_CUDA(h, cudaGetLastError());
  HSB_CUDA(h, cudaMemcpyAsync(hs + o_out, ds + o_out, out_end - o_out, cudaMemcpyDeviceToHost, st));
  HSB_CUDA(h, cudaStreamSynchronize(st));
  if (kind == SCORE_MATCH) {
    memcpy(match->out_poses, hs + o_out, (size_t)Q * 12);
    if (match->out_cov) memcpy(match->out_cov, hs + o_cov, (size_t)Q * 36);
  } else if (kind == SCORE_COVARIANCE) {
    if (out_map) memcpy(out_map, hs + o_map, (size_t)Q * 36);
    if (out_world) memcpy(out_world, hs + o_world, (size_t)Q * 36);
  } else {
    if (out_lh) memcpy(out_lh, hs + o_lh, (size_t)Q * 4);
    if (out_best4) memcpy(out_best4, hs + o_best4, (size_t)K * 16);   // (given with SCORE_BEST only)
    if (out_best_index) memcpy(out_best_index, hs + o_index, (size_t)K * 4);
  }
  return HSB_OK;
}

// hsb_likelihood_batch / hsb_covariance_batch on h's level, on h->stream, staged through the handle's scan staging as
// the ray queries are (see hsb_raycast_batch).  Every session is on member 0.  Without offsets: one session of all B
// poses whose scan is the shared one, n points long (none are staged if n < 0); with offsets: B sessions of one pose
// each, session b's scan [offsets[b], offsets[b+1]) of the offsets[B] staged points.
int single_score(hsb_handle* h, ScoreKind kind, int level, int B, const float* poses, const float* pts, const int* offsets,
                 int n, float* out_lh, float* out_map, float* out_world) {
  const size_t total = offsets ? (size_t)offsets[B] : (size_t)(n > 0 ? n : 0);
  if (total > 0 && !pts) return fail(h, HSB_ERR_INVALID_ARG, "points pointer is NULL");
  const int K = offsets ? B : 1;
  auto sessions = [&](HsbScoreSessionDev* sess, int* pose_offsets, const float2* staged) {
    for (int k = 0; k < K; ++k) {
      sess[k].pts = staged + (offsets ? offsets[k] : 0);
      sess[k].n = offsets ? offsets[k + 1] - offsets[k] : n;
      sess[k].member = 0;
      sess[k].cell_length = h->lv[level].cell_length;
      pose_offsets[k] = k;
    }
    pose_offsets[K] = B;
  };
  return score_query(h, h->stream, h->h_stage, h->h_stage_bytes, h->d_pts, nullptr, 1, level, kind, K, B, poses, pts,
                     total, sessions, nullptr, out_lh, out_map, out_world, nullptr, nullptr);
}

}  // namespace

extern "C" {

// A negative n_shared scores against no points in both calls, but as the length of the scan the likelihood sees 0
// (1 - 0/0: NaN) and the covariance's sigma points see n_shared itself (1 - 0/n_shared: 1).
int hsb_likelihood_batch(hsb_handle* h, int level, int B, const float* poses, const float* pts, const int* offsets,
                         int n_shared, float* out) {
  if (!h || level < 0 || level >= h->levels || B < 0 || !poses || !out) return HSB_ERR_INVALID_ARG;
  if (B == 0) return HSB_OK;
  HandleScope guard(h);
  return single_score(h, SCORE_LIKELIHOOD, level, B, poses, pts, offsets, n_shared > 0 ? n_shared : 0, out, nullptr,
                      nullptr);
}

int hsb_covariance_batch(hsb_handle* h, int level, int B, const float* poses, const float* pts, const int* offsets, int n_shared,
                         float* out_cov_map, float* out_cov_world) {
  if (!h || level < 0 || level >= h->levels || B < 0 || !poses || (!out_cov_map && !out_cov_world)) return HSB_ERR_INVALID_ARG;
  if (B == 0) return HSB_OK;
  HandleScope guard(h);
  return single_score(h, SCORE_COVARIANCE, level, B, poses, pts, offsets, n_shared, nullptr, out_cov_map, out_cov_world);
}

// A level's replication rectangle as a host reader sees it: the whole level while the cleared flag is set (the level
// was cleared by hsb_group_reset and not shipped since), so the two-step protocol ships what it ships after hsb_reset.
static void replication_rect(const Level& L, const int* words, int* rect) {
  if (words[HSB_DIRTY_CLEARED]) {
    const int full[4] = {0, 0, L.sx - 1, L.sy - 1};
    memcpy(rect, full, sizeof(full));
  } else {
    memcpy(rect, words, 4 * sizeof(int));
  }
}

static int get_dirty(hsb_handle* h, int level, int which, int rect[4], int reset) {
  if (!h || level < 0 || level >= h->levels || !rect) return HSB_ERR_INVALID_ARG;
  HandleScope guard(h);
  Level& L = h->lv[level];
  int* src = L.dirty + 4 * which;
  int* pin = h->h_pin->dirty;
  HSB_CUDA(h, cudaMemcpyAsync(pin, L.dirty, HSB_DIRTY_WORDS * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  if (reset) {
    static const int clean[4] = {INT_MAX, INT_MAX, -1, -1};
    HSB_CUDA(h, cudaMemcpyAsync(src, clean, sizeof(clean), cudaMemcpyHostToDevice, h->stream));
    if (which == 0) HSB_CUDA(h, cudaMemsetAsync(L.dirty + HSB_DIRTY_CLEARED, 0, sizeof(int), h->stream));
  }
  HSB_CUDA(h, cudaStreamSynchronize(h->stream));
  if (which == 0) replication_rect(L, pin, rect);
  else memcpy(rect, pin + 4, 4 * sizeof(int));
  return HSB_OK;
}
int hsb_get_dirty_rect(hsb_handle* h, int level, int rect[4], int reset) { return get_dirty(h, level, 0, rect, reset); }
int hsb_get_mirror_dirty_rect(hsb_handle* h, int level, int rect[4], int reset) { return get_dirty(h, level, 1, rect, reset); }

// All levels' replication rectangles with one copy and one synchronize (levels x 4 ints).
int hsb_get_dirty_rects(hsb_handle* h, int* rects, int reset) {
  if (!h || !rects) return HSB_ERR_INVALID_ARG;
  HandleScope guard(h);
  int all[kOverflowWord];
  HSB_CUDA(h, cudaMemcpyAsync(all, h->d_dirty_all, sizeof(all), cudaMemcpyDeviceToHost, h->stream));
  HSB_CUDA(h, cudaStreamSynchronize(h->stream));
  for (int l = 0; l < h->levels; ++l) replication_rect(h->lv[l], all + HSB_DIRTY_WORDS * l, rects + 4 * l);
  if (reset) {
    for (int l = 0; l < h->levels; ++l) {
      int* w = all + HSB_DIRTY_WORDS * l;
      w[0] = w[1] = INT_MAX;
      w[2] = w[3] = -1;
      w[HSB_DIRTY_CLEARED] = 0;
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
  HandleScope guard(h);
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
  HandleScope guard(h);
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
  T.capacity_words = std::min<size_t>(capacity_bytes / 4, 0xffffffffu);
  T.error_count = h->d_dirty_all + kOverflowWord;
  T.K = 1;
  T.M = 1;
}

int hsb_pack_dirty_device(hsb_handle* h, float* d_buf, size_t capacity_bytes, int reset, void* stream) {
  if (!h || !d_buf || capacity_bytes < HSB_TILE_HEADER_WORDS * 4) return HSB_ERR_INVALID_ARG;
  HandleScope guard(h);
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
  HandleScope guard(h);
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
  HandleScope guard(h);
  int* d = h->d_dirty_all + kOverflowWord;
  HSB_CUDA(h, cudaDeviceSynchronize());
  HSB_CUDA(h, cudaMemcpy(count, d, sizeof(int), cudaMemcpyDeviceToHost));
  if (reset) HSB_CUDA(h, cudaMemset(d, 0, sizeof(int)));
  return HSB_OK;
}

// h's level as a ray query sees it (HsbRayLevelDev): getDist's transform computed exactly as the single calls have
// always computed it.
static void fill_ray_level(const hsb_handle* h, int level, HsbRayLevelDev& d) {
  const Level& L = h->lv[level];
  float origo[2];
  hsb_get_map_origin(h, level, origo);
  volatile float inv_scale = 1.0f / L.cell_length;   // CoordinateTransformer::setTransforms, HectorMapTools.h:64
  d.plane = L.logodds;
  d.sx = L.sx;
  d.sy = L.sy;
  d.origo_x = origo[0];
  d.origo_y = origo[1];
  d.scale = L.cell_length;
  d.inv_scale = inv_scale;
}

// Every ray query's host body (hsb_raycast_batch, hsb_get_dist_batch and their group forms): Q = offsets[K] rays of K
// sessions, session k's rays [offsets[k], offsets[k+1]) cast on member members[k]'s level `level`, described by the
// device table lv[member * levels + level] (plane, size, getDist's transform) — or, with lv NULL, h's own level, staged
// with the rays as a one-entry table.  One host-to-device copy of member list, offsets, (level) and rays from the pinned
// staging hs, one launch on `st`, one device-to-host copy of the results into the staging and one synchronise; the
// results are then copied into the caller's arrays on the host.  The launch and any error are counted on h.
// world: getDist rays, otherwise ray-cast rays.
static int ray_query(hsb_handle* h, cudaStream_t st, float*& hs_buf, size_t& hs_bytes, DevBuf& d_stage,
                     const HsbRayLevelDev* lv, int levels, int level, bool world, int K, const int* members,
                     const int* offsets, const void* begin, const void* end, float* out_dist, void* out_hit,
                     int* out_found) {
  const int Q = offsets[K];
  // staging: member list | offsets | (level) | begin | end, then the results: dist | hit | found (getDist)
  auto al = [](size_t x) { return (x + 15) & ~(size_t)15; };
  const size_t o_off = al((size_t)K * 4), o_lv = al(o_off + (size_t)(K + 1) * 4);
  const size_t o_begin = lv ? o_lv : al(o_lv + sizeof(HsbRayLevelDev));
  const size_t o_end = o_begin + (size_t)Q * 8, o_dist = al(o_end + (size_t)Q * 8);
  const size_t o_hit = al(o_dist + (size_t)Q * 4), o_found = o_hit + (size_t)Q * 8;
  const size_t out_end = out_found ? o_found + (size_t)Q * 4 : out_hit ? o_found : o_dist + (size_t)Q * 4;
  int s;
  if ((s = ensure_pinned(h, hs_buf, hs_bytes, out_end)) != HSB_OK) return s;
  if ((s = ensure(h, d_stage, out_end)) != HSB_OK) return s;
  char* hs = reinterpret_cast<char*>(hs_buf);
  char* ds = static_cast<char*>(d_stage.p);
  memcpy(hs, members, (size_t)K * 4);
  memcpy(hs + o_off, offsets, (size_t)(K + 1) * 4);
  if (!lv) {
    HsbRayLevelDev R;
    fill_ray_level(h, level, R);
    memcpy(hs + o_lv, &R, sizeof(R));
  }
  memcpy(hs + o_begin, begin, (size_t)Q * 8);
  memcpy(hs + o_end, end, (size_t)Q * 8);
  HSB_CUDA(h, cudaMemcpyAsync(ds, hs, o_end + (size_t)Q * 8, cudaMemcpyHostToDevice, st));

  HsbRayParams P;
  P.lv = lv ? lv : reinterpret_cast<const HsbRayLevelDev*>(ds + o_lv);
  P.members = reinterpret_cast<const int*>(ds);
  P.offsets = reinterpret_cast<const int*>(ds + o_off);
  P.begin = ds + o_begin;
  P.end = ds + o_end;
  P.out_dist = reinterpret_cast<float*>(ds + o_dist);
  P.out_hit = out_hit ? ds + o_hit : nullptr;
  P.out_found = out_found ? reinterpret_cast<int*>(ds + o_found) : nullptr;
  P.levels = lv ? levels : 1;
  P.level = lv ? level : 0;
  P.K = K;
  P.Q = Q;
  const int blocks = std::min((Q + 7) / 8, h->sm_count * 8);
  if (world) hsb::ray_kernel<true><<<blocks, 256, 0, st>>>(P);
  else hsb::ray_kernel<false><<<blocks, 256, 0, st>>>(P);
  h->launches++;
  HSB_CUDA(h, cudaGetLastError());
  HSB_CUDA(h, cudaMemcpyAsync(hs + o_dist, ds + o_dist, out_end - o_dist, cudaMemcpyDeviceToHost, st));
  HSB_CUDA(h, cudaStreamSynchronize(st));
  memcpy(out_dist, hs + o_dist, (size_t)Q * 4);
  if (out_hit) memcpy(out_hit, hs + o_hit, (size_t)Q * 8);
  if (out_found) memcpy(out_found, hs + o_found, (size_t)Q * 4);
  return HSB_OK;
}

// The single calls stage through the handle's scan staging: every call that fills h_stage either synchronises or, a
// nowait SLAM step, returns once its pose is published, which comes after the staging's host-to-device copy.
int hsb_raycast_batch(hsb_handle* h, int level, int B, const int* begin_cells, const int* end_cells, float* out_dist,
                      int* out_hit) {
  if (!h || level < 0 || level >= h->levels || B < 0 || !begin_cells || !end_cells || !out_dist) return HSB_ERR_INVALID_ARG;
  if (B == 0) return HSB_OK;
  HandleScope guard(h);
  const int members[1] = {0}, offsets[2] = {0, B};
  return ray_query(h, h->stream, h->h_stage, h->h_stage_bytes, h->d_pts, nullptr, 1, level, false, 1, members, offsets,
                   begin_cells, end_cells, out_dist, out_hit, nullptr);
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
  HandleScope guard(h);
  const int members[1] = {0}, offsets[2] = {0, B};
  return ray_query(h, h->stream, h->h_stage, h->h_stage_bytes, h->d_pts, nullptr, 1, level, true, 1, members, offsets,
                   begin_world, end_world, out_dist, out_hit_world, out_found);
}

void* hsb_level_logodds_device_ptr(hsb_handle* h, int level) {
  if (!h || level < 0 || level >= h->levels) return nullptr;
  return h->lv[level].logodds;
}

int hsb_refresh_level(hsb_handle* h, int level, void* stream) {
  if (!h || level < 0 || level >= h->levels) return HSB_ERR_INVALID_ARG;
  HandleScope guard(h);
  int s = refresh_level(h, level, (cudaStream_t)stream);
  if (s != HSB_OK) return s;
  // the plane was written from outside (a full-plane broadcast): the host mirror has to re-read the whole level, so the
  // mirror rectangle becomes the level, in order on `stream`.  The replication rectangle is left alone: marking it
  // would make a replica re-ship a whole plane it has only received.
  Level& L = h->lv[level];
  if (!L.dirty) return HSB_OK;
  const int full[4] = {0, 0, L.sx - 1, L.sy - 1};
  HSB_CUDA(h, cudaMemcpyAsync(L.dirty + 4, full, sizeof(full), cudaMemcpyHostToDevice, (cudaStream_t)stream));
  return HSB_OK;
}

}  // extern "C"

// ---- group SLAM step: HectorSlamProcessor::update for M handles in one device pass ----------------------------------
// One host-to-device copy (hints, thresholds, offsets, per-session descriptors, all scans) and three launches on the
// group's stream, whatever M is: the match kernel with one 8-warp CTA per session (the shape hsb_slam_update uses, so
// every session's pose, Hessian and gate decision are the single call's bits) and the gate of each session in its
// epilogue, then mark and apply over (session, level).  The per-step handle state the single call keeps on the host
// (stamp bases, writer slots, the last match's container size and origo) advances through the functions the single
// call uses: step_session, record_match, fill_update_levels and step_results.

struct hsb_group {
  std::vector<hsb_handle*> m;      // the members, in the order hsb_group_create(_mixed / _heterogeneous) was given them
  std::vector<int> all;            // 0 .. M-1: the member list of a step of every member
  std::vector<unsigned char> listed;   // scratch of a step's member-list check, M flags
  int device = 0;
  // the largest level count of the members (the stride of every member-major table); every member's but in a
  // heterogeneous group, whose members may each have their own (ragged) and their own gather mode (any_mode: both
  // occur, so the kernels take the gather path from each level descriptor, MODE_ANY).  Both stay false in groups of
  // the other two constructors, which require the members to agree.
  int levels = 0;
  bool ragged = false, any_mode = false;
  int* d_member_levels = nullptr;  // ragged: the members' level counts (the *_ragged tile and reset kernels)
  cudaStream_t stream = nullptr;   // every step of the group runs here
  cudaEvent_t ev = nullptr;        // recorded behind every step; members wait on it lazily (HandleScope)
  // M x levels match-kernel level descriptors, member-major (a handle's planes never move); a session reads its
  // member's row (HsbGroupSessionDev::member)
  HsbLevelDev* d_lv = nullptr;
  // per session (at most M) 4 floats (pose, write flag) for the map writer, the finished-session counter (4 words), then
  // the sessions' kept-endpoint counts of a converted step (ints, the map writer's n_dev)
  float* d_res = nullptr;
  // mapped pinned, per session: 4 (pose, flag), then 9 Hessian; the sequence number (4 words), kept-endpoint counts (ints)
  float* h_res = nullptr;
  float* h_res_dev = nullptr;      // device alias of h_res
  char* h_stage = nullptr;         // pinned staging of the step's host-to-device copy
  size_t h_stage_bytes = 0;
  DevBuf d_stage;
  unsigned seq = 0;
  // occupancy sync (hsb_group_sync_occupancy): M x levels pointers to the members' mirror rectangles (Level::dirty + 4),
  // member-major like d_lv; the call's member list, gathered rectangles and row table (device and pinned twin, sized
  // for M sessions); the packed rows of one chunk (device and pinned staging)
  int** d_mirror = nullptr;
  char* d_occ_meta = nullptr;
  char* h_occ_meta = nullptr;
  DevBuf d_occ_rows;
  int8_t* h_occ_rows = nullptr;
  size_t h_occ_rows_bytes = 0;
  // ray queries (hsb_group_raycast, hsb_group_get_dist): M x levels descriptors of the members' levels (plane, size,
  // getDist's transform), member-major like d_lv; the call's staging (member list, offsets and rays, then the results),
  // pinned and on the device
  HsbRayLevelDev* d_ray_lv = nullptr;
  float* h_ray_stage = nullptr;
  size_t h_ray_stage_bytes = 0;
  DevBuf d_ray_stage;
  // pose scoring (hsb_group_likelihood, hsb_group_covariance, hsb_group_best_hypothesis) stages through the ray queries'
  // staging above (every call that fills it returns synchronised); M arg-max accumulators of the best hypothesis,
  // zeroed once (every call re-arms the ones it used)
  unsigned long long* d_best = nullptr;
  // map replication (hsb_group_pack_dirty_device, hsb_group_unpack_dirty_device): M x levels tile descriptors,
  // member-major like d_lv, and the members' replication-overflow counters; two events ordering the caller's stream
  // against the group's
  HsbTileLevelDev* d_tile_lv = nullptr;
  int** d_tile_counters = nullptr;
  cudaEvent_t ev_tile[2] = {nullptr, nullptr};
  // map reset (hsb_group_reset): per member its stamp planes and gate state, next to its row of d_tile_lv
  HsbResetMemberDev* d_reset = nullptr;
};

namespace {

// hsb_group_create's errors: hsb_last_error(NULL), and hsb_last_error(handles[0]) when that is a handle
int group_fail(hsb_handle* h, int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_create_error = buf;
  if (h) h->err = buf;
  return code;
}

// Layout of hsb_group::d_occ_meta / h_occ_meta for up to K sessions: member list | gathered rectangles | row table
struct OccMeta {
  size_t members = 0, rects, rows, bytes;
  explicit OccMeta(int K) {
    rects = ((size_t)K * sizeof(int) + 15) & ~(size_t)15;
    rows = rects + (size_t)K * sizeof(int4);
    bytes = rows + (size_t)K * sizeof(HsbOccRowsDev);
  }
};

}  // namespace

extern "C" {

int hsb_group_destroy(hsb_group* g) {
  if (!g) return HSB_OK;
  DeviceGuard guard(g->device);
  if (g->stream) cudaStreamSynchronize(g->stream);
  for (hsb_handle* h : g->m)
    if (h->group_ev == g->ev) h->group_ev = nullptr;   // the step it would wait for is complete
  if (g->d_lv) cudaFree(g->d_lv);
  if (g->d_mirror) cudaFree(g->d_mirror);
  if (g->d_occ_meta) cudaFree(g->d_occ_meta);
  if (g->d_occ_rows.p) cudaFree(g->d_occ_rows.p);
  if (g->h_occ_meta) cudaFreeHost(g->h_occ_meta);
  if (g->h_occ_rows) cudaFreeHost(g->h_occ_rows);
  if (g->d_ray_lv) cudaFree(g->d_ray_lv);
  if (g->d_best) cudaFree(g->d_best);
  if (g->d_tile_lv) cudaFree(g->d_tile_lv);
  if (g->d_tile_counters) cudaFree(g->d_tile_counters);
  if (g->d_reset) cudaFree(g->d_reset);
  if (g->d_member_levels) cudaFree(g->d_member_levels);
  for (cudaEvent_t e : g->ev_tile)
    if (e) cudaEventDestroy(e);
  if (g->d_ray_stage.p) cudaFree(g->d_ray_stage.p);
  if (g->h_ray_stage) cudaFreeHost(g->h_ray_stage);
  if (g->d_res) cudaFree(g->d_res);
  if (g->d_stage.p) cudaFree(g->d_stage.p);
  if (g->h_res) cudaFreeHost(g->h_res);
  if (g->h_stage) cudaFreeHost(g->h_stage);
  if (g->ev) cudaEventDestroy(g->ev);
  if (g->stream) cudaStreamDestroy(g->stream);
  delete g;
  return HSB_OK;
}

}  // extern "C"

namespace {

// What a group's members may differ in: nothing but their maps' contents (hsb_group_create), their map size, resolution
// and start (hsb_group_create_mixed), or also their level count, per-level iteration counts and gather mode
// (hsb_group_create_heterogeneous).
enum GroupKind { GROUP_SAME, GROUP_MIXED, GROUP_HETERO };

// hsb_group_create, hsb_group_create_mixed and hsb_group_create_heterogeneous (see GroupKind).  fn names the entry point
// in the error messages.
int group_create(hsb_handle* const* handles, int M, hsb_group** out, GroupKind kind, const char* fn) {
  const bool mixed = kind == GROUP_MIXED;
  if (!out) return group_fail(nullptr, HSB_ERR_INVALID_ARG, "%s: out is NULL", fn);
  *out = nullptr;
  hsb_handle* h0 = (handles && M > 0) ? handles[0] : nullptr;
  if (!handles || M < 1) return group_fail(h0, HSB_ERR_INVALID_ARG, "%s: a group needs M >= 1 handles (M = %d)", fn, M);
  for (int s = 0; s < M; ++s)
    if (!handles[s]) return group_fail(h0, HSB_ERR_INVALID_ARG, "%s: handle %d is NULL", fn, s);
  {
    std::vector<hsb_handle*> sorted(handles, handles + M);
    std::sort(sorted.begin(), sorted.end());
    if (std::adjacent_find(sorted.begin(), sorted.end()) != sorted.end())
      return group_fail(h0, HSB_ERR_INVALID_ARG, "%s: a handle is listed twice", fn);
  }
  for (int s = 1; s < M; ++s) {
    const hsb_handle* h = handles[s];
    if (h->device != h0->device)
      return group_fail(h0, HSB_ERR_INVALID_ARG, "%s: handle %d is on device %d, handle 0 on device %d", fn, s,
                        h->device, h0->device);
    if (kind == GROUP_HETERO) continue;   // each member runs its own levels, iterations and gather path
    if (mixed) {   // what every group launch shares: the level count, the per-level iteration counts, the gather mode
      if (h->levels != h0->levels)
        return group_fail(h0, HSB_ERR_INVALID_ARG, "%s: handle %d has %d levels, handle 0 has %d", fn, s, h->levels,
                          h0->levels);
      for (int l = 0; l < h0->levels; ++l)
        if (h->lv[l].evals != h0->lv[l].evals)
          return group_fail(h0, HSB_ERR_INVALID_ARG,
                            "%s: handle %d differs from handle 0 in the resolved max_iterations of level %d (%d, %d)", fn,
                            s, l, h->lv[l].evals - 1, h0->lv[l].evals - 1);
      if (h->gather_mode != h0->gather_mode)
        return group_fail(h0, HSB_ERR_INVALID_ARG,
                          "%s: handle %d differs from handle 0 in the resolved gather mode (%d, %d)", fn, s,
                          h->gather_mode, h0->gather_mode);
      continue;
    }
    bool same = h->levels == h0->levels && h->cfg.map_size_x == h0->cfg.map_size_x &&
                h->cfg.map_size_y == h0->cfg.map_size_y && h->cfg.map_resolution == h0->cfg.map_resolution &&
                h->cfg.start_x == h0->cfg.start_x && h->cfg.start_y == h0->cfg.start_y && h->gather_mode == h0->gather_mode;
    for (int l = 0; same && l < h0->levels; ++l) same = h->lv[l].evals == h0->lv[l].evals;
    if (!same)
      return group_fail(h0, HSB_ERR_INVALID_ARG,
                        "%s: handle %d differs from handle 0 in levels, map size, resolution, start, "
                        "max_iterations or gather mode", fn, s);
  }
  DeviceGuard guard(h0->device);
  hsb_group* g = new (std::nothrow) hsb_group();
  if (!g) return group_fail(h0, HSB_ERR_OUT_OF_MEMORY, "%s: out of host memory", fn);
  g->m.assign(handles, handles + M);
  g->all.resize(M);
  for (int s = 0; s < M; ++s) g->all[s] = s;
  g->listed.assign(M, 0);
  g->device = h0->device;
  g->levels = h0->levels;
  for (int s = 1; s < M; ++s) {
    g->levels = std::max(g->levels, handles[s]->levels);
    g->ragged |= handles[s]->levels != h0->levels;
    g->any_mode |= handles[s]->gather_mode != h0->gather_mode;
  }
#define HSB_GROUP_CUDA(expr)                                                                                 \
  do {                                                                                                       \
    cudaError_t _e = (expr);                                                                                 \
    if (_e != cudaSuccess) {                                                                                 \
      const int _code = _e == cudaErrorMemoryAllocation ? HSB_ERR_OUT_OF_MEMORY : HSB_ERR_CUDA;              \
      group_fail(h0, _code, "%s: %s failed: %s", fn, #expr, cudaGetErrorString(_e));                         \
      hsb_group_destroy(g);                                                                                  \
      return _code;                                                                                          \
    }                                                                                                        \
  } while (0)
  HSB_GROUP_CUDA(cudaStreamCreateWithFlags(&g->stream, cudaStreamNonBlocking));
  HSB_GROUP_CUDA(cudaEventCreateWithFlags(&g->ev, cudaEventDisableTiming));
  {
    std::vector<HsbLevelDev> lv((size_t)M * g->levels);
    memset(lv.data(), 0, lv.size() * sizeof(HsbLevelDev));
    for (int s = 0; s < M; ++s)   // (a member's rows past its own levels stay zero: nothing reads them)
      for (int l = 0; l < g->m[s]->levels; ++l) fill_level_dev(g->m[s], l, lv[(size_t)s * g->levels + l]);
    HSB_GROUP_CUDA(cudaMalloc(&g->d_lv, lv.size() * sizeof(HsbLevelDev)));
    HSB_GROUP_CUDA(cudaMemcpy(g->d_lv, lv.data(), lv.size() * sizeof(HsbLevelDev), cudaMemcpyHostToDevice));
    std::vector<int*> mirror((size_t)M * g->levels);
    for (int s = 0; s < M; ++s)
      for (int l = 0; l < g->m[s]->levels; ++l) mirror[(size_t)s * g->levels + l] = g->m[s]->lv[l].dirty + 4;
    HSB_GROUP_CUDA(cudaMalloc(&g->d_mirror, mirror.size() * sizeof(int*)));
    HSB_GROUP_CUDA(cudaMemcpy(g->d_mirror, mirror.data(), mirror.size() * sizeof(int*), cudaMemcpyHostToDevice));
    std::vector<HsbRayLevelDev> ray((size_t)M * g->levels);
    for (int s = 0; s < M; ++s)
      for (int l = 0; l < g->m[s]->levels; ++l) fill_ray_level(g->m[s], l, ray[(size_t)s * g->levels + l]);
    HSB_GROUP_CUDA(cudaMalloc(&g->d_ray_lv, ray.size() * sizeof(HsbRayLevelDev)));
    HSB_GROUP_CUDA(cudaMemcpy(g->d_ray_lv, ray.data(), ray.size() * sizeof(HsbRayLevelDev), cudaMemcpyHostToDevice));
    HSB_GROUP_CUDA(cudaMalloc(&g->d_best, (size_t)M * sizeof(unsigned long long)));
    HSB_GROUP_CUDA(cudaMemset(g->d_best, 0, (size_t)M * sizeof(unsigned long long)));
    std::vector<HsbTileLevelDev> tile((size_t)M * g->levels);
    std::vector<int*> counters(M);
    for (int s = 0; s < M; ++s) {
      HsbTileParams T;
      fill_tile_params(g->m[s], T, nullptr, 0);
      for (int l = 0; l < g->m[s]->levels; ++l) tile[(size_t)s * g->levels + l] = T.lv[l];
      counters[s] = T.error_count;
    }
    HSB_GROUP_CUDA(cudaMalloc(&g->d_tile_lv, tile.size() * sizeof(HsbTileLevelDev)));
    HSB_GROUP_CUDA(cudaMemcpy(g->d_tile_lv, tile.data(), tile.size() * sizeof(HsbTileLevelDev), cudaMemcpyHostToDevice));
    HSB_GROUP_CUDA(cudaMalloc(&g->d_tile_counters, counters.size() * sizeof(int*)));
    HSB_GROUP_CUDA(cudaMemcpy(g->d_tile_counters, counters.data(), counters.size() * sizeof(int*), cudaMemcpyHostToDevice));
    std::vector<HsbResetMemberDev> reset(M);
    memset(reset.data(), 0, reset.size() * sizeof(HsbResetMemberDev));
    for (int s = 0; s < M; ++s) {
      reset[s].gate = g->m[s]->d_gate;
      for (int l = 0; l < g->m[s]->levels; ++l) reset[s].stamp[l] = g->m[s]->lv[l].stamp;
    }
    HSB_GROUP_CUDA(cudaMalloc(&g->d_reset, reset.size() * sizeof(HsbResetMemberDev)));
    HSB_GROUP_CUDA(cudaMemcpy(g->d_reset, reset.data(), reset.size() * sizeof(HsbResetMemberDev), cudaMemcpyHostToDevice));
    if (g->ragged) {
      std::vector<int> nl(M);
      for (int s = 0; s < M; ++s) nl[s] = g->m[s]->levels;
      HSB_GROUP_CUDA(cudaMalloc(&g->d_member_levels, nl.size() * sizeof(int)));
      HSB_GROUP_CUDA(cudaMemcpy(g->d_member_levels, nl.data(), nl.size() * sizeof(int), cudaMemcpyHostToDevice));
    }
    for (cudaEvent_t& e : g->ev_tile) HSB_GROUP_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    HSB_GROUP_CUDA(cudaMalloc(&g->d_occ_meta, OccMeta(M).bytes));
    HSB_GROUP_CUDA(cudaMallocHost(reinterpret_cast<void**>(&g->h_occ_meta), OccMeta(M).bytes));
  }
  HSB_GROUP_CUDA(cudaMalloc(&g->d_res, ((size_t)M * 5 + 4) * sizeof(float)));
  HSB_GROUP_CUDA(cudaMemset(g->d_res, 0, ((size_t)M * 5 + 4) * sizeof(float)));
  HSB_GROUP_CUDA(cudaHostAlloc(&g->h_res, ((size_t)M * 14 + 4) * sizeof(float), cudaHostAllocMapped));
  memset(g->h_res, 0, ((size_t)M * 14 + 4) * sizeof(float));
  HSB_GROUP_CUDA(cudaHostGetDevicePointer(&g->h_res_dev, g->h_res, 0));
#undef HSB_GROUP_CUDA
  *out = g;
  return HSB_OK;
}

}  // namespace

extern "C" {

int hsb_group_create(hsb_handle* const* handles, int M, hsb_group** out) {
  return group_create(handles, M, out, GROUP_SAME, "hsb_group_create");
}

int hsb_group_create_mixed(hsb_handle* const* handles, int M, hsb_group** out) {
  return group_create(handles, M, out, GROUP_MIXED, "hsb_group_create_mixed");
}

int hsb_group_create_heterogeneous(hsb_handle* const* handles, int M, hsb_group** out) {
  return group_create(handles, M, out, GROUP_HETERO, "hsb_group_create_heterogeneous");
}

}  // extern "C"

namespace {

// What a group step's sessions bring: level-0 endpoints (hsb_group_slam_update), the node's projected point clouds
// (hsb_group_slam_update_cloud), raw LaserScan ranges (hsb_group_slam_update_ranges) or raw ranges to project
// (hsb_group_slam_update_projected).  All but endpoints are converted in the match kernel's staging step as
// hsb_slam_update_cloud / _ranges / _projected convert them.  Every array has one entry per session (K).
struct GroupInput {
  HsbInputKind kind;
  const char* fn;              // the entry point, for the error messages
  const float* hints;          // K x 3
  const float* pts;            // endpoints: xy pairs; cloud: Point32 triples; ranges: one float per beam
  const int* offsets;          // K + 1, in points (ranges: in beams)
  const float* origo;          // endpoints: K x 2 (NULL = 0, 0)
  const double* transforms;    // cloud / projected: K x 12 (NULL = every session's member's hsb_set_cloud_format transform)
};

// warps per session of the group match kernel: the shape the single SLAM steps take, so results are theirs bit for bit
constexpr int kGroupW = 8;

// The group step's match launch in gather mode `mode`; MODE_ANY only with GRP_STEP_HET (a heterogeneous group holding
// both gather modes).
template <int GRP, bool PROJ>
int launch_group_step(hsb_handle* h0, HsbMatchParams& P, int max_n, cudaStream_t st, int mode) {
  if constexpr (GRP == hsb::GRP_STEP_HET) {
    if (mode == hsb::MODE_ANY)
      return launch_match_t<kGroupW, 1, hsb::MODE_ANY, 4, false, false, GRP, PROJ>(h0, P, max_n, st, 1);
  }
  return mode == hsb::MODE_TEX ? launch_match_t<kGroupW, 1, hsb::MODE_TEX, 4, false, false, GRP, PROJ>(h0, P, max_n, st, 1)
                               : launch_match_t<kGroupW, 1, hsb::MODE_LDG, 4, false, false, GRP, PROJ>(h0, P, max_n, st, 1);
}

// The member list of a group call over K sessions: 0 <= K <= M, and with K > 0 a list of distinct indices in [0, M).
int check_members(hsb_group* g, const char* fn, int K, const int* members) {
  hsb_handle* h0 = g->m[0];
  const int M = (int)g->m.size();
  if (K < 0 || K > M) return fail(h0, HSB_ERR_INVALID_ARG, "%s: K is %d, must be in [0, %d]", fn, K, M);
  if (K == 0) return HSB_OK;
  if (!members) return fail(h0, HSB_ERR_INVALID_ARG, "%s: members is NULL with K = %d", fn, K);
  std::fill(g->listed.begin(), g->listed.end(), 0);
  for (int k = 0; k < K; ++k) {
    const int j = members[k];
    if (j < 0 || j >= M)
      return fail(h0, HSB_ERR_INVALID_ARG, "%s: session %d: member %d is outside [0, %d)", fn, k, j, M);
    if (g->listed[j]) return fail(h0, HSB_ERR_INVALID_ARG, "%s: session %d: member %d is listed twice", fn, k, j);
    g->listed[j] = 1;
  }
  return HSB_OK;
}

// The level rule of a heterogeneous group's level-taking calls: every listed member has level `level` (members not
// listed are not checked).  Checked before anything is queued.  In a group whose members share their level count the
// group's own range check (level < hsb_group::levels) is the whole rule.
int check_member_level(hsb_group* g, const char* fn, int K, const int* members, int level) {
  if (!g->ragged) return HSB_OK;
  for (int k = 0; k < K; ++k) {
    const hsb_handle* h = g->m[members[k]];
    if (level >= h->levels)
      return fail(g->m[0], HSB_ERR_INVALID_ARG, "%s: session %d: member %d has %d levels, level %d is not one of them",
                  fn, k, members[k], h->levels, level);
  }
  return HSB_OK;
}

// The K + 1 offsets `name` of a group call's sessions: given, starting at 0, never decreasing.
int check_offsets(hsb_handle* h0, const char* fn, const char* name, int K, const int* offsets) {
  if (!offsets) return fail(h0, HSB_ERR_INVALID_ARG, "%s: %s is NULL", fn, name);
  if (offsets[0] != 0) return fail(h0, HSB_ERR_INVALID_ARG, "%s: %s[0] is %d, must be 0", fn, name, offsets[0]);
  for (int k = 0; k < K; ++k)
    if (offsets[k + 1] < offsets[k])
      return fail(h0, HSB_ERR_INVALID_ARG, "%s: %s decrease at session %d (%d -> %d)", fn, name, k, offsets[k],
                  offsets[k + 1]);
  return HSB_OK;
}

// Orders the group's stream behind everything queued for the listed members: the work they queued themselves, and a
// pending step of another group they belong to.
int order_members(hsb_group* g, int K, const int* members) {
  hsb_handle* h0 = g->m[0];
  for (int k = 0; k < K; ++k) {
    hsb_handle* h = g->m[members[k]];
    if (h->group_ev && h->group_ev != g->ev) HSB_CUDA(h0, cudaStreamWaitEvent(g->stream, h->group_ev, 0));
    if (h->queued) {
      const int s = order_before(h, g->stream, true);
      if (s != HSB_OK) return s;
      h->queued = false;
    }
  }
  return HSB_OK;
}

// One group step of any input kind over K of the group's members: session k steps member members[k] (a step of every
// member passes K = M and g->all).  Members not listed are neither read nor changed.  Everything that can reject the
// step is checked before any member's state moves.
int group_step(hsb_group* g, const GroupInput& in, int K, const int* members, const int* map_without_matching,
               int nowait, float* out_poses, float* cov_inout, int* map_updated, int* out_kept) {
  hsb_handle* h0 = g->m[0];   // launches and errors are accounted on handles[0], whether or not it is stepped
  const int M = (int)g->m.size(), levels = g->levels;
  int s = check_members(g, in.fn, K, members);
  if (s != HSB_OK || K == 0) return s;
  const bool cloud = in.kind == HSB_IN_CLOUD;
  const bool conv = in.kind != HSB_IN_ENDPOINTS;   // converted on the device: the kept count decides what the session had
  const bool tf = cloud || in.kind == HSB_IN_PROJECTED;   // with a laser transform per session
  const int* offsets = in.offsets;
  if (!in.hints || !offsets || !out_poses)
    return fail(h0, HSB_ERR_INVALID_ARG, "%s: hints, offsets and out_poses must not be NULL", in.fn);
  if ((s = check_offsets(h0, in.fn, "offsets", K, offsets)) != HSB_OK) return s;
  int max_n = 0;
  for (int k = 0; k < K; ++k) max_n = std::max(max_n, offsets[k + 1] - offsets[k]);
  const int total = offsets[K];
  if (total > 0 && !in.pts)
    return fail(h0, HSB_ERR_INVALID_ARG, "%s: %s is NULL", in.fn, cloud ? "points_xyz" : conv ? "ranges" : "points_xy");
  for (int k = 0; conv && k < K; ++k) {
    if ((s = check_input(g->m[members[k]], h0, in.kind, in.fn, k, offsets[k + 1] - offsets[k], false)) != HSB_OK)
      return s;
  }
  // every scan is converted whole into shared memory: the launcher's limit for the group kernel's shape
  if (conv && !staging_fits<kGroupW, 1>(whole_scan_slots(max_n), 1)) return fail_fused_too_long(h0, max_n);
  DeviceGuard guard(g->device);
  cudaStream_t st = g->stream;
  if ((s = order_members(g, K, members)) != HSB_OK) return s;

  // staging: hints | gate inputs | offsets | session descriptors | map-writer descriptors | increments |
  // laser transforms (cloud, projected) | scans
  auto al = [](size_t x) { return (x + 15) & ~(size_t)15; };
  const size_t o_gin = al((size_t)K * 12), o_off = al(o_gin + (size_t)K * 12), o_sess = al(o_off + (size_t)(K + 1) * 4);
  const size_t o_upd = al(o_sess + (size_t)K * sizeof(HsbGroupSessionDev));
  const size_t o_lo = al(o_upd + (size_t)K * levels * sizeof(HsbUpdateLevelDev)), o_tf = al(o_lo + (size_t)K * 8);
  const size_t o_pts = al(o_tf + (tf ? (size_t)K * 12 * sizeof(double) : 0));
  const size_t pt_bytes = cloud ? 12 : conv ? 4 : 8;
  const size_t bytes = o_pts + (size_t)total * pt_bytes;
  if ((s = ensure_pinned(h0, g->h_stage, g->h_stage_bytes, bytes)) != HSB_OK) return s;
  if ((s = ensure(h0, g->d_stage, bytes)) != HSB_OK) return s;
  char* hs = g->h_stage;
  const char* ds = static_cast<const char*>(g->d_stage.p);
  float* s_gin = reinterpret_cast<float*>(hs + o_gin);
  HsbGroupSessionDev* s_sess = reinterpret_cast<HsbGroupSessionDev*>(hs + o_sess);
  HsbUpdateLevelDev* s_upd = reinterpret_cast<HsbUpdateLevelDev*>(hs + o_upd);
  float2* s_lo = reinterpret_cast<float2*>(hs + o_lo);
  double* s_tf = reinterpret_cast<double*>(hs + o_tf);
  const char* d_in = ds + o_pts;
  memcpy(hs, in.hints, (size_t)K * 12);
  memcpy(hs + o_off, offsets, (size_t)(K + 1) * 4);
  if (total > 0) memcpy(hs + o_pts, in.pts, (size_t)total * pt_bytes);
  // a converted session's kept-endpoint count: in device memory for the map writer, in mapped host memory for the host
  int* kept_dev = reinterpret_cast<int*>(g->d_res + 4 * (size_t)M + 4);
  int* kept_mapped = reinterpret_cast<int*>(g->h_res_dev + 13 * (size_t)M + 4);
  int max_upd = 0;
  for (int k = 0; k < K; ++k) {
    hsb_handle* h = g->m[members[k]];
    const int n = offsets[k + 1] - offsets[k];   // a cloud's size / a scan's beams: an upper bound of the endpoints kept
    const bool matched = !(map_without_matching && map_without_matching[k]);
    const double* T = nullptr;
    if (tf) {
      T = in.transforms ? in.transforms + 12 * (size_t)k : h->cfmt.laser_transform;
      memcpy(s_tf + 12 * (size_t)k, T, 12 * sizeof(double));
    }
    StepSession ss;
    if ((s = step_session(h, in.kind, n, T, in.origo ? in.origo + 2 * k : nullptr, matched, kept_dev + k, kept_mapped + k,
                          ss)) != HSB_OK)
      return s;
    memcpy(s_gin + 3 * k, ss.gate_in, sizeof(ss.gate_in));
    s_lo[k] = make_float2(h->log_odds_free, h->log_odds_occ);
    HsbGroupSessionDev& gs = s_sess[k];
    memset(&gs, 0, sizeof(gs));
    gs.gate_state = h->d_gate;
    gs.member = members[k];
    gs.levels = h->levels;
    gs.conv = ss.conv;
    h->stepped = true;
    h->step_rec_matched = h->step_rec_on && matched;
    gs.record = h->step_rec_matched ? h->h_step_rec_dev : nullptr;
    if (matched && !conv) gs.last_pts = reinterpret_cast<float2*>(scan_points(*ss.sink));   // the match copies the scan there
    if (matched) record_match(h, n, ss.origo);
    // level 0 reads the staged endpoints, or a converted scan where it was converted to, with its count on the device
    const float2* pts0 = conv ? ss.conv.out_pts : reinterpret_cast<const float2*>(d_in) + offsets[k];
    if ((s = fill_update_levels(h, s_upd + (size_t)k * levels, pts0, n, ss.conv.out_n, ss.origo, matched, st, &max_upd)) !=
        HSB_OK)
      return s;
    // a member with fewer levels than the group: its writer slots past them are inactive
    if (h->levels < levels)
      memset(s_upd + (size_t)k * levels + h->levels, 0, (size_t)(levels - h->levels) * sizeof(HsbUpdateLevelDev));
  }
  HSB_CUDA(h0, cudaMemcpyAsync(g->d_stage.p, hs, bytes, cudaMemcpyHostToDevice, st));

  // K1: (conversion +) match + gate, one session per CTA; the last session to finish publishes the step's sequence number
  HsbMatchParams P;
  fill_match_params(h0, P);
  P.levels = levels;   // the stride of group_lv (the sessions' own level counts: GRP_STEP_HET)
  P.B = K;
  P.hints = reinterpret_cast<const float*>(ds);
  // (a converted session converts with its own descriptor, HsbGroupSessionDev::conv)
  fill_scan(h0, {in.kind, reinterpret_cast<const float*>(d_in), reinterpret_cast<const int*>(ds + o_off), 0, max_n,
                 tf ? reinterpret_cast<const double*>(ds + o_tf) : nullptr}, P);
  P.out_poses = g->d_res;
  P.out_cov = g->h_res_dev + 4 * (size_t)M;
  P.gate_in = reinterpret_cast<const float*>(ds + o_gin);
  P.gate_out_host = g->h_res_dev;
  P.seq_host = reinterpret_cast<unsigned*>(g->h_res_dev + 13 * (size_t)M);
  P.seq_value = ++g->seq;
  P.group_lv = g->d_lv;
  P.group_sess = reinterpret_cast<const HsbGroupSessionDev*>(ds + o_sess);
  P.group_done = reinterpret_cast<unsigned*>(g->d_res + 4 * (size_t)M);
  {
    // each session on its member's levels (GRP_STEP_HET) when the members differ in level count or gather mode, in the
    // members' one gather mode, or MODE_ANY when they hold both
    const int mode = g->any_mode ? hsb::MODE_ANY : h0->gather_mode == HSB_GATHER_TEX ? hsb::MODE_TEX : hsb::MODE_LDG;
    const bool proj = in.kind == HSB_IN_PROJECTED;
    if (g->ragged || g->any_mode)
      s = proj ? launch_group_step<hsb::GRP_STEP_HET, true>(h0, P, max_n, st, mode)
               : launch_group_step<hsb::GRP_STEP_HET, false>(h0, P, max_n, st, mode);
    else
      s = proj ? launch_group_step<hsb::GRP_STEP, true>(h0, P, max_n, st, mode)
               : launch_group_step<hsb::GRP_STEP, false>(h0, P, max_n, st, mode);
  }
  if (s != HSB_OK) return s;

  // K2: mark and apply over (session, level), behind the match with programmatic dependent launch, in the single
  // write's grids shared out among the sessions (a cloud's size or a scan's beam count bounds its endpoints: the grids
  // are sized by it)
  HsbGroupUpdateParams U;
  U.lv = reinterpret_cast<const HsbUpdateLevelDev*>(ds + o_upd);
  U.log_odds = reinterpret_cast<const float2*>(ds + o_lo);
  U.res = g->d_res;
  U.levels = levels;
  s = launch_map_write<hsb::update_mark_group_kernel<kMarkTeam>, hsb::update_apply_group_kernel>(h0, st, U, levels, K,
                                                                                                 max_upd, true);
  if (s != HSB_OK) return s;
  HSB_CUDA(h0, cudaEventRecord(g->ev, st));
  // every later operation of a stepped member waits for this step (HandleScope).  A member left out keeps its own
  // group_ev: a map write still pending from an earlier nowait step of this group is waited for through the event,
  // now recorded behind this step on the same stream.
  for (int k = 0; k < K; ++k) {
    hsb_handle* h = g->m[members[k]];
    h->group_ev = nowait ? g->ev : nullptr;
    h->map_write_pending = nowait != 0;
  }

  if (nowait) {   // return when every pose has arrived; the map writes continue on the group's stream
    volatile unsigned* seq = reinterpret_cast<volatile unsigned*>(g->h_res + 13 * (size_t)M);
    if ((s = wait_published(h0, seq, P.seq_value, st, "group step finished without publishing its poses")) != HSB_OK) return s;
  } else {
    HSB_CUDA(h0, cudaStreamSynchronize(st));   // :93 onMapUpdated for every stepped member
  }
  const int* kept_host = reinterpret_cast<const int*>(g->h_res + 13 * (size_t)M + 4);
  for (int k = 0; k < K; ++k) {
    const bool matched = !(map_without_matching && map_without_matching[k]);
    step_results(g->m[members[k]], matched, conv ? kept_host[k] : offsets[k + 1] - offsets[k], g->h_res + 4 * (size_t)k,
                 g->h_res + 4 * (size_t)M + 9 * (size_t)k, out_poses + 3 * (size_t)k, map_updated ? map_updated + k : nullptr,
                 cov_inout ? cov_inout + 9 * (size_t)k : nullptr, out_kept ? out_kept + k : nullptr);
  }
  return HSB_OK;
}

// Packed bytes of one device-to-host copy of a group occupancy sync (pinned staging owned by the group).  A larger total
// goes in chunks split at row boundaries; hsb_set_tuning(handles[0], "occupancy_chunk", bytes) overrides it.  A chunk
// always holds at least one whole row of the widest level among the call's changed members (in a group of one geometry,
// handles[0]'s row), so every rectangle's row fits one.
constexpr size_t kOccChunkBytes = 32u << 20;

// publishMap's grid for K members in one pass: gather (and clear) their mirror rectangles of `level` with one launch,
// one synchronise to size the payload, then per chunk one threshold launch, one device-to-host copy and one synchronise,
// and the rows scattered into grids[k] on the host.
int group_sync_occupancy(hsb_group* g, const char* fn, int K, const int* members, int level, int8_t* const* grids,
                         int* out_rects, int reset) {
  hsb_handle* h0 = g->m[0];   // launches and errors are accounted on handles[0], whether or not it is listed
  int s = check_members(g, fn, K, members);
  if (s != HSB_OK || K == 0) return s;
  if (level < 0 || level >= g->levels)
    return fail(h0, HSB_ERR_INVALID_ARG, "%s: level %d is outside [0, %d)", fn, level, g->levels);
  if ((s = check_member_level(g, fn, K, members, level)) != HSB_OK) return s;
  if (!grids) return fail(h0, HSB_ERR_INVALID_ARG, "%s: grids is NULL", fn);
  for (int k = 0; k < K; ++k)
    if (!grids[k]) return fail(h0, HSB_ERR_INVALID_ARG, "%s: session %d: grid is NULL", fn, k);
  DeviceGuard guard(g->device);
  cudaStream_t st = g->stream;
  if ((s = order_members(g, K, members)) != HSB_OK) return s;

  // pass 1: the rectangles, gathered and (reset) cleared in order behind the members' queued map writes
  const OccMeta lay(K);
  memcpy(g->h_occ_meta, members, (size_t)K * sizeof(int));
  HSB_CUDA(h0, cudaMemcpyAsync(g->d_occ_meta, g->h_occ_meta, (size_t)K * sizeof(int), cudaMemcpyHostToDevice, st));
  hsb::gather_mirror_rects_kernel<<<(K + 127) / 128, 128, 0, st>>>(
      g->d_mirror, g->levels, level, reinterpret_cast<const int*>(g->d_occ_meta), K, reset,
      reinterpret_cast<int4*>(g->d_occ_meta + lay.rects));
  h0->launches++;
  HSB_CUDA(h0, cudaGetLastError());
  HSB_CUDA(h0, cudaMemcpyAsync(g->h_occ_meta + lay.rects, g->d_occ_meta + lay.rects, (size_t)K * sizeof(int4),
                               cudaMemcpyDeviceToHost, st));
  HSB_CUDA(h0, cudaStreamSynchronize(st));
  const int* rects = reinterpret_cast<const int*>(g->h_occ_meta + lay.rects);
  if (out_rects) memcpy(out_rects, rects, (size_t)K * 4 * sizeof(int));

  // the row table of the non-empty rectangles, in session order
  HsbOccRowsDev* rows = reinterpret_cast<HsbOccRowsDev*>(g->h_occ_meta + lay.rows);
  std::vector<int> sess;   // session of each row-table entry
  int n_rows = 0, total_rows = 0, max_sx = 0;
  size_t total = 0;
  for (int k = 0; k < K; ++k) {
    const int* r = rects + 4 * k;
    if (r[2] < r[0] || r[3] < r[1]) continue;   // clean: the map did not change
    hsb_handle* h = g->m[members[k]];
    HsbOccRowsDev& e = rows[n_rows++];
    e.logodds = h->lv[level].logodds;
    e.sx = h->lv[level].sx;   // (the member's own row pitch: members of a mixed group differ)
    max_sx = std::max(max_sx, e.sx);
    e.x0 = r[0];
    e.y0 = r[1];
    e.w = r[2] - r[0] + 1;
    e.row0 = total_rows;
    e.off = total;
    const int hgt = r[3] - r[1] + 1;
    total_rows += hgt;
    total += (size_t)e.w * hgt;
    h->d2h_bytes += (size_t)e.w * hgt;
    sess.push_back(k);
  }
  if (n_rows == 0) return HSB_OK;
  HSB_CUDA(h0, cudaMemcpyAsync(g->d_occ_meta + lay.rows, rows, (size_t)n_rows * sizeof(HsbOccRowsDev),
                               cudaMemcpyHostToDevice, st));

  // pass 2: chunks of whole rows
  const size_t cap = std::max<size_t>(h0->tune_occ_chunk > 0 ? (size_t)h0->tune_occ_chunk : kOccChunkBytes, (size_t)max_sx);
  if (std::min(cap, total) > g->h_occ_rows_bytes) {   // grown geometrically: dirty areas creep up from call to call
    const size_t stage = std::min(cap, std::max(total, 2 * g->h_occ_rows_bytes));
    if (g->h_occ_rows) cudaFreeHost(g->h_occ_rows);
    g->h_occ_rows = nullptr;
    g->h_occ_rows_bytes = 0;
    HSB_CUDA(h0, cudaMallocHost(reinterpret_cast<void**>(&g->h_occ_rows), stage));
    g->h_occ_rows_bytes = stage;
    if ((s = ensure(h0, g->d_occ_rows, stage)) != HSB_OK) return s;
  }
  int8_t* d_out = static_cast<int8_t*>(g->d_occ_rows.p);
  int e = 0, y = 0;   // the chunk starts at row y of row-table entry e
  while (e < n_rows) {
    const int e_begin = e, y_begin = y;
    const size_t base = rows[e].off + (size_t)y * rows[e].w;
    size_t bytes = 0;
    while (e < n_rows) {   // whole rectangles while they fit, then as many rows of the next one as fit
      const int w = rows[e].w, left = rects[4 * sess[e] + 3] - rects[4 * sess[e] + 1] + 1 - y;
      const size_t fit = (cap - bytes) / (size_t)w;
      if (fit >= (size_t)left) {
        bytes += (size_t)left * w;
        ++e;
        y = 0;
      } else {
        bytes += fit * w;
        y += (int)fit;
        break;
      }
    }
    const int r_begin = rows[e_begin].row0 + y_begin, r_end = (e < n_rows ? rows[e].row0 + y : total_rows);
    const int blocks = (int)std::min<long>(((long)(r_end - r_begin) + 7) / 8, (long)h0->sm_count * 16);
    hsb::occupancy_rows_kernel<<<blocks, 256, 0, st>>>(reinterpret_cast<const HsbOccRowsDev*>(g->d_occ_meta + lay.rows),
                                                       n_rows, r_begin, r_end, base, d_out);
    h0->launches++;
    HSB_CUDA(h0, cudaGetLastError());
    HSB_CUDA(h0, cudaMemcpyAsync(g->h_occ_rows, d_out, bytes, cudaMemcpyDeviceToHost, st));
    HSB_CUDA(h0, cudaStreamSynchronize(st));
    // scatter the chunk's rows into the callers' grids
    const int8_t* src = g->h_occ_rows;
    for (int ee = e_begin, yy = y_begin; src < g->h_occ_rows + bytes; ++ee, yy = 0) {
      const HsbOccRowsDev& d = rows[ee];
      const int hgt = rects[4 * sess[ee] + 3] - d.y0 + 1;
      for (; yy < hgt && src < g->h_occ_rows + bytes; ++yy, src += d.w)
        memcpy(grids[sess[ee]] + (size_t)(d.y0 + yy) * d.sx + d.x0, src, (size_t)d.w);
    }
  }
  return HSB_OK;
}

// hsb_raycast_batch (world: hsb_get_dist_batch) for K members in one pass: session k's rays [offsets[k], offsets[k+1])
// on member members[k], behind the members' queued work, through the group's pinned staging and plane table (ray_query:
// one copy each way and one synchronise, whatever K is).  No member's state changes.
int group_rays(hsb_group* g, const char* fn, bool world, int K, const int* members, int level, const int* offsets,
               const void* begin, const void* end, float* out_dist, void* out_hit, int* out_found) {
  hsb_handle* h0 = g->m[0];   // launches and errors are accounted on handles[0], whether or not it is listed
  int s = check_members(g, fn, K, members);
  if (s != HSB_OK || K == 0) return s;
  if (level < 0 || level >= g->levels)
    return fail(h0, HSB_ERR_INVALID_ARG, "%s: level %d is outside [0, %d)", fn, level, g->levels);
  if ((s = check_member_level(g, fn, K, members, level)) != HSB_OK) return s;
  if ((s = check_offsets(h0, fn, "offsets", K, offsets)) != HSB_OK) return s;
  const int Q = offsets[K];
  if (Q == 0) return HSB_OK;
  if (!begin || !end || !out_dist)
    return fail(h0, HSB_ERR_INVALID_ARG, "%s: %s, %s and out_dist must not be NULL", fn,
                world ? "begin_world" : "begin_cells", world ? "end_world" : "end_cells");
  DeviceGuard guard(g->device);
  if ((s = order_members(g, K, members)) != HSB_OK) return s;
  return ray_query(h0, g->stream, g->h_ray_stage, g->h_ray_stage_bytes, g->d_ray_stage, g->d_ray_lv, g->levels, level,
                   world, K, members, offsets, begin, end, out_dist, out_hit, out_found);
}

// The scans of a group pose query (scoring or match): session k's is pts[scan_offsets[k] .. scan_offsets[k+1]), staged
// with the call, or, with pts and scan_offsets both NULL, its member's last-match container as it is on the device when
// the call runs.
int check_scans(hsb_handle* h0, const char* fn, int K, const float* pts, const int* scan_offsets) {
  if (!pts != !scan_offsets)
    return fail(h0, HSB_ERR_INVALID_ARG, "%s: points_xy and scan_offsets must both be given or both be NULL", fn);
  return pts ? check_offsets(h0, fn, "scan_offsets", K, scan_offsets) : HSB_OK;
}

// The length of session k's scan on member h by check_scans' rule (a member that never matched has no container: 0).
int scan_length(const hsb_handle* h, const int* scan_offsets, int k) {
  if (scan_offsets) return scan_offsets[k + 1] - scan_offsets[k];
  return h->d_last_pts.p ? h->last_n : 0;
}

// score_query's `sessions` for a group pose query: session k is member members[k] with its scan by check_scans' rule
// (`staged`: where score_query puts the scans sent with the call) and the k-th of the K + 1 `offsets` of its poses or
// hints; its cell length is its member's of `level`.
auto group_sessions(hsb_group* g, int K, const int* members, int level, const int* offsets, const int* scan_offsets) {
  return [=](HsbScoreSessionDev* sess, int* staged_offsets, const float2* staged) {
    for (int k = 0; k < K; ++k) {
      hsb_handle* h = g->m[members[k]];
      if (scan_offsets) sess[k].pts = staged + scan_offsets[k];
      else sess[k].pts = h->d_last_pts.p ? reinterpret_cast<const float2*>(scan_points(h->d_last_pts)) : nullptr;
      sess[k].n = scan_length(h, scan_offsets, k);
      sess[k].member = members[k];
      sess[k].cell_length = h->lv[level].cell_length;
      sess[k].levels = h->levels;
    }
    memcpy(staged_offsets, offsets, (size_t)(K + 1) * 4);
  };
}

// hsb_likelihood_batch / hsb_covariance_batch / hsb_best_hypothesis_device for K members in one pass: session k's poses
// [pose_offsets[k], pose_offsets[k+1]) scored on member members[k]'s map of `level` against the session's scan
// (check_scans).  Behind the members' queued work, through the group's pinned query staging and descriptor table
// (score_query: one copy each way, one launch, two for the best hypothesis, and one synchronise, whatever K is).  No
// member's state changes.
int group_score(hsb_group* g, const char* fn, ScoreKind kind, int K, const int* members, int level, const int* pose_offsets,
                const float* poses, const float* pts, const int* scan_offsets, float* out_lh, float* out_map,
                float* out_world, float* out_best4, int* out_best_index) {
  hsb_handle* h0 = g->m[0];   // launches and errors are accounted on handles[0], whether or not it is listed
  int s = check_members(g, fn, K, members);
  if (s != HSB_OK || K == 0) return s;
  if (level < 0 || level >= g->levels)
    return fail(h0, HSB_ERR_INVALID_ARG, "%s: level %d is outside [0, %d)", fn, level, g->levels);
  if ((s = check_member_level(g, fn, K, members, level)) != HSB_OK) return s;
  if ((s = check_offsets(h0, fn, "pose_offsets", K, pose_offsets)) != HSB_OK) return s;
  if ((s = check_scans(h0, fn, K, pts, scan_offsets)) != HSB_OK) return s;
  const int Q = pose_offsets[K];
  if (Q == 0) {   // nothing to score: every session's best hypothesis is the empty batch's
    for (int k = 0; kind == SCORE_BEST && out_best4 && k < K; ++k) {
      out_best4[4 * k] = -1.0f;
      out_best4[4 * k + 1] = out_best4[4 * k + 2] = out_best4[4 * k + 3] = 0.0f;
      if (out_best_index) out_best_index[k] = -1;
    }
    return HSB_OK;
  }
  if (!poses) return fail(h0, HSB_ERR_INVALID_ARG, "%s: poses_world is NULL", fn);
  if (kind == SCORE_LIKELIHOOD && !out_lh) return fail(h0, HSB_ERR_INVALID_ARG, "%s: out_likelihood is NULL", fn);
  if (kind == SCORE_COVARIANCE && !out_map && !out_world)
    return fail(h0, HSB_ERR_INVALID_ARG, "%s: out_cov_map and out_cov_world are both NULL", fn);
  if (kind == SCORE_BEST && !out_best4) return fail(h0, HSB_ERR_INVALID_ARG, "%s: out_best4 is NULL", fn);
  DeviceGuard guard(g->device);
  if ((s = order_members(g, K, members)) != HSB_OK) return s;
  // (h0's gather mode is every member's unless the group is heterogeneous and holds both: any_mode)
  return score_query(h0, g->stream, g->h_ray_stage, g->h_ray_stage_bytes, g->d_ray_stage, g->d_lv, g->levels, level, kind,
                     K, Q, poses, pts, pts ? (size_t)scan_offsets[K] : 0,
                     group_sessions(g, K, members, level, pose_offsets, scan_offsets), g->d_best, out_lh, out_map,
                     out_world, out_best4, out_best_index, nullptr, g->ragged, g->any_mode);
}

// hsb_match_batch in shared-scan mode for K members in one pass: session k's hints [hint_offsets[k], hint_offsets[k+1])
// each matched over all levels on member members[k]'s maps with the session's one scan (check_scans).  One match-kernel
// launch (GRP_MATCH: one hint per scan) in the shape hsb_match_batch would take for Q hints, behind the members' queued
// work, through the group's pinned query staging (score_query: one copy each way and one synchronise, whatever K is).
// The launch shape is chosen, and a tuning without a group match kernel rejected, before anything is queued.  No
// member's state changes.
int group_match(hsb_group* g, const char* fn, int K, const int* members, const int* hint_offsets, const float* hints,
                const float* pts, const int* scan_offsets, float* out_poses, float* out_cov) {
  hsb_handle* h0 = g->m[0];   // launches, launch shape and errors are accounted on handles[0], whether or not it is listed
  int s = check_members(g, fn, K, members);
  if (s != HSB_OK || K == 0) return s;
  if ((s = check_offsets(h0, fn, "hint_offsets", K, hint_offsets)) != HSB_OK) return s;
  if ((s = check_scans(h0, fn, K, pts, scan_offsets)) != HSB_OK) return s;
  const int Q = hint_offsets[K];
  if (Q == 0) return HSB_OK;
  if (!hints) return fail(h0, HSB_ERR_INVALID_ARG, "%s: hints_world is NULL", fn);
  if (!out_poses) return fail(h0, HSB_ERR_INVALID_ARG, "%s: out_poses_world is NULL", fn);
  // the launch shape: hsb_match_batch's for Q hints (launch_match), among the shapes the group match is compiled for —
  // W in {1, 2, 4, 8}, one scan per CTA, 4 gathers in flight, unpacked (with one warp per scan, grouping scans into
  // CTAs does not change a bit, so the auto-group shapes need no twin)
  const int W = h0->tune_warps_per_scan > 0 ? h0->tune_warps_per_scan : auto_warps_per_scan(h0, Q);
  const int G = h0->tune_scans_per_block > 0 ? h0->tune_scans_per_block : 1;
  const int U = h0->tune_unroll > 0 ? h0->tune_unroll : 4;
  if (!has_projected_kernel(h0, W, G, U))   // (the same set of shapes)
    return fail(h0, HSB_ERR_UNSUPPORTED, "%s: no group match kernel for tuning warps_per_scan=%d scans_per_block=%d "
                "unroll=%d packed=%d", fn, W, G, U, h0->tune_packed);
  MatchQuery mq = {W, 0, out_poses, out_cov};
  // (only a session with hints launches work: an unused long scan must not shrink the staging of the others)
  for (int k = 0; k < K; ++k)
    if (hint_offsets[k + 1] > hint_offsets[k])
      mq.max_n = std::max(mq.max_n, scan_length(g->m[members[k]], scan_offsets, k));
  DeviceGuard guard(g->device);
  if ((s = order_members(g, K, members)) != HSB_OK) return s;
  // (the match reads no cell length: the sessions carry level 0's)
  return score_query(h0, g->stream, g->h_ray_stage, g->h_ray_stage_bytes, g->d_ray_stage, g->d_lv, g->levels, 0,
                     SCORE_MATCH, K, Q, hints, pts, pts ? (size_t)scan_offsets[K] : 0,
                     group_sessions(g, K, members, 0, hint_offsets, scan_offsets), nullptr, nullptr, nullptr, nullptr,
                     nullptr, nullptr, &mq, g->ragged, g->any_mode);
}

}  // namespace

extern "C" {

int hsb_group_likelihood(hsb_group* g, int level, const int* pose_offsets, const float* poses_world, const float* points_xy,
                         const int* scan_offsets, float* out_likelihood) {
  if (!g) return HSB_ERR_INVALID_ARG;
  return group_score(g, "hsb_group_likelihood", SCORE_LIKELIHOOD, (int)g->m.size(), g->all.data(), level, pose_offsets,
                     poses_world, points_xy, scan_offsets, out_likelihood, nullptr, nullptr, nullptr, nullptr);
}

int hsb_group_likelihood_subset(hsb_group* g, int K, const int* members, int level, const int* pose_offsets,
                                const float* poses_world, const float* points_xy, const int* scan_offsets,
                                float* out_likelihood) {
  if (!g) return HSB_ERR_INVALID_ARG;
  return group_score(g, "hsb_group_likelihood_subset", SCORE_LIKELIHOOD, K, members, level, pose_offsets, poses_world,
                     points_xy, scan_offsets, out_likelihood, nullptr, nullptr, nullptr, nullptr);
}

int hsb_group_covariance(hsb_group* g, int level, const int* pose_offsets, const float* poses_world, const float* points_xy,
                         const int* scan_offsets, float* out_cov_map, float* out_cov_world) {
  if (!g) return HSB_ERR_INVALID_ARG;
  return group_score(g, "hsb_group_covariance", SCORE_COVARIANCE, (int)g->m.size(), g->all.data(), level, pose_offsets,
                     poses_world, points_xy, scan_offsets, nullptr, out_cov_map, out_cov_world, nullptr, nullptr);
}

int hsb_group_covariance_subset(hsb_group* g, int K, const int* members, int level, const int* pose_offsets,
                                const float* poses_world, const float* points_xy, const int* scan_offsets,
                                float* out_cov_map, float* out_cov_world) {
  if (!g) return HSB_ERR_INVALID_ARG;
  return group_score(g, "hsb_group_covariance_subset", SCORE_COVARIANCE, K, members, level, pose_offsets, poses_world,
                     points_xy, scan_offsets, nullptr, out_cov_map, out_cov_world, nullptr, nullptr);
}

int hsb_group_best_hypothesis(hsb_group* g, int level, const int* pose_offsets, const float* poses_world,
                              const float* points_xy, const int* scan_offsets, float* out_likelihood, float* out_best4,
                              int* out_best_index) {
  if (!g) return HSB_ERR_INVALID_ARG;
  return group_score(g, "hsb_group_best_hypothesis", SCORE_BEST, (int)g->m.size(), g->all.data(), level, pose_offsets,
                     poses_world, points_xy, scan_offsets, out_likelihood, nullptr, nullptr, out_best4, out_best_index);
}

int hsb_group_best_hypothesis_subset(hsb_group* g, int K, const int* members, int level, const int* pose_offsets,
                                     const float* poses_world, const float* points_xy, const int* scan_offsets,
                                     float* out_likelihood, float* out_best4, int* out_best_index) {
  if (!g) return HSB_ERR_INVALID_ARG;
  return group_score(g, "hsb_group_best_hypothesis_subset", SCORE_BEST, K, members, level, pose_offsets, poses_world,
                     points_xy, scan_offsets, out_likelihood, nullptr, nullptr, out_best4, out_best_index);
}

int hsb_group_match_batch(hsb_group* g, const int* hint_offsets, const float* hints_world, const float* points_xy,
                          const int* scan_offsets, float* out_poses_world, float* out_cov) {
  if (!g) return HSB_ERR_INVALID_ARG;
  return group_match(g, "hsb_group_match_batch", (int)g->m.size(), g->all.data(), hint_offsets, hints_world, points_xy,
                     scan_offsets, out_poses_world, out_cov);
}

int hsb_group_match_batch_subset(hsb_group* g, int K, const int* members, const int* hint_offsets,
                                 const float* hints_world, const float* points_xy, const int* scan_offsets,
                                 float* out_poses_world, float* out_cov) {
  if (!g) return HSB_ERR_INVALID_ARG;
  return group_match(g, "hsb_group_match_batch_subset", K, members, hint_offsets, hints_world, points_xy, scan_offsets,
                     out_poses_world, out_cov);
}

int hsb_group_raycast(hsb_group* g, int level, const int* offsets, const int* begin_cells, const int* end_cells,
                      float* out_dist, int* out_hit) {
  if (!g) return HSB_ERR_INVALID_ARG;
  return group_rays(g, "hsb_group_raycast", false, (int)g->m.size(), g->all.data(), level, offsets, begin_cells,
                    end_cells, out_dist, out_hit, nullptr);
}

int hsb_group_raycast_subset(hsb_group* g, int K, const int* members, int level, const int* offsets,
                             const int* begin_cells, const int* end_cells, float* out_dist, int* out_hit) {
  if (!g) return HSB_ERR_INVALID_ARG;
  return group_rays(g, "hsb_group_raycast_subset", false, K, members, level, offsets, begin_cells, end_cells, out_dist,
                    out_hit, nullptr);
}

int hsb_group_get_dist(hsb_group* g, int level, const int* offsets, const float* begin_world, const float* end_world,
                       float* out_dist, float* out_hit_world, int* out_found) {
  if (!g) return HSB_ERR_INVALID_ARG;
  return group_rays(g, "hsb_group_get_dist", true, (int)g->m.size(), g->all.data(), level, offsets, begin_world,
                    end_world, out_dist, out_hit_world, out_found);
}

int hsb_group_get_dist_subset(hsb_group* g, int K, const int* members, int level, const int* offsets,
                              const float* begin_world, const float* end_world, float* out_dist, float* out_hit_world,
                              int* out_found) {
  if (!g) return HSB_ERR_INVALID_ARG;
  return group_rays(g, "hsb_group_get_dist_subset", true, K, members, level, offsets, begin_world, end_world, out_dist,
                    out_hit_world, out_found);
}

int hsb_group_sync_occupancy(hsb_group* g, int level, int8_t* const* grids, int* out_rects, int reset) {
  if (!g) return HSB_ERR_INVALID_ARG;
  return group_sync_occupancy(g, "hsb_group_sync_occupancy", (int)g->m.size(), g->all.data(), level, grids, out_rects,
                              reset);
}

int hsb_group_sync_occupancy_subset(hsb_group* g, int K, const int* members, int level, int8_t* const* grids,
                                    int* out_rects, int reset) {
  if (!g) return HSB_ERR_INVALID_ARG;
  return group_sync_occupancy(g, "hsb_group_sync_occupancy_subset", K, members, level, grids, out_rects, reset);
}

int hsb_group_slam_update(hsb_group* g, const float* hints, const float* points_xy, const int* offsets, const float* origo,
                          const int* map_without_matching, int nowait, float* out_poses, float* cov_inout, int* map_updated) {
  if (!g) return HSB_ERR_INVALID_ARG;
  const GroupInput in = {HSB_IN_ENDPOINTS, "hsb_group_slam_update", hints, points_xy, offsets, origo, nullptr};
  return group_step(g, in, (int)g->m.size(), g->all.data(), map_without_matching, nowait, out_poses, cov_inout,
                    map_updated, nullptr);
}

int hsb_group_slam_update_cloud(hsb_group* g, const float* hints, const float* points_xyz, const int* offsets,
                                const double* transforms, const int* map_without_matching, int nowait, float* out_poses,
                                float* cov_inout, int* map_updated, int* out_kept) {
  if (!g) return HSB_ERR_INVALID_ARG;
  const GroupInput in = {HSB_IN_CLOUD, "hsb_group_slam_update_cloud", hints, points_xyz, offsets, nullptr, transforms};
  return group_step(g, in, (int)g->m.size(), g->all.data(), map_without_matching, nowait, out_poses, cov_inout,
                    map_updated, out_kept);
}

int hsb_group_slam_update_ranges(hsb_group* g, const float* hints, const float* ranges, const int* offsets,
                                 const int* map_without_matching, int nowait, float* out_poses, float* cov_inout,
                                 int* map_updated, int* out_kept) {
  if (!g) return HSB_ERR_INVALID_ARG;
  const GroupInput in = {HSB_IN_RANGES, "hsb_group_slam_update_ranges", hints, ranges, offsets, nullptr, nullptr};
  return group_step(g, in, (int)g->m.size(), g->all.data(), map_without_matching, nowait, out_poses, cov_inout,
                    map_updated, out_kept);
}

int hsb_group_slam_update_projected(hsb_group* g, const float* hints, const float* ranges, const int* offsets,
                                    const double* transforms, const int* map_without_matching, int nowait,
                                    float* out_poses, float* cov_inout, int* map_updated, int* out_kept) {
  if (!g) return HSB_ERR_INVALID_ARG;
  const GroupInput in = {HSB_IN_PROJECTED, "hsb_group_slam_update_projected", hints, ranges, offsets, nullptr, transforms};
  return group_step(g, in, (int)g->m.size(), g->all.data(), map_without_matching, nowait, out_poses, cov_inout,
                    map_updated, out_kept);
}

int hsb_group_slam_update_subset(hsb_group* g, int K, const int* members, const float* hints, const float* points_xy,
                                 const int* offsets, const float* origo, const int* map_without_matching, int nowait,
                                 float* out_poses, float* cov_inout, int* map_updated) {
  if (!g) return HSB_ERR_INVALID_ARG;
  const GroupInput in = {HSB_IN_ENDPOINTS, "hsb_group_slam_update_subset", hints, points_xy, offsets, origo, nullptr};
  return group_step(g, in, K, members, map_without_matching, nowait, out_poses, cov_inout, map_updated, nullptr);
}

int hsb_group_slam_update_cloud_subset(hsb_group* g, int K, const int* members, const float* hints,
                                       const float* points_xyz, const int* offsets, const double* transforms,
                                       const int* map_without_matching, int nowait, float* out_poses, float* cov_inout,
                                       int* map_updated, int* out_kept) {
  if (!g) return HSB_ERR_INVALID_ARG;
  const GroupInput in = {HSB_IN_CLOUD, "hsb_group_slam_update_cloud_subset", hints, points_xyz, offsets, nullptr,
                         transforms};
  return group_step(g, in, K, members, map_without_matching, nowait, out_poses, cov_inout, map_updated, out_kept);
}

int hsb_group_slam_update_ranges_subset(hsb_group* g, int K, const int* members, const float* hints, const float* ranges,
                                        const int* offsets, const int* map_without_matching, int nowait,
                                        float* out_poses, float* cov_inout, int* map_updated, int* out_kept) {
  if (!g) return HSB_ERR_INVALID_ARG;
  const GroupInput in = {HSB_IN_RANGES, "hsb_group_slam_update_ranges_subset", hints, ranges, offsets, nullptr, nullptr};
  return group_step(g, in, K, members, map_without_matching, nowait, out_poses, cov_inout, map_updated, out_kept);
}

int hsb_group_slam_update_projected_subset(hsb_group* g, int K, const int* members, const float* hints,
                                           const float* ranges, const int* offsets, const double* transforms,
                                           const int* map_without_matching, int nowait, float* out_poses,
                                           float* cov_inout, int* map_updated, int* out_kept) {
  if (!g) return HSB_ERR_INVALID_ARG;
  const GroupInput in = {HSB_IN_PROJECTED, "hsb_group_slam_update_projected_subset", hints, ranges, offsets, nullptr,
                         transforms};
  return group_step(g, in, K, members, map_without_matching, nowait, out_poses, cov_inout, map_updated, out_kept);
}

}  // extern "C"

// ---- group map replication: every session's dirty tiles in one buffer, one pack launch and one unpack launch --------
namespace {

// A subset pack lists its sessions' members in the launch parameters (no host-to-device copy whose pinned source a later
// call could overwrite before it runs): up to 128 in a 512-byte block, up to 4096 in a 16 KB one.
constexpr int kTileSubsetSmall = 128, kTileSubsetMax = 4096;

// The caller's stream behind everything queued on the sessions' members (members == nullptr: all M in order): a pending
// step of any group they belong to, and, for a member that queued work of its own since, its stream (all_streams: its
// copy streams too).  group_stream: also behind everything queued on this group's stream.
int tile_order_before(hsb_group* g, cudaStream_t user, int K, const int* members, bool all_streams, bool group_stream) {
  hsb_handle* h0 = g->m[0];
  if (group_stream) {
    HSB_CUDA(h0, cudaEventRecord(g->ev_tile[0], g->stream));
    HSB_CUDA(h0, cudaStreamWaitEvent(user, g->ev_tile[0], 0));
  }
  std::vector<cudaEvent_t> waited;
  for (int k = 0; k < K; ++k) {
    hsb_handle* h = g->m[members ? members[k] : k];
    if (h->group_ev && std::find(waited.begin(), waited.end(), h->group_ev) == waited.end()) {
      HSB_CUDA(h0, cudaStreamWaitEvent(user, h->group_ev, 0));
      waited.push_back(h->group_ev);
    }
    if (h->queued) {
      const int s = order_before(h, user, all_streams);
      if (s != HSB_OK) return s;
    }
  }
  return HSB_OK;
}

// Everything the sessions' members queue after the call waits for it: the group's stream waits for the caller's, and the
// members take the group's event, recorded behind that wait, as they take a nowait step's (HandleScope, order_members).
// map_write: the members' planes were written (a match on a copy stream waits for the handle's stream, launch_match).
int tile_order_after(hsb_group* g, cudaStream_t user, int K, const int* members, bool map_write) {
  hsb_handle* h0 = g->m[0];
  HSB_CUDA(h0, cudaEventRecord(g->ev_tile[1], user));
  HSB_CUDA(h0, cudaStreamWaitEvent(g->stream, g->ev_tile[1], 0));
  HSB_CUDA(h0, cudaEventRecord(g->ev, g->stream));
  for (int k = 0; k < K; ++k) {
    hsb_handle* h = g->m[members ? members[k] : k];
    h->group_ev = g->ev;
    if (map_write) h->map_write_pending = true;
  }
  return HSB_OK;
}

void fill_group_tile_params(hsb_group* g, HsbTileParams& T, float* d_buf, size_t capacity_bytes, int K) {
  memset(&T, 0, sizeof(T));
  T.levels = g->levels;
  T.buf = d_buf;
  T.capacity_words = std::min<size_t>(capacity_bytes / 4, 0xffffffffu);
  T.error_count = g->m[0]->d_dirty_all + kOverflowWord;
  T.table = g->d_tile_lv;
  T.counters = g->d_tile_counters;
  T.K = K;
  T.M = (int)g->m.size();
}

// hsb_pack_dirty_device for K sessions (members == g->all: every member in order) into one buffer.
int group_pack_dirty(hsb_group* g, const char* fn, int K, const int* members, float* d_buf, size_t capacity_bytes,
                     int reset, cudaStream_t user) {
  hsb_handle* h0 = g->m[0];   // launches and errors are accounted on handles[0], whether or not it is listed
  const bool all = members == g->all.data();   // the full form: session k is member k, no list in the launch
  int s = check_members(g, fn, K, members);
  if (s != HSB_OK || K == 0) return s;
  if (all) members = nullptr;
  if (!d_buf) return fail(h0, HSB_ERR_INVALID_ARG, "%s: d_buf is NULL", fn);
  const size_t min_bytes = 4 * (size_t)(hsb_tile_group_header_words(K) + (unsigned long long)HSB_TILE_HEADER_WORDS * K);
  if (capacity_bytes < min_bytes)
    return fail(h0, HSB_ERR_INVALID_ARG, "%s: capacity_bytes is %zu, below the minimum of %zu bytes for K = %d", fn,
                capacity_bytes, min_bytes, K);
  if (members && K > kTileSubsetMax)
    return fail(h0, HSB_ERR_INVALID_ARG, "%s: K is %d, a subset pack lists at most %d sessions", fn, K, kTileSubsetMax);
  DeviceGuard guard(g->device);
  if ((s = tile_order_before(g, user, K, members, false, false)) != HSB_OK) return s;
  HsbTileParams T;
  fill_group_tile_params(g, T, d_buf, capacity_bytes, K);
  T.reset = reset;
  const int blocks = h0->sm_count * 4;
  const int* nl = g->d_member_levels;   // a ragged group's blocks each carry their member's level count
  if (!members) {
    if (nl) hsb::pack_dirty_group_ragged_kernel<<<blocks, 256, 0, user>>>(T, nl);
    else hsb::pack_dirty_group_kernel<<<blocks, 256, 0, user>>>(T);
  } else if (K <= kTileSubsetSmall) {
    hsb::TileMembers<kTileSubsetSmall> S;
    memcpy(S.idx, members, (size_t)K * sizeof(int));
    if (nl) hsb::pack_dirty_subset_ragged_kernel<kTileSubsetSmall><<<blocks, 256, 0, user>>>(T, S, nl);
    else hsb::pack_dirty_subset_kernel<kTileSubsetSmall><<<blocks, 256, 0, user>>>(T, S);
  } else {
    std::unique_ptr<hsb::TileMembers<kTileSubsetMax>> S(new hsb::TileMembers<kTileSubsetMax>());   // 16 KB: not on the stack
    memcpy(S->idx, members, (size_t)K * sizeof(int));
    if (nl) hsb::pack_dirty_subset_ragged_kernel<kTileSubsetMax><<<blocks, 256, 0, user>>>(T, *S, nl);
    else hsb::pack_dirty_subset_kernel<kTileSubsetMax><<<blocks, 256, 0, user>>>(T, *S);
  }
  if (reset) {
    const int threads = K * 4 * g->levels;
    if (nl) hsb::reset_dirty_ragged_kernel<<<(threads + 255) / 256, 256, 0, user>>>(T, nl);
    else hsb::reset_dirty_kernel<<<(threads + 255) / 256, 256, 0, user>>>(T);
  }
  h0->launches += reset ? 2 : 1;
  HSB_CUDA(h0, cudaGetLastError());
  return tile_order_after(g, user, K, members, false);
}

}  // namespace

extern "C" {

int hsb_group_pack_dirty_device(hsb_group* g, float* d_buf, size_t capacity_bytes, int reset, void* stream) {
  if (!g) return HSB_ERR_INVALID_ARG;
  return group_pack_dirty(g, "hsb_group_pack_dirty_device", (int)g->m.size(), g->all.data(), d_buf, capacity_bytes,
                          reset, (cudaStream_t)stream);
}

int hsb_group_pack_dirty_device_subset(hsb_group* g, int K, const int* members, float* d_buf, size_t capacity_bytes,
                                       int reset, void* stream) {
  if (!g) return HSB_ERR_INVALID_ARG;
  return group_pack_dirty(g, "hsb_group_pack_dirty_device_subset", K, members, d_buf, capacity_bytes, reset,
                          (cudaStream_t)stream);
}

int hsb_group_unpack_dirty_device(hsb_group* g, const float* d_buf, size_t capacity_bytes, void* stream) {
  if (!g) return HSB_ERR_INVALID_ARG;
  hsb_handle* h0 = g->m[0];
  const char* fn = "hsb_group_unpack_dirty_device";
  if (!d_buf) return fail(h0, HSB_ERR_INVALID_ARG, "%s: d_buf is NULL", fn);
  const size_t min_bytes = 4 * (size_t)(hsb_tile_group_header_words(1) + HSB_TILE_HEADER_WORDS);
  if (capacity_bytes < min_bytes)
    return fail(h0, HSB_ERR_INVALID_ARG, "%s: capacity_bytes is %zu, below the minimum of %zu bytes (one block)", fn,
                capacity_bytes, min_bytes);
  DeviceGuard guard(g->device);
  const int M = (int)g->m.size();
  cudaStream_t user = (cudaStream_t)stream;
  int s;
  if ((s = tile_order_before(g, user, M, nullptr, true, true)) != HSB_OK) return s;
  HsbTileParams T;
  fill_group_tile_params(g, T, const_cast<float*>(d_buf), capacity_bytes, 0);
  if (g->d_member_levels) hsb::unpack_dirty_ragged_kernel<<<h0->sm_count * 4, 256, 0, user>>>(T, g->d_member_levels);
  else hsb::unpack_dirty_kernel<<<h0->sm_count * 4, 256, 0, user>>>(T);
  h0->launches++;
  HSB_CUDA(h0, cudaGetLastError());
  return tile_order_after(g, user, M, nullptr, true);
}

}  // extern "C"

// ---- group map reset: hsb_reset for K members in one launch, replicated as a clear record ---------------------------
namespace {

// hsb_reset for the K members members[k] (members == g->all: every member, no list in the launch) with one launch on
// the group's stream and no synchronise; the replication rectangles are left clean with the cleared flags set.
int group_reset(hsb_group* g, const char* fn, int K, const int* members) {
  hsb_handle* h0 = g->m[0];   // launches and errors are accounted on handles[0], whether or not it is listed
  const bool all = members == g->all.data();
  int s = check_members(g, fn, K, members);
  if (s != HSB_OK || K == 0) return s;
  if (!all && K > kTileSubsetMax)
    return fail(h0, HSB_ERR_INVALID_ARG, "%s: K is %d, a subset reset lists at most %d sessions", fn, K, kTileSubsetMax);
  DeviceGuard guard(g->device);
  cudaStream_t st = g->stream;
  if ((s = order_members(g, K, members)) != HSB_OK) return s;
  HsbResetParams P;
  P.table = g->d_tile_lv;
  P.mem = g->d_reset;
  P.levels = g->levels;
  P.K = K;
  // blockIdx.y: session; blockIdx.x: about four waves of the device's CTAs over all sessions, no more than a level-0
  // plane has 256-cell stretches
  size_t max_cells = 0;
  for (int k = 0; k < K; ++k) {
    const Level& L0 = g->m[members[k]]->lv[0];
    max_cells = std::max(max_cells, (size_t)L0.sx * L0.sy);
  }
  const size_t want = ((size_t)h0->sm_count * 32 + K - 1) / K;
  const dim3 grid((unsigned)std::max<size_t>(1, std::min(want, (max_cells + 255) / 256)), (unsigned)std::min(K, 65535));
  const int* nl = g->d_member_levels;   // a ragged group: each member's own levels
  if (all) {
    if (nl) hsb::group_reset_ragged_kernel<<<grid, 256, 0, st>>>(P, nl);
    else hsb::group_reset_kernel<<<grid, 256, 0, st>>>(P);
  } else if (K <= kTileSubsetSmall) {
    hsb::TileMembers<kTileSubsetSmall> S;
    memcpy(S.idx, members, (size_t)K * sizeof(int));
    if (nl) hsb::group_reset_subset_ragged_kernel<kTileSubsetSmall><<<grid, 256, 0, st>>>(P, S, nl);
    else hsb::group_reset_subset_kernel<kTileSubsetSmall><<<grid, 256, 0, st>>>(P, S);
  } else {
    std::unique_ptr<hsb::TileMembers<kTileSubsetMax>> S(new hsb::TileMembers<kTileSubsetMax>());   // 16 KB: not on the stack
    memcpy(S->idx, members, (size_t)K * sizeof(int));
    if (nl) hsb::group_reset_subset_ragged_kernel<kTileSubsetMax><<<grid, 256, 0, st>>>(P, *S, nl);
    else hsb::group_reset_subset_kernel<kTileSubsetMax><<<grid, 256, 0, st>>>(P, *S);
  }
  h0->launches++;
  HSB_CUDA(h0, cudaGetLastError());
  HSB_CUDA(h0, cudaEventRecord(g->ev, st));
  // every later call on a reset member runs after the reset (HandleScope; a match on a copy stream through
  // map_write_pending), as after a nowait step; clear_level's host part
  for (int k = 0; k < K; ++k) {
    hsb_handle* h = g->m[members[k]];
    for (int l = 0; l < h->levels; ++l) h->lv[l].stamp_base = 0;
    h->group_ev = g->ev;
    h->map_write_pending = true;
  }
  return HSB_OK;
}

}  // namespace

extern "C" {

int hsb_group_reset(hsb_group* g) {
  if (!g) return HSB_ERR_INVALID_ARG;
  return group_reset(g, "hsb_group_reset", (int)g->m.size(), g->all.data());
}

int hsb_group_reset_subset(hsb_group* g, int K, const int* members) {
  if (!g) return HSB_ERR_INVALID_ARG;
  return group_reset(g, "hsb_group_reset_subset", K, members);
}

}  // extern "C"
