// hsb_internal.h — shared host/device declarations of the H100 scan matcher (not installed).
#ifndef HSB_INTERNAL_H
#define HSB_INTERNAL_H

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/hector_slam_b200.h"

// Per-level constants the kernels need.  The two affine maps are kept as the full 2x3 matrices
// the reference builds (GridMapBase.h:265-280) so that device code can evaluate them term by
// term in the same order as the oracle (oracle/hs_oracle.c affine2_apply).
struct HsbLevelDev {
  const float* prob;         // probability plane, row-major [sy][sx]
  cudaTextureObject_t tex;   // same plane as a gather-capable 2-D texture (0 if unused)
  int sx, sy;
  float lim_x, lim_y;        // size - 2 (MapDimensionProperties.h:73)
  float mtw[6];              // map_T_world  m[2][3] row-major
  float wtm[6];              // world_T_map  m[2][3] row-major
  int evals;                 // maxIterations + 1 (ScanMatcher.h:74,94)
  float pt_scale;            // 2^-level (MapRepMultiMap.h:127)
  int rec_off;               // where this level's part of a scan's per-evaluation record starts (HsbMatchParams::record)
};

struct HsbMatchParams {
  HsbLevelDev lv[HSB_MAX_LEVELS];
  int levels;
  int B;
  const float* hints;   // B x 3
  const float2* pts;    // all scans, interleaved xy
  const int* offsets;   // B + 1, or nullptr in shared-scan mode
  int n_shared;
  float* out_poses;     // B x 3
  float* out_cov;       // B x 9 or nullptr
  int pts_cap;          // points of smem staging per scan group (0 = read points from global)
  // raw-range input (N2: rosLaserScanToDataContainer fused into the staging step); ranges == nullptr
  // selects the endpoint input above
  const float* ranges;      // B x n_beams
  const float2* beam_cs;    // n_beams x (cos, sin) of the accumulated beam angle
  int n_beams;
  float range_min, range_max_c;  // keep range_min < r < range_max - 0.1
  float scale_to_map;
  // point-cloud input (N2, the node's default path: rosPointCloudToDataContainer fused into the staging step);
  // cloud == nullptr selects one of the inputs above.  Scan b is the Point32 triples cloud[3*cloud_offsets[b] ..
  // 3*cloud_offsets[b+1]); its laser transform is cloud_tf + 12*b (rows of [R | t], double) or, if that is null, cloud_tf0.
  const float* cloud;
  const int* cloud_offsets;
  const double* cloud_tf;
  double cloud_tf0[12];
  float sqr_min_dist, sqr_max_dist, z_min, z_max;
  float* out_origo;         // B x 2 (may be null): dataContainer origo = laser position * scaleToMap
  // fused single-scan SLAM step from a point cloud (B == 1): the converted endpoints are also written out for the map
  // writer, their number goes to device memory (out_n) and to mapped host memory (out_n_host)
  float2* out_pts;
  int* out_n;
  int* out_n_host;
  // fused SLAM step (B == 1): the gate of HectorSlamProcessor::update evaluated in the kernel's epilogue
  float* gate_state;        // [0..2] lastMapUpdatePose, [3] flag out; nullptr = no gate
  const float* gate_in;     // minDist, minAngle, force
  float* gate_out_host;     // mapped host memory for pose + flag (may be nullptr)
  unsigned* seq_host;       // mapped host memory: seq_value is stored here (system-scope release) once pose, flag and
  unsigned seq_value;       // covariance of the step are visible to the host — the host may poll it instead of synchronising
  int stagger_ns;           // > 0: the warps sharing an SM start this many ns apart (see match_kernel: phase-locking)
  int sm_count;             // SMs of the device (the one-scan-per-CTA shapes derive a warp's rank on its SM from blockIdx)
  int pace_slack;           // > 0: groups of a CTA keep within this many evaluations of the slowest one (see match_kernel)
  int prefetch;             // != 0: L2 bulk prefetch of the part of a scan that is read from global memory
  // diagnostics (hsb_set_tuning "trace"): per scan 8 x u64 = {start, after coarsest level, ..., end (slot 1+levels), -, smid (slot 7)}
  unsigned long long* trace;
  // per-evaluation record (hsb_match_data_record / hsb_match_batch_record_device), nullptr = none.  Scan b owns
  // record[b * record_floats ..], record_floats = R = sum over levels of (3 + 15 * evals).  Per level, coarsest first:
  //   [3]  the world pose the level starts from (ScanMatcher::matchData's beginEstimateWorld)
  //   then for every evaluation e = 0 .. evals-1, 15 floats:
  //   [9]  H row-major, [3] dTr, [3] the estimate after e's step in the level's map cells, angle not normalised
  //        (equal to the estimate before it when the H(0,0) != 0 && H(1,1) != 0 gate skipped the step)
  // An empty scan writes the level start poses (all the hint) and zeros in every evaluation slot.
  float* record;
  int record_floats;
};

struct HsbUpdateLevelDev {
  float* logodds;
  float* prob;
  uint32_t* stamp;
  cudaSurfaceObject_t surf;  // 0 if the level has no CUDA-array twin
  int sx, sy;
  float mtw[6];
  float pt_scale;            // applied to points and origo (2^-level), 1 for per-level calls
  const float2* pts;         // scan used for this level
  int n;                     // number of endpoints — an upper bound when n_dev is set
  const int* n_dev;          // if set, the number of endpoints is read from device memory (fused point-cloud step)
  float origo_x, origo_y;    // already in the units of `pts` before pt_scale
  uint32_t stamp_base;       // this scan's stamps: base+1 free, base+2 occupied
  int active;
  int* dirty;                // two rectangles {xmin, ymin, xmax, ymax} of cells written since their last reset (device)
  // per-scan scratch of the two-phase writer (device): two slots of 8 ints, {-, x0, y0, x1, y1, -, -, -}; the mark
  // phase of a scan leaves the bounding box of its start and end cells in slot `slot`, the apply phase consumes it and
  // clears the OTHER slot for the next scan
  int* scratch;
  int slot;
};

// One-shot, host-free tile transport (hsb_pack_dirty_device / hsb_unpack_dirty_device): buffer layout in 4-byte words —
// [0] magic, [1] levels, [2] overflow (1 = the dirty area did not fit, nothing packed), [3] total cells,
// [4 + 4 l ..] rectangle {x0, y0, x1, y1} of level l (x1 < x0: clean), [HSB_TILE_HEADER_WORDS ..] the log-odds rows of
// level 0's rectangle, then level 1's, ...
#define HSB_TILE_HEADER_WORDS 64
#define HSB_TILE_MAGIC 0x48534254
struct HsbTileLevelDev {
  float* logodds;
  float* prob;
  cudaSurfaceObject_t surf;
  int sx, sy;
  int* dirty;   // [0..3] replication rectangle, [4..7] host-mirror rectangle
};
struct HsbTileParams {
  HsbTileLevelDev lv[HSB_MAX_LEVELS];
  int levels;
  float* buf;
  unsigned capacity_words;   // whole buffer, header included
  int reset;                 // pack: clear the replication rectangles afterwards (unless overflowed)
  int* error_count;          // unpack: incremented when an overflowed buffer arrives
};

struct HsbUpdateParams {
  HsbUpdateLevelDev lv[HSB_MAX_LEVELS];
  int levels;
  float pose_world[3];
  float log_odds_free, log_odds_occ;
  const float* pose_dev;     // if set, the pose is read from device memory (fused SLAM step) instead of pose_world
  const float* gate_flag;    // if set, *gate_flag == 0 turns the launch into a no-op (slam_gate_kernel in update_kernel.cuh)
};

#endif
