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

// What a scan arrives as: level-0 endpoints, or an input the match kernel's staging step converts to them —
// LaserScan ranges (rosLaserScanToDataContainer), a Point32 cloud in the laser frame (rosPointCloudToDataContainer) or
// LaserScan ranges projected by laser_geometry and then converted as a cloud.
enum HsbInputKind { HSB_IN_ENDPOINTS, HSB_IN_RANGES, HSB_IN_CLOUD, HSB_IN_PROJECTED };

// How a handle converts a scan (its hsb_set_scan_format / _cloud_format / _laser_projection at call time), and where
// the converted endpoints go.  Only the fields of the scan's kind are set.  (A scan of ranges has exactly the format's
// beam count, checked on the host: the kernels take it from the scan's length.)
struct HsbConvDev {
  // ranges: the (cos, sin) table of the accumulated beam angle, kept where range_min < r < range_max_c;
  // projected: kept where (double)r < range_cutoff && r >= range_min, projected with proj_unit (double (cos, sin))
  const float2* beam_cs;
  const double2* proj_unit;
  float range_min, range_max_c;
  double range_cutoff;
  // cloud and projected: the thresholds of the cloud rule
  float sqr_min_dist, sqr_max_dist, z_min, z_max;
  float scale_to_map;
  // the sink (SLAM steps and the stand-alone conversion; null for batch matches): the compacted endpoints go to
  // out_pts, their number to device memory (out_n, the map writer's n_dev) and, if set, to a second place (out_n_host:
  // a step's mapped host memory, written before the step's sequence number is published; a group match's result block)
  float2* out_pts;
  int* out_n;
  int* out_n_host;
};

// One scan of a stand-alone conversion (conv_to_points_kernel, one CTA per entry): n_in inputs of the launch's kind at
// `in` (ranges: one float per beam; cloud: Point32 triples), laser transform T (cloud and projected: 12 doubles, rows
// of [R | t]), converted by conv into conv's sink.
struct HsbConvScanDev {
  HsbConvDev conv;
  const float* in;
  const double* T;
  int n_in;
};

// One session of a group SLAM step (hsb_group_slam_update / _cloud / _ranges / _projected and their _subset forms): the
// member handle's state the match kernel touches.
struct HsbGroupSessionDev {
  float* gate_state;   // the member's lastMapUpdatePose[3] and write flag (hsb_handle::d_gate)
  float2* last_pts;    // the member's "containers of the last match": a matched scan's endpoints are copied here
  // converted input: the member's format; the sink is its last-match container when the session matches, its
  // update-scan buffer when not
  HsbConvDev conv;
  // the member's position in the group (its row of HsbMatchParams::group_lv).  Kept here rather than in HsbMatchParams
  // so that the parameter block, and with it every other instantiation of the match kernel, is unchanged.
  int member;
  // the member's level count: the step starts the session at its member's coarsest level; its rows of group_lv past
  // that are never read.  (Fills the descriptor's tail padding: its size is unchanged.)
  int levels;
  // the member's per-evaluation record of this step's match (HsbMatchParams::record's layout for the member's own levels:
  // group_lv's rec_off), in the member's mapped host buffer (hsb_set_step_record); null: the session records nothing
  float* record;
};

// One session of a pose-scoring call or of a group batch match: the scan its poses are scored against (its hints are
// matched with) and the member whose map they are scored (matched) on.
struct HsbScoreSessionDev {
  const float2* pts;   // the session's slice of the staged scans, or the member's last-match container
  int n;
  int member;
  float cell_length;   // of the member's level of a scoring call (covariance: the world matrix); unused by the match
  int levels;          // the member's level count: a group match starts the session's hints at its coarsest
};

struct HsbMatchParams {
  HsbLevelDev lv[HSB_MAX_LEVELS];
  int levels;
  int B;
  const float* hints;   // B x 3
  // Scan b's input is [offsets[b], offsets[b+1]) — endpoints, ranges or cloud points — or, without offsets, n_shared
  // inputs: the same endpoints for every scan (shared-scan mode), or scan b's own converted input at b * n_shared.
  HsbInputKind kind;
  const float2* pts;    // endpoints, interleaved xy
  const float* conv_in; // converted input: one float per range, or Point32 (x, y, z) triples
  const int* offsets;   // B + 1, or nullptr
  int n_shared;
  float* out_poses;     // B x 3
  float* out_cov;       // B x 9 or nullptr
  int pts_cap;          // points of smem staging per scan group (0 = read points from global)
  // how converted input becomes endpoints (N2: the node's conversions fused into the staging step), and where the
  // endpoints go (fused single SLAM step; with an inline scan, where its endpoints go)
  HsbConvDev conv;
  // cloud and projected: scan b's laser transform is cloud_tf + 12*b (rows of [R | t], double) or, if that is null,
  // cloud_tf0
  const double* cloud_tf;
  double cloud_tf0[12];
  float* out_origo;         // cloud and projected: B x 2 (may be null): dataContainer origo = laser position * scaleToMap
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
  int fixpoint;             // != 0: a level's Gauss-Newton loop ends at the first evaluation that leaves the pose
                            // bitwise unchanged (the later ones would repeat it exactly; see match_kernel)
  // diagnostics (hsb_set_tuning "trace"): per scan 8 x u64 =
  //   [0] start, [1 .. levels] after each level (coarsest first), [1 + levels] end,
  //   [5] evaluations the scan actually ran (written with <= 3 levels, where slot 5 is free), [6] %warpid, [7] %smid
  // The layout holds up to HSB_TRACE_MAX_LEVELS levels (the end time then sits in slot 5); with more the host leaves
  // the pointer null (hsb_api.cu launch_match), so no store of the kernel can land outside a scan's 8 slots.
  unsigned long long* trace;
  // per-evaluation record (hsb_match_data_record / hsb_match_batch_record_device), nullptr = none.  Scan b owns
  // record[b * record_floats ..], record_floats = R = sum over levels of (3 + 15 * evals).  Per level, coarsest first:
  //   [3]  the world pose the level starts from (ScanMatcher::matchData's beginEstimateWorld)
  //   then for every evaluation e = 0 .. evals-1, 15 floats:
  //   [9]  H row-major, [3] dTr, [3] the estimate after e's step in the level's map cells, angle not normalised
  //        (equal to the estimate before it when the H(0,0) != 0 && H(1,1) != 0 gate skipped the step)
  // An empty scan writes the level start poses (all the hint) and zeros in every evaluation slot.  A group SLAM step
  // leaves this null: each session records into its own HsbGroupSessionDev::record.
  float* record;
  int record_floats;
  // group SLAM step (match_kernel<..., GRP = GRP_STEP>): scan b is session b of the step, which steps member
  // group_sess[b].member of the group.  Its level descriptors are group_lv[member * levels ..] (built once per group;
  // `levels` is then the group's largest level count, and each scan runs its own member's)
  // instead of lv[], its gate thresholds and map_without_matching flag
  // gate_in[3b ..] (a set flag skips the match: the hint passes through the gate), its gate state and last-match
  // container group_sess[b]; out_poses and gate_out_host hold 4 floats per session (pose, write flag).  group_done
  // counts the sessions that have finished: the last one publishes seq_value to seq_host.  A converted session converts
  // with group_sess[b].conv (conv above is unused); a set map_without_matching flag still converts the scan for the map
  // writer: only the match is skipped.
  // group batch match (match_kernel<..., GRP = GRP_MATCH>, hsb_group_match_batch): scan b is hint b of session k, the
  // last one with match_offsets[k] <= b (match_offsets: match_K + 1 hint bounds).  The hint is matched with the
  // session's scan match_sess[k].pts / .n (endpoints; offsets, n_shared and pts above are unused) on member
  // match_sess[k].member's maps, group_lv[member * levels ..].  The epilogue is the plain batch one: pose and covariance
  // out, no gate, no sequence number, no container copy.  match_K fills the padding after record_floats and the two
  // arrays share storage with the step's, so the block keeps its size and layout: the inline-scan kernels' second
  // parameter stays where it was.
  int match_K;
  const HsbLevelDev* group_lv;
  union {
    const HsbGroupSessionDev* group_sess;
    const HsbScoreSessionDev* match_sess;
  };
  union {
    unsigned* group_done;
    const int* match_offsets;
  };
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

// A level's replication words in device memory (hsb_handle::d_dirty_all, one run of HSB_DIRTY_WORDS per level):
// [0..3] replication rectangle {xmin, ymin, xmax, ymax} (hsb_get_dirty_rect), [4..7] host-mirror rectangle
// (hsb_get_mirror_dirty_rect), [8] cleared flag: hsb_group_reset cleared the level since its last shipped pack, so a
// pack ships the clear record plus the replication rectangle (written since the clear) instead of the whole level.
#define HSB_DIRTY_WORDS 9
#define HSB_DIRTY_CLEARED 8

// One-shot, host-free tile transport (hsb_pack_dirty_device / hsb_unpack_dirty_device): buffer layout in 4-byte words —
// [0] magic, [1] levels, [2] overflow (1 = the dirty area did not fit, nothing packed), [3] total cells,
// [4 + 4 l ..] rectangle {x0, y0, x1, y1} of level l (x1 < x0: clean), [HSB_TILE_CLEARED_WORD] the clear record: bit l
// set = level l was cleared (hsb_group_reset) before the cells of its rectangle were written, so a replica clears the
// level outside the rectangle (0 when nothing was cleared; every pack writes it), [HSB_TILE_HEADER_WORDS ..] the
// log-odds rows of level 0's rectangle, then level 1's, ...
#define HSB_TILE_HEADER_WORDS 64
#define HSB_TILE_CLEARED_WORD (4 + 4 * HSB_MAX_LEVELS)
#define HSB_TILE_MAGIC 0x48534254
// A group's buffer (hsb_group_pack_dirty_device / hsb_group_unpack_dirty_device): a group header of G words —
// [0] HSB_TILE_GROUP_MAGIC, [1] K, [2] levels, [3] deferred blocks, [4] words used (G + 64 K + shipped cells),
// [5 + 2k], [6 + 2k] session k's {member index in the group, word offset of its block}, zeros up to G = 5 + 2K rounded
// up to a multiple of 4 — then K blocks in session order, each exactly the buffer hsb_pack_dirty_device writes for that
// member alone (HSB_TILE_HEADER_WORDS of header, then its rows).  A deferred block (overflow = 1) has no rows.  The
// blocks' rows are placed first-fit in session order: a block whose rows fit behind those already placed is shipped.
#define HSB_TILE_GROUP_MAGIC 0x48534247
#define HSB_TILE_GROUP_FIXED_WORDS 5
__host__ __device__ inline unsigned long long hsb_tile_group_header_words(int K) {
  return (HSB_TILE_GROUP_FIXED_WORDS + 2ull * (unsigned long long)K + 3ull) & ~3ull;
}
struct HsbTileLevelDev {
  float* logodds;
  float* prob;
  cudaSurfaceObject_t surf;
  int sx, sy;
  int* dirty;   // the level's HSB_DIRTY_WORDS: [0..3] replication rectangle, [4..7] host-mirror rectangle, [8] cleared flag
};
// What a group reset (hsb_group_reset) clears beyond a member's tile descriptors: its stamp planes and its gate state
// (hsb_handle::d_gate: lastMapUpdatePose[3], write flag).  One entry per member (hsb_group::d_reset).
struct HsbResetMemberDev {
  float* gate;
  uint32_t* stamp[HSB_MAX_LEVELS];
};
// A group reset: session k (blockIdx.y) clears every level of member S.member(k).
struct HsbResetParams {
  const HsbTileLevelDev* table;     // M x levels, member-major (hsb_group::d_tile_lv)
  const HsbResetMemberDev* mem;     // M (hsb_group::d_reset)
  int levels, K;
};
struct HsbTileParams {
  HsbTileLevelDev lv[HSB_MAX_LEVELS];   // a single handle's levels (table == nullptr)
  int levels;
  float* buf;
  unsigned long long capacity_words;    // whole buffer, headers included
  int reset;                 // pack: clear the replication rectangles afterwards (unless overflowed)
  int* error_count;          // unpack: incremented once when a buffer arrives that does not fit (a single handle's
                             // counter also takes its overflowed buffers)
  // group form: M x levels descriptors, member-major (hsb_group::d_tile_lv), each member's overflow counter (a deferred
  // block is counted there), the sessions of a pack (K) and the group's size; a single handle passes table = nullptr
  // and K = 1
  const HsbTileLevelDev* table;
  int* const* counters;
  int K, M;
};

struct HsbUpdateParams {
  HsbUpdateLevelDev lv[HSB_MAX_LEVELS];
  int levels;
  float pose_world[3];
  float log_odds_free, log_odds_occ;
  const float* pose_dev;     // if set, the pose is read from device memory (fused SLAM step) instead of pose_world
  const float* gate_flag;    // if set, *gate_flag == 0 turns the launch into a no-op (slam_gate_kernel in update_kernel.cuh)
};

// One non-empty rectangle of a group occupancy sync (hsb_group_sync_occupancy): the rows of all the call's rectangles are
// numbered consecutively in session order; this one owns rows [row0, row0 + its height) and the packed bytes from off on
// (w bytes per row).
struct HsbOccRowsDev {
  const float* logodds;   // the member's log-odds plane of the level
  int sx, x0, y0, w;
  int row0;
  size_t off;
};

// One member's level as a ray query sees it: the log-odds plane, its size, and getDist's transform — the map origin
// (hsb_get_map_origin), the cell length and 1 / cell length, all computed on the host as the single calls compute them.
struct HsbRayLevelDev {
  const float* plane;
  int sx, sy;
  float origo_x, origo_y, scale, inv_scale;
};

// A ray query (ray_kernel: hsb_raycast_batch, hsb_get_dist_batch and their group forms): Q rays of K sessions, session
// k's rays [offsets[k], offsets[k+1]) cast on member members[k]'s level `level`.  Arrays in device memory, in ray order.
struct HsbRayParams {
  const HsbRayLevelDev* lv;     // members x levels, member-major (hsb_group::d_ray_lv; one entry for a single handle)
  const int* members;           // K
  const int* offsets;           // K + 1
  const void* begin;            // Q: int2 cells (ray cast) or float2 world points (getDist)
  const void* end;
  float* out_dist;              // Q
  void* out_hit;                // Q int2 hit cells / float2 hit points, or null
  int* out_found;               // Q (getDist), or null
  int levels, level, K, Q;
};

// A pose-scoring call from host buffers (likelihood_group_kernel, best_group_finish_kernel, covariance_kernel:
// hsb_likelihood_batch, hsb_covariance_batch and the group calls): Q poses of K sessions, session k's poses
// [pose_offsets[k], pose_offsets[k+1]).  Arrays in device memory; outputs in pose order.
struct HsbScoreParams {
  const HsbLevelDev* lv;            // members x levels, member-major (hsb_group::d_lv; one entry for a single handle)
  const HsbScoreSessionDev* sess;   // K
  const int* pose_offsets;          // K + 1
  const float* poses;               // Q x 3, world
  float* out;                       // Q likelihoods, or null
  unsigned long long* best;         // K arg-max accumulators (best hypothesis), or null
  float* out_best4;                 // K x 4 (best hypothesis)
  int* out_best_index;              // K (best hypothesis)
  float* out_map;                   // Q x 9 (covariance), or null
  float* out_world;                 // Q x 9 (covariance), or null
  int levels, level, K, Q;
};

// Map write of a group SLAM step (update_mark_group_kernel / update_apply_group_kernel): blockIdx.z = session,
// blockIdx.y = level.  Everything per session lives in device memory, uploaded with the step's scans.
struct HsbGroupUpdateParams {
  const HsbUpdateLevelDev* lv;   // sessions x levels, session-major
  const float2* log_odds;        // per session: the member's (free, occupied) log-odds increments
  const float* res;              // per session 4 floats: the step's pose and write flag (the match kernel's gate)
  int levels;
};

#endif
