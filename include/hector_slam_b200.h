/* hector_slam_b200.h — C-ABI of the H100-native (sm_90a) scan matcher / map writer.
 *
 * This is the drop-in boundary for hector_mapping's hot path.  The reference has no FFI of its
 * own: its seam is the pure-virtual C++ class hectorslam::MapRepresentationInterface
 * (hector_mapping/include/hector_slam_lib/slam_main/MapRepresentationInterface.h:38-62), whose
 * only implementation, MapRepMultiMap, is created at slam_main/HectorSlamProcessor.h:58.  Each
 * entry point below replaces one virtual of that interface (or one function the matcher is built
 * from) and says which.  The host-side adaptor that plugs these calls back into the reference
 * (class MapRepB200 : public hectorslam::MapRepresentationInterface) is
 * hector_slam_b200/host/MapRepB200.h; INTEGRATION.md shows the three-line change a maintainer
 * makes.
 *
 * Conventions
 *   - plain C: pointers and sizes only, no C++/torch types; every call returns an hsb_status
 *     (0 = ok, < 0 = error) and never throws; hsb_last_error() gives a message.
 *   - poses are (x [m], y [m], psi [rad]) in the world frame, float32            (Eigen::Vector3f)
 *   - scan endpoints are n x 2 float32, interleaved x,y, robot frame, in LEVEL-0 CELL units
 *     (metres * hsb_get_scale_to_map()) — exactly DataContainer's memory layout
 *     (scan/DataPointContainer.h:92-96; filled at src/HectorMappingRos.cpp:501-502,538)
 *   - 3x3 matrices are 9 float32; H is symmetric so row/column order is moot.
 *   - "host" entry points take host pointers and return when the result is in the output
 *     buffers; "_device" entry points take device pointers and a CUDA stream (cudaStream_t cast
 *     to void*) and are asynchronous on that stream.
 *   - a handle is single-writer, like the reference (one spinner thread calls update()): calls on
 *     one handle must not overlap, and work queued by a "_device" entry point on a caller stream
 *     must have completed (or be ordered by the caller) before a call that writes the map.
 *   - numerical edge cases keep the reference's silent semantics: empty scan -> pose = hint and
 *     the covariance buffer is left untouched (ScanMatcher.h:68,189); H(0,0)==0 or H(1,1)==0 ->
 *     the Gauss-Newton step is skipped (ScanMatcher.h:201); endpoints outside [0, S-2] add
 *     nothing (OccGridMapUtil.h:290-292); beams leaving the grid are dropped
 *     (OccGridMapBase.h:176,186).  One deliberate difference: a NON-FINITE map coordinate is
 *     treated as out of map instead of indexing memory with it (the reference crashes there,
 *     SURVEY.md Q4).
 */
#ifndef HECTOR_SLAM_B200_H
#define HECTOR_SLAM_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HSB_MAX_LEVELS 8

typedef struct hsb_handle hsb_handle;

typedef enum hsb_status {
  HSB_OK = 0,
  HSB_ERR_INVALID_ARG = -1,
  HSB_ERR_CUDA = -2,
  HSB_ERR_OUT_OF_MEMORY = -3,
  HSB_ERR_NO_DEVICE = -4,
  HSB_ERR_UNSUPPORTED = -5
} hsb_status;

/* How the four probability cells under an endpoint are fetched by the match kernel. */
typedef enum hsb_gather_mode {
  HSB_GATHER_AUTO = 0,   /* TEX, or LDG when the map exceeds the device's texture gather limit     */
  HSB_GATHER_LDG = 1,    /* four 32-bit loads from the linear probability plane              */
  HSB_GATHER_TEX = 2     /* one tex2Dgather on a block-linear CUDA array (point-sampled 2x2) */
} hsb_gather_mode;

/* Constructor arguments of HectorSlamProcessor / MapRepMultiMap
 * (slam_main/HectorSlamProcessor.h:54, slam_main/MapRepMultiMap.h:48). */
typedef struct hsb_config {
  float map_resolution;   /* level-0 cell length [m]                                        */
  int   map_size_x;       /* level-0 cells; level k has size >> k (MapRepMultiMap.h:67)     */
  int   map_size_y;
  float start_x;          /* startCoords: where world (0,0) sits in the map, as a fraction  */
  float start_y;
  int   levels;           /* multi_res_size, 1..HSB_MAX_LEVELS                              */
  int   device;           /* CUDA device ordinal                                            */
  /* maxIterations handed to ScanMatcher::matchData per level (the matcher then runs
   * maxIterations + 1 evaluations, ScanMatcher.h:74,94).  A zero entry selects the reference's
   * literal: 5 at level 0, 3 at coarser levels (MapRepMultiMap.h:125,128). Use -1 for "0". */
  int   max_iterations[HSB_MAX_LEVELS];
  float update_factor_free;      /* 0 -> 0.4 (GridMapLogOdds.h:117)                         */
  float update_factor_occupied;  /* 0 -> 0.6 (GridMapLogOdds.h:118); the ROS node sets 0.9  */
  int   gather_mode;             /* hsb_gather_mode                                         */
  int   reserved[7];
} hsb_config;

/* ---- lifetime -------------------------------------------------------------------------------*/
/* new MapRepMultiMap(...) — slam_main/MapRepMultiMap.h:48-72.  All level planes are allocated in
 * HBM and cleared (log-odds 0, probability 0.5). */
int hsb_create(const hsb_config* cfg, hsb_handle** out);
/* ~MapRepMultiMap — slam_main/MapRepMultiMap.h:74-81 */
int hsb_destroy(hsb_handle* h);
/* MapRepresentationInterface::reset — MapRepMultiMap.h:83-90 (every level cleared) */
int hsb_reset(hsb_handle* h);
/* setUpdateFactorFree / setUpdateFactorOccupied — MapRepMultiMap.h:149-167 */
int hsb_set_update_factor_free(hsb_handle* h, float factor);
int hsb_set_update_factor_occupied(hsb_handle* h, float factor);
/* the two log-odds increments currently in force: out[0] = free, out[1] = occupied */
int hsb_get_logodds_increments(hsb_handle* h, float out[2]);

/* ---- getters --------------------------------------------------------------------------------*/
/* getScaleToMap — MapRepMultiMap.h:92 ; getMapLevels — :94 */
float hsb_get_scale_to_map(const hsb_handle* h);
int   hsb_get_map_levels(const hsb_handle* h);
/* dimensions and cell length of one level (GridMapBase::getSizeX/getSizeY/getCellLength) */
int   hsb_get_level_info(const hsb_handle* h, int level, int* size_x, int* size_y, float* cell_length);
/* GridMapBase::getMapCoordsPose / getWorldCoordsPose — map/GridMapBase.h:226-239 (host arithmetic,
 * the same the kernels use) */
int   hsb_map_coords_pose(const hsb_handle* h, int level, const float world[3], float out[3]);
int   hsb_world_coords_pose(const hsb_handle* h, int level, const float map[3], float out[3]);

/* ---- the hot path: matching -----------------------------------------------------------------*/
/* MapRepresentationInterface::matchData — MapRepMultiMap.h:116-132: coarse-to-fine Gauss-Newton
 * over all levels, on the device without a host round trip.  `cov_inout` receives the Hessian of
 * the last evaluation (ScanMatcher.h:184) and is left untouched for n == 0.  The scan is also
 * remembered as "the containers of the last match", which hsb_update_by_scan uses for the
 * coarse levels exactly like MapRepMultiMap.h:143 does. `origo` may be NULL (= 0,0). */
int hsb_match_data(hsb_handle* h, const float begin_estimate_world[3], const float* points_xy, int n,
                   const float origo[2], float out_pose_world[3], float cov_inout[9]);

/* B independent matchData calls against the current (frozen) map: scan b is
 * points_xy[offsets[b] .. offsets[b+1]) with hint hints[3b..3b+2].  If `offsets` is NULL every
 * item uses the one scan points_xy[0 .. n_shared) (pose-hypothesis mode).  Outputs: out_poses
 * B x 3, out_cov B x 9 (may be NULL).  Host buffers (pinned memory lets the copies overlap the
 * kernel).  Does not touch the "last match" containers.  An empty scan returns its hint as the
 * pose and an all-zero out_cov entry (the batch buffer is write-only; the single-scan call above
 * keeps the reference's "untouched" behaviour). */
int hsb_match_batch(hsb_handle* h, int B, const float* hints_world, const float* points_xy, const int* offsets,
                    int n_shared, float* out_poses_world, float* out_cov);

/* Same with everything resident in device memory; asynchronous on `stream`.  `total_points` is
 * offsets[B] (ignored in shared-scan mode). */
int hsb_match_batch_device(hsb_handle* h, int B, const float* d_hints_world, const float* d_points_xy,
                           const int* d_offsets, int n_shared, int max_points_per_scan, float* d_out_poses_world,
                           float* d_out_cov, void* stream);

/* ---- the match, evaluation by evaluation ---------------------------------------------------------*/
/* What ScanMatcher::matchData (matcher/ScanMatcher.h:54-190) shows its DrawInterface and HectorDebugInfoInterface,
 * and a little more: every Gauss-Newton evaluation of every level, written by the match kernel from the values it
 * already holds (results are bit-identical with and without the record).  One scan's record is R floats,
 *   R = sum over levels l of (3 + 15 * (maxIterations_l + 1))          (hsb_get_match_record_floats)
 * and holds, per level, COARSEST FIRST:
 *   [3]   the world pose the level starts from (matchData's beginEstimateWorld);
 *   then for each evaluation e = 0 .. maxIterations_l, 15 floats:
 *   [9]   H, row-major (getCompleteHessianDerivs at the estimate before e's step),
 *   [3]   dTr,
 *   [3]   the estimate after e's step, in the level's map cells, angle not normalised (equal to the estimate before
 *         it when the H(0,0) != 0 && H(1,1) != 0 gate skipped the step).
 * Evaluation 0 is the one before the loop (ScanMatcher.h:74); the hooks report evaluations 1 .. maxIterations.
 * The last estimate of level 0, normalised and converted to world coordinates, is the returned pose, and its H is
 * the covariance.  An empty scan writes the level start poses (all equal to the hint) and zeros in every
 * evaluation slot. */
int hsb_get_match_record_floats(const hsb_handle* h);
/* hsb_match_data plus the record of that scan into `record_out` (host, R floats).  Same "last match" containers,
 * same latency paths (tuning keys host_out, inline_scan); the record costs one extra device-to-host copy. */
int hsb_match_data_record(hsb_handle* h, const float begin_estimate_world[3], const float* points_xy, int n,
                          const float origo[2], float out_pose_world[3], float cov_inout[9], float* record_out);
/* hsb_match_batch_device plus the records of all scans: d_record (device) receives B x R floats, scan b at b * R. */
int hsb_match_batch_record_device(hsb_handle* h, int B, const float* d_hints_world, const float* d_points_xy,
                                  const int* d_offsets, int n_shared, int max_points_per_scan, float* d_out_poses_world,
                                  float* d_out_cov, float* d_record, void* stream);

/* ---- raw laser ranges in (the step before the path: scan -> DataContainer) ---------------------*/
/* The sensor_msgs/LaserScan fields HectorMappingRos::rosLaserScanToDataContainer reads
 * (hector_mapping/src/HectorMappingRos.cpp:483-507).  Setting a format builds the per-beam
 * (cos, sin) table on the host exactly as the node does (fp32 `angle += angle_increment`, cos/sin of
 * the float angle) and keeps it on the device. */
typedef struct hsb_scan_format {
  int   n_beams;          /* ranges.size()                                   */
  float angle_min;        /* scan.angle_min                                  */
  float angle_increment;  /* scan.angle_increment                            */
  float range_min;        /* scan.range_min   (kept: range_min < r)          */
  float range_max;        /* scan.range_max   (kept: r < range_max - 0.1)    */
} hsb_scan_format;
int hsb_set_scan_format(hsb_handle* h, const hsb_scan_format* fmt);
/* rosLaserScanToDataContainer for one scan: ranges[n_beams] (host) -> compacted endpoints in
 * level-0 cell units, beam order (host, capacity n_beams x 2), *out_n = number kept. */
int hsb_scan_to_points(hsb_handle* h, const float* ranges, float* out_points_xy, int* out_n);
/* hsb_match_batch / hsb_match_batch_device with the conversion fused into the match kernel's
 * staging step: scan b is ranges[b*n_beams .. (b+1)*n_beams).  Halves the bytes per scan that have
 * to cross PCIe (4 B per beam instead of 8 B per endpoint). */
int hsb_match_batch_ranges(hsb_handle* h, int B, const float* hints_world, const float* ranges, float* out_poses_world,
                           float* out_cov);
int hsb_match_batch_ranges_device(hsb_handle* h, int B, const float* d_hints_world, const float* d_ranges,
                                  float* d_out_poses_world, float* d_out_cov, void* stream);

/* ---- point clouds in (the node's DEFAULT input path) ---------------------------------------------*/
/* HectorMappingRos::rosPointCloudToDataContainer (hector_mapping/src/HectorMappingRos.cpp:509-542), which a default
 * node (use_tf_scan_transformation = true, :82) runs on the cloud laser_geometry projected from the scan (:274-283).
 * The four parameters are the node's (:98-108: laser_min_dist^2, laser_max_dist^2 as floats, laser_z_min/max_value);
 * laser_transform is tf's base_frame <- laser frame as 12 doubles, rows of [R | t] (tfScalar is double). */
typedef struct hsb_cloud_format {
  double laser_transform[12];
  float  sqr_laser_min_dist;   /* keep sqr_min < x*x + y*y            (:526) */
  float  sqr_laser_max_dist;   /*      x*x + y*y < sqr_max                   */
  float  laser_z_min_value;    /* keep z_min < z(base) - z(laser) < z_max (:534-536) */
  float  laser_z_max_value;
} hsb_cloud_format;
int hsb_set_cloud_format(hsb_handle* h, const hsb_cloud_format* fmt);
/* The conversion alone for one cloud: points_xyz = n Point32 triples (x, y, z float32, laser frame, exactly
 * sensor_msgs/PointCloud::points' memory) -> kept endpoints in level-0 cell units, input order (capacity n x 2),
 * *out_n = number kept, out_origo (may be NULL) = the container's origo (:516-517).  Host buffers. */
int hsb_cloud_to_points(hsb_handle* h, const float* points_xyz, int n, float* out_points_xy, int* out_n, float out_origo[2]);
/* hsb_match_batch with that conversion fused into the match kernel's staging step: cloud b is the triples
 * points_xyz[3*offsets[b] .. 3*offsets[b+1]).  `transforms` (B x 12 doubles, may be NULL) gives every cloud its own
 * laser transform (a tf lookup per scan stamp, :262); NULL uses the format's.  out_origo (B x 2, may be NULL)
 * receives each container's origo, which hsb_update_by_scan needs.  Host buffers / device buffers + stream. */
int hsb_match_batch_cloud(hsb_handle* h, int B, const float* hints_world, const float* points_xyz, const int* offsets,
                          const double* transforms, float* out_poses_world, float* out_cov, float* out_origo);
int hsb_match_batch_cloud_device(hsb_handle* h, int B, const float* d_hints_world, const float* d_points_xyz,
                                 const int* d_offsets, int max_points_per_scan, const double* d_transforms,
                                 float* d_out_poses_world, float* d_out_cov, float* d_out_origo, void* stream);

/* ---- streams of batches: submit / wait ---------------------------------------------------------*/
/* The three host-buffer batch calls above are `submit` followed by `wait`.  Used separately they let a caller keep
 * the PCIe link busy across calls: the handle owns TWO sets of device staging buffers that alternate between calls,
 * so the copies of call k+1 travel while the last chunk of call k is still being matched.
 *   submit  queues the copies and kernels of one batch and returns a ticket (it blocks only while the staging set it
 *           is about to reuse — the one from two submits ago — has not delivered yet);
 *   wait    returns when that batch's results are in its output buffers.
 * Rules: at most two submits may be outstanding; input AND output buffers of a submit belong to the library until
 * its wait returns (pinned host memory, e.g. hsb_alloc_pinned, is what makes the copies asynchronous — with pageable
 * memory the calls still work but serialise); no map-writing call (hsb_update_by_scan, hsb_slam_update, hsb_reset,
 * uploads) between a submit and its wait.  Results are identical to the blocking calls. */
int hsb_match_batch_submit(hsb_handle* h, int B, const float* hints_world, const float* points_xy, const int* offsets,
                           int n_shared, float* out_poses_world, float* out_cov, int* ticket);
int hsb_match_batch_ranges_submit(hsb_handle* h, int B, const float* hints_world, const float* ranges,
                                  float* out_poses_world, float* out_cov, int* ticket);
int hsb_match_batch_cloud_submit(hsb_handle* h, int B, const float* hints_world, const float* points_xyz, const int* offsets,
                                 const double* transforms, float* out_poses_world, float* out_cov, float* out_origo,
                                 int* ticket);
int hsb_match_batch_wait(hsb_handle* h, int ticket);
/* Page-locked host memory for those buffers (cudaHostAlloc, allocated by the calling thread: bind the thread to the
 * GPU's NUMA node first if the host has several).  NULL on failure. */
void* hsb_alloc_pinned(size_t bytes);
/* diagnostic: host->device copy rate of `bytes` from `host` (reps back-to-back copies timed with CUDA events) —
 * bench.py reports it next to e2e so that a slow host path shows up as such */
int hsb_measure_h2d_gbs(hsb_handle* h, const void* host, size_t bytes, int reps, float* out_gbs);
int hsb_free_pinned(void* p);

/* OccGridMapUtil::getCompleteHessianDerivs — map/OccGridMapUtil.h:64-104, one evaluation on one
 * level: `pose_map` and `points_level_xy` are in that level's cell units.  This is the finest
 * seam (SURVEY.md §8b): the reference's own ScanMatcher can drive it one evaluation at a time. */
int hsb_hessian_derivs(hsb_handle* h, int level, const float pose_map[3], const float* points_level_xy, int n,
                       float H_out[9], float dTr_out[3]);

/* ---- the hot path: map writing --------------------------------------------------------------*/
/* MapRepresentationInterface::updateByScan — MapRepMultiMap.h:134-147 -> OccGridMapBase.h:121-168:
 * Bresenham free/occupied log-odds update of every level, once per cell per scan.  Level 0 uses
 * the scan given here; level k > 0 uses the scan of the last hsb_match_data scaled by 2^-k
 * (MapRepMultiMap.h:143).  The probability planes of the touched cells are refreshed in the same
 * pass. */
int hsb_update_by_scan(hsb_handle* h, const float* points_xy, int n, const float origo[2],
                       const float robot_pose_world[3]);
/* OccGridMapBase::updateByScan on ONE level with that level's own container (points/origo in the
 * level's cell units) — map/OccGridMapBase.h:121-168. */
int hsb_update_level_by_scan(hsb_handle* h, int level, const float* points_level_xy, int n,
                             const float origo_level[2], const float robot_pose_world[3]);
/* ---- the hot path, one SLAM step ------------------------------------------------------------*/
/* HectorSlamProcessor::update — slam_main/HectorSlamProcessor.h:71-113 — as ONE stream-ordered
 * sequence without a host round trip between its parts: matchData (:78; skipped and the hint taken
 * as the pose when map_without_matching != 0, :80), the poseDifferenceLargerThan gate against the
 * pose of the last map write (:89, util/UtilFunctions.h:73-92) evaluated on the device,
 * updateByScan at the new pose when the gate fires (:91) and onMapUpdated (:93).  The pose of the
 * last map write lives in the handle (FLT_MAX after hsb_create / hsb_reset, :117); the thresholds
 * are HectorSlamProcessor::setMapUpdateMinDistDiff / setMapUpdateMinAngleDiff (:141-142, defaults
 * 0.4 m / 0.13 rad as in :62-63).  Results equal hsb_match_data followed by a host-side gate and
 * hsb_update_by_scan + hsb_on_map_updated.  `cov_inout` as in hsb_match_data (untouched when
 * nothing was matched); `map_updated` (may be NULL) tells whether the map was written. */
int hsb_set_map_update_min_dist_diff(hsb_handle* h, float min_dist);
int hsb_set_map_update_min_angle_diff(hsb_handle* h, float min_angle);
int hsb_slam_update(hsb_handle* h, const float pose_hint_world[3], const float* points_xy, int n,
                    const float origo[2], int map_without_matching, float out_pose_world[3],
                    float cov_inout[9], int* map_updated);
/* The same step, returning as soon as the step's pose, covariance and gate decision have arrived in host memory (the
 * match kernel publishes them itself; the host polls a sequence number instead of synchronising the stream) — the map
 * write, if the gate fired, is still running on the handle's stream.  Every later call on the handle is ordered
 * behind it, so results are identical to hsb_slam_update; hsb_on_map_updated(h) is the explicit completion point
 * (what HectorSlamProcessor::update calls at :93).  This is the latency a robot sees for its pose estimate; the
 * sustained step rate is that of hsb_slam_update. */
int hsb_slam_update_nowait(hsb_handle* h, const float pose_hint_world[3], const float* points_xy, int n,
                           const float origo[2], int map_without_matching, float out_pose_world[3],
                           float cov_inout[9], int* map_updated);
/* The DEFAULT branch of HectorMappingRos::scanCallback in one call: rosPointCloudToDataContainer
 * (hector_mapping/src/HectorMappingRos.cpp:283, 509-542) followed by HectorSlamProcessor::update (:297).  points_xyz =
 * the n Point32 triples of the projected cloud, `transform` = the tf laser transform of this scan (12 doubles, rows of
 * [R | t]; NULL = the format's), thresholds from hsb_set_cloud_format.  The conversion runs in the match kernel's staging
 * step, the converted endpoints are handed to the map writer on the device and their number is counted there: no host
 * round trip between conversion, match, gate and map write.  nowait != 0: return when the pose has arrived (as
 * hsb_slam_update_nowait).  *out_kept (may be NULL) = number of endpoints the conversion kept.  Results equal
 * hsb_cloud_to_points followed by hsb_slam_update with the returned origo. */
int hsb_slam_update_cloud(hsb_handle* h, const float pose_hint_world[3], const float* points_xyz, int n,
                          const double* transform, int map_without_matching, int nowait, float out_pose_world[3],
                          float cov_inout[9], int* map_updated, int* out_kept);
/* lastMapUpdatePose of the fused step (HectorSlamProcessor.h:151) */
int hsb_get_last_map_update_pose(hsb_handle* h, float out[3]);
/* ... and its setter, for a host that wrote the map itself (hsb_update_by_scan) between fused steps: the gate of the
 * next hsb_slam_update then compares against this pose, as HectorSlamProcessor.h:94 would have left it. */
int hsb_set_last_map_update_pose(hsb_handle* h, const float pose[3]);

/* MapRepresentationInterface::onMapUpdated — MapRepMultiMap.h:107-114.  The reference bumps its
 * probability-cache epoch here; on the device the probability planes are already current, so this
 * only orders the stream (kept so the host façade reads like the reference). */
int hsb_on_map_updated(hsb_handle* h);

/* ---- map planes (checkpoint / parity / replication) -----------------------------------------*/
/* log-odds plane of one level, row-major [size_y][size_x] float32 (GridMapBase.h:141-149).
 * Upload refreshes that level's probability plane. */
int hsb_upload_level(hsb_handle* h, int level, const float* logodds_host);
int hsb_download_level(hsb_handle* h, int level, float* logodds_host_out);
/* probability plane P = e^l / (e^l + 1) (GridMapLogOdds.h:163-166) as the match kernel sees it */
int hsb_download_prob(hsb_handle* h, int level, float* prob_host_out);
/* device address of the level's log-odds plane (for NCCL broadcast of map replicas) and a full
 * recompute of the probability planes after such an external write */
void* hsb_level_logodds_device_ptr(hsb_handle* h, int level);
int hsb_refresh_level(hsb_handle* h, int level, void* stream);

/* Dirty-rectangle replication (multi-GPU: the owner of the map writes, replicas receive tiles).
 * hsb_get_dirty_rect: bounding box {x0, y0, x1, y1} (inclusive, level cells) of everything
 * hsb_update_by_scan wrote on `level` since the last reset (x1 < x0: nothing); `reset` != 0 clears
 * it.  hsb_pack_rect_device copies that rectangle of the log-odds plane row by row into a
 * contiguous device buffer ((x1-x0+1)*(y1-y0+1) floats) — the payload of an NCCL broadcast;
 * hsb_unpack_rect_device writes such a buffer into this handle's plane and refreshes the
 * probability plane (and texture twin) of the rectangle.  Asynchronous on `stream`. */
int hsb_get_dirty_rect(hsb_handle* h, int level, int rect[4], int reset);
/* the same for every level with one device-to-host copy: rects = levels x 4 ints */
int hsb_get_dirty_rects(hsb_handle* h, int* rects, int reset);
/* Ordering: `stream` may be any stream of the caller.  pack waits for the map writes the handle has queued and the
 * handle's next map write waits for pack; unpack waits for everything the handle has queued (matches still reading
 * the planes) and everything the handle queues afterwards waits for unpack — no synchronisation is needed around
 * them.  After hsb_reset / hsb_upload_level the dirty rectangle is the whole level. */
int hsb_pack_rect_device(hsb_handle* h, int level, const int rect[4], float* d_buf, void* stream);
int hsb_unpack_rect_device(hsb_handle* h, int level, const int rect[4], const float* d_buf, void* stream);

/* One-shot tile transport without the host in the loop.  hsb_pack_dirty_device reads the dirty rectangles of ALL levels
 * on the device and writes a self-describing buffer: a 256-byte header (magic, levels, overflow flag, cell count, the
 * rectangles) followed by the rectangles' log-odds rows; with `reset` the replication rectangles are cleared afterwards.
 * hsb_unpack_dirty_device applies such a buffer on a replica (rows, probabilities, texture twin, mirror rectangles),
 * reading everything it needs from the buffer itself.  Between them ONE collective of a fixed size (`capacity_bytes`,
 * e.g. 4 MB — a scan dirties 0.3-1 MB) moves the buffer: no size passes through a host, the whole replication step is
 * stream-ordered.  If the dirty area does not fit, pack sets the overflow flag, ships nothing and keeps the rectangles;
 * replicas count such buffers (hsb_get_replication_overflows; synchronises) and the caller falls back to the two-step
 * protocol above (hsb_get_dirty_rects + hsb_pack_rect_device) or a full plane broadcast.  Stream ordering as for
 * hsb_pack_rect_device / hsb_unpack_rect_device. */
int hsb_pack_dirty_device(hsb_handle* h, float* d_buf, size_t capacity_bytes, int reset, void* stream);
int hsb_unpack_dirty_device(hsb_handle* h, const float* d_buf, size_t capacity_bytes, void* stream);
int hsb_get_replication_overflows(hsb_handle* h, int* count, int reset);

/* ---- after the path: what the node does with the results -------------------------------------*/
/* nav_msgs/OccupancyGrid cell values of one level, as HectorMappingRos::publishMap derives them
 * (hector_mapping/src/HectorMappingRos.cpp:448-468): 0 where the cell is free (log-odds < 0,
 * GridMapLogOdds.h:81-84), 100 where occupied (> 0, :76-79), -1 otherwise.  Thresholded on the
 * device, so one byte per cell crosses PCIe instead of four.  out: [size_y][size_x] int8 (host). */
int hsb_download_occupancy(hsb_handle* h, int level, int8_t* occupancy_host_out);
/* Dirty-rectangle variants (the "dirty-rect download" of SURVEY.md N1): a second rectangle per level accumulates what
 * was written since the HOST last looked (independent of the replication rectangle above; whole level after a reset
 * or an upload).  hsb_download_level_rect / hsb_download_occupancy_rect copy only rect = {x0, y0, x1, y1} (inclusive),
 * packed row by row ((x1-x0+1) * (y1-y0+1) values) — bytes over PCIe proportional to the touched area, which is what
 * MapRepB200::getGridMap's mirror sync and a publishMap that keeps its data vector (HectorMappingRos.cpp:445) need.
 * hsb_get_d2h_bytes: bytes the download entry points have copied to the host so far (tests assert the proportionality). */
int hsb_get_mirror_dirty_rect(hsb_handle* h, int level, int rect[4], int reset);
int hsb_download_level_rect(hsb_handle* h, int level, const int rect[4], float* logodds_rows_out);
int hsb_download_occupancy_rect(hsb_handle* h, int level, const int rect[4], int8_t* occupancy_rows_out);
uint64_t hsb_get_d2h_bytes(const hsb_handle* h);
/* OccGridMapUtil::getLikelihoodForState — map/OccGridMapUtil.h:189-221: 1 - residual / n with
 * residual = sum_i (1 - interpMapValue(T(state) * p_i)) (an out-of-map endpoint counts 1), for B
 * poses (world frame; converted with getMapCoordsPose of `level`) against scan b of the batch
 * (same scan layout as hsb_match_batch: offsets == NULL -> one shared scan of n_shared points,
 * given in LEVEL-0 cell units and scaled by 2^-level like the matcher does).  Ranks relocalisation
 * hypotheses; the reference only uses it in its (dead) sigma-point covariance.  Host buffers. */
int hsb_likelihood_batch(hsb_handle* h, int level, int B, const float* poses_world, const float* points_xy,
                         const int* offsets, int n_shared, float* out_likelihood);
/* The same on DEVICE pointers, enqueued on `stream` (ordered behind a pending map write of the handle, nothing is
 * synchronised): scores the output of hsb_match_batch_device where it lies — a relocalisation step is match -> score ->
 * arg-max without a host round trip.  Same values as the host call. */
int hsb_likelihood_batch_device(hsb_handle* h, int level, int B, const float* d_poses_world, const float* d_points_xy,
                                const int* d_offsets, int n_shared, float* d_out_likelihood, void* stream);
/* Score AND pick (Monte-Carlo relocalisation, BASELINE config 4): the likelihood launch above with an arg-max folded
 * in — d_best4 receives {likelihood, x, y, psi} of the most likely pose of the batch (lowest index among equals; a
 * non-finite pose scores -1; an empty batch gives likelihood -1).  d_out_likelihood may be NULL.  Two launches on
 * `stream`, nothing is synchronised: a multi-GPU caller all-gathers the 16 bytes. */
int hsb_best_hypothesis_device(hsb_handle* h, int level, int B, const float* d_poses_world, const float* d_points_xy,
                               const int* d_offsets, int n_shared, float* d_out_likelihood, float* d_best4, void* stream);

/* OccGridMapUtil::getCovarianceForPose — map/OccGridMapUtil.h:106-160 — the sigma-point covariance of a pose: the
 * likelihoods (above) of the pose and of six neighbours (+-1.5 cells in x / y, +-0.05 rad) weight a mean and a 3x3
 * covariance in the level's MAP units; out_cov_world additionally applies getCovMatrixWorldCoords (:162-187: cell
 * length squared on the translation block, cell length on the mixed terms).  Poses are world poses (converted with
 * getMapCoordsPose of `level`); scans as in hsb_likelihood_batch.  Either output may be NULL.  Row-major 3x3 each.
 * (Dead code in the reference's own node, but part of the library interface; the reference prints the seven
 * likelihoods to stdout at :139 — not reproduced.)  Host buffers. */
int hsb_covariance_batch(hsb_handle* h, int level, int B, const float* poses_world, const float* points_xy,
                         const int* offsets, int n_shared, float* out_cov_map, float* out_cov_world);

/* hector_map_tools' DistanceMeasurementProvider::checkOccupancyBresenhami
 * (hector_map_tools/include/hector_map_tools/HectorMapTools.h:133-216, bresenham2D :200-216), B rays
 * at once on one level: walk the Bresenham line from begin cell to end cell (start included, end
 * excluded, at most 5000 steps) and stop at the first OCCUPIED cell (occupancy value 100, i.e.
 * log-odds > 0).  out_dist[b] = (int) Euclidean distance begin -> hit in cells, as a float, or -1
 * if nothing is hit or begin / end lies outside the level; out_hit (may be NULL) receives the hit
 * cell (x, y) or (-1, -1).  begin_cells / end_cells: B x 2 int32 (x, y).  Host buffers. */
int hsb_raycast_batch(hsb_handle* h, int level, int B, const int* begin_cells, const int* end_cells, float* out_dist,
                      int* out_hit);

/* The origin a nav_msgs/OccupancyGrid of `level` carries (HectorMappingRos::setServiceGetMapData,
 * hector_mapping/src/HectorMappingRos.cpp:546-550): world coordinates of cell (0,0) minus half a cell. */
int hsb_get_map_origin(const hsb_handle* h, int level, float out[2]);
/* DistanceMeasurementProvider::getDist (HectorMapTools.h:133-147), B world-frame rays at once: both end points go
 * through CoordinateTransformer<float>::getC2Coords ((w - origin) * (1.0f / resolution), truncated to int), the ray is
 * cast as in hsb_raycast_batch, out_dist[b] = resolution * cells (or resolution * -1 if nothing was hit, as the
 * reference returns), out_hit_world (B x 2, may be NULL) = origin + hit cell * resolution, out_found (may be NULL) =
 * 1 where something was hit (the reference leaves the hit undefined otherwise; (0, 0) here).  This is what
 * hector_map_server's get_distance_to_obstacle service calls (hector_map_server.cpp:123).  Host buffers. */
int hsb_get_dist_batch(hsb_handle* h, int level, int B, const float* begin_world, const float* end_world, float* out_dist,
                       float* out_hit_world, int* out_found);

/* ---- diagnostics ----------------------------------------------------------------------------*/
const char* hsb_last_error(const hsb_handle* h);
const char* hsb_status_string(int status);
/* number of CUDA kernels this handle has launched since creation (bench.py's gpu_launches) */
uint64_t hsb_get_launch_count(const hsb_handle* h);
/* the gather mode actually in use (after HSB_GATHER_AUTO resolution) */
int hsb_get_gather_mode(const hsb_handle* h);
/* launch-shape knobs for experiments: "warps_per_scan" (0 = auto), "scans_per_block" (0 = auto),
 * "stage_smem" (1 = stage scan endpoints in shared memory), "chunk" (scans per pipeline chunk of
 * hsb_match_batch, 0 = auto), "partial" (1 = stage a prefix of each scan when the whole scan would cost a wave),
 * "prefetch" (1 = L2 bulk prefetch of the unstaged part of a scan), "unroll", "trace" (see hsb_read_trace),
 * "inline_scan" (1: hsb_match_data / hsb_slam_update send scans of up to 1280 endpoints inside the kernel launch
 * instead of through a host-to-device copy — slower per step in measurement, higher back-to-back rate; default 0),
 * "host_out".  Results never depend on them beyond summation order. */
int hsb_set_tuning(hsb_handle* h, const char* key, int value);
/* Shape of the last match-kernel launch of this handle: {warps per scan, scans per CTA, gather batch (unroll),
 * endpoints of each scan staged in shared memory (0 = read through L1), grid size, resident CTAs per SM}.
 * Lets tests assert WHICH instantiation they compared with the oracle. */
int hsb_get_last_launch_shape(const hsb_handle* h, int out[6]);
/* Device time of the last map write's two kernels (mark + apply, CUDA events on the handle's stream), available when
 * the tuning key "time_update" was set before the write — bench.py's K2 roofline. */
int hsb_get_last_update_device_ms(hsb_handle* h, float* ms);
/* Timeline of the last match launch when the tuning key "trace" is set: per scan 8 x uint64 =
 * {%globaltimer at start, after each level (coarsest first), at the end (slot 1 + levels), ..., %smid (slot 7)}.
 * Synchronises the device; returns the number of scans copied (<= max_scans) or a negative status. */
int hsb_read_trace(hsb_handle* h, uint64_t* out, int max_scans);
/* library build identification, e.g. "hector_slam_b200 0.1 (sm_90a)" */
const char* hsb_version(void);

#ifdef __cplusplus
}
#endif
#endif /* HECTOR_SLAM_B200_H */
