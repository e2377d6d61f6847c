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
/* the most levels a scan's 8-slot trace record can describe (tuning key "trace", hsb_read_trace) */
#define HSB_TRACE_MAX_LEVELS 4

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
  int   levels;           /* multi_res_size, 1..HSB_MAX_LEVELS: every depth 1..8 is tested   */
                          /* (4..8: tests/deep_cases.py); the coarsest level has >= 4 cells   */
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
/* Gauss-Newton evaluations of one level's match: maxIterations + 1 (the defaults 5 / 3 for a zero entry of
 * hsb_config::max_iterations).  Returns the count, or HSB_ERR_INVALID_ARG for a level the handle does not have. */
int hsb_get_level_evals(const hsb_handle* h, int level);

/* The record of the fused SLAM steps, for the node's pub_drawings / pub_debug_output hooks without leaving the fused
 * or group step.  on != 0: every matched fused SLAM step of this handle writes the per-evaluation record of its match
 * (the layout above, R = hsb_get_match_record_floats floats).  This covers hsb_slam_update* and the handle's session in
 * any hsb_group_slam_update*, full or subset, waiting or nowait.  Recording changes no result and adds no launch,
 * copy or synchronise: the match kernel stores the record into mapped pinned host memory owned by the handle before
 * the step's pose is published, so a nowait step's record is complete when the step returns.  The handle's next
 * fused step overwrites it.  Turning the switch on allocates that memory (once). */
int hsb_set_step_record(hsb_handle* h, int on);
/* the record of the handle's last fused step (R floats).  *matched = 0 when that step ran no match
 * (map_without_matching, or no step since the switch was turned on; record_out is then left untouched): the reference
 * calls no hook then.  Rejected with a message: a NULL record_out or matched, a handle that took no fused step. */
int hsb_get_step_record(hsb_handle* h, float* record_out, int* matched);
/* the level-0 container of the handle's last matched scan (endpoints in level-0 cells, and origo): what drawScan
 * draws, needed after a converted step (cloud, ranges, projected), whose endpoints exist only on the device.  *n_out
 * receives the count even when `capacity` is below it (then HSB_ERR_INVALID_ARG).  Rejected with a message: a NULL
 * n_out or origo_out, a NULL points_xy_out for a non-empty container, a handle that has matched no scan. */
int hsb_get_last_match_scan(hsb_handle* h, float* points_xy_out, int capacity, int* n_out, float origo_out[2]);

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

/* ---- the node's default path from the LaserScan itself ------------------------------------------*/
/* A default node (use_tf_scan_transformation = true, HectorMappingRos.cpp:258-297) projects every scan into a
 * sensor_msgs/PointCloud with laser_geometry, projector_.projectLaser(scan, cloud, 30.0) (:273), and converts that cloud
 * with rosPointCloudToDataContainer (:283).  These calls take the scan's ranges and run both on the device.  The
 * projection restates laser_geometry's LaserProjection::projectLaser_ / getUnitVectors_ (ROS1 Melodic / Noetic) for the
 * PointCloud output:
 *   unit vectors  c_i = cos((double)angle_min + (double)i * (double)angle_increment), s_i likewise with sin — libm's
 *                 double functions, evaluated on the host once per hsb_set_laser_projection;
 *   beam i kept   iff (double)range < cutoff && range >= range_min (float compare: NaN and +-inf are dropped);
 *   Point32       ((float)((double)range * c_i), (float)((double)range * s_i), 0.0f), beam order kept.
 * The cloud then takes the hsb_cloud_format rule of the handle as it is at the call (thresholds and, unless a call
 * passes its own, the laser transform).  The two filters compose into one over the beams in beam order. */
typedef struct hsb_laser_projection {
  int    n_beams;          /* ranges.size()                                                                   */
  float  angle_min;        /* scan.angle_min                                                                  */
  float  angle_increment;  /* scan.angle_increment                                                            */
  float  range_min;        /* scan.range_min   (kept: range >= range_min)                                     */
  float  range_max;        /* scan.range_max   (the cutoff when range_cutoff < 0)                             */
  double range_cutoff;     /* projectLaser's third argument (the node passes 30.0, :273); < 0 means range_max.
                            * Releases differ on whether range_max also caps it: pass the value the robot's
                            * release uses.                                                                   */
} hsb_laser_projection;
/* Builds the unit-vector table on the host and keeps it on the device (16 bytes per beam).  HSB_ERR_INVALID_ARG, and
 * the handle keeps its previous projection, for n_beams outside [1, 2^20], a non-finite angle_min, angle_increment or
 * range_min, a NaN cutoff, or a negative cutoff with a NaN range_max. */
int hsb_set_laser_projection(hsb_handle* h, const hsb_laser_projection* proj);
/* Projection + cloud conversion alone for one scan: ranges[n] (host, n = the projection's n_beams) -> kept endpoints
 * in level-0 cell units, beam order (capacity n x 2), *out_n = number kept, out_origo (may be NULL) = laser position *
 * scaleToMap.  transform: 12 doubles, rows of [R | t], NULL = the cloud format's.  Equal bit for bit to
 * hsb_cloud_to_points on the projected cloud.  Needs hsb_set_laser_projection and hsb_set_cloud_format
 * (HSB_ERR_INVALID_ARG, the message names what is missing); a scan longer than the fused SLAM step can stage fails with
 * HSB_ERR_UNSUPPORTED. */
int hsb_projected_scan_to_points(hsb_handle* h, const float* ranges, int n, const double* transform,
                                 float* out_points_xy, int* out_n, float out_origo[2]);
/* hsb_match_batch with both conversions fused into the match kernel's staging step, for replaying or relocalising a
 * default node's LaserScans: scan b is ranges[b*n_beams .. (b+1)*n_beams), n_beams = the laser projection's.
 * `transforms` (B x 12 doubles, rows of [R | t], may be NULL) and out_origo (B x 2, may be NULL: each container's
 * origo, laser position * scaleToMap) as in hsb_match_batch_cloud.  4 bytes per beam cross PCIe instead of 12 per
 * projected point.  An all-dropped scan returns its hint and an all-zero covariance; the "last match" containers are not
 * touched.  Each scan's pose, covariance and origo are bit-identical to hsb_match_batch_cloud on the cloud the
 * restatement above projects from that scan, with the same transforms, in the same launch shape, and to
 * hsb_match_batch on the endpoints hsb_projected_scan_to_points returns.  Rejected before anything is queued:
 * HSB_ERR_INVALID_ARG for NULL pointers, B < 0 or a handle without hsb_set_laser_projection or hsb_set_cloud_format
 * (the message names what is missing); HSB_ERR_UNSUPPORTED for a projection longer than the fused conversion can stage,
 * and for a tuning that selects a match shape without the projection — the projection is compiled into the shapes a
 * batch takes by default (1, 2, 4 or 8 warps per scan, one scan per CTA, 4 gathers in flight, unpacked).  B = 0 returns
 * HSB_OK.  Host buffers (submit / wait form below) / device buffers + stream. */
int hsb_match_batch_projected(hsb_handle* h, int B, const float* hints_world, const float* ranges,
                              const double* transforms, float* out_poses_world, float* out_cov, float* out_origo);
int hsb_match_batch_projected_device(hsb_handle* h, int B, const float* d_hints_world, const float* d_ranges,
                                     const double* d_transforms, float* d_out_poses_world, float* d_out_cov,
                                     float* d_out_origo, void* stream);

/* ---- streams of batches: submit / wait ---------------------------------------------------------*/
/* The four host-buffer batch calls above are `submit` followed by `wait`.  Used separately they let a caller keep
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
int hsb_match_batch_projected_submit(hsb_handle* h, int B, const float* hints_world, const float* ranges,
                                     const double* transforms, float* out_poses_world, float* out_cov,
                                     float* out_origo, int* ticket);
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
/* The branch WITHOUT the laser tf (use_tf_scan_transformation = false, HectorMappingRos.cpp:248-254) in one call:
 * rosLaserScanToDataContainer (:483-507, origo zero, :491) followed by HectorSlamProcessor::update with the last match
 * as the start estimate.  ranges = the LaserScan's n ranges; n must equal the n_beams of the handle's scan format
 * (hsb_set_scan_format, read at the call), otherwise HSB_ERR_INVALID_ARG.  The conversion runs in the match kernel's
 * staging step and its endpoints stay on the device for the map writer, as in hsb_slam_update_cloud: 4 bytes per beam
 * cross PCIe, no host round trip, three launches.  With map_without_matching the stand-alone conversion kernel
 * converts the scan for level 0 and the coarse levels keep the last match's containers.  nowait and *out_kept as in
 * hsb_slam_update_cloud.  A format longer than the fused conversion can stage fails with HSB_ERR_UNSUPPORTED.
 * Pose, covariance, gate decision, kept count, every plane and the handle's end state (gate pose, last match's
 * container, size and origo, stamps, both dirty rectangles, the pending write after nowait) are bit-identical to
 * hsb_scan_to_points followed by hsb_slam_update(h, hint, points, kept, origo = {0, 0}, ...). */
int hsb_slam_update_ranges(hsb_handle* h, const float pose_hint_world[3], const float* ranges, int n,
                           int map_without_matching, int nowait, float out_pose_world[3], float cov_inout[9],
                           int* map_updated, int* out_kept);
/* The DEFAULT branch of scanCallback from the LaserScan it receives (HectorMappingRos.cpp:258-297): laser_geometry's
 * projection (:273, see hsb_laser_projection), rosPointCloudToDataContainer (:283) and HectorSlamProcessor::update (:297)
 * in one call.  ranges = the scan's n ranges, n = the projection's n_beams (HSB_ERR_INVALID_ARG otherwise); transform
 * as in hsb_slam_update_cloud (NULL = the cloud format's).  Both conversions run in the match kernel's staging step:
 * 4 bytes per beam cross PCIe instead of 12 per projected point, one host-to-device copy and three launches.
 * map_without_matching, nowait and *out_kept as in hsb_slam_update_cloud.  Needs hsb_set_laser_projection and
 * hsb_set_cloud_format (HSB_ERR_INVALID_ARG, the message names what is missing); a scan longer than the fused
 * conversion can stage fails with HSB_ERR_UNSUPPORTED, and so does a handle whose tuning selects a match shape other
 * than the single step's default (8 warps, 4 gathers in flight, unpacked), the only one compiled with the projection.
 * Pose, covariance, gate decision, kept count, every plane and the handle's end state are bit-identical to
 * hsb_slam_update_cloud(h, hint, project(ranges), m, transform, ...), project being the restatement above and m the
 * number of projected points. */
int hsb_slam_update_projected(hsb_handle* h, const float pose_hint_world[3], const float* ranges, int n,
                              const double* transform, int map_without_matching, int nowait, float out_pose_world[3],
                              float cov_inout[9], int* map_updated, int* out_kept);
/* ---- many SLAM sessions in one device pass ------------------------------------------------------*/
/* N robots that each build their own map are N independent HectorSlamProcessors, i.e. N handles.  A group steps
 * them together: one host-to-device copy and three kernel launches per step whatever the number of members, instead
 * of N single steps in series.  (The batch matchers above serve many scans against ONE shared map.)
 * A group of existing handles stepped together.  The group does not own the handles.  Destroy the group before any of
 * its handles.  Members must have the same geometry: levels, map_size_x/y, map_resolution, start_x/y, the resolved
 * max_iterations of every level and the resolved gather mode, and sit on one device; update factors and the two gate
 * thresholds are per handle and may differ.  A group made by hsb_group_create_mixed may hold members that differ in
 * map_size_x/y, map_resolution and start_x/y; every group call then takes each member's own sizes: grids[k] of the
 * occupancy sync is member k's own size_y x size_x at `level`, session k's endpoints and scans are in member k's own
 * level-0 cell units, and a world ray, pose or hint is mapped into each member's own grid.  A handle may belong to
 * several groups.  Errors of hsb_group_create(_mixed): hsb_last_error(NULL) and hsb_last_error(handles[0]); of the other
 * group calls: hsb_last_error(handles[0]). */
typedef struct hsb_group hsb_group;
int hsb_group_create(hsb_handle* const* handles, int M, hsb_group** out);
/* hsb_group_create for members of different maps: robots at different sites, at different resolutions, started at
 * different map_start_x/y.  Members may differ in map_size_x, map_size_y, map_resolution, start_x and start_y; they must
 * still agree on the level count, the resolved max_iterations of every level and the resolved gather mode (an
 * HSB_GATHER_AUTO member larger than the texture limit resolves to LDG), and sit on one device — a mismatch is rejected
 * with HSB_ERR_INVALID_ARG, the message naming the member and the field.  Every other rejection and error rule of
 * hsb_group_create applies.  Every group call on such a group has exactly the contract documented for it: each
 * session's results and each stepped member's end state are bit-identical to the single-handle call on that member, and
 * a step is still one host-to-device copy and three launches counted on handles[0].  hsb_group_unpack_dirty_device
 * treats a shipped block whose rectangle on any level lies outside that level of the member it lands on as a buffer
 * that does not fit the group: counted once on handles[0], nothing of it applied. */
int hsb_group_create_mixed(hsb_handle* const* handles, int M, hsb_group** out);
/* hsb_group_create for members that differ in everything a robot's node sets per robot: members may differ in all that
 * hsb_group_create_mixed allows, and also in the level count (1 .. HSB_MAX_LEVELS), the resolved max_iterations of
 * every level and the resolved gather mode (TEX or LDG).  They must still sit on one device.  NULL, duplicate and
 * other-device handles are rejected as hsb_group_create_mixed rejects them.  Every group call keeps the contract
 * documented for it: each session's results and each member's end state are bit-identical to the single-handle call on
 * that member — its own levels, its own iteration counts, its own gather path — and a step is still one host-to-device
 * copy and three launches counted on handles[0].
 * Level rule: a call that takes a `level` (hsb_group_sync_occupancy, hsb_group_get_dist, hsb_group_raycast,
 * hsb_group_likelihood, hsb_group_covariance, hsb_group_best_hypothesis and their _subset forms) accepts any level below
 * the largest level count of the members, and rejects with HSB_ERR_INVALID_ARG, before anything is queued, cleared or
 * written, a listed member that does not have that level; the message names the session and the member's level count.
 * Members that are not listed are not checked.  hsb_group_match_batch runs each hint over its member's own levels with
 * its member's iteration counts (W chosen from handles[0] as for every group).  Tile replication: each block is exactly
 * the member's hsb_pack_dirty_device buffer, its own level count in block word 1; group-header word 2 is the largest
 * level count; on unpack a block whose level count differs from the member it lands on makes the buffer not fit the
 * group (counted once on handles[0], nothing of it applied).  hsb_group_reset clears each member's own levels. */
int hsb_group_create_heterogeneous(hsb_handle* const* handles, int M, hsb_group** out);
int hsb_group_destroy(hsb_group* g);
/* HectorSlamProcessor::update for every member at once. Session s is handles[s] with hint hints[3s..], the scan
 * points_xy[offsets[s] .. offsets[s+1]) (level-0 cells, DataContainer layout), origo[2s..] (NULL = 0,0) and
 * map_without_matching[s] (NULL = all 0). Host buffers. out_poses M x 3. cov_inout M x 9 (may be NULL; an entry is
 * left untouched where the single call leaves it untouched). map_updated M (may be NULL). nowait != 0: return once all
 * M poses have arrived, as hsb_slam_update_nowait does.
 * Every member is left in exactly the state hsb_slam_update with the same inputs would have left it in (gate pose,
 * last match's containers, stamps, both dirty rectangles, the pending map write after nowait), and each session's
 * results are bit-identical to that call's, so group steps, single steps and every other call may be mixed freely on a
 * member.  Ordering: a group step runs after everything already queued on its members' streams; every later call on a
 * member runs after the group step (hsb_on_map_updated(member) is the completion point after nowait), and "_device"
 * calls on caller streams are ordered as after hsb_slam_update_nowait.  The step runs on the group's own stream; its
 * kernel launches are counted on handles[0] (hsb_get_launch_count), three per step. */
int hsb_group_slam_update(hsb_group* g, const float* hints_world, const float* points_xy, const int* offsets,
                          const float* origo, const int* map_without_matching, int nowait,
                          float* out_poses_world, float* cov_inout, int* map_updated);
/* The same group step from the node's DEFAULT input: hsb_slam_update_cloud for every member at once.  Session s takes
 * the Point32 triples points_xyz[3*offsets[s] .. 3*offsets[s+1]) and the laser transform transforms[12s..] (12 doubles,
 * rows of [R | t]; transforms == NULL: every member's hsb_set_cloud_format transform).  Each session converts with its
 * own member's format thresholds (sqr_laser_min/max_dist, laser_z_min/max_value) as they are at the call, so robots
 * may differ in laser mount and filter settings.  out_kept (M ints, may be NULL) = the endpoints each conversion kept;
 * hints, map_without_matching, nowait, cov_inout and map_updated as in hsb_group_slam_update.  The conversion runs in
 * the group's match kernel (still one host-to-device copy and three launches per step; a map_without_matching session
 * is converted for the map writer and not matched, and its endpoints do not replace the last match's container).
 * Every session's pose, covariance, gate decision and kept count are bit-identical to hsb_slam_update_cloud on its
 * handle with the same inputs, and every member is left in the state that call leaves (gate pose, last match's
 * container and origo = laser position * scaleToMap, stamps, both dirty rectangles, the pending map write after
 * nowait); ordering as in hsb_group_slam_update.  Rejected before any member changes: a member without a cloud format
 * (HSB_ERR_INVALID_ARG, the message names the session), bad offsets (HSB_ERR_INVALID_ARG), a cloud longer than the
 * fused conversion can stage (HSB_ERR_UNSUPPORTED, the limit of hsb_slam_update_cloud). */
int hsb_group_slam_update_cloud(hsb_group* g, const float* hints_world, const float* points_xyz, const int* offsets,
                                const double* transforms, const int* map_without_matching, int nowait,
                                float* out_poses_world, float* cov_inout, int* map_updated, int* out_kept);
/* The same group step from raw LaserScan ranges: hsb_slam_update_ranges for every member at once.  Session s takes
 * ranges[offsets[s] .. offsets[s+1]), whose length must equal its member's n_beams.  Each session converts with its own
 * member's scan format as it is at the call (beam table, beam count, range window), so robots may differ in all of
 * these.  out_kept, hints, map_without_matching, nowait, cov_inout and map_updated as in hsb_group_slam_update_cloud;
 * one host-to-device copy and three launches per step.  Every session's pose, covariance, gate decision and kept count
 * are bit-identical to hsb_slam_update_ranges on its handle with the same inputs, and every member is left in the
 * state that call leaves.  Rejected before any member changes: a member without a scan format (HSB_ERR_INVALID_ARG,
 * the message names the session), offsets that disagree with the members' n_beams (HSB_ERR_INVALID_ARG), a scan
 * longer than the fused conversion can stage (HSB_ERR_UNSUPPORTED, the limit and message of hsb_slam_update_ranges). */
int hsb_group_slam_update_ranges(hsb_group* g, const float* hints_world, const float* ranges, const int* offsets,
                                 const int* map_without_matching, int nowait, float* out_poses_world, float* cov_inout,
                                 int* map_updated, int* out_kept);
/* The same group step from the LaserScans of default-configured nodes: hsb_slam_update_projected for every member at
 * once.  Session s takes ranges[offsets[s] .. offsets[s+1]), whose length must equal its member's projection n_beams,
 * and the laser transform transforms[12s..] (NULL: every member's cloud format transform).  Each session projects and
 * converts with its own member's projection and cloud format as they are at the call.  out_kept, hints,
 * map_without_matching, nowait, cov_inout and map_updated as in hsb_group_slam_update_cloud; one host-to-device copy
 * and three launches per step.  Every session's results and every member's end state are bit-identical to
 * hsb_slam_update_projected on its handle with the same inputs.  Rejected before any member changes: a member without
 * a projection or a cloud format (HSB_ERR_INVALID_ARG, the message names the session and what is missing), offsets that
 * disagree with the members' n_beams (HSB_ERR_INVALID_ARG), a scan longer than the fused conversion can stage
 * (HSB_ERR_UNSUPPORTED, the limit and message of hsb_slam_update_projected). */
int hsb_group_slam_update_projected(hsb_group* g, const float* hints_world, const float* ranges, const int* offsets,
                                    const double* transforms, const int* map_without_matching, int nowait,
                                    float* out_poses_world, float* cov_inout, int* map_updated, int* out_kept);
/* The four group steps above for K of the group's members, for robots whose scans do not arrive in step: session k
 * steps members[k], an index into the handles given to hsb_group_create, in any order.  Every per-session array
 * (hints_world, offsets (K + 1), origo, transforms, map_without_matching, out_poses_world, cov_inout, map_updated,
 * out_kept) has K entries in session order; otherwise each call takes the arguments of its full form.
 * Each session's pose, covariance, gate decision and kept count are bit-identical to the single-handle call on its
 * member (hsb_slam_update / _cloud / _ranges / _projected) with the same inputs, and each stepped member is left in the
 * state that call leaves.  A member not listed is neither read nor changed: its planes, texture twin, stamps, dirty
 * rectangles, gate pose and last match's container stay as they are, its formats are not checked (a member without a
 * cloud format may be left out of a cloud step), and work queued on its own stream does not delay the step.
 * Ordering: the step runs after everything queued on the listed members and after any pending group step that
 * involves them; every later call on a listed member runs after it.  Later calls on a member left out keep the
 * ordering they had (they may also be ordered behind this step), so a map write still pending from an earlier nowait
 * step of that member is still waited for.
 * Rejected with HSB_ERR_INVALID_ARG before any member changes: K < 0 or K > M; members == NULL with K > 0; an index
 * outside [0, M) or listed twice (the message names the session); and every rejection of the full form, applied to the
 * listed members.  K = 0 returns HSB_OK, reads no other argument and queues nothing.  A step of K >= 1 is one
 * host-to-device copy and three launches, counted on handles[0] whether or not it is listed. */
int hsb_group_slam_update_subset(hsb_group* g, int K, const int* members, const float* hints_world,
                                 const float* points_xy, const int* offsets, const float* origo,
                                 const int* map_without_matching, int nowait, float* out_poses_world, float* cov_inout,
                                 int* map_updated);
int hsb_group_slam_update_cloud_subset(hsb_group* g, int K, const int* members, const float* hints_world,
                                       const float* points_xyz, const int* offsets, const double* transforms,
                                       const int* map_without_matching, int nowait, float* out_poses_world,
                                       float* cov_inout, int* map_updated, int* out_kept);
int hsb_group_slam_update_ranges_subset(hsb_group* g, int K, const int* members, const float* hints_world,
                                        const float* ranges, const int* offsets, const int* map_without_matching,
                                        int nowait, float* out_poses_world, float* cov_inout, int* map_updated,
                                        int* out_kept);
int hsb_group_slam_update_projected_subset(hsb_group* g, int K, const int* members, const float* hints_world,
                                           const float* ranges, const int* offsets, const double* transforms,
                                           const int* map_without_matching, int nowait, float* out_poses_world,
                                           float* cov_inout, int* map_updated, int* out_kept);
/* HectorMappingRos::publishMap (hector_mapping/src/HectorMappingRos.cpp:435-481) for K of the group's members in one
 * pass.  Session k is member members[k] (the full form: every member, in order).  grids[k] is the caller's whole-level
 * grid of that member, size_y x size_x int8 row-major, kept between calls as the node keeps map_.map.data (:445-448).
 * Let r be member k's mirror rectangle of `level` (hsb_get_mirror_dirty_rect) after all work already queued for it:
 * out_rects[4k .. 4k+3] = r (out_rects may be NULL); x1 < x0 means the map did not change, so the caller skips
 * publishing that robot (:440).  Every cell of r gets publishMap's value in grids[k][y * size_x + x] (0 where the
 * log-odds l < 0, 100 where l > 0, -1 otherwise: +-0 and NaN), bit-identical to hsb_get_mirror_dirty_rect +
 * hsb_download_occupancy_rect + a row-by-row copy; no other byte of grids[k] is read or written.  reset != 0 clears the
 * mirror rectangle as hsb_get_mirror_dirty_rect(..., 1) does (the replication rectangle is untouched).  This call
 * consumes the same rectangle that hsb_get_mirror_dirty_rect and MapRepB200::getGridMap consume: one consumer per
 * handle.  A member not listed is neither read nor changed.
 * Ordering: the call runs on the group's stream after everything queued on the listed members (their own work and a
 * pending step of any group they belong to), and returns when every grid is written, so every later call on a member —
 * its next step included, whose map write grows the rectangle this call cleared — runs after it.
 * Cost: one launch gathers the K rectangles (one synchronise sizes the payload), then per chunk of at most 32 MiB of
 * packed rows (rectangles are split at row boundaries) one threshold launch, one device-to-host copy into the group's
 * pinned staging and one synchronise.  Launches are counted on handles[0]; hsb_get_d2h_bytes of each listed member
 * grows by the area of its rectangle.
 * Rejected with HSB_ERR_INVALID_ARG before anything is queued or cleared: K < 0 or K > M; members == NULL with K > 0;
 * an index outside [0, M) or listed twice; level outside [0, levels); grids == NULL or a NULL grids[k] (the message
 * names the session).  K = 0 returns HSB_OK, reads no other argument and queues nothing. */
/* Level rule (a group from hsb_group_create_heterogeneous): a listed member without `level` is rejected with
 * HSB_ERR_INVALID_ARG before anything is queued, cleared or written; the message names the session and the member's level count. */
int hsb_group_sync_occupancy(hsb_group* g, int level, int8_t* const* grids, int* out_rects, int reset);
int hsb_group_sync_occupancy_subset(hsb_group* g, int K, const int* members, int level, int8_t* const* grids,
                                    int* out_rects, int reset);
/* hector_map_server's get_distance_to_obstacle queries (hector_map_server.cpp:91-165, getDist at :123) for K of the
 * group's members in one pass: hsb_group_get_dist is hsb_get_dist_batch, hsb_group_raycast is hsb_raycast_batch.
 * Session k is member members[k] (the full form: every member, in order); its rays are [offsets[k], offsets[k+1]) of
 * begin_* / end_* (Q x 2 each, Q = offsets[K]; a session may hold none).  The outputs are in ray order: out_dist Q,
 * out_hit_world / out_hit Q x 2, out_found Q; the ones the single calls let be NULL may be NULL here.  Every ray's
 * distance, hit and found flag are bit-identical to the single call on its member with the same ray (misses, edges,
 * NaN and absurd world coordinates and the 5000-step cap included).  No member's state changes; a member not listed
 * is neither read nor waited for.
 * Ordering: the call runs on the group's stream after everything queued on the listed members (their own work and a
 * pending step of any group they belong to, so a query right after a nowait step sees that step's map write), and
 * returns when the results are in the caller's arrays.
 * Cost: one host-to-device copy of member list, offsets and rays from the group's pinned staging (grown geometrically),
 * one launch, one device-to-host copy of the results and one synchronise, whatever K is.  The launch is counted on
 * handles[0].
 * Rejected with HSB_ERR_INVALID_ARG before anything is queued: K < 0 or K > M; members == NULL with K > 0; an index
 * outside [0, M) or listed twice (the message names the session); level outside [0, levels); offsets == NULL,
 * offsets[0] != 0 or decreasing offsets (the message names the session); begin, end or out_dist NULL with Q > 0.
 * K = 0 returns HSB_OK and reads no other argument; Q = 0 returns HSB_OK and queues nothing. */
/* Level rule (a group from hsb_group_create_heterogeneous): a listed member without `level` is rejected with
 * HSB_ERR_INVALID_ARG before anything is queued; the message names the session and the member's level count. */
int hsb_group_get_dist(hsb_group* g, int level, const int* offsets, const float* begin_world, const float* end_world,
                       float* out_dist, float* out_hit_world, int* out_found);
int hsb_group_get_dist_subset(hsb_group* g, int K, const int* members, int level, const int* offsets,
                              const float* begin_world, const float* end_world, float* out_dist, float* out_hit_world,
                              int* out_found);
/* Level rule (a group from hsb_group_create_heterogeneous): a listed member without `level` is rejected with
 * HSB_ERR_INVALID_ARG before anything is queued; the message names the session and the member's level count. */
int hsb_group_raycast(hsb_group* g, int level, const int* offsets, const int* begin_cells, const int* end_cells,
                      float* out_dist, int* out_hit);
int hsb_group_raycast_subset(hsb_group* g, int K, const int* members, int level, const int* offsets,
                             const int* begin_cells, const int* end_cells, float* out_dist, int* out_hit);
/* Scoring poses for K of the group's members in one pass: hsb_group_likelihood is hsb_likelihood_batch
 * (getLikelihoodForState, OccGridMapUtil.h:189-221), hsb_group_covariance is hsb_covariance_batch (getCovarianceForPose,
 * :106-187) and hsb_group_best_hypothesis is hsb_best_hypothesis_device.  A server scores the poses a group step
 * returned (the step's own "covariance" is the raw Hessian; the likelihood of the returned pose is the reference's measure
 * of a match gone wrong) or picks the best of many hypotheses for each lost robot.
 * Session k is member members[k] (the full form: every member, in order).  Its poses are [pose_offsets[k],
 * pose_offsets[k+1]) of poses_world (Q x 3, Q = pose_offsets[K]; a session may hold none).  All of a session's poses are
 * scored against that session's ONE scan, on that member's map, at `level`.  The outputs are in pose order:
 * out_likelihood Q (may be NULL for the best hypothesis), out_cov_map / out_cov_world Q x 9 (either may be NULL, not
 * both), out_best4 K x 4 {likelihood, x, y, psi} and out_best_index K (may be NULL; the winner's index within its
 * session, -1 for an empty session).
 * The scan of session k:
 *  - points_xy and scan_offsets given: points_xy[scan_offsets[k] .. scan_offsets[k+1]), level-0 cell units, DataContainer
 *    layout, as hsb_likelihood_batch takes them;
 *  - points_xy == NULL and scan_offsets == NULL: the member's last-match container as it is on the device when the call
 *    runs on the group's stream, that is the endpoints of the member's last matched step of any input kind (single or
 *    group).  No scan crosses the bus.  A step with map_without_matching set does not replace the container: the scan of
 *    the last MATCHED step stays in force.  A member that has never matched has n = 0, which gives the reference's
 *    1 - 0/0 NaN as the single call does for an empty scan.
 * Bits: every likelihood equals hsb_likelihood_batch(member, level, ...) on the same pose and scan bit for bit, every
 * covariance equals hsb_covariance_batch bit for bit (NaN patterns included), and every session's out_best4 equals
 * hsb_best_hypothesis_device on that member with the session's poses: the highest score, the lowest index among equals;
 * a non-finite pose and a NaN likelihood score -1; an empty session gives {-1, 0, 0, 0}.  With the last-match container
 * the scan is the one hsb_cloud_to_points / hsb_scan_to_points / hsb_projected_scan_to_points returns for the stepped
 * input, or the endpoints given to an endpoint step.
 * No member's state changes; a member not listed is neither read nor waited for.
 * Ordering: the call runs on the group's stream after everything queued on the listed members (their own work and a
 * pending step of any group they belong to, so a call right after a nowait step sees that step's map write and its
 * last-match container), and returns when the results are in the caller's arrays.
 * Cost, whatever K is: one host-to-device copy from the group's pinned staging (grown geometrically) of the sessions'
 * descriptors (member, scan address and length), the pose offsets, the poses and, when given, the scans; one launch
 * (two for the best hypothesis); one device-to-host copy of one result block; one synchronise.  Launches are counted on
 * handles[0].
 * Rejected with HSB_ERR_INVALID_ARG before anything is queued: K < 0 or K > M; members == NULL with K > 0; an index
 * outside [0, M) or listed twice (the message names the session); level outside [0, levels); pose_offsets == NULL,
 * pose_offsets[0] != 0 or decreasing (the message names the session); exactly one of points_xy / scan_offsets NULL;
 * scan_offsets[0] != 0 or decreasing; poses_world, out_likelihood (likelihood), both covariance outputs or out_best4
 * NULL with Q > 0.  K = 0 returns HSB_OK and reads no other argument; Q = 0 returns HSB_OK and queues nothing (the best
 * hypothesis of every session is then the empty session's, written if out_best4 is given). */
/* Level rule (a group from hsb_group_create_heterogeneous): a listed member without `level` is rejected with
 * HSB_ERR_INVALID_ARG before anything is queued; the message names the session and the member's level count. */
int hsb_group_likelihood(hsb_group* g, int level, const int* pose_offsets, const float* poses_world,
                         const float* points_xy, const int* scan_offsets, float* out_likelihood);
int hsb_group_likelihood_subset(hsb_group* g, int K, const int* members, int level, const int* pose_offsets,
                                const float* poses_world, const float* points_xy, const int* scan_offsets,
                                float* out_likelihood);
/* Level rule (a group from hsb_group_create_heterogeneous): a listed member without `level` is rejected with
 * HSB_ERR_INVALID_ARG before anything is queued; the message names the session and the member's level count. */
int hsb_group_covariance(hsb_group* g, int level, const int* pose_offsets, const float* poses_world,
                         const float* points_xy, const int* scan_offsets, float* out_cov_map, float* out_cov_world);
int hsb_group_covariance_subset(hsb_group* g, int K, const int* members, int level, const int* pose_offsets,
                                const float* poses_world, const float* points_xy, const int* scan_offsets,
                                float* out_cov_map, float* out_cov_world);
/* Level rule (a group from hsb_group_create_heterogeneous): a listed member without `level` is rejected with
 * HSB_ERR_INVALID_ARG before anything is queued; the message names the session and the member's level count. */
int hsb_group_best_hypothesis(hsb_group* g, int level, const int* pose_offsets, const float* poses_world,
                              const float* points_xy, const int* scan_offsets, float* out_likelihood, float* out_best4,
                              int* out_best_index);
int hsb_group_best_hypothesis_subset(hsb_group* g, int K, const int* members, int level, const int* pose_offsets,
                                     const float* poses_world, const float* points_xy, const int* scan_offsets,
                                     float* out_likelihood, float* out_best4, int* out_best_index);
/* MapRepMultiMap::matchData (MapRepMultiMap.h:116-132) from many start poses for K of the group's members in one pass:
 * hsb_match_batch in shared-scan mode for each member.  A server re-matches a lost robot's last scan from a spread of
 * hints on that robot's own map, then picks the winner with hsb_group_best_hypothesis on the returned poses.
 * Session k is member members[k] (the full form: every member, in order).  Its hints are [hint_offsets[k],
 * hint_offsets[k+1]) of hints_world (Q x 3, Q = hint_offsets[K]; a session may hold none).  Each hint runs the full
 * coarse-to-fine matchData over all levels, on that member's current map, with the session's ONE scan.
 * The scan of session k:
 *  - points_xy and scan_offsets given: points_xy[scan_offsets[k] .. scan_offsets[k+1]), level-0 cell units, DataContainer
 *    layout, as hsb_match_batch takes them;
 *  - points_xy == NULL and scan_offsets == NULL: the member's last-match container as it is on the device when the call
 *    runs, by the rule hsb_group_likelihood documents (the endpoints of the last MATCHED step of any input kind; n = 0
 *    for a member that has never matched).  No scan crosses the bus.
 * The outputs are in hint order: out_poses_world Q x 3, out_cov Q x 9 (may be NULL), the Hessian of the last evaluation
 * (ScanMatcher.h:184).  An empty scan returns the hint and an all-zero covariance, as hsb_match_batch does.
 * Bits: every pose and covariance equals hsb_match_batch(member, B = the session's hint count, its hints, its scan,
 * offsets = NULL, n_shared = n) run with the same warps per scan W, bit for bit.  The reduction order follows W, and the
 * call takes W as hsb_match_batch would for ONE batch of Q hints (or handles[0]'s tuning warps_per_scan), so it may
 * differ from what each member's own call would take; hsb_get_last_launch_shape(handles[0]) reports it.
 * No member's state changes: no planes, stamps, dirty rectangles or gate pose, and the last-match container is not
 * replaced.  A member not listed is neither read nor waited for.
 * Ordering: the call runs on the group's stream after everything queued on the listed members (their own work and a
 * pending step of any group they belong to, so a call right after a nowait step sees that step's map write and its
 * last-match container), and returns when the results are in the caller's arrays.
 * Cost, whatever K is: one host-to-device copy from the group's pinned staging (grown geometrically) of the sessions'
 * descriptors (member, scan address and length), the hint offsets, the hints and, when given, the scans; one match
 * launch, counted on handles[0]; one device-to-host copy of the poses (and covariances, if asked for); one synchronise.
 * Rejected with HSB_ERR_INVALID_ARG before anything is queued, no output byte written: K < 0 or K > M; members == NULL
 * with K > 0; an index outside [0, M) or listed twice (the message names the session); hint_offsets == NULL,
 * hint_offsets[0] != 0 or decreasing (the message names the session); exactly one of points_xy / scan_offsets NULL;
 * scan_offsets[0] != 0 or decreasing; hints_world or out_poses_world NULL with Q > 0.  Rejected with
 * HSB_ERR_UNSUPPORTED: a handles[0] tuning whose launch shape has no group match kernel (the shapes are W in {1, 2, 4,
 * 8}, one scan per CTA, 4 gathers in flight, unpacked; the message names the tuning).  K = 0 returns HSB_OK and reads no
 * other argument; Q = 0 returns HSB_OK and queues nothing. */
int hsb_group_match_batch(hsb_group* g, const int* hint_offsets, const float* hints_world, const float* points_xy,
                          const int* scan_offsets, float* out_poses_world, float* out_cov);
int hsb_group_match_batch_subset(hsb_group* g, int K, const int* members, const int* hint_offsets,
                                 const float* hints_world, const float* points_xy, const int* scan_offsets,
                                 float* out_poses_world, float* out_cov);
/* hsb_group_match_batch from each session's new raw scan, with the pick: the relocalisation round of a lost robot from
 * what a node receives (LaserScan ranges, a Point32 cloud, or LaserScan ranges the default node projects), in one pass.
 * Sessions and hints are hsb_group_match_batch's.  Session k's ONE scan is [scan_offsets[k], scan_offsets[k+1]) of
 * `ranges` (one float per beam: _ranges, _projected) or of `points_xyz` (Point32 triples: _cloud); transforms holds 12
 * doubles per session, rows of [R | t] (NULL: each member's hsb_set_cloud_format transform, as in the group steps).
 * The scan is converted once with its member's scan format, cloud format or laser projection as they are at the call
 * (members may differ in all of these, and in map geometry and pyramid), then each hint runs the full coarse-to-fine
 * matchData with it on the member's own levels.
 * Outputs: out_poses_world Q x 3, out_cov Q x 9 (may be NULL) and out_likelihood Q, in hint order; out_kept K: the
 * endpoints each conversion kept (may be NULL).  Scoring runs only when asked for: out_likelihood scores every matched
 * pose at level 0 against the session's converted scan; out_best4 K x 4 {likelihood, x, y, psi} and out_best_index K
 * pick each session's winner by hsb_group_best_hypothesis's rule (any of the three may be NULL; all NULL: no scoring
 * launch).
 * Bits: out_kept[k] equals hsb_scan_to_points / hsb_cloud_to_points / hsb_projected_scan_to_points on member members[k]
 * with the same input and transform; every pose and Hessian equals hsb_group_match_batch(_subset) on the same hints with
 * points_xy set to those endpoints, in the same launch shape (W from Q and handles[0]'s tuning, reported by
 * hsb_get_last_launch_shape(handles[0])); every likelihood, best4 and index equals hsb_group_best_hypothesis(_subset) at
 * level 0 on the returned poses with those endpoints (NaN likelihoods and non-finite poses score -1; an empty session
 * gives {-1, 0, 0, 0} and index -1; an all-dropped scan returns its hints and all-zero Hessians).
 * No member's state changes: planes, texture twin, stamps, dirty rectangles and gate pose stay, and the new scan does
 * not replace the last-match container.  A member not listed is neither read nor waited for.  Ordering is
 * hsb_group_match_batch's.
 * Cost, whatever K is: one host-to-device copy from the group's pinned query staging of the sessions' descriptors,
 * offsets, hints, conversion table, transforms and raw scans (scans past the staging chunk: a second copy straight from
 * the caller's memory); one conversion launch (one CTA of 8 warps per session, into a group-owned device scratch of
 * one endpoint slot per input), one match launch, and one (likelihood) or two (best hypothesis) scoring launches on the
 * matched poses where they lie on the device, all counted on handles[0]; one device-to-host copy of one result block;
 * one synchronise.  No endpoint crosses the bus.
 * Rejected before anything is queued, no output byte written: every rejection of hsb_group_match_batch(_subset)
 * (HSB_ERR_UNSUPPORTED tuning rule included); scan_offsets NULL, not starting at 0 or decreasing; a NULL ranges /
 * points_xyz with scan_offsets[K] > 0; a listed member without the format its kind needs (the message names the
 * session); ranges / projected scan offsets that disagree with a member's n_beams.  K = 0 returns HSB_OK and reads no
 * other argument; Q = 0 returns HSB_OK and queues nothing (out_best4 / out_best_index get the empty session's values
 * if given, out_kept is not written).  No scan-length limit beyond the group match's. */
int hsb_group_match_batch_ranges(hsb_group* g, const int* hint_offsets, const float* hints_world, const float* ranges,
                                 const int* scan_offsets, float* out_poses_world, float* out_cov, float* out_likelihood,
                                 float* out_best4, int* out_best_index, int* out_kept);
int hsb_group_match_batch_cloud(hsb_group* g, const int* hint_offsets, const float* hints_world, const float* points_xyz,
                                const int* scan_offsets, const double* transforms, float* out_poses_world, float* out_cov,
                                float* out_likelihood, float* out_best4, int* out_best_index, int* out_kept);
int hsb_group_match_batch_projected(hsb_group* g, const int* hint_offsets, const float* hints_world, const float* ranges,
                                    const int* scan_offsets, const double* transforms, float* out_poses_world,
                                    float* out_cov, float* out_likelihood, float* out_best4, int* out_best_index,
                                    int* out_kept);
int hsb_group_match_batch_ranges_subset(hsb_group* g, int K, const int* members, const int* hint_offsets,
                                        const float* hints_world, const float* ranges, const int* scan_offsets,
                                        float* out_poses_world, float* out_cov, float* out_likelihood, float* out_best4,
                                        int* out_best_index, int* out_kept);
int hsb_group_match_batch_cloud_subset(hsb_group* g, int K, const int* members, const int* hint_offsets,
                                       const float* hints_world, const float* points_xyz, const int* scan_offsets,
                                       const double* transforms, float* out_poses_world, float* out_cov,
                                       float* out_likelihood, float* out_best4, int* out_best_index, int* out_kept);
int hsb_group_match_batch_projected_subset(hsb_group* g, int K, const int* members, const int* hint_offsets,
                                           const float* hints_world, const float* ranges, const int* scan_offsets,
                                           const double* transforms, float* out_poses_world, float* out_cov,
                                           float* out_likelihood, float* out_best4, int* out_best_index,
                                           int* out_kept);
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
 * recompute of the probability plane and texture twin after such an external write, on `stream`.
 * hsb_refresh_level also sets the level's mirror rectangle (hsb_get_mirror_dirty_rect) to the whole
 * level, in order on `stream`, so that a host mirror re-reads the plane; the replication rectangle
 * (hsb_get_dirty_rect) is left as it is, so a replica does not ship back a plane it only received.
 * Ordering as for hsb_unpack_rect_device: the refresh runs after everything the handle has queued (a pending map write
 * of a nowait step, single or group, and matches still reading the planes) and everything the handle queues afterwards
 * waits for it, on any stream.  The external write itself is the caller's: it must be ordered before the refresh on
 * `stream`, and after whatever the handle queued before it. */
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
 * them.  After hsb_reset / hsb_upload_level the dirty rectangle is the whole level; after hsb_group_reset it reads as the
 * whole level until a reset consumes it (the cleared flag, see hsb_group_reset). */
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

/* The same transport for a group: K sessions' dirty tiles in ONE buffer, one pack launch (plus one with `reset`) and one
 * unpack launch, counted on handles[0], whatever K is; nothing is synchronised or copied to the host.  Session k packs
 * member members[k] (hsb_group_pack_dirty_device: every member in order).
 * Buffer, in 4-byte words: a group header of G words — [0] group magic 0x48534247, [1] K, [2] levels, [3] deferred
 * blocks, [4] words used, then K pairs {member index in the group, word offset of its block}, zero-padded to
 * G = 5 + 2K rounded up to a multiple of 4 — then K blocks in session order.  Each block is exactly the buffer
 * hsb_pack_dirty_device writes for that member alone (256-byte header, then its rows), so one block can also be applied
 * with hsb_unpack_dirty_device.  Every block's header is written; the words left (capacity - G - 64 K) go to the
 * blocks' rows first-fit in session order: a block whose rows fit behind those already placed is shipped, one whose
 * rows do not is deferred (overflow = 1, no rows) and later blocks may still ship.  A deferred member keeps its
 * replication rectangles even with `reset` (the next pack ships the union); `reset` clears the shipped members' ones.
 * Mirror rectangles on the owner are not touched.  Only a member larger than the whole buffer needs the two-step
 * protocol.
 * hsb_group_unpack_dirty_device applies every shipped block on member `member index` of g (a replica group listing its
 * handles in the owner group's order) as hsb_unpack_dirty_device does (log-odds, probability, texture twin, mirror
 * rectangle; the replication rectangle stays clean) and counts a deferred block once on that member's
 * hsb_get_replication_overflows counter.  A buffer that does not fit g (wrong magic, another level count, a member index
 * >= M, a block offset or size past the capacity, a shipped rectangle outside its level of the member it lands on — in a
 * mixed group, an owner that lists its handles in another order) is counted once on handles[0]'s counter and nothing of
 * it is applied.  (The size check only guards bounds: it cannot tell apart two members whose rectangles both fit.)
 * Ordering, with `stream` in the role hsb_pack_dirty_device gives it: pack runs after everything queued on the listed
 * members (including a pending step of any group they belong to, so a pack right after a nowait step ships its map
 * write) and their next map write waits for it; a member not listed is neither read nor changed.  Unpack runs after
 * everything queued on every member of g (all their streams) and everything a member queues afterwards waits for it.
 * Rejected with HSB_ERR_INVALID_ARG before anything is queued: K < 0 or K > M; members == NULL with K > 0; an index
 * outside [0, M) or listed twice (the message names the session); a subset of more than 4096 sessions; d_buf == NULL; a
 * capacity below 4 (G + 64 K) bytes (unpack: below one block's, 4 (8 + 64)); the message names the minimum.  K = 0
 * returns HSB_OK and queues nothing. */
int hsb_group_pack_dirty_device(hsb_group* g, float* d_buf, size_t capacity_bytes, int reset, void* stream);
int hsb_group_pack_dirty_device_subset(hsb_group* g, int K, const int* members, float* d_buf, size_t capacity_bytes,
                                       int reset, void* stream);
int hsb_group_unpack_dirty_device(hsb_group* g, const float* d_buf, size_t capacity_bytes, void* stream);
/* MapRepresentationInterface::reset (MapRepMultiMap.h:83-90) for K of the group's members in one launch: the node's
 * reset_map service, a "reset" system message, and restart_mapping_with_new_pose (reset, then pass the new pose as the
 * member's next step hint) for many robots.  Session k resets member members[k] (hsb_group_reset: every member).
 * End state: each listed member is left in the state hsb_reset leaves — every level's log-odds 0 and probability 0.5,
 * texture twin 0.5, stamps 0, lastMapUpdatePose FLT_MAX^3 and write flag 0, mirror rectangle (hsb_get_mirror_dirty_rect)
 * the whole level; its last match's container, formats, update factors and gate thresholds stay as they are — with one
 * difference in the replication state: each level's replication rectangle is left clean and the level's cleared flag
 * is set; the map writer grows the rectangle from clean as usual.  The tile transport ships the clear record instead of
 * the whole level: every block hsb_pack_dirty_device / hsb_group_pack_dirty_device(_subset) writes carries in header
 * word 36 the mask of its member's levels cleared since their last shipped pack (0: none), its rows are only the cells
 * written since the reset (a reset with nothing written after it ships a 256-byte header), and first fit counts only
 * those cells; `reset` clears a shipped block's flags with its rectangles, a deferred block keeps both.  Unpack (single
 * or group) applies a shipped block with bit l set by resetting every cell of level l outside the shipped rectangle
 * (log-odds 0, probability 0.5, texture twin 0.5) and writing the shipped rows inside it, in its one launch; the
 * replica's mirror rectangle of level l becomes the whole level and its replication rectangle and flags stay clean.  A
 * block with a mask bit >= levels makes the buffer one that does not fit (counted once on handles[0], nothing applied).
 * hsb_get_dirty_rect and hsb_get_dirty_rects report the whole level while its flag is set, and their `reset` clears the
 * flag with the rectangle, so the two-step protocol ships what it ships after hsb_reset.  hsb_reset and
 * hsb_upload_level leave the flag clear (whole-level rectangles, as before).
 * A member not listed is neither read nor changed.
 * Ordering: the reset runs on the group's stream after everything queued on the listed members (their own work and a
 * pending step of any group they belong to) and returns once queued, without a synchronise; every later call on a
 * listed member runs after it.
 * Cost: one launch, counted on handles[0], whatever K is; the member list travels in the launch parameters (no
 * host-to-device copy), at most 4096 sessions in a subset.
 * Rejected with HSB_ERR_INVALID_ARG before anything is queued: K < 0 or K > M; members == NULL with K > 0; an index
 * outside [0, M) or listed twice (the message names the session); a subset of more than 4096 sessions.  K = 0 returns
 * HSB_OK and queues nothing. */
int hsb_group_reset(hsb_group* g);
int hsb_group_reset_subset(hsb_group* g, int K, const int* members);

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
 * non-finite pose and a NaN likelihood — an empty scan, 1 - 0/0 — score -1, so neither wins over a real score; an empty
 * batch gives likelihood -1).  d_out_likelihood may be NULL; it keeps the reference's NaN.  Two launches on
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
 * "host_out", "occupancy_chunk" (bytes of packed rows per chunk of a group occupancy sync whose handles[0] this handle
 * is, 0 = 32 MiB; at least one row).  Results never depend on them beyond summation order.
 * "trace" is refused with HSB_ERR_UNSUPPORTED on a handle of more than HSB_TRACE_MAX_LEVELS levels: the 8-slot
 * record has no room for their level times. */
int hsb_set_tuning(hsb_handle* h, const char* key, int value);
/* Shape of the last match-kernel launch of this handle: {warps per scan, scans per CTA, gather batch (unroll),
 * endpoints of each scan staged in shared memory (0 = read through L1), grid size, resident CTAs per SM}.
 * Lets tests assert WHICH instantiation they compared with the oracle. */
int hsb_get_last_launch_shape(const hsb_handle* h, int out[6]);
/* Device time of the last map write's two kernels (mark + apply, CUDA events on the handle's stream), available when
 * the tuning key "time_update" was set before the write — bench.py's K2 roofline. */
int hsb_get_last_update_device_ms(hsb_handle* h, float* ms);
/* Timeline of the last match launch when the tuning key "trace" is set: per scan 8 x uint64 =
 * {%globaltimer at start, after each level (coarsest first), at the end (slot 1 + levels), ..., %warpid (slot 6),
 * %smid (slot 7)}; with up to 3 levels slot 5 holds the evaluations the scan ran.  Handles of at most
 * HSB_TRACE_MAX_LEVELS levels only (with 4 the end time is slot 5); deeper ones cannot set the key and record nothing.
 * Synchronises the device; returns the number of scans copied (<= max_scans) or a negative status. */
int hsb_read_trace(hsb_handle* h, uint64_t* out, int max_scans);
/* library build identification, e.g. "hector_slam_b200 0.1 (sm_90a)" */
const char* hsb_version(void);

#ifdef __cplusplus
}
#endif
#endif /* HECTOR_SLAM_B200_H */
