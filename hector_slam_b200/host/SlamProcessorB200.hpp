// SlamProcessorB200.hpp — standalone C++ host façade over the C-ABI (no Eigen, no ROS).
//
// Mirrors hectorslam::HectorSlamProcessor (hector_mapping/include/hector_slam_lib/slam_main/
// HectorSlamProcessor.h:50-154) method for method — update(), reset(), the getters and setters —
// for callers that do not have the reference's headers around.  update() is one C-ABI call
// (hsb_slam_update): match, gate on pose difference, map write and epoch bump run back to back on
// the GPU; updateUnfused() keeps the reference's host-side control flow over the two heavy calls.  Where the reference's own
// headers are available, use MapRepB200.h instead: it plugs into the unmodified reference façade.
#ifndef HECTOR_SLAM_B200_SLAMPROCESSOR_HPP
#define HECTOR_SLAM_B200_SLAMPROCESSOR_HPP

#include <cfloat>
#include <cmath>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "hector_slam_b200.h"

namespace hsb200 {

struct Pose {
  float x, y, psi;
};

class SlamProcessor {
 public:
  // HectorSlamProcessor.h:54
  SlamProcessor(float mapResolution, int mapSizeX, int mapSizeY, float startX, float startY, int multi_res_size,
                int device = 0)
      : h_(0), group_(0), groupOwner_(0), heterogeneous_(false) {
    hsb_config cfg = hsb_config();
    cfg.map_resolution = mapResolution;
    cfg.map_size_x = mapSizeX;
    cfg.map_size_y = mapSizeY;
    cfg.start_x = startX;
    cfg.start_y = startY;
    cfg.levels = multi_res_size;
    cfg.device = device;
    if (hsb_create(&cfg, &h_) != HSB_OK) throw std::runtime_error(std::string("hsb_create: ") + hsb_last_error(0));
    reset();
    setMapUpdateMinDistDiff(0.4f * 1.0f);    // :62
    setMapUpdateMinAngleDiff(0.13f * 1.0f);  // :63
    for (int i = 0; i < 9; ++i) lastScanMatchCov_[i] = 0.f;
  }
  ~SlamProcessor() {
    if (groupOwner_) groupOwner_->dropGroup();   // a group goes before its handles
    dropGroup();
    hsb_destroy(h_);
  }
  SlamProcessor(const SlamProcessor&) = delete;
  SlamProcessor& operator=(const SlamProcessor&) = delete;

  // HectorSlamProcessor.h:71-113.  points: n x 2 floats in level-0 cell units (DataContainer).
  void update(const float* points_xy, int n, const float origo[2], const Pose& poseHintWorld,
              bool map_without_matching = false) {
    // one fused call: match (:78), gate (:89), updateByScan (:91), onMapUpdated (:93) run back to back on the
    // device; the host only mirrors the two poses the getters expose
    const float hint[3] = {poseHintWorld.x, poseHintWorld.y, poseHintWorld.psi};
    float out[3];
    int updated = 0;
    check(hsb_slam_update(h_, hint, points_xy, n, origo, map_without_matching ? 1 : 0, out, lastScanMatchCov_, &updated));
    lastScanMatchPose_ = Pose{out[0], out[1], out[2]};  // :83
    if (updated) lastMapUpdatePose_ = lastScanMatchPose_;  // :94
  }

  // update() for M processors at once — M robots, each with its own map — in one device pass (hsb_group_slam_update):
  // processor s takes the scan points_xy[offsets[s] .. offsets[s+1]) with origo[2s..] (origo may be null), the hint
  // poseHintsWorld[s] and map_without_matching[s] (may be null).  Every processor ends exactly as its own update() would
  // have left it.  The group is kept by ps[0] for as long as the same processors are stepped together in the same order.
  static void updateMany(SlamProcessor* const* ps, int M, const float* points_xy, const int* offsets, const float* origo,
                         const Pose* poseHintsWorld, const int* map_without_matching = 0) {
    stepMany(ps, M, 0, M, poseHintsWorld, "updateMany",
             [&](hsb_group* g, const float* hints, float* poses, float* cov, int* updated) {
               return hsb_group_slam_update(g, hints, points_xy, offsets, origo, map_without_matching, 0, poses, cov,
                                            updated);
             });
  }

  // updateMany() for the K processors ps[members[0..K)] of ps[0..M) that have a new scan (hsb_group_slam_update_subset):
  // processor ps[members[k]] takes the scan points_xy[offsets[k] .. offsets[k+1]), origo[2k..], poseHintsWorld[k] and
  // map_without_matching[k].  The cached group stays the one of ps[0..M), so steps over changing subsets reuse it; the
  // processors not listed are left exactly as they are.
  static void updateMany(SlamProcessor* const* ps, int M, const int* members, int K, const float* points_xy,
                         const int* offsets, const float* origo, const Pose* poseHintsWorld,
                         const int* map_without_matching = 0) {
    stepMany(ps, M, members, K, poseHintsWorld, "updateMany",
             [&](hsb_group* g, const float* hints, float* poses, float* cov, int* updated) {
               return hsb_group_slam_update_subset(g, K, members, hints, points_xy, offsets, origo, map_without_matching,
                                                   0, poses, cov, updated);
             });
  }

  // The node's default input (use_tf_scan_transformation, HectorMappingRos.cpp:283, 509-542): update() from the projected
  // point cloud of a scan, converted on the device (hsb_slam_update_cloud).  points_xyz: n Point32 triples in the laser
  // frame; transform: the scan's tf laser transform (12 doubles, rows of [R | t]), null = the cloud format's.  Returns
  // the number of endpoints the conversion kept.
  int updateCloud(const float* points_xyz, int n, const double* transform, const Pose& poseHintWorld,
                  bool map_without_matching = false) {
    const float hint[3] = {poseHintWorld.x, poseHintWorld.y, poseHintWorld.psi};
    float out[3];
    int updated = 0, kept = 0;
    check(hsb_slam_update_cloud(h_, hint, points_xyz, n, transform, map_without_matching ? 1 : 0, 0, out, lastScanMatchCov_,
                                &updated, &kept));
    lastScanMatchPose_ = Pose{out[0], out[1], out[2]};  // :83
    if (updated) lastMapUpdatePose_ = lastScanMatchPose_;  // :94
    return kept;
  }

  // updateCloud() for M processors in one device pass (hsb_group_slam_update_cloud): processor s takes the cloud
  // points_xyz[3*offsets[s] .. 3*offsets[s+1]) with transforms[12s..] (transforms may be null: each processor's cloud
  // format), the hint poseHintsWorld[s] and map_without_matching[s] (may be null); kept (M ints, may be null) receives
  // each conversion's endpoint count.  Same group cache and end state as updateMany.
  static void updateManyCloud(SlamProcessor* const* ps, int M, const float* points_xyz, const int* offsets,
                              const double* transforms, const Pose* poseHintsWorld, const int* map_without_matching = 0,
                              int* kept = 0) {
    stepMany(ps, M, 0, M, poseHintsWorld, "updateManyCloud",
             [&](hsb_group* g, const float* hints, float* poses, float* cov, int* updated) {
               return hsb_group_slam_update_cloud(g, hints, points_xyz, offsets, transforms, map_without_matching, 0,
                                                  poses, cov, updated, kept);
             });
  }

  // updateManyCloud() for the processors ps[members[0..K)] (hsb_group_slam_update_cloud_subset); every per-session
  // array has K entries, as in the subset form of updateMany.
  static void updateManyCloud(SlamProcessor* const* ps, int M, const int* members, int K, const float* points_xyz,
                              const int* offsets, const double* transforms, const Pose* poseHintsWorld,
                              const int* map_without_matching = 0, int* kept = 0) {
    stepMany(ps, M, members, K, poseHintsWorld, "updateManyCloud",
             [&](hsb_group* g, const float* hints, float* poses, float* cov, int* updated) {
               return hsb_group_slam_update_cloud_subset(g, K, members, hints, points_xyz, offsets, transforms,
                                                         map_without_matching, 0, poses, cov, updated, kept);
             });
  }

  // the cloud format of updateCloud / updateManyCloud (the node's laser transform and filter parameters)
  void setCloudFormat(const hsb_cloud_format& fmt) { check(hsb_set_cloud_format(h_, &fmt)); }

  // The node's branch without the laser tf (use_tf_scan_transformation = false, HectorMappingRos.cpp:248-254): update()
  // from a LaserScan's raw ranges, converted on the device (hsb_slam_update_ranges).  n must equal the scan format's
  // n_beams; poseHintWorld is the node's getLastScanMatchPose().  Returns the number of endpoints the conversion kept.
  int updateRanges(const float* ranges, int n, const Pose& poseHintWorld, bool map_without_matching = false) {
    const float hint[3] = {poseHintWorld.x, poseHintWorld.y, poseHintWorld.psi};
    float out[3];
    int updated = 0, kept = 0;
    check(hsb_slam_update_ranges(h_, hint, ranges, n, map_without_matching ? 1 : 0, 0, out, lastScanMatchCov_, &updated,
                                 &kept));
    lastScanMatchPose_ = Pose{out[0], out[1], out[2]};  // :83
    if (updated) lastMapUpdatePose_ = lastScanMatchPose_;  // :94
    return kept;
  }

  // updateRanges() for M processors in one device pass (hsb_group_slam_update_ranges): processor s takes the ranges
  // ranges[offsets[s] .. offsets[s+1]) (as many as its scan format's n_beams), the hint poseHintsWorld[s] and
  // map_without_matching[s] (may be null); kept (M ints, may be null) receives each conversion's endpoint count.  Same
  // group cache and end state as updateMany.
  static void updateManyRanges(SlamProcessor* const* ps, int M, const float* ranges, const int* offsets,
                               const Pose* poseHintsWorld, const int* map_without_matching = 0, int* kept = 0) {
    stepMany(ps, M, 0, M, poseHintsWorld, "updateManyRanges",
             [&](hsb_group* g, const float* hints, float* poses, float* cov, int* updated) {
               return hsb_group_slam_update_ranges(g, hints, ranges, offsets, map_without_matching, 0, poses, cov,
                                                   updated, kept);
             });
  }

  // updateManyRanges() for the processors ps[members[0..K)] (hsb_group_slam_update_ranges_subset); every per-session
  // array has K entries, as in the subset form of updateMany.
  static void updateManyRanges(SlamProcessor* const* ps, int M, const int* members, int K, const float* ranges,
                               const int* offsets, const Pose* poseHintsWorld, const int* map_without_matching = 0,
                               int* kept = 0) {
    stepMany(ps, M, members, K, poseHintsWorld, "updateManyRanges",
             [&](hsb_group* g, const float* hints, float* poses, float* cov, int* updated) {
               return hsb_group_slam_update_ranges_subset(g, K, members, hints, ranges, offsets, map_without_matching, 0,
                                                          poses, cov, updated, kept);
             });
  }

  // the scan format of updateRanges / updateManyRanges (the LaserScan's beam geometry and range window)
  void setScanFormat(const hsb_scan_format& fmt) { check(hsb_set_scan_format(h_, &fmt)); }

  // The node's default branch from the LaserScan it receives (HectorMappingRos.cpp:258-297): laser_geometry's
  // projection (:273), the cloud conversion (:283) and update() (:297) on the device (hsb_slam_update_projected).  n
  // must equal the laser projection's n_beams; transform: the scan's tf laser transform, null = the cloud format's.
  // Returns the number of endpoints the conversion kept.
  int updateProjected(const float* ranges, int n, const double* transform, const Pose& poseHintWorld,
                      bool map_without_matching = false) {
    const float hint[3] = {poseHintWorld.x, poseHintWorld.y, poseHintWorld.psi};
    float out[3];
    int updated = 0, kept = 0;
    check(hsb_slam_update_projected(h_, hint, ranges, n, transform, map_without_matching ? 1 : 0, 0, out,
                                    lastScanMatchCov_, &updated, &kept));
    lastScanMatchPose_ = Pose{out[0], out[1], out[2]};  // :83
    if (updated) lastMapUpdatePose_ = lastScanMatchPose_;  // :94
    return kept;
  }

  // updateProjected() for M processors in one device pass (hsb_group_slam_update_projected): processor s takes the
  // ranges ranges[offsets[s] .. offsets[s+1]) (as many as its projection's n_beams) with transforms[12s..] (may be null:
  // each processor's cloud format), the hint poseHintsWorld[s] and map_without_matching[s] (may be null); kept (M ints,
  // may be null) receives each conversion's endpoint count.  Same group cache and end state as updateMany.
  static void updateManyProjected(SlamProcessor* const* ps, int M, const float* ranges, const int* offsets,
                                  const double* transforms, const Pose* poseHintsWorld, const int* map_without_matching = 0,
                                  int* kept = 0) {
    stepMany(ps, M, 0, M, poseHintsWorld, "updateManyProjected",
             [&](hsb_group* g, const float* hints, float* poses, float* cov, int* updated) {
               return hsb_group_slam_update_projected(g, hints, ranges, offsets, transforms, map_without_matching, 0,
                                                      poses, cov, updated, kept);
             });
  }

  // updateManyProjected() for the processors ps[members[0..K)] (hsb_group_slam_update_projected_subset); every
  // per-session array has K entries, as in the subset form of updateMany.
  static void updateManyProjected(SlamProcessor* const* ps, int M, const int* members, int K, const float* ranges,
                                  const int* offsets, const double* transforms, const Pose* poseHintsWorld,
                                  const int* map_without_matching = 0, int* kept = 0) {
    stepMany(ps, M, members, K, poseHintsWorld, "updateManyProjected",
             [&](hsb_group* g, const float* hints, float* poses, float* cov, int* updated) {
               return hsb_group_slam_update_projected_subset(g, K, members, hints, ranges, offsets, transforms,
                                                             map_without_matching, 0, poses, cov, updated, kept);
             });
  }

  // the laser projection of updateProjected / updateManyProjected (the LaserScan's beam geometry and projectLaser's
  // cutoff); the cloud format (setCloudFormat) supplies the rest
  void setLaserProjection(const hsb_laser_projection& proj) { check(hsb_set_laser_projection(h_, &proj)); }

  // The same step with the control flow on the host (two C-ABI calls and a round trip in between), as the
  // reference's own HectorSlamProcessor drives MapRepB200; kept for comparison and tests.
  void updateUnfused(const float* points_xy, int n, const float origo[2], const Pose& poseHintWorld,
                     bool map_without_matching = false) {
    Pose newPose;
    if (!map_without_matching) {
      const float hint[3] = {poseHintWorld.x, poseHintWorld.y, poseHintWorld.psi};
      float out[3];
      check(hsb_match_data(h_, hint, points_xy, n, origo, out, lastScanMatchCov_));  // :78
      newPose = Pose{out[0], out[1], out[2]};
    } else {
      newPose = poseHintWorld;  // :80
    }
    lastScanMatchPose_ = newPose;  // :83
    if (poseDifferenceLargerThan(newPose, lastMapUpdatePose_, minDist_, minAngle_) || map_without_matching) {  // :89
      const float p[3] = {newPose.x, newPose.y, newPose.psi};
      check(hsb_update_by_scan(h_, points_xy, n, origo, p));  // :91
      check(hsb_on_map_updated(h_));                          // :93
      lastMapUpdatePose_ = newPose;                           // :94
      check(hsb_set_last_map_update_pose(h_, p));             // keep the fused path's gate state in step (mixing allowed)
    }
  }

  // HectorSlamProcessor.h:115-124
  void reset() {
    lastMapUpdatePose_ = Pose{FLT_MAX, FLT_MAX, FLT_MAX};
    lastScanMatchPose_ = Pose{0.f, 0.f, 0.f};
    check(hsb_reset(h_));
  }

  // Opt-in, on the processor that is ps[0] of the …Many calls: its cached group of ps[0..M) is made with
  // hsb_group_create_heterogeneous, so the processors may differ in map size, resolution, start, level count
  // (map_multi_res_levels), per-level iteration counts and gather mode.  Off (the default), the group is made with
  // hsb_group_create and the …Many calls throw for processors that differ.  Changing it drops the cached group.
  void setHeterogeneousGroups(bool on) {
    if (on == heterogeneous_) return;
    dropGroup();
    heterogeneous_ = on;
  }
  bool heterogeneousGroups() const { return heterogeneous_; }

  // reset() for the processors ps[members[0..K)] of ps[0..M) in one launch (hsb_group_reset_subset, through the group
  // updateMany keeps; members null: all M, hsb_group_reset, and K is not read): the node's reset_map service or "reset"
  // system message for a fleet.  restart_mapping_with_new_pose for K robots is resetMany() followed by their next step
  // with the new poses as hints.  Returns once the reset is queued; every later call on a reset processor runs after it.
  static void resetMany(SlamProcessor* const* ps, int M, const int* members = 0, int K = 0) {
    SlamProcessor& owner = groupOwnerOf(ps, M, "resetMany");
    hsb_group* g = owner.groupFor(ps, M);
    owner.check(members ? hsb_group_reset_subset(g, K, members) : hsb_group_reset(g));
    for (int k = 0; k < (members ? K : M); ++k) {
      SlamProcessor& p = *ps[members ? members[k] : k];
      p.lastMapUpdatePose_ = Pose{FLT_MAX, FLT_MAX, FLT_MAX};   // as reset()
      p.lastScanMatchPose_ = Pose{0.f, 0.f, 0.f};
    }
  }

  // The node's pub_drawings / pub_debug_output for the fused and group steps (hsb_set_step_record): on, every matched
  // update*() and this processor's session of every updateMany*() records its match; the results are unchanged.
  // stepRecord() fetches the record of the last step (false: that step ran no match, the reference calls no hook);
  // lastMatchScan() the level-0 container it matched (n endpoints, 2n floats, and origo).  With the reference's headers,
  // replayMatchHooks (MatchHooksB200.h) turns the two into the matcher's hook calls.
  void setStepRecord(bool on) { check(hsb_set_step_record(h_, on ? 1 : 0)); }
  bool stepRecord(std::vector<float>& record) const {
    const int R = hsb_get_match_record_floats(h_);
    if (R < 0) check(R);
    record.resize((size_t)R);
    int matched = 0;
    check(hsb_get_step_record(h_, record.data(), &matched));
    return matched != 0;
  }
  int lastMatchScan(std::vector<float>& pointsXY, float origo[2]) const {
    int n = 0;
    if (hsb_get_last_match_scan(h_, 0, 0, &n, origo) != HSB_OK && n == 0) check(HSB_ERR_INVALID_ARG);
    pointsXY.resize(2 * (size_t)n);
    check(hsb_get_last_match_scan(h_, pointsXY.data(), n, &n, origo));
    return n;
  }

  const Pose& getLastScanMatchPose() const { return lastScanMatchPose_; }
  const float* getLastScanMatchCovariance() const { return lastScanMatchCov_; }
  float getScaleToMap() const { return hsb_get_scale_to_map(h_); }
  int getMapLevels() const { return hsb_get_map_levels(h_); }
  void setUpdateFactorFree(float f) { check(hsb_set_update_factor_free(h_, f)); }
  void setUpdateFactorOccupied(float f) { check(hsb_set_update_factor_occupied(h_, f)); }
  void setMapUpdateMinDistDiff(float minDist) {
    minDist_ = minDist;
    check(hsb_set_map_update_min_dist_diff(h_, minDist));
  }
  void setMapUpdateMinAngleDiff(float angleChange) {
    minAngle_ = angleChange;
    check(hsb_set_map_update_min_angle_diff(h_, angleChange));
  }
  // getGridMap(level): the log-odds plane, row-major [sizeY][sizeX]
  void getGridMap(int level, float* logodds_out) const { check(hsb_download_level(h_, level, logodds_out)); }

  // HectorMappingRos::publishMap's grid kept up to date (HectorMappingRos.cpp:435-481): grid is this processor's whole
  // level, sizeY x sizeX int8 row-major, kept between calls as the node keeps map_.map.data.  The cells written since the
  // last call (the mirror rectangle, which this consumes) get publishMap's values (0 free, 100 occupied, -1 unknown); no
  // other byte is touched.  rect (may be null) receives {x0, y0, x1, y1}; x1 < x0: nothing changed, nothing to publish.
  void syncOccupancy(int level, int8_t* grid, int rect[4] = 0) {
    int r[4];
    check(hsb_get_mirror_dirty_rect(h_, level, r, 1));
    if (rect) std::memcpy(rect, r, sizeof(r));
    if (r[2] < r[0] || r[3] < r[1]) return;
    int sx = 0, sy = 0;
    float cl = 0.f;
    check(hsb_get_level_info(h_, level, &sx, &sy, &cl));
    const int w = r[2] - r[0] + 1, hgt = r[3] - r[1] + 1;
    std::vector<int8_t> rows((size_t)w * hgt);
    check(hsb_download_occupancy_rect(h_, level, r, rows.data()));
    for (int y = 0; y < hgt; ++y) std::memcpy(grid + (size_t)(r[1] + y) * sx + r[0], &rows[(size_t)y * w], (size_t)w);
  }

  // syncOccupancy() for M processors in one pass (hsb_group_sync_occupancy, through the group updateMany keeps):
  // grids[s] is processor s's grid, rects (4M ints, may be null) receives each rectangle.
  static void syncOccupancyMany(SlamProcessor* const* ps, int M, int level, int8_t* const* grids, int* rects = 0) {
    SlamProcessor& owner = groupOwnerOf(ps, M, "syncOccupancyMany");
    owner.check(hsb_group_sync_occupancy(owner.groupFor(ps, M), level, grids, rects, 1));
  }

  // syncOccupancyMany() for the processors ps[members[0..K)] (hsb_group_sync_occupancy_subset): grids[k] and
  // rects[4k..] belong to ps[members[k]]; the processors not listed are left as they are.
  static void syncOccupancyMany(SlamProcessor* const* ps, int M, const int* members, int K, int level,
                                int8_t* const* grids, int* rects = 0) {
    SlamProcessor& owner = groupOwnerOf(ps, M, "syncOccupancyMany");
    owner.check(hsb_group_sync_occupancy_subset(owner.groupFor(ps, M), K, members, level, grids, rects, 1));
  }

  // hector_map_tools' DistanceMeasurementProvider::getDist (HectorMapTools.h:133-147) for n world-frame rays on this
  // processor's level, as hector_map_server's get_distance_to_obstacle calls it (hector_map_server.cpp:123):
  // dist[i] = distance to the first occupied cell in metres (-cell length: nothing hit), hitWorld[2i..] (may be null)
  // the hit point ((0, 0) if none), found[i] (may be null) whether something was hit.  beginWorld / endWorld: n x 2.
  void getDist(int level, int n, const float* beginWorld, const float* endWorld, float* dist, float* hitWorld = 0,
               int* found = 0) {
    check(hsb_get_dist_batch(h_, level, n, beginWorld, endWorld, dist, hitWorld, found));
  }

  // getDist() for M processors in one pass (hsb_group_get_dist, through the group updateMany keeps): processor s casts
  // the rays [offsets[s], offsets[s+1]) of beginWorld / endWorld; the outputs are in ray order.
  static void getDistMany(SlamProcessor* const* ps, int M, int level, const int* offsets, const float* beginWorld,
                          const float* endWorld, float* dist, float* hitWorld = 0, int* found = 0) {
    SlamProcessor& owner = groupOwnerOf(ps, M, "getDistMany");
    owner.check(hsb_group_get_dist(owner.groupFor(ps, M), level, offsets, beginWorld, endWorld, dist, hitWorld, found));
  }

  // getDistMany() for the processors ps[members[0..K)] (hsb_group_get_dist_subset): the rays [offsets[k],
  // offsets[k+1]) belong to ps[members[k]]; the processors not listed are neither read nor waited for.
  static void getDistMany(SlamProcessor* const* ps, int M, const int* members, int K, int level, const int* offsets,
                          const float* beginWorld, const float* endWorld, float* dist, float* hitWorld = 0,
                          int* found = 0) {
    SlamProcessor& owner = groupOwnerOf(ps, M, "getDistMany");
    owner.check(hsb_group_get_dist_subset(owner.groupFor(ps, M), K, members, level, offsets, beginWorld, endWorld, dist,
                                          hitWorld, found));
  }
  // getLikelihoodForState (OccGridMapUtil.h:189-221) for M processors in one pass (hsb_group_likelihood, through the
  // group updateMany keeps): processor s's world poses [poseOffsets[s], poseOffsets[s+1]) of posesWorld (x, y, psi) are
  // scored on its map of `level` against its scan pointsXY[scanOffsets[s] .. scanOffsets[s+1]) (level-0 cells), or,
  // with pointsXY and scanOffsets null, against the scan of its last matched update as it is on the device.
  // likelihood: one per pose, in pose order.
  static void likelihoodMany(SlamProcessor* const* ps, int M, int level, const int* poseOffsets, const float* posesWorld,
                             const float* pointsXY, const int* scanOffsets, float* likelihood) {
    SlamProcessor& owner = groupOwnerOf(ps, M, "likelihoodMany");
    owner.check(hsb_group_likelihood(owner.groupFor(ps, M), level, poseOffsets, posesWorld, pointsXY, scanOffsets,
                                     likelihood));
  }

  // likelihoodMany() for the processors ps[members[0..K)] (hsb_group_likelihood_subset): session k's poses and scan
  // belong to ps[members[k]]; the processors not listed are neither read nor waited for.
  static void likelihoodMany(SlamProcessor* const* ps, int M, const int* members, int K, int level,
                             const int* poseOffsets, const float* posesWorld, const float* pointsXY,
                             const int* scanOffsets, float* likelihood) {
    SlamProcessor& owner = groupOwnerOf(ps, M, "likelihoodMany");
    owner.check(hsb_group_likelihood_subset(owner.groupFor(ps, M), K, members, level, poseOffsets, posesWorld, pointsXY,
                                            scanOffsets, likelihood));
  }

  // getCovarianceForPose and getCovMatrixWorldCoords (OccGridMapUtil.h:106-187) for M processors in one pass
  // (hsb_group_covariance); poses and scans as in likelihoodMany.  covMap / covWorld: 9 floats per pose, row-major;
  // either may be null, not both.
  static void covarianceMany(SlamProcessor* const* ps, int M, int level, const int* poseOffsets, const float* posesWorld,
                             const float* pointsXY, const int* scanOffsets, float* covMap, float* covWorld) {
    SlamProcessor& owner = groupOwnerOf(ps, M, "covarianceMany");
    owner.check(hsb_group_covariance(owner.groupFor(ps, M), level, poseOffsets, posesWorld, pointsXY, scanOffsets, covMap,
                                     covWorld));
  }

  // covarianceMany() for the processors ps[members[0..K)] (hsb_group_covariance_subset).
  static void covarianceMany(SlamProcessor* const* ps, int M, const int* members, int K, int level,
                             const int* poseOffsets, const float* posesWorld, const float* pointsXY,
                             const int* scanOffsets, float* covMap, float* covWorld) {
    SlamProcessor& owner = groupOwnerOf(ps, M, "covarianceMany");
    owner.check(hsb_group_covariance_subset(owner.groupFor(ps, M), K, members, level, poseOffsets, posesWorld, pointsXY,
                                            scanOffsets, covMap, covWorld));
  }

  // The most likely of each processor's pose hypotheses in one pass (hsb_group_best_hypothesis): relocalising several
  // lost robots at once; poses and scans as in likelihoodMany.  best4: per processor {likelihood, x, y, psi} of its
  // winner (the lowest index among equals; likelihood -1 without hypotheses); bestIndex (may be null): the winner's
  // index among the processor's poses, -1 without hypotheses; likelihood (may be null): one per pose.
  static void bestHypothesisMany(SlamProcessor* const* ps, int M, int level, const int* poseOffsets,
                                 const float* posesWorld, const float* pointsXY, const int* scanOffsets, float* best4,
                                 int* bestIndex = 0, float* likelihood = 0) {
    SlamProcessor& owner = groupOwnerOf(ps, M, "bestHypothesisMany");
    owner.check(hsb_group_best_hypothesis(owner.groupFor(ps, M), level, poseOffsets, posesWorld, pointsXY, scanOffsets,
                                          likelihood, best4, bestIndex));
  }

  // bestHypothesisMany() for the processors ps[members[0..K)] (hsb_group_best_hypothesis_subset).
  static void bestHypothesisMany(SlamProcessor* const* ps, int M, const int* members, int K, int level,
                                 const int* poseOffsets, const float* posesWorld, const float* pointsXY,
                                 const int* scanOffsets, float* best4, int* bestIndex = 0, float* likelihood = 0) {
    SlamProcessor& owner = groupOwnerOf(ps, M, "bestHypothesisMany");
    owner.check(hsb_group_best_hypothesis_subset(owner.groupFor(ps, M), K, members, level, poseOffsets, posesWorld,
                                                 pointsXY, scanOffsets, likelihood, best4, bestIndex));
  }

  // MapRepMultiMap::matchData (MapRepMultiMap.h:116-132) from many start poses for M processors in one pass
  // (hsb_group_match_batch, through the group updateMany keeps): processor s's world hints [hintOffsets[s],
  // hintOffsets[s+1]) of hintsWorld (x, y, psi) are each matched over all levels on its map with its scan
  // pointsXY[scanOffsets[s] .. scanOffsets[s+1]) (level-0 cells), or, with pointsXY and scanOffsets null, with the scan
  // of its last matched update as it is on the device.  posesWorld: one pose per hint, in hint order; cov (may be null):
  // the Hessian of each hint's last evaluation, 9 floats row-major.  No processor's state changes.
  static void matchMany(SlamProcessor* const* ps, int M, const int* hintOffsets, const float* hintsWorld,
                        const float* pointsXY, const int* scanOffsets, float* posesWorld, float* cov = 0) {
    SlamProcessor& owner = groupOwnerOf(ps, M, "matchMany");
    owner.check(hsb_group_match_batch(owner.groupFor(ps, M), hintOffsets, hintsWorld, pointsXY, scanOffsets, posesWorld,
                                      cov));
  }

  // matchMany() for the processors ps[members[0..K)] (hsb_group_match_batch_subset): session k's hints and scan
  // belong to ps[members[k]]; the processors not listed are neither read nor waited for.
  static void matchMany(SlamProcessor* const* ps, int M, const int* members, int K, const int* hintOffsets,
                        const float* hintsWorld, const float* pointsXY, const int* scanOffsets, float* posesWorld,
                        float* cov = 0) {
    SlamProcessor& owner = groupOwnerOf(ps, M, "matchMany");
    owner.check(hsb_group_match_batch_subset(owner.groupFor(ps, M), K, members, hintOffsets, hintsWorld, pointsXY,
                                             scanOffsets, posesWorld, cov));
  }

  // matchMany() from each processor's new LaserScan ranges[scanOffsets[s] .. scanOffsets[s+1]), converted on the device
  // with its scan format, followed by the pick (hsb_group_match_batch_ranges): relocalising lost robots from the scans
  // they just sent, before anything writes them into a map.  likelihood (one per hint), best4 ({likelihood, x, y, psi}
  // per processor), bestIndex (per processor) and kept (endpoints each conversion kept, per processor) may be null; the
  // scoring runs only when one of the first three is given.  No processor's state changes.
  static void matchManyRanges(SlamProcessor* const* ps, int M, const int* hintOffsets, const float* hintsWorld,
                              const float* ranges, const int* scanOffsets, float* posesWorld, float* cov = 0,
                              float* likelihood = 0, float* best4 = 0, int* bestIndex = 0, int* kept = 0) {
    SlamProcessor& owner = groupOwnerOf(ps, M, "matchManyRanges");
    owner.check(hsb_group_match_batch_ranges(owner.groupFor(ps, M), hintOffsets, hintsWorld, ranges, scanOffsets,
                                             posesWorld, cov, likelihood, best4, bestIndex, kept));
  }
  // matchManyRanges() for the processors ps[members[0..K)] (hsb_group_match_batch_ranges_subset).
  static void matchManyRanges(SlamProcessor* const* ps, int M, const int* members, int K, const int* hintOffsets,
                              const float* hintsWorld, const float* ranges, const int* scanOffsets, float* posesWorld,
                              float* cov = 0, float* likelihood = 0, float* best4 = 0, int* bestIndex = 0,
                              int* kept = 0) {
    SlamProcessor& owner = groupOwnerOf(ps, M, "matchManyRanges");
    owner.check(hsb_group_match_batch_ranges_subset(owner.groupFor(ps, M), K, members, hintOffsets, hintsWorld, ranges,
                                                    scanOffsets, posesWorld, cov, likelihood, best4, bestIndex, kept));
  }
  // matchManyRanges() from Point32 clouds in the laser frame, pointsXYZ[scanOffsets[s] .. scanOffsets[s+1]) with laser
  // transforms (12 doubles per processor, null: each processor's cloud format), each converted with its cloud format
  // (hsb_group_match_batch_cloud).
  static void matchManyCloud(SlamProcessor* const* ps, int M, const int* hintOffsets, const float* hintsWorld,
                             const float* pointsXYZ, const int* scanOffsets, const double* transforms, float* posesWorld,
                             float* cov = 0, float* likelihood = 0, float* best4 = 0, int* bestIndex = 0, int* kept = 0) {
    SlamProcessor& owner = groupOwnerOf(ps, M, "matchManyCloud");
    owner.check(hsb_group_match_batch_cloud(owner.groupFor(ps, M), hintOffsets, hintsWorld, pointsXYZ, scanOffsets,
                                            transforms, posesWorld, cov, likelihood, best4, bestIndex, kept));
  }
  // matchManyCloud() for the processors ps[members[0..K)] (hsb_group_match_batch_cloud_subset).
  static void matchManyCloud(SlamProcessor* const* ps, int M, const int* members, int K, const int* hintOffsets,
                             const float* hintsWorld, const float* pointsXYZ, const int* scanOffsets,
                             const double* transforms, float* posesWorld, float* cov = 0, float* likelihood = 0,
                             float* best4 = 0, int* bestIndex = 0, int* kept = 0) {
    SlamProcessor& owner = groupOwnerOf(ps, M, "matchManyCloud");
    owner.check(hsb_group_match_batch_cloud_subset(owner.groupFor(ps, M), K, members, hintOffsets, hintsWorld, pointsXYZ,
                                                   scanOffsets, transforms, posesWorld, cov, likelihood, best4,
                                                   bestIndex, kept));
  }
  // matchManyRanges() from the LaserScans of default-configured nodes: each processor projects its ranges with its laser
  // projection and converts them with its cloud format; transforms as in matchManyCloud (hsb_group_match_batch_projected).
  static void matchManyProjected(SlamProcessor* const* ps, int M, const int* hintOffsets, const float* hintsWorld,
                                 const float* ranges, const int* scanOffsets, const double* transforms,
                                 float* posesWorld, float* cov = 0, float* likelihood = 0, float* best4 = 0,
                                 int* bestIndex = 0, int* kept = 0) {
    SlamProcessor& owner = groupOwnerOf(ps, M, "matchManyProjected");
    owner.check(hsb_group_match_batch_projected(owner.groupFor(ps, M), hintOffsets, hintsWorld, ranges, scanOffsets,
                                                transforms, posesWorld, cov, likelihood, best4, bestIndex, kept));
  }
  // matchManyProjected() for the processors ps[members[0..K)] (hsb_group_match_batch_projected_subset).
  static void matchManyProjected(SlamProcessor* const* ps, int M, const int* members, int K, const int* hintOffsets,
                                 const float* hintsWorld, const float* ranges, const int* scanOffsets,
                                 const double* transforms, float* posesWorld, float* cov = 0, float* likelihood = 0,
                                 float* best4 = 0, int* bestIndex = 0, int* kept = 0) {
    SlamProcessor& owner = groupOwnerOf(ps, M, "matchManyProjected");
    owner.check(hsb_group_match_batch_projected_subset(owner.groupFor(ps, M), K, members, hintOffsets, hintsWorld,
                                                       ranges, scanOffsets, transforms, posesWorld, cov, likelihood,
                                                       best4, bestIndex, kept));
  }
  hsb_handle* handle() { return h_; }

  // util::poseDifferenceLargerThan, util/UtilFunctions.h:73-92 (float norm, double pi arithmetic)
  static bool poseDifferenceLargerThan(const Pose& p1, const Pose& p2, float distThresh, float angleThresh) {
    const float dx = p1.x - p2.x, dy = p1.y - p2.y;
    if (std::sqrt(dx * dx + dy * dy) > distThresh) return true;
    float angleDiff = p1.psi - p2.psi;
    if (angleDiff > M_PI) {
      angleDiff -= M_PI * 2.0f;
    } else if (angleDiff < -M_PI) {
      angleDiff += M_PI * 2.0f;
    }
    return std::fabs(angleDiff) > angleThresh;
  }

 private:
  void check(int st) const {
    if (st != HSB_OK) throw std::runtime_error(std::string("hector_slam_b200: ") + hsb_last_error(h_));
  }
  // One group step of the group of ps[0..M) over the K processors ps[members[k]] (members null: all M, in order):
  // `step(group, hints, poses, cov, updated)` makes the C-ABI call; the stepped processors' poses and covariances are
  // kept as update() keeps them.
  template <class Step>
  static void stepMany(SlamProcessor* const* ps, int M, const int* members, int K, const Pose* poseHintsWorld,
                       const char* what, Step step) {
    SlamProcessor& owner = groupOwnerOf(ps, M, what);
    if (K < 0 || K > M || (K > 0 && !members && K != M))
      throw std::invalid_argument(std::string("hector_slam_b200: ") + what + " needs 0 <= K <= M and a member list");
    for (int k = 0; members && k < K; ++k)
      if (members[k] < 0 || members[k] >= M)
        throw std::invalid_argument(std::string("hector_slam_b200: ") + what + ": a member index is outside [0, M)");
    hsb_group* g = owner.groupFor(ps, M);
    std::vector<float> hints(3 * (size_t)K), poses(3 * (size_t)K), cov(9 * (size_t)K);
    std::vector<int> updated(K);
    for (int s = 0; s < K; ++s) {
      const SlamProcessor& p = *ps[members ? members[s] : s];
      hints[3 * s] = poseHintsWorld[s].x;
      hints[3 * s + 1] = poseHintsWorld[s].y;
      hints[3 * s + 2] = poseHintsWorld[s].psi;
      std::memcpy(&cov[9 * s], p.lastScanMatchCov_, sizeof(p.lastScanMatchCov_));   // untouched where unmatched
    }
    owner.check(step(g, hints.data(), poses.data(), cov.data(), updated.data()));
    for (int s = 0; s < K; ++s) {
      SlamProcessor& p = *ps[members ? members[s] : s];
      p.lastScanMatchPose_ = Pose{poses[3 * s], poses[3 * s + 1], poses[3 * s + 2]};  // :83
      if (updated[s]) p.lastMapUpdatePose_ = p.lastScanMatchPose_;                    // :94
      std::memcpy(p.lastScanMatchCov_, &cov[9 * s], sizeof(p.lastScanMatchCov_));
    }
  }
  // ps[0], which keeps the group of ps[0..M)
  static SlamProcessor& groupOwnerOf(SlamProcessor* const* ps, int M, const char* what) {
    if (!ps || M < 1 || !ps[0])
      throw std::invalid_argument(std::string("hector_slam_b200: ") + what + " needs M >= 1 processors");
    return *ps[0];
  }
  // the cached group of updateMany: rebuilt only when the member list changes.  A processor belongs to at most one
  // cached group (its groupOwner_), so that destroying any member destroys that group first.
  hsb_group* groupFor(SlamProcessor* const* ps, int M) {
    bool same = group_ && (int)groupMembers_.size() == M;
    for (int s = 0; same && s < M; ++s) same = groupMembers_[s] == ps[s];
    if (same) return group_;
    dropGroup();
    std::vector<hsb_handle*> hs(M);
    for (int s = 0; s < M; ++s) {
      if (!ps[s]) throw std::invalid_argument("hector_slam_b200: updateMany: processor is null");
      if (ps[s]->groupOwner_) ps[s]->groupOwner_->dropGroup();
      hs[s] = ps[s]->h_;
    }
    hsb_group* g = 0;
    const int st = heterogeneous_ ? hsb_group_create_heterogeneous(hs.data(), M, &g) : hsb_group_create(hs.data(), M, &g);
    if (st != HSB_OK)
      throw std::runtime_error(std::string("hector_slam_b200: ") + hsb_last_error(0));
    group_ = g;
    groupMembers_.assign(ps, ps + M);
    for (int s = 0; s < M; ++s) ps[s]->groupOwner_ = this;
    return group_;
  }
  void dropGroup() {
    if (!group_) return;
    hsb_group_destroy(group_);
    group_ = 0;
    for (size_t s = 0; s < groupMembers_.size(); ++s)
      if (groupMembers_[s]->groupOwner_ == this) groupMembers_[s]->groupOwner_ = 0;
    groupMembers_.clear();
  }
  hsb_handle* h_;
  hsb_group* group_;                           // updateMany's group, when this processor is its ps[0]
  std::vector<SlamProcessor*> groupMembers_;
  SlamProcessor* groupOwner_;                  // the processor whose cached group contains this one
  bool heterogeneous_;                         // setHeterogeneousGroups
  Pose lastMapUpdatePose_, lastScanMatchPose_;
  float lastScanMatchCov_[9];
  float minDist_, minAngle_;
};

}  // namespace hsb200
#endif
