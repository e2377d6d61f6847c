// host_capi.cpp — extern "C" shim over hsb200::SlamProcessor so that the C++ host façade can be
// driven from ctypes in the tests (the façade itself is header-only C++).
#include "SlamProcessorB200.hpp"

#include <cstring>
#include <vector>

extern "C" {

void* hsbp_create(float res, int sx, int sy, float startx, float starty, int levels, int device) {
  try {
    return new hsb200::SlamProcessor(res, sx, sy, startx, starty, levels, device);
  } catch (const std::exception&) {
    return 0;
  }
}
void hsbp_destroy(void* p) { delete static_cast<hsb200::SlamProcessor*>(p); }

int hsbp_update(void* p, const float* pts, int n, const float* origo, const float hint[3], int map_without_matching,
                float out_pose[3], float out_cov[9]) {
  hsb200::SlamProcessor* s = static_cast<hsb200::SlamProcessor*>(p);
  try {
    s->update(pts, n, origo, hsb200::Pose{hint[0], hint[1], hint[2]}, map_without_matching != 0);
  } catch (const std::exception&) {
    return -1;
  }
  const hsb200::Pose& q = s->getLastScanMatchPose();
  out_pose[0] = q.x;
  out_pose[1] = q.y;
  out_pose[2] = q.psi;
  if (out_cov) std::memcpy(out_cov, s->getLastScanMatchCovariance(), 9 * sizeof(float));
  return 0;
}
int hsbp_update_many(void* const* ps, int M, const float* pts, const int* offsets, const float* origo, const float* hints,
                     const int* map_without_matching) {
  std::vector<hsb200::SlamProcessor*> procs(M > 0 ? M : 0);
  std::vector<hsb200::Pose> poses(M > 0 ? M : 0);
  for (int s = 0; s < M; ++s) {
    procs[s] = static_cast<hsb200::SlamProcessor*>(ps[s]);
    poses[s] = hsb200::Pose{hints[3 * s], hints[3 * s + 1], hints[3 * s + 2]};
  }
  try {
    hsb200::SlamProcessor::updateMany(procs.data(), M, pts, offsets, origo, poses.data(), map_without_matching);
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
int hsbp_set_cloud_format(void* p, const double transform[12], float sqr_min_dist, float sqr_max_dist, float z_min,
                          float z_max) {
  hsb_cloud_format fmt;
  std::memcpy(fmt.laser_transform, transform, sizeof(fmt.laser_transform));
  fmt.sqr_laser_min_dist = sqr_min_dist;
  fmt.sqr_laser_max_dist = sqr_max_dist;
  fmt.laser_z_min_value = z_min;
  fmt.laser_z_max_value = z_max;
  try {
    static_cast<hsb200::SlamProcessor*>(p)->setCloudFormat(fmt);
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
int hsbp_update_cloud(void* p, const float* points_xyz, int n, const double* transform, const float hint[3],
                      int map_without_matching, int* out_kept) {
  try {
    const int kept = static_cast<hsb200::SlamProcessor*>(p)->updateCloud(
        points_xyz, n, transform, hsb200::Pose{hint[0], hint[1], hint[2]}, map_without_matching != 0);
    if (out_kept) *out_kept = kept;
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
int hsbp_update_many_cloud(void* const* ps, int M, const float* points_xyz, const int* offsets, const double* transforms,
                           const float* hints, const int* map_without_matching, int* out_kept) {
  std::vector<hsb200::SlamProcessor*> procs(M > 0 ? M : 0);
  std::vector<hsb200::Pose> poses(M > 0 ? M : 0);
  for (int s = 0; s < M; ++s) {
    procs[s] = static_cast<hsb200::SlamProcessor*>(ps[s]);
    poses[s] = hsb200::Pose{hints[3 * s], hints[3 * s + 1], hints[3 * s + 2]};
  }
  try {
    hsb200::SlamProcessor::updateManyCloud(procs.data(), M, points_xyz, offsets, transforms, poses.data(),
                                           map_without_matching, out_kept);
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
int hsbp_set_scan_format(void* p, int n_beams, float angle_min, float angle_increment, float range_min, float range_max) {
  hsb_scan_format fmt;
  fmt.n_beams = n_beams;
  fmt.angle_min = angle_min;
  fmt.angle_increment = angle_increment;
  fmt.range_min = range_min;
  fmt.range_max = range_max;
  try {
    static_cast<hsb200::SlamProcessor*>(p)->setScanFormat(fmt);
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
int hsbp_update_ranges(void* p, const float* ranges, int n, const float hint[3], int map_without_matching, int* out_kept) {
  try {
    const int kept = static_cast<hsb200::SlamProcessor*>(p)->updateRanges(
        ranges, n, hsb200::Pose{hint[0], hint[1], hint[2]}, map_without_matching != 0);
    if (out_kept) *out_kept = kept;
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
int hsbp_update_many_ranges(void* const* ps, int M, const float* ranges, const int* offsets, const float* hints,
                            const int* map_without_matching, int* out_kept) {
  std::vector<hsb200::SlamProcessor*> procs(M > 0 ? M : 0);
  std::vector<hsb200::Pose> poses(M > 0 ? M : 0);
  for (int s = 0; s < M; ++s) {
    procs[s] = static_cast<hsb200::SlamProcessor*>(ps[s]);
    poses[s] = hsb200::Pose{hints[3 * s], hints[3 * s + 1], hints[3 * s + 2]};
  }
  try {
    hsb200::SlamProcessor::updateManyRanges(procs.data(), M, ranges, offsets, poses.data(), map_without_matching,
                                            out_kept);
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
int hsbp_set_laser_projection(void* p, int n_beams, float angle_min, float angle_increment, float range_min,
                              float range_max, double range_cutoff) {
  hsb_laser_projection proj;
  proj.n_beams = n_beams;
  proj.angle_min = angle_min;
  proj.angle_increment = angle_increment;
  proj.range_min = range_min;
  proj.range_max = range_max;
  proj.range_cutoff = range_cutoff;
  try {
    static_cast<hsb200::SlamProcessor*>(p)->setLaserProjection(proj);
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
int hsbp_update_projected(void* p, const float* ranges, int n, const double* transform, const float hint[3],
                          int map_without_matching, int* out_kept) {
  try {
    const int kept = static_cast<hsb200::SlamProcessor*>(p)->updateProjected(
        ranges, n, transform, hsb200::Pose{hint[0], hint[1], hint[2]}, map_without_matching != 0);
    if (out_kept) *out_kept = kept;
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
int hsbp_update_many_projected(void* const* ps, int M, const float* ranges, const int* offsets, const double* transforms,
                               const float* hints, const int* map_without_matching, int* out_kept) {
  std::vector<hsb200::SlamProcessor*> procs(M > 0 ? M : 0);
  std::vector<hsb200::Pose> poses(M > 0 ? M : 0);
  for (int s = 0; s < M; ++s) {
    procs[s] = static_cast<hsb200::SlamProcessor*>(ps[s]);
    poses[s] = hsb200::Pose{hints[3 * s], hints[3 * s + 1], hints[3 * s + 2]};
  }
  try {
    hsb200::SlamProcessor::updateManyProjected(procs.data(), M, ranges, offsets, transforms, poses.data(),
                                               map_without_matching, out_kept);
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
// The subset overloads: processor ps[members[k]] takes session k; hints and every per-session array have K entries.
int hsbp_update_many_subset(void* const* ps, int M, const int* members, int K, const float* pts, const int* offsets,
                            const float* origo, const float* hints, const int* map_without_matching) {
  std::vector<hsb200::SlamProcessor*> procs(M > 0 ? M : 0);
  std::vector<hsb200::Pose> poses(K > 0 ? K : 0);
  for (int s = 0; s < M; ++s) procs[s] = static_cast<hsb200::SlamProcessor*>(ps[s]);
  for (int k = 0; k < K; ++k) poses[k] = hsb200::Pose{hints[3 * k], hints[3 * k + 1], hints[3 * k + 2]};
  try {
    hsb200::SlamProcessor::updateMany(procs.data(), M, members, K, pts, offsets, origo, poses.data(),
                                      map_without_matching);
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
int hsbp_update_many_cloud_subset(void* const* ps, int M, const int* members, int K, const float* points_xyz,
                                  const int* offsets, const double* transforms, const float* hints,
                                  const int* map_without_matching, int* out_kept) {
  std::vector<hsb200::SlamProcessor*> procs(M > 0 ? M : 0);
  std::vector<hsb200::Pose> poses(K > 0 ? K : 0);
  for (int s = 0; s < M; ++s) procs[s] = static_cast<hsb200::SlamProcessor*>(ps[s]);
  for (int k = 0; k < K; ++k) poses[k] = hsb200::Pose{hints[3 * k], hints[3 * k + 1], hints[3 * k + 2]};
  try {
    hsb200::SlamProcessor::updateManyCloud(procs.data(), M, members, K, points_xyz, offsets, transforms, poses.data(),
                                           map_without_matching, out_kept);
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
int hsbp_update_many_ranges_subset(void* const* ps, int M, const int* members, int K, const float* ranges,
                                   const int* offsets, const float* hints, const int* map_without_matching,
                                   int* out_kept) {
  std::vector<hsb200::SlamProcessor*> procs(M > 0 ? M : 0);
  std::vector<hsb200::Pose> poses(K > 0 ? K : 0);
  for (int s = 0; s < M; ++s) procs[s] = static_cast<hsb200::SlamProcessor*>(ps[s]);
  for (int k = 0; k < K; ++k) poses[k] = hsb200::Pose{hints[3 * k], hints[3 * k + 1], hints[3 * k + 2]};
  try {
    hsb200::SlamProcessor::updateManyRanges(procs.data(), M, members, K, ranges, offsets, poses.data(),
                                            map_without_matching, out_kept);
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
int hsbp_update_many_projected_subset(void* const* ps, int M, const int* members, int K, const float* ranges,
                                      const int* offsets, const double* transforms, const float* hints,
                                      const int* map_without_matching, int* out_kept) {
  std::vector<hsb200::SlamProcessor*> procs(M > 0 ? M : 0);
  std::vector<hsb200::Pose> poses(K > 0 ? K : 0);
  for (int s = 0; s < M; ++s) procs[s] = static_cast<hsb200::SlamProcessor*>(ps[s]);
  for (int k = 0; k < K; ++k) poses[k] = hsb200::Pose{hints[3 * k], hints[3 * k + 1], hints[3 * k + 2]};
  try {
    hsb200::SlamProcessor::updateManyProjected(procs.data(), M, members, K, ranges, offsets, transforms, poses.data(),
                                               map_without_matching, out_kept);
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
int hsbp_sync_occupancy(void* p, int level, int8_t* grid, int* rect) {
  try {
    static_cast<hsb200::SlamProcessor*>(p)->syncOccupancy(level, grid, rect);
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
int hsbp_sync_occupancy_many(void* const* ps, int M, int level, int8_t* const* grids, int* rects) {
  std::vector<hsb200::SlamProcessor*> procs(M > 0 ? M : 0);
  for (int s = 0; s < M; ++s) procs[s] = static_cast<hsb200::SlamProcessor*>(ps[s]);
  try {
    hsb200::SlamProcessor::syncOccupancyMany(procs.data(), M, level, grids, rects);
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
int hsbp_sync_occupancy_many_subset(void* const* ps, int M, const int* members, int K, int level, int8_t* const* grids,
                                    int* rects) {
  std::vector<hsb200::SlamProcessor*> procs(M > 0 ? M : 0);
  for (int s = 0; s < M; ++s) procs[s] = static_cast<hsb200::SlamProcessor*>(ps[s]);
  try {
    hsb200::SlamProcessor::syncOccupancyMany(procs.data(), M, members, K, level, grids, rects);
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
int hsbp_get_dist(void* p, int level, int n, const float* begin_world, const float* end_world, float* dist,
                  float* hit_world, int* found) {
  try {
    static_cast<hsb200::SlamProcessor*>(p)->getDist(level, n, begin_world, end_world, dist, hit_world, found);
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
int hsbp_get_dist_many(void* const* ps, int M, int level, const int* offsets, const float* begin_world,
                       const float* end_world, float* dist, float* hit_world, int* found) {
  std::vector<hsb200::SlamProcessor*> procs(M > 0 ? M : 0);
  for (int s = 0; s < M; ++s) procs[s] = static_cast<hsb200::SlamProcessor*>(ps[s]);
  try {
    hsb200::SlamProcessor::getDistMany(procs.data(), M, level, offsets, begin_world, end_world, dist, hit_world, found);
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
int hsbp_get_dist_many_subset(void* const* ps, int M, const int* members, int K, int level, const int* offsets,
                              const float* begin_world, const float* end_world, float* dist, float* hit_world,
                              int* found) {
  std::vector<hsb200::SlamProcessor*> procs(M > 0 ? M : 0);
  for (int s = 0; s < M; ++s) procs[s] = static_cast<hsb200::SlamProcessor*>(ps[s]);
  try {
    hsb200::SlamProcessor::getDistMany(procs.data(), M, members, K, level, offsets, begin_world, end_world, dist,
                                       hit_world, found);
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
int hsbp_likelihood_many(void* const* ps, int M, int level, const int* pose_offsets, const float* poses_world,
                         const float* points_xy, const int* scan_offsets, float* likelihood) {
  std::vector<hsb200::SlamProcessor*> procs(M > 0 ? M : 0);
  for (int s = 0; s < M; ++s) procs[s] = static_cast<hsb200::SlamProcessor*>(ps[s]);
  try {
    hsb200::SlamProcessor::likelihoodMany(procs.data(), M, level, pose_offsets, poses_world, points_xy, scan_offsets,
                                          likelihood);
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
int hsbp_likelihood_many_subset(void* const* ps, int M, const int* members, int K, int level, const int* pose_offsets,
                                const float* poses_world, const float* points_xy, const int* scan_offsets,
                                float* likelihood) {
  std::vector<hsb200::SlamProcessor*> procs(M > 0 ? M : 0);
  for (int s = 0; s < M; ++s) procs[s] = static_cast<hsb200::SlamProcessor*>(ps[s]);
  try {
    hsb200::SlamProcessor::likelihoodMany(procs.data(), M, members, K, level, pose_offsets, poses_world, points_xy,
                                          scan_offsets, likelihood);
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
int hsbp_covariance_many(void* const* ps, int M, int level, const int* pose_offsets, const float* poses_world,
                         const float* points_xy, const int* scan_offsets, float* cov_map, float* cov_world) {
  std::vector<hsb200::SlamProcessor*> procs(M > 0 ? M : 0);
  for (int s = 0; s < M; ++s) procs[s] = static_cast<hsb200::SlamProcessor*>(ps[s]);
  try {
    hsb200::SlamProcessor::covarianceMany(procs.data(), M, level, pose_offsets, poses_world, points_xy, scan_offsets,
                                          cov_map, cov_world);
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
int hsbp_covariance_many_subset(void* const* ps, int M, const int* members, int K, int level, const int* pose_offsets,
                                const float* poses_world, const float* points_xy, const int* scan_offsets, float* cov_map,
                                float* cov_world) {
  std::vector<hsb200::SlamProcessor*> procs(M > 0 ? M : 0);
  for (int s = 0; s < M; ++s) procs[s] = static_cast<hsb200::SlamProcessor*>(ps[s]);
  try {
    hsb200::SlamProcessor::covarianceMany(procs.data(), M, members, K, level, pose_offsets, poses_world, points_xy,
                                          scan_offsets, cov_map, cov_world);
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
int hsbp_best_hypothesis_many(void* const* ps, int M, int level, const int* pose_offsets, const float* poses_world,
                              const float* points_xy, const int* scan_offsets, float* best4, int* best_index,
                              float* likelihood) {
  std::vector<hsb200::SlamProcessor*> procs(M > 0 ? M : 0);
  for (int s = 0; s < M; ++s) procs[s] = static_cast<hsb200::SlamProcessor*>(ps[s]);
  try {
    hsb200::SlamProcessor::bestHypothesisMany(procs.data(), M, level, pose_offsets, poses_world, points_xy, scan_offsets,
                                              best4, best_index, likelihood);
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
int hsbp_best_hypothesis_many_subset(void* const* ps, int M, const int* members, int K, int level,
                                     const int* pose_offsets, const float* poses_world, const float* points_xy,
                                     const int* scan_offsets, float* best4, int* best_index, float* likelihood) {
  std::vector<hsb200::SlamProcessor*> procs(M > 0 ? M : 0);
  for (int s = 0; s < M; ++s) procs[s] = static_cast<hsb200::SlamProcessor*>(ps[s]);
  try {
    hsb200::SlamProcessor::bestHypothesisMany(procs.data(), M, members, K, level, pose_offsets, poses_world, points_xy,
                                              scan_offsets, best4, best_index, likelihood);
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
int hsbp_match_many(void* const* ps, int M, const int* hint_offsets, const float* hints_world, const float* points_xy,
                    const int* scan_offsets, float* out_poses_world, float* out_cov) {
  std::vector<hsb200::SlamProcessor*> procs(M > 0 ? M : 0);
  for (int s = 0; s < M; ++s) procs[s] = static_cast<hsb200::SlamProcessor*>(ps[s]);
  try {
    hsb200::SlamProcessor::matchMany(procs.data(), M, hint_offsets, hints_world, points_xy, scan_offsets,
                                     out_poses_world, out_cov);
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
int hsbp_match_many_subset(void* const* ps, int M, const int* members, int K, const int* hint_offsets,
                           const float* hints_world, const float* points_xy, const int* scan_offsets,
                           float* out_poses_world, float* out_cov) {
  std::vector<hsb200::SlamProcessor*> procs(M > 0 ? M : 0);
  for (int s = 0; s < M; ++s) procs[s] = static_cast<hsb200::SlamProcessor*>(ps[s]);
  try {
    hsb200::SlamProcessor::matchMany(procs.data(), M, members, K, hint_offsets, hints_world, points_xy, scan_offsets,
                                     out_poses_world, out_cov);
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
// matchManyRanges / matchManyCloud / matchManyProjected (kind 0 / 1 / 2), over ps[members[0..K)] or, with members
// NULL, all M processors; `in` is the ranges or the Point32 triples, transforms is ignored for ranges
int hsbp_match_many_scans(void* const* ps, int M, int kind, const int* members, int K, const int* hint_offsets,
                          const float* hints_world, const float* in, const int* scan_offsets, const double* transforms,
                          float* out_poses_world, float* out_cov, float* likelihood, float* best4, int* best_index,
                          int* kept) {
  std::vector<hsb200::SlamProcessor*> procs(M > 0 ? M : 0);
  for (int s = 0; s < M; ++s) procs[s] = static_cast<hsb200::SlamProcessor*>(ps[s]);
  using P = hsb200::SlamProcessor;
  try {
    if (kind == 0 && !members)
      P::matchManyRanges(procs.data(), M, hint_offsets, hints_world, in, scan_offsets, out_poses_world, out_cov,
                         likelihood, best4, best_index, kept);
    else if (kind == 0)
      P::matchManyRanges(procs.data(), M, members, K, hint_offsets, hints_world, in, scan_offsets, out_poses_world,
                         out_cov, likelihood, best4, best_index, kept);
    else if (kind == 1 && !members)
      P::matchManyCloud(procs.data(), M, hint_offsets, hints_world, in, scan_offsets, transforms, out_poses_world,
                        out_cov, likelihood, best4, best_index, kept);
    else if (kind == 1)
      P::matchManyCloud(procs.data(), M, members, K, hint_offsets, hints_world, in, scan_offsets, transforms,
                        out_poses_world, out_cov, likelihood, best4, best_index, kept);
    else if (!members)
      P::matchManyProjected(procs.data(), M, hint_offsets, hints_world, in, scan_offsets, transforms, out_poses_world,
                            out_cov, likelihood, best4, best_index, kept);
    else
      P::matchManyProjected(procs.data(), M, members, K, hint_offsets, hints_world, in, scan_offsets, transforms,
                            out_poses_world, out_cov, likelihood, best4, best_index, kept);
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
int hsbp_get_pose_and_cov(void* p, float out_pose[3], float out_cov[9]) {
  hsb200::SlamProcessor* s = static_cast<hsb200::SlamProcessor*>(p);
  const hsb200::Pose& q = s->getLastScanMatchPose();
  out_pose[0] = q.x;
  out_pose[1] = q.y;
  out_pose[2] = q.psi;
  std::memcpy(out_cov, s->getLastScanMatchCovariance(), 9 * sizeof(float));
  return 0;
}
int hsbp_reset(void* p) {
  try {
    static_cast<hsb200::SlamProcessor*>(p)->reset();
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
void hsbp_set_heterogeneous_groups(void* p, int on) {
  static_cast<hsb200::SlamProcessor*>(p)->setHeterogeneousGroups(on != 0);
}
int hsbp_reset_many(void* const* ps, int M, const int* members, int K) {
  std::vector<hsb200::SlamProcessor*> procs(M > 0 ? M : 0);
  for (int s = 0; s < M; ++s) procs[s] = static_cast<hsb200::SlamProcessor*>(ps[s]);
  try {
    hsb200::SlamProcessor::resetMany(procs.data(), M, members, K);
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
void hsbp_set_update_factors(void* p, float ffree, float focc) {
  static_cast<hsb200::SlamProcessor*>(p)->setUpdateFactorFree(ffree);
  static_cast<hsb200::SlamProcessor*>(p)->setUpdateFactorOccupied(focc);
}
void hsbp_set_map_update_thresholds(void* p, float dist, float ang) {
  static_cast<hsb200::SlamProcessor*>(p)->setMapUpdateMinDistDiff(dist);
  static_cast<hsb200::SlamProcessor*>(p)->setMapUpdateMinAngleDiff(ang);
}
int hsbp_get_grid_map(void* p, int level, float* out) {
  try {
    static_cast<hsb200::SlamProcessor*>(p)->getGridMap(level, out);
  } catch (const std::exception&) {
    return -1;
  }
  return 0;
}
int hsbp_pose_difference_larger_than(const float a[3], const float b[3], float dist, float ang) {
  return hsb200::SlamProcessor::poseDifferenceLargerThan(hsb200::Pose{a[0], a[1], a[2]}, hsb200::Pose{b[0], b[1], b[2]},
                                                         dist, ang)
             ? 1
             : 0;
}
void* hsbp_handle(void* p) { return static_cast<hsb200::SlamProcessor*>(p)->handle(); }
}
