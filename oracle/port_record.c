/* oracle/port_record.c — TEST INFRASTRUCTURE, not product code.
 *
 * The plain-C port (hs_oracle.c, compiled into this library as one translation unit) plus the per-evaluation record
 * of matchData in the layout of include/hector_slam_b200.h (hsb_match_data_record).  Built by oracle/record.mk into
 * oracle/_build/libhsoracle_record.so; every hso_ entry point of libhsoracle.so is exported here too.
 *
 * Per level, coarsest first: the world pose the level starts from, then for each evaluation H (9, row-major), dTr (3)
 * and the estimate after that evaluation's step (3, the level's map cells, angle not normalised).  An empty scan
 * writes the start poses and zeros. */
#include "hs_oracle.c"

/* ScanMatcher.h:54-190 matchData, as scan_matcher_match, with the level's part of the record written to rec */
static void scan_matcher_match_rec(level_t* L, const float begin_world[3], const container_t* dc, float cov[9],
                                   int max_iterations, float out_world[3], float* rec) {
  memcpy(rec, begin_world, 3 * sizeof(float));
  memset(rec + 3, 0, sizeof(float) * 15 * (size_t)(max_iterations + 1));
  if (dc->n != 0) { /* :68 */
    float estimate[3], H[9], dTr[3];
    map_coords_pose(L, begin_world, estimate); /* :70 */
    for (int e = 0; e <= max_iterations; ++e) { /* :74, then :94-97 */
      estimate_transformation_log_lh(L, estimate, dc, H, dTr);
      float* r = rec + 3 + 15 * e;
      memcpy(r, H, 9 * sizeof(float));
      memcpy(r + 9, dTr, 3 * sizeof(float));
      memcpy(r + 12, estimate, 3 * sizeof(float));
    }
    estimate[2] = normalize_angle(estimate[2]); /* :170 */
    for (int i = 0; i < 9; ++i) cov[i] = H[i];  /* :184 */
    world_coords_pose(L, estimate, out_world);  /* :186 */
    return;
  }
  out_world[0] = begin_world[0]; /* :189 */
  out_world[1] = begin_world[1];
  out_world[2] = begin_world[2];
}

/* maxIterations of a level as hsb_config::max_iterations gives it: 0 = the reference's 5 / 3, negative = 0 */
static int record_level_iterations(const int* iters, int index) {
  int mi = iters ? iters[index] : 0;
  if (mi == 0) mi = index == 0 ? 5 : 3; /* MapRepMultiMap.h:125,128 */
  return mi < 0 ? 0 : mi;
}

/* MapRepMultiMap.h:116-132 matchData (as maprep_match) with the record.  iters may be NULL (the reference's 5 / 3). */
void hso_match_record(void* hv, const float hint[3], const float* pts, int n, const float* origo, const int* iters,
                      float out_pose[3], float cov_inout[9], float* rec) {
  hso_t* h = (hso_t*)hv;
  container_t dc;
  wrap_container(&dc, pts, n, origo);
  float cov[9];
  for (int i = 0; i < 9; ++i) cov[i] = cov_inout ? cov_inout[i] : 0.0f;
  float tmp[3] = {hint[0], hint[1], hint[2]};
  for (int index = h->levels - 1; index >= 0; --index) {
    float r[3];
    const int mi = record_level_iterations(iters, index);
    if (index == 0) {
      scan_matcher_match_rec(&h->lv[0], tmp, &dc, cov, mi, r, rec);
    } else {
      container_set_from(&h->dc[index - 1], &dc, (float)(1.0 / pow(2.0, (double)index))); /* :127 */
      scan_matcher_match_rec(&h->lv[index], tmp, &h->dc[index - 1], cov, mi, r, rec);
    }
    rec += 3 + 15 * (mi + 1);
    tmp[0] = r[0];
    tmp[1] = r[1];
    tmp[2] = r[2];
  }
  memcpy(out_pose, tmp, sizeof(tmp));
  if (cov_inout) memcpy(cov_inout, cov, sizeof(cov));
}
