/* oracle/hs_oracle.c — TEST INFRASTRUCTURE, not product code.
 *
 * Plain-C restatement ("port") of hector_mapping's scan-matching / map-writing path, one function
 * per reference function, each citing the reference file:line it follows (paths relative to
 * /root/reference/hector_mapping/include/hector_slam_lib/).  No Eigen: every small fixed-size
 * operation is written out in the evaluation order oracle/shim fixes for it (see shim/Eigen/Core
 * and shim/Eigen/Geometry), so that this file and oracle/_ref/libhsref.so (the unmodified
 * reference headers on the shim) agree BIT FOR BIT — tests/test_oracle_golden.py
 * asserts exactly that wherever /root/reference or the prebuilt _ref library is available.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's CPU-baseline / `--impl reference` legs may
 * build, load or call this file.  The product (hector_slam_b200/csrc) never does.
 *
 * Parity pinning: the reference ships no tests or golden vectors (SURVEY.md §4); this port is
 * pinned against the compiled reference itself and against tests/golden/ fixtures generated
 * from the compiled reference by oracle/gen_golden.py.
 *
 * Build: see oracle/Makefile (gcc -O2 -std=c99, no -ffast-math, no -march: no FMA contraction).
 */
#define _GNU_SOURCE
#include <float.h>
#include <math.h>
#include <pthread.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#define HSO_MAX_LEVELS 8

/* ---- tiny affine helper: the shim's Transform * vector -------------------------------------
 * out[r] = M[r][0]*v0 + (M[r][1]*v1 + M[r][2]*1)   (three products, halving sum a0+(a1+a2);
 * shim/Eigen/Geometry `Transform::operator*`).                                               */
typedef struct {
  float m[2][3];
} affine2;

static void affine2_apply(const affine2* t, float vx, float vy, float* ox, float* oy) {
  float p0 = t->m[0][0] * vx, p1 = t->m[0][1] * vy, p2 = t->m[0][2] * 1.0f;
  float q0 = t->m[1][0] * vx, q1 = t->m[1][1] * vy, q2 = t->m[1][2] * 1.0f;
  *ox = p0 + (p1 + p2);
  *oy = q0 + (q1 + q2);
}

/* Affine-mode inverse (shim `Transform::inverse`): 2x2 cofactor inverse of the linear part,
 * translation = (-Linv) * t with the 2-term product sum.  GridMapBase.h:279.                  */
static void affine2_inverse(const affine2* a, affine2* r) {
  float invdet = 1.0f / (a->m[0][0] * a->m[1][1] - a->m[1][0] * a->m[0][1]);
  float l00 = a->m[1][1] * invdet;
  float l10 = -a->m[1][0] * invdet;
  float l01 = -a->m[0][1] * invdet;
  float l11 = a->m[0][0] * invdet;
  r->m[0][0] = l00;
  r->m[0][1] = l01;
  r->m[1][0] = l10;
  r->m[1][1] = l11;
  r->m[0][2] = (-l00) * a->m[0][2] + (-l01) * a->m[1][2];
  r->m[1][2] = (-l10) * a->m[0][2] + (-l11) * a->m[1][2];
}

/* ---- one grid level: GridMapBase + OccGridMapBase + OccGridMapUtil(+cache) ------------------ */
typedef struct {
  int size_x, size_y;
  float cell_length;   /* MapDimensionProperties::cellLength */
  float scale_to_map;  /* GridMapBase.h:270 */
  float limit_x, limit_y; /* mapLimitsf = dims - 2, MapDimensionProperties.h:73 */
  affine2 map_T_world; /* GridMapBase.h:272 */
  affine2 world_T_map; /* GridMapBase.h:279 */
  float* logodds;      /* LogOddsCell::logOddsVal, GridMapLogOdds.h:99 */
  int* update_index;   /* LogOddsCell::updateIndex, GridMapLogOdds.h:100 */
  float* cache_val;    /* GridMapCacheArray: CachedMapElement::val   GridMapCacheArray.h:34-39 */
  int* cache_index;    /*                    CachedMapElement::index */
  int curr_cache_index;
  int curr_update_index, curr_mark_occ, curr_mark_free; /* OccGridMapBase.h:263-265 */
  int last_update_index;                                /* GridMapBase.h:398 */
  float log_odds_free, log_odds_occ;                    /* GridMapLogOdds.h:205-206 */
} level_t;

typedef struct {
  int n;
  float* xy; /* n x 2 */
  float origo[2];
  int cap;
} container_t;

typedef struct {
  int levels;
  float res;
  int sx, sy;
  float startx, starty;
  float ffree, focc;
  level_t lv[HSO_MAX_LEVELS];
  container_t dc[HSO_MAX_LEVELS]; /* MapRepMultiMap::dataContainers (index level-1), :171 */
  /* HectorSlamProcessor state, HectorSlamProcessor.h:145-150 */
  float last_map_update_pose[3];
  float last_scan_match_pose[3];
  float last_scan_match_cov[9];
  float min_dist, min_ang;
} hso_t;

/* GridMapLogOdds.h:197-201 probToLogOdds: odds = p/(1-p); log(odds) in float. */
static float prob_to_log_odds(float prob) {
  float odds = prob / (1.0f - prob);
  return logf(odds);
}

/* GridMapBase.h:265-280 setMapTransformation + MapDimensionProperties.h:70-74 */
static void level_init(level_t* L, float cell_length, int sx, int sy, float off_x, float off_y) {
  memset(L, 0, sizeof(*L));
  L->size_x = sx;
  L->size_y = sy;
  L->cell_length = cell_length;
  L->limit_x = (float)sx - 2.0f;
  L->limit_y = (float)sy - 2.0f;
  L->scale_to_map = 1.0f / cell_length;
  /* AlignedScaling2f(s,s) * Translation2f(off): linear diag(s,s), translation (s*off.x, s*off.y) */
  L->map_T_world.m[0][0] = L->scale_to_map;
  L->map_T_world.m[0][1] = 0.0f;
  L->map_T_world.m[1][0] = 0.0f;
  L->map_T_world.m[1][1] = L->scale_to_map;
  L->map_T_world.m[0][2] = L->scale_to_map * off_x;
  L->map_T_world.m[1][2] = L->scale_to_map * off_y;
  affine2_inverse(&L->map_T_world, &L->world_T_map);
  size_t n = (size_t)sx * (size_t)sy;
  L->logodds = (float*)calloc(n, sizeof(float));
  L->update_index = (int*)malloc(n * sizeof(int));
  L->cache_val = (float*)malloc(n * sizeof(float));
  L->cache_index = (int*)malloc(n * sizeof(int));
  for (size_t i = 0; i < n; ++i) {
    L->update_index[i] = -1; /* resetGridCell, GridMapLogOdds.h:89-93 */
    L->cache_index[i] = -1;  /* GridMapCacheArray.h:130-132 */
  }
  L->curr_cache_index = 0;  /* GridMapCacheArray.h:53 */
  L->curr_update_index = 0; /* OccGridMapBase.h:52 */
  L->curr_mark_occ = -1;
  L->curr_mark_free = -1;
  L->last_update_index = -1; /* GridMapBase.h:99 */
  L->log_odds_free = prob_to_log_odds(0.4f); /* GridMapLogOdds.h:117 */
  L->log_odds_occ = prob_to_log_odds(0.6f);  /* GridMapLogOdds.h:118 */
}

static void level_free(level_t* L) {
  free(L->logodds);
  free(L->update_index);
  free(L->cache_val);
  free(L->cache_index);
}

/* GridMapBase.h:71-82 clear(): every cell resetGridCell().  (currUpdateIndex is NOT reset.) */
static void level_clear(level_t* L) {
  size_t n = (size_t)L->size_x * (size_t)L->size_y;
  for (size_t i = 0; i < n; ++i) {
    L->logodds[i] = 0.0f;
    L->update_index[i] = -1;
  }
}

/* GridMapBase.h:235-239 getMapCoordsPose */
static void map_coords_pose(const level_t* L, const float w[3], float out[3]) {
  affine2_apply(&L->map_T_world, w[0], w[1], &out[0], &out[1]);
  out[2] = w[2];
}
/* GridMapBase.h:226-230 getWorldCoordsPose */
static void world_coords_pose(const level_t* L, const float m[3], float out[3]) {
  affine2_apply(&L->world_T_map, m[0], m[1], &out[0], &out[1]);
  out[2] = m[2];
}

/* GridMapLogOdds.h:163-166 getGridProbability via the cache GridMapCacheArray.h:80-102 */
static float cached_prob(level_t* L, int index) {
  if (L->cache_index[index] == L->curr_cache_index) return L->cache_val[index];
  float odds = expf(L->logodds[index]);
  float p = odds / (odds + 1.0f);
  L->cache_index[index] = L->curr_cache_index;
  L->cache_val[index] = p;
  return p;
}

/* OccGridMapUtil.h:287-347 interpMapValueWithDerivatives; bounds MapDimensionProperties.h:65-68 */
static void interp_with_derivs(level_t* L, float cx, float cy, float out[3]) {
  /* a NaN coordinate (a NaN pose or endpoint) passes the reference's four comparisons and indexes the grid with
   * (int)NaN; here it is out of the map, as on the device, so that a NaN step can be followed */
  if (!((cx >= 0.0f) && (cx <= L->limit_x) && (cy >= 0.0f) && (cy <= L->limit_y))) {
    out[0] = out[1] = out[2] = 0.0f;
    return;
  }
  int ix = (int)cx, iy = (int)cy;                 /* :295 */
  float fx = cx - (float)ix, fy = cy - (float)iy; /* :298 */
  int size_x = L->size_x;
  int index = iy * size_x + ix; /* :302 */
  float i0 = cached_prob(L, index);
  ++index;
  float i1 = cached_prob(L, index);
  index += size_x - 1;
  float i2 = cached_prob(L, index);
  ++index;
  float i3 = cached_prob(L, index);
  float dx1 = i0 - i1, dx2 = i2 - i3; /* :332-333 */
  float dy1 = i0 - i2, dy2 = i1 - i3; /* :335-336 */
  float x_inv = 1.0f - fx, y_inv = 1.0f - fy;
  out[0] = ((i0 * x_inv + i1 * fx) * y_inv) + ((i2 * x_inv + i3 * fx) * fy); /* :342-343 */
  out[1] = -((dx1 * x_inv) + (dx2 * fx));                                    /* :344 */
  out[2] = -((dy1 * y_inv) + (dy2 * fy));                                    /* :345 */
}

/* OccGridMapUtil.h:349-352 getTransformForState: Translation2f(x,y) * Rotation2Df(psi) */
static void transform_for_state(const float pose[3], affine2* t) {
  float s = sinf(pose[2]), c = cosf(pose[2]);
  t->m[0][0] = c;
  t->m[0][1] = -s;
  t->m[1][0] = s;
  t->m[1][1] = c;
  t->m[0][2] = pose[0];
  t->m[1][2] = pose[1];
}

/* OccGridMapUtil.h:64-104 getCompleteHessianDerivs.  H is 3x3 (row-major here; symmetric). */
static void complete_hessian_derivs(level_t* L, const float pose[3], const container_t* dc, float H[9], float dTr[3]) {
  affine2 T;
  transform_for_state(pose, &T);
  float sin_rot = sinf(pose[2]); /* :70 */
  float cos_rot = cosf(pose[2]); /* :71 */
  for (int i = 0; i < 9; ++i) H[i] = 0.0f;
  dTr[0] = dTr[1] = dTr[2] = 0.0f;
  for (int i = 0; i < dc->n; ++i) {
    float px = dc->xy[2 * i], py = dc->xy[2 * i + 1];
    float qx, qy, d[3];
    affine2_apply(&T, px, py, &qx, &qy); /* :80 */
    interp_with_derivs(L, qx, qy, d);
    float fun_val = 1.0f - d[0]; /* :82 */
    dTr[0] += d[1] * fun_val;
    dTr[1] += d[2] * fun_val;
    float rot_deriv = ((-sin_rot * px - cos_rot * py) * d[1] + (cos_rot * px - sin_rot * py) * d[2]); /* :87 */
    dTr[2] += rot_deriv * fun_val;
    H[0] += d[1] * d[1];           /* (0,0) :91 */
    H[4] += d[2] * d[2];           /* (1,1) */
    H[8] += rot_deriv * rot_deriv; /* (2,2) */
    H[1] += d[1] * d[2];           /* (0,1) :95 */
    H[2] += d[1] * rot_deriv;      /* (0,2) */
    H[5] += d[2] * rot_deriv;      /* (1,2) */
  }
  H[3] = H[1]; /* :100-102 */
  H[6] = H[2];
  H[7] = H[5];
}

/* Eigen fixed 3x3 inverse times vector, ScanMatcher.h:205 `H.inverse() * dTr` — shim/Eigen/Core
 * Matrix::inverse (cyclic cofactors, det = c00*m00 + (c10*m10 + c20*m20), inv(i,j)=cof(j,i)/det
 * via *invdet) followed by the coefficient-based product with the halving sum.                 */
static float cof3(const float m[9], int i, int j) {
  int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
  return m[3 * i1 + j1] * m[3 * i2 + j2] - m[3 * i1 + j2] * m[3 * i2 + j1];
}
static void inverse3_times(const float m[9], const float v[3], float out[3]) {
  float c0 = cof3(m, 0, 0), c1 = cof3(m, 1, 0), c2 = cof3(m, 2, 0);
  float p0 = c0 * m[0], p1 = c1 * m[3], p2 = c2 * m[6];
  float det = p0 + (p1 + p2);
  float invdet = 1.0f / det;
  float inv[9];
  inv[0] = c0 * invdet;
  inv[1] = c1 * invdet;
  inv[2] = c2 * invdet;
  inv[3] = cof3(m, 0, 1) * invdet;
  inv[4] = cof3(m, 1, 1) * invdet;
  inv[5] = cof3(m, 2, 1) * invdet;
  inv[6] = cof3(m, 0, 2) * invdet;
  inv[7] = cof3(m, 1, 2) * invdet;
  inv[8] = cof3(m, 2, 2) * invdet;
  for (int r = 0; r < 3; ++r) {
    float a0 = inv[3 * r] * v[0], a1 = inv[3 * r + 1] * v[1], a2 = inv[3 * r + 2] * v[2];
    out[r] = a0 + (a1 + a2);
  }
}

/* ScanMatcher.h:194-221 estimateTransformationLogLh (the stdout print at :211,214 is dropped) */
static int estimate_transformation_log_lh(level_t* L, float estimate[3], const container_t* dc, float H[9], float dTr[3]) {
  complete_hessian_derivs(L, estimate, dc, H, dTr);
  if ((H[0] != 0.0f) && (H[4] != 0.0f)) { /* :201 */
    float dir[3];
    inverse3_times(H, dTr, dir); /* :205 */
    if (dir[2] > 0.2f) {         /* :209-215 */
      dir[2] = 0.2f;
    } else if (dir[2] < -0.2f) {
      dir[2] = -0.2f;
    }
    estimate[0] += dir[0]; /* :217 -> :223-226 */
    estimate[1] += dir[1];
    estimate[2] += dir[2];
    return 1;
  }
  return 0;
}

/* UtilFunctions.h:37-49 normalize_angle (double arithmetic: M_PI is double) */
static float normalize_angle_pos(float angle) { return (float)fmod(fmod(angle, 2.0f * M_PI) + 2.0f * M_PI, 2.0f * M_PI); }
static float normalize_angle(float angle) {
  float a = normalize_angle_pos(angle);
  if (a > M_PI) {
    a -= 2.0f * M_PI;
  }
  return a;
}

/* ScanMatcher.h:54-190 matchData.  cov is written only when the scan is non-empty. */
static void scan_matcher_match(level_t* L, const float begin_world[3], const container_t* dc, float cov[9],
                               int max_iterations, float out_world[3]) {
  if (dc->n != 0) { /* :68 */
    float estimate[3], H[9], dTr[3];
    map_coords_pose(L, begin_world, estimate);              /* :70 */
    estimate_transformation_log_lh(L, estimate, dc, H, dTr); /* :74 */
    for (int i = 0; i < max_iterations; ++i) {               /* :94-97 */
      estimate_transformation_log_lh(L, estimate, dc, H, dTr);
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

static void container_reserve(container_t* c, int n) {
  if (n > c->cap) {
    c->xy = (float*)realloc(c->xy, sizeof(float) * 2 * (size_t)n);
    c->cap = n;
  }
}
/* DataPointContainer.h:46-58 setFrom */
static void container_set_from(container_t* c, const container_t* o, float factor) {
  container_reserve(c, o->n);
  c->origo[0] = o->origo[0] * factor;
  c->origo[1] = o->origo[1] * factor;
  c->n = o->n;
  for (int i = 0; i < 2 * o->n; ++i) c->xy[i] = o->xy[i] * factor;
}

/* MapRepMultiMap.h:116-132 matchData */
static void maprep_match(hso_t* h, const float begin_world[3], const container_t* dc, float cov[9], float out[3]) {
  float tmp[3] = {begin_world[0], begin_world[1], begin_world[2]};
  for (int index = h->levels - 1; index >= 0; --index) {
    float r[3];
    if (index == 0) {
      scan_matcher_match(&h->lv[0], tmp, dc, cov, 5, r); /* :125 */
    } else {
      container_set_from(&h->dc[index - 1], dc, (float)(1.0 / pow(2.0, (double)index))); /* :127 */
      scan_matcher_match(&h->lv[index], tmp, &h->dc[index - 1], cov, 3, r);               /* :128 */
    }
    tmp[0] = r[0];
    tmp[1] = r[1];
    tmp[2] = r[2];
  }
  out[0] = tmp[0];
  out[1] = tmp[1];
  out[2] = tmp[2];
}

/* OccGridMapBase.h:216-224 bresenhamCellFree; GridMapLogOdds.h:146-151 */
static void cell_free(level_t* L, unsigned int offset) {
  if (L->update_index[offset] < L->curr_mark_free) {
    L->logodds[offset] += L->log_odds_free;
    L->update_index[offset] = L->curr_mark_free;
  }
}
/* OccGridMapBase.h:226-241 bresenhamCellOcc; GridMapLogOdds.h:135-140,153-156 */
static void cell_occ(level_t* L, unsigned int offset) {
  if (L->update_index[offset] < L->curr_mark_occ) {
    if (L->update_index[offset] == L->curr_mark_free) {
      L->logodds[offset] -= L->log_odds_free;
    }
    if (L->logodds[offset] < 50.0f) {
      L->logodds[offset] += L->log_odds_occ;
    }
    L->update_index[offset] = L->curr_mark_occ;
  }
}
/* OccGridMapBase.h:243-260 bresenham2D */
static void bresenham2d(level_t* L, unsigned int abs_da, unsigned int abs_db, int error_b, int offset_a, int offset_b,
                        unsigned int offset) {
  cell_free(L, offset);
  unsigned int end = abs_da - 1;
  for (unsigned int i = 0; i < end; ++i) {
    offset += offset_a;
    error_b += abs_db;
    if ((unsigned int)error_b >= abs_da) {
      offset += offset_b;
      error_b -= abs_da;
    }
    cell_free(L, offset);
  }
}
static int sign_i(int x) { return x > 0 ? 1 : -1; } /* UtilFunctions.h:56-59 (sign(0) = -1) */

/* OccGridMapBase.h:170-214 updateLineBresenhami */
static void update_line(level_t* L, int x0, int y0, int x1, int y1) {
  if ((x0 < 0) || (x0 >= L->size_x) || (y0 < 0) || (y0 >= L->size_y)) return; /* :176 */
  if ((x1 < 0) || (x1 >= L->size_x) || (y1 < 0) || (y1 >= L->size_y)) return; /* :186 */
  int dx = x1 - x0, dy = y1 - y0;
  unsigned int abs_dx = abs(dx), abs_dy = abs(dy);
  int offset_dx = sign_i(dx);
  int offset_dy = sign_i(dy) * L->size_x;
  unsigned int start_offset = y0 * L->size_x + x0;
  if (abs_dx >= abs_dy) { /* :202 */
    int error_y = abs_dx / 2;
    bresenham2d(L, abs_dx, abs_dy, error_y, offset_dx, offset_dy, start_offset);
  } else {
    int error_x = abs_dy / 2;
    bresenham2d(L, abs_dy, abs_dx, error_x, offset_dy, offset_dx, start_offset);
  }
  unsigned int end_offset = y1 * L->size_x + x1; /* :211 */
  cell_occ(L, end_offset);
}

/* OccGridMapBase.h:121-168 updateByScan */
static void grid_update_by_scan(level_t* L, const container_t* dc, const float pose_world[3]) {
  L->curr_mark_free = L->curr_update_index + 1; /* :123-124 */
  L->curr_mark_occ = L->curr_update_index + 2;
  float map_pose[3];
  map_coords_pose(L, pose_world, map_pose); /* :127 */
  affine2 T;
  transform_for_state(map_pose, &T); /* :130-131 */
  float bx, by;
  affine2_apply(&T, dc->origo[0], dc->origo[1], &bx, &by); /* :134 */
  int bxi = (int)(bx + 0.5f), byi = (int)(by + 0.5f);      /* :137 */
  for (int i = 0; i < dc->n; ++i) {
    float ex, ey;
    affine2_apply(&T, dc->xy[2 * i], dc->xy[2 * i + 1], &ex, &ey); /* :148 */
    ex += 0.5f;                                                   /* :152 */
    ey += 0.5f;
    int exi = (int)ex, eyi = (int)ey;  /* :155 */
    if (bxi != exi || byi != eyi) {    /* :158 */
      update_line(L, bxi, byi, exi, eyi);
    }
  }
  L->last_update_index++;    /* :164 setUpdated */
  L->curr_update_index += 3; /* :167 */
}

/* UtilFunctions.h:73-92 poseDifferenceLargerThan */
static int pose_difference_larger_than(const float p1[3], const float p2[3], float dist_thresh, float ang_thresh) {
  float dx = p1[0] - p2[0], dy = p1[1] - p2[1];
  if (sqrtf(dx * dx + dy * dy) > dist_thresh) return 1;
  float angle_diff = p1[2] - p2[2];
  if (angle_diff > M_PI) {
    angle_diff -= M_PI * 2.0f;
  } else if (angle_diff < -M_PI) {
    angle_diff += M_PI * 2.0f;
  }
  if (fabsf(angle_diff) > ang_thresh) return 1;
  return 0;
}

/* the two util:: functions on their own, n at a time (oracle/pose32.py is tied to them) */
void hso_normalize_angle(const float* in, int n, float* out) {
  for (int i = 0; i < n; ++i) out[i] = normalize_angle(in[i]);
}
void hso_pose_difference_larger_than(const float* p1, const float* p2, const float* dist, const float* ang, int n,
                                     int* out) {
  for (int i = 0; i < n; ++i) out[i] = pose_difference_larger_than(p1 + 3 * i, p2 + 3 * i, dist[i], ang[i]);
}
/* the Gauss-Newton step's `H.inverse() * dTr` on its own, n at a time: m n x 9 (row-major 3x3), v n x 3, out n x 3 */
void hso_inverse3_times(const float* m, const float* v, int n, float* out) {
  for (int i = 0; i < n; ++i) inverse3_times(m + 9 * i, v + 3 * i, out + 3 * i);
}

/* MapRepMultiMap.h:134-147 updateByScan (coarse levels use the containers left by matchData) */
static void maprep_update_by_scan(hso_t* h, const container_t* dc, const float pose[3]) {
  for (int i = 0; i < h->levels; ++i) {
    if (i == 0)
      grid_update_by_scan(&h->lv[0], dc, pose);
    else
      grid_update_by_scan(&h->lv[i], &h->dc[i - 1], pose);
  }
}
/* MapRepMultiMap.h:107-114 onMapUpdated -> GridMapCacheArray::resetCache :69-72 */
static void maprep_on_map_updated(hso_t* h) {
  for (int i = 0; i < h->levels; ++i) h->lv[i].curr_cache_index++;
}

static void wrap_container(container_t* c, const float* pts, int n, const float* origo) {
  c->n = n;
  c->xy = (float*)pts;
  c->cap = 0;
  c->origo[0] = origo ? origo[0] : 0.0f;
  c->origo[1] = origo ? origo[1] : 0.0f;
}

/* ============================ exported entry points (same as hsref_*) ======================== */

void* hso_create(float res, int sx, int sy, float startx, float starty, int levels) {
  hso_t* h = (hso_t*)calloc(1, sizeof(hso_t));
  h->levels = levels;
  h->res = res;
  h->sx = sx;
  h->sy = sy;
  h->startx = startx;
  h->starty = starty;
  h->ffree = 0.4f;
  h->focc = 0.6f;
  /* MapRepMultiMap.h:48-72 */
  float total_x = res * (float)sx;
  float mid_x = total_x * startx;
  float total_y = res * (float)sy;
  float mid_y = total_y * starty;
  float r = res;
  int dx = sx, dy = sy;
  for (int i = 0; i < levels; ++i) {
    level_init(&h->lv[i], r, dx, dy, mid_x, mid_y);
    dx /= 2; /* :67 */
    dy /= 2;
    r *= 2.0f; /* :68 */
  }
  /* HectorSlamProcessor.h:60-63 */
  h->last_map_update_pose[0] = h->last_map_update_pose[1] = h->last_map_update_pose[2] = FLT_MAX;
  h->min_dist = 0.4f * 1.0f;
  h->min_ang = 0.13f * 1.0f;
  return h;
}

void hso_destroy(void* hv) {
  hso_t* h = (hso_t*)hv;
  for (int i = 0; i < h->levels; ++i) level_free(&h->lv[i]);
  for (int i = 0; i < HSO_MAX_LEVELS; ++i) free(h->dc[i].xy);
  free(h);
}

/* HectorSlamProcessor.h:115-124 reset -> MapRepMultiMap::reset :83-90 -> MapProcContainer::reset :67-71 */
void hso_reset(void* hv) {
  hso_t* h = (hso_t*)hv;
  h->last_map_update_pose[0] = h->last_map_update_pose[1] = h->last_map_update_pose[2] = FLT_MAX;
  h->last_scan_match_pose[0] = h->last_scan_match_pose[1] = h->last_scan_match_pose[2] = 0.0f;
  for (int i = 0; i < h->levels; ++i) {
    level_clear(&h->lv[i]);
    h->lv[i].curr_cache_index++;
  }
}

void hso_set_update_factors(void* hv, float ffree, float focc) {
  hso_t* h = (hso_t*)hv;
  h->ffree = ffree;
  h->focc = focc;
  for (int i = 0; i < h->levels; ++i) { /* MapRepMultiMap.h:149-167 */
    h->lv[i].log_odds_free = prob_to_log_odds(ffree);
    h->lv[i].log_odds_occ = prob_to_log_odds(focc);
  }
}

void hso_set_map_update_thresholds(void* hv, float dist, float ang) {
  hso_t* h = (hso_t*)hv;
  h->min_dist = dist;
  h->min_ang = ang;
}

int hso_levels(void* hv) { return ((hso_t*)hv)->levels; }
int hso_size_x(void* hv, int level) { return ((hso_t*)hv)->lv[level].size_x; }
int hso_size_y(void* hv, int level) { return ((hso_t*)hv)->lv[level].size_y; }
float hso_cell_length(void* hv, int level) { return ((hso_t*)hv)->lv[level].cell_length; }
float hso_scale_to_map(void* hv) { return ((hso_t*)hv)->lv[0].scale_to_map; }

void hso_map_coords_pose(void* hv, int level, const float w[3], float out[3]) {
  map_coords_pose(&((hso_t*)hv)->lv[level], w, out);
}
void hso_world_coords_pose(void* hv, int level, const float m[3], float out[3]) {
  world_coords_pose(&((hso_t*)hv)->lv[level], m, out);
}

/* HectorSlamProcessor.h:71-113 update */
void hso_update(void* hv, const float* pts, int n, const float* origo, const float hint[3], int map_without_matching,
                float out_pose[3], float out_cov[9]) {
  hso_t* h = (hso_t*)hv;
  container_t dc;
  wrap_container(&dc, pts, n, origo);
  float new_pose[3];
  if (!map_without_matching) {
    maprep_match(h, hint, &dc, h->last_scan_match_cov, new_pose); /* :78 */
  } else {
    new_pose[0] = hint[0];
    new_pose[1] = hint[1];
    new_pose[2] = hint[2];
  }
  memcpy(h->last_scan_match_pose, new_pose, sizeof(new_pose)); /* :83 */
  if (pose_difference_larger_than(new_pose, h->last_map_update_pose, h->min_dist, h->min_ang) || map_without_matching) {
    maprep_update_by_scan(h, &dc, new_pose); /* :91 */
    maprep_on_map_updated(h);                /* :93 */
    memcpy(h->last_map_update_pose, new_pose, sizeof(new_pose));
  }
  memcpy(out_pose, new_pose, sizeof(new_pose));
  if (out_cov) memcpy(out_cov, h->last_scan_match_cov, sizeof(h->last_scan_match_cov));
}

void hso_match(void* hv, const float hint[3], const float* pts, int n, const float* origo, float out_pose[3],
               float cov_inout[9]) {
  hso_t* h = (hso_t*)hv;
  container_t dc;
  wrap_container(&dc, pts, n, origo);
  float cov[9];
  for (int i = 0; i < 9; ++i) cov[i] = cov_inout ? cov_inout[i] : 0.0f;
  maprep_match(h, hint, &dc, cov, out_pose);
  if (cov_inout) memcpy(cov_inout, cov, sizeof(cov));
}

void hso_update_by_scan(void* hv, const float* pts, int n, const float* origo, const float pose[3]) {
  hso_t* h = (hso_t*)hv;
  container_t dc;
  wrap_container(&dc, pts, n, origo);
  maprep_update_by_scan(h, &dc, pose);
}

void hso_on_map_updated(void* hv) { maprep_on_map_updated((hso_t*)hv); }

void hso_get_logodds(void* hv, int level, float* out) {
  level_t* L = &((hso_t*)hv)->lv[level];
  memcpy(out, L->logodds, sizeof(float) * (size_t)L->size_x * L->size_y);
}
void hso_set_logodds(void* hv, int level, const float* in) {
  hso_t* h = (hso_t*)hv;
  level_t* L = &h->lv[level];
  memcpy(L->logodds, in, sizeof(float) * (size_t)L->size_x * L->size_y);
  maprep_on_map_updated(h);
}
void hso_get_prob(void* hv, int level, float* out) {
  level_t* L = &((hso_t*)hv)->lv[level];
  size_t n = (size_t)L->size_x * L->size_y;
  for (size_t i = 0; i < n; ++i) {
    float odds = expf(L->logodds[i]); /* GridMapLogOdds.h:165-166 */
    out[i] = odds / (odds + 1.0f);
  }
}
void hso_get_logodds_increments(void* hv, float out[2]) {
  hso_t* h = (hso_t*)hv;
  out[0] = 0.0f + h->lv[0].log_odds_free;
  out[1] = 0.0f + h->lv[0].log_odds_occ;
}

void hso_hessian_derivs(void* hv, int level, const float pose_map[3], const float* pts_level, int n, float H[9],
                        float dTr[3]) {
  hso_t* h = (hso_t*)hv;
  container_t dc;
  wrap_container(&dc, pts_level, n, 0);
  complete_hessian_derivs(&h->lv[level], pose_map, &dc, H, dTr);
}

void hso_match_level(void* hv, int level, const float hint_world[3], const float* pts_level, int n, int max_iterations,
                     float out_pose[3], float out_cov[9]) {
  hso_t* h = (hso_t*)hv;
  container_t dc;
  wrap_container(&dc, pts_level, n, 0);
  float cov[9] = {0};
  scan_matcher_match(&h->lv[level], hint_world, &dc, cov, max_iterations, out_pose);
  if (out_cov) memcpy(out_cov, cov, sizeof(cov));
}

void hso_update_level(void* hv, int level, const float* pts_level, int n, const float* origo_level,
                      const float pose_world[3]) {
  hso_t* h = (hso_t*)hv;
  container_t dc;
  wrap_container(&dc, pts_level, n, origo_level);
  grid_update_by_scan(&h->lv[level], &dc, pose_world);
  maprep_on_map_updated(h);
}

/* OccGridMapUtil.h:233-285 interpMapValue */
static float interp_value(level_t* L, float cx, float cy) {
  if (!((cx >= 0.0f) && (cx <= L->limit_x) && (cy >= 0.0f) && (cy <= L->limit_y))) return 0.0f;   /* NaN: out */
  int ix = (int)cx, iy = (int)cy;
  float fx = cx - (float)ix, fy = cy - (float)iy;
  int size_x = L->size_x;
  int index = iy * size_x + ix;
  float i0 = cached_prob(L, index);
  ++index;
  float i1 = cached_prob(L, index);
  index += size_x - 1;
  float i2 = cached_prob(L, index);
  ++index;
  float i3 = cached_prob(L, index);
  float x_inv = 1.0f - fx, y_inv = 1.0f - fy;
  return ((i0 * x_inv + i1 * fx) * y_inv) + ((i2 * x_inv + i3 * fx) * fy);
}

/* OccGridMapUtil.h:189-221 getLikelihoodForState = getLikelihoodForResidual(getResidualForState) */
float hso_likelihood(void* hv, int level, const float pose_map[3], const float* pts_level, int n) {
  hso_t* h = (hso_t*)hv;
  level_t* L = &h->lv[level];
  affine2 T;
  transform_for_state(pose_map, &T);
  float residual = 0.0f;
  for (int i = 0; i < n; ++i) {
    float qx, qy;
    affine2_apply(&T, pts_level[2 * i], pts_level[2 * i + 1], &qx, &qy);
    float funval = 1.0f - interp_value(L, qx, qy); /* :216 */
    residual += funval;
  }
  float sizef = (float)n; /* :205-206 */
  return 1 - (residual / sizef);
}

/* OccGridMapUtil::getCovarianceForPose — map/OccGridMapUtil.h:106-160 — and getCovMatrixWorldCoords — :162-187.
 * Seven sigma points (+-1.5 cells, +-0.05 rad, the pose itself), their likelihoods, the likelihood-weighted mean and
 * the weighted sum of outer products.  Fixed-size Eigen operations in the shim's order: likelihoods.sum() of 7 by
 * recursive halving = (l0 + (l1 + l2)) + ((l3 + l4) + (l5 + l6)); vector * scalar and matrix += element-wise. */
void hso_covariance_for_pose(void* hv, int level, const float pose_map[3], const float* pts_level, int n, float out_map[9],
                             float out_world[9]) {
  hso_t* h = (hso_t*)hv;
  const float dtx = 1.5f, dty = 1.5f, dang = 0.05f; /* :109-111 */
  const float x = pose_map[0], y = pose_map[1], ang = pose_map[2];
  float sp[7][3] = {{x + dtx, y, ang}, {x - dtx, y, ang}, {x, y + dty, ang}, {x, y - dty, ang},
                    {x, y, ang + dang}, {x, y, ang - dang}, {x, y, ang}}; /* :119-125 */
  float lh[7];
  for (int i = 0; i < 7; ++i) lh[i] = hso_likelihood(hv, level, sp[i], pts_level, n); /* :129-135 */
  float sum = (lh[0] + (lh[1] + lh[2])) + ((lh[3] + lh[4]) + (lh[5] + lh[6]));
  float inv = 1 / sum; /* :137 */
  float mean[3] = {0.0f, 0.0f, 0.0f};
  for (int i = 0; i < 7; ++i)
    for (int k = 0; k < 3; ++k) mean[k] += sp[i][k] * lh[i]; /* :144 */
  for (int k = 0; k < 3; ++k) mean[k] *= inv;                 /* :147 */
  float cov[9] = {0};
  for (int i = 0; i < 7; ++i) { /* :151-154 */
    float d[3] = {sp[i][0] - mean[0], sp[i][1] - mean[1], sp[i][2] - mean[2]};
    float wgt = lh[i] * inv;
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) {
        float outer = d[r] * d[c];
        cov[3 * r + c] += wgt * outer;
      }
  }
  memcpy(out_map, cov, sizeof(cov));
  float st = h->lv[level].cell_length, st2 = st * st; /* :169-170 util::sqr */
  out_world[0] = cov[0] * st2;                        /* :172 */
  out_world[4] = cov[4] * st2;
  out_world[3] = cov[3] * st2;                        /* (1,0) :175 */
  out_world[1] = out_world[3];
  out_world[6] = cov[6] * st;                         /* (2,0) :178 */
  out_world[2] = out_world[6];
  out_world[7] = cov[7] * st;                         /* (2,1) :181 */
  out_world[5] = out_world[7];
  out_world[8] = cov[8];                              /* :184 */
}

/* hector_map_tools DistanceMeasurementProvider::checkOccupancyBresenhami + bresenham2D
 * (/root/reference/hector_map_tools/include/hector_map_tools/HectorMapTools.h:133-216), on a level's
 * log-odds plane: a cell's nav_msgs value is 100 iff its log-odds is > 0 (HectorMappingRos.cpp:462-465).
 * (The header needs nav_msgs / ROS and cannot be compiled here: pinned by restatement only.) */
float hso_raycast(void* hv, int level, int x0, int y0, int x1, int y1, int hit[2]) {
  level_t* L = &((hso_t*)hv)->lv[level];
  int size_x = L->size_x, size_y = L->size_y;
  hit[0] = hit[1] = -1;
  if ((x0 < 0) || (x0 >= size_x) || (y0 < 0) || (y0 >= size_y)) return -1.0f; /* :141 */
  if ((x1 < 0) || (x1 >= size_x) || (y1 < 0) || (y1 >= size_y)) return -1.0f; /* :152 */
  int dx = x1 - x0, dy = y1 - y0;
  unsigned int abs_dx = abs(dx), abs_dy = abs(dy);
  int offset_dx = dx > 0 ? 1 : -1;
  int offset_dy = (dy > 0 ? 1 : -1) * size_x;
  unsigned int offset = y0 * size_x + x0;
  unsigned int abs_da, abs_db;
  int error_b, offset_a, offset_b;
  if (abs_dx >= abs_dy) { /* :170 */
    abs_da = abs_dx; abs_db = abs_dy; error_b = abs_dx / 2; offset_a = offset_dx; offset_b = offset_dy;
  } else {
    abs_da = abs_dy; abs_db = abs_dx; error_b = abs_dy / 2; offset_a = offset_dy; offset_b = offset_dx;
  }
  unsigned int end = abs_da < 5000u ? abs_da : 5000u; /* :203 std::min(max_length, abs_da) */
  int end_offset = -1;
  for (unsigned int i = 0; i < end; ++i) { /* :207-216 */
    if (L->logodds[offset] > 0.0f) {
      end_offset = (int)offset;
      break;
    }
    offset += offset_a;
    error_b += abs_db;
    if ((unsigned int)error_b >= abs_da) {
      offset += offset_b;
      error_b -= abs_da;
    }
  }
  if (end_offset != -1) {
    int ex = end_offset % size_x, ey = end_offset / size_x; /* :182 */
    float fx = (float)(x0 - ex), fy = (float)(y0 - ey);
    int dist_map = (int)sqrtf(fx * fx + fy * fy); /* :184 */
    hit[0] = ex;
    hit[1] = ey;
    return (float)dist_map;
  }
  return -1.0f;
}

/* The nav_msgs/OccupancyGrid origin of a level as HectorMappingRos::setServiceGetMapData derives it
 * (hector_mapping/src/HectorMappingRos.cpp:546-550): getWorldCoords(0, 0) - cellLength * 0.5 in float. */
void hso_map_origin(void* hv, int level, float out[2]) {
  level_t* L = &((hso_t*)hv)->lv[level];
  float wx, wy;
  affine2_apply(&L->world_T_map, 0.0f, 0.0f, &wx, &wy);
  float half = L->cell_length * 0.5f;
  out[0] = wx - half;
  out[1] = wy - half;
}

/* DistanceMeasurementProvider::getDist — hector_map_tools/HectorMapTools.h:133-147 with CoordinateTransformer<float>
 * (:41-116): getC2Coords = (world - origo) * inv_scale then cast<int> (truncation, :136-137), the ray cast above,
 * getC1Coords = origo + cells * scale for the hit (:141), getC1Scale = scale * dist (:144).  inv_scale = 1.0f /
 * resolution (:64).  *found = 0 when nothing was hit (the value returned is then scale * -1). */
float hso_get_dist(void* hv, int level, const float begin_world[2], const float end_world[2], float hit_world[2], int* found) {
  level_t* L = &((hso_t*)hv)->lv[level];
  float origo[2];
  hso_map_origin(hv, level, origo);
  float scale = L->cell_length, inv_scale = 1.0f / L->cell_length;
  int bx = (int)((begin_world[0] - origo[0]) * inv_scale), by = (int)((begin_world[1] - origo[1]) * inv_scale);
  int ex = (int)((end_world[0] - origo[0]) * inv_scale), ey = (int)((end_world[1] - origo[1]) * inv_scale);
  int hit[2];
  float dist = hso_raycast(hv, level, bx, by, ex, ey, hit);
  *found = dist >= 0.0f;
  hit_world[0] = hit_world[1] = 0.0f;
  if (*found) {
    hit_world[0] = origo[0] + (float)hit[0] * scale;
    hit_world[1] = origo[1] + (float)hit[1] * scale;
  }
  return scale * dist;
}

/* HectorMappingRos::rosLaserScanToDataContainer — hector_mapping/src/HectorMappingRos.cpp:483-507.
 * (That file needs ROS and cannot be compiled here, so this row of the path is pinned by this
 * restatement only.)  `cos(angle)` / `sin(angle)` are called on a float with the <cmath> overloads
 * visible, i.e. cosf / sinf.  out_xy has room for n_beams x 2; returns the number of endpoints. */
int hso_scan_to_points(const float* ranges, int n_beams, float angle_min, float angle_increment, float range_min,
                       float range_max, float scale_to_map, float* out_xy) {
  float angle = angle_min;                         /* :487 */
  float max_range_for_container = range_max - 0.1f; /* :493 */
  int n = 0;
  for (int i = 0; i < n_beams; ++i) {
    float dist = ranges[i];
    if ((dist > range_min) && (dist < max_range_for_container)) { /* :499 */
      dist *= scale_to_map;                                       /* :501 */
      out_xy[2 * n] = cosf(angle) * dist;
      out_xy[2 * n + 1] = sinf(angle) * dist;
      ++n;
    }
    angle += angle_increment; /* :505 */
  }
  return n;
}

/* HectorMappingRos::rosPointCloudToDataContainer — hector_mapping/src/HectorMappingRos.cpp:509-542: the node's
 * DEFAULT input path (use_tf_scan_transformation = true, :82; called at :283).  Point32 fields are float, tf is
 * double (tfScalar): `laserTransform * tf::Vector3(x, y, z)` is row.dot(v) + origin per row with
 * dot = r0*x + r1*y + r2*z (tf/LinearMath/Transform.h, Vector3.h), narrowed to float by Eigen::Vector2f(double,
 * double) (:538) and by the `float pointPosLaserFrameZ` declaration (:534).  transform: 12 doubles, rows of [R | t].
 * out_xy has room for n x 2; returns the number of endpoints kept, origo (:516-517) in out_origo. */
int hso_cloud_to_points(const float* xyz, int n, const double* T, float sqr_min_dist, float sqr_max_dist, float z_min,
                        float z_max, float scale_to_map, float* out_xy, float* out_origo) {
  const double lx = T[3], ly = T[7], lz = T[11]; /* laserPos = getOrigin()  :515 */
  if (out_origo) {                               /* :517 Vector2f(laserPos.x(), laserPos.y()) * scaleToMap */
    out_origo[0] = (float)lx * scale_to_map;
    out_origo[1] = (float)ly * scale_to_map;
  }
  int kept = 0;
  for (int i = 0; i < n; ++i) {
    const float x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    float dist_sqr = x * x + y * y;                                   /* :524 */
    if ((dist_sqr > sqr_min_dist) && (dist_sqr < sqr_max_dist)) {     /* :526 */
      if ((x < 0.0f) && (dist_sqr < 0.50f)) continue;                 /* :528-530 */
      const double vx = (double)x, vy = (double)y, vz = (double)z;
      const double bx = (T[0] * vx + T[1] * vy + T[2] * vz) + lx;     /* :532 */
      const double by = (T[4] * vx + T[5] * vy + T[6] * vz) + ly;
      const double bz = (T[8] * vx + T[9] * vy + T[10] * vz) + lz;
      float z_laser = (float)(bz - lz);                               /* :534 */
      if (z_laser > z_min && z_laser < z_max) {                       /* :536 */
        out_xy[2 * kept] = (float)bx * scale_to_map;                  /* :538 */
        out_xy[2 * kept + 1] = (float)by * scale_to_map;
        ++kept;
      }
    }
  }
  return kept;
}

/* ---- batch of independent matches (timing harness; same contract as hsref_match_batch) ------ */
typedef struct {
  hso_t* master;
  int B, t, nthreads;
  const float* hints;
  const float* pts;
  const int* offsets;
  float* out_poses;
  float* out_cov;
  double secs;
  pthread_barrier_t* bar;
} worker_t;

static double now_s(void) {
  struct timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec;
}

static void run_range(hso_t* h, const worker_t* w, int b0, int b1) {
  for (int b = b0; b < b1; ++b) {
    container_t dc;
    wrap_container(&dc, w->pts + 2 * (size_t)w->offsets[b], w->offsets[b + 1] - w->offsets[b], 0);
    float cov[9] = {0};
    maprep_match(h, w->hints + 3 * b, &dc, cov, w->out_poses + 3 * b);
    if (w->out_cov) memcpy(w->out_cov + 9 * b, cov, sizeof(cov));
  }
}

static void* worker_main(void* arg) {
  worker_t* w = (worker_t*)arg;
  hso_t* m = w->master;
  /* private instance (own probability cache and scaled containers), planes cloned untimed */
  hso_t* h = (hso_t*)hso_create(m->res, m->sx, m->sy, m->startx, m->starty, m->levels);
  for (int l = 0; l < m->levels; ++l)
    memcpy(h->lv[l].logodds, m->lv[l].logodds, sizeof(float) * (size_t)m->lv[l].size_x * m->lv[l].size_y);
  int b0 = (int)((long long)w->B * w->t / w->nthreads), b1 = (int)((long long)w->B * (w->t + 1) / w->nthreads);
  run_range(h, w, b0, b1); /* untimed warm pass: private planes touched, probability cache filled */
  pthread_barrier_wait(w->bar);
  double t0 = now_s();
  run_range(h, w, b0, b1);
  w->secs = now_s() - t0;
  hso_destroy(h);
  return 0;
}

double hso_match_batch(void* hv, int B, const float* hints, const float* pts, const int* offsets, float* out_poses,
                       float* out_cov, int nthreads) {
  hso_t* h = (hso_t*)hv;
  worker_t base;
  memset(&base, 0, sizeof(base));
  base.master = h;
  base.B = B;
  base.hints = hints;
  base.pts = pts;
  base.offsets = offsets;
  base.out_poses = out_poses;
  base.out_cov = out_cov;
  if (nthreads <= 1) {
    double t0 = now_s();
    run_range(h, &base, 0, B);
    return now_s() - t0;
  }
  pthread_barrier_t bar;
  pthread_barrier_init(&bar, 0, (unsigned)nthreads);
  worker_t* ws = (worker_t*)calloc((size_t)nthreads, sizeof(worker_t));
  pthread_t* th = (pthread_t*)calloc((size_t)nthreads, sizeof(pthread_t));
  for (int t = 0; t < nthreads; ++t) {
    ws[t] = base;
    ws[t].t = t;
    ws[t].nthreads = nthreads;
    ws[t].bar = &bar;
    pthread_create(&th[t], 0, worker_main, &ws[t]);
  }
  double mx = 0.0;
  for (int t = 0; t < nthreads; ++t) {
    pthread_join(th[t], 0);
    if (ws[t].secs > mx) mx = ws[t].secs;
  }
  pthread_barrier_destroy(&bar);
  free(ws);
  free(th);
  return mx;
}
