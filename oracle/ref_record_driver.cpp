// oracle/ref_record_driver.cpp — TEST INFRASTRUCTURE, not product code.
//
// ref_driver.cpp (compiled into this library as one translation unit, so every hsref_ entry point of libhsref.so is
// exported here too) plus hsref_match_record: what the reference's ScanMatcher::matchData (matcher/ScanMatcher.h:54-190)
// reports to a DrawInterface and a HectorDebugInfoInterface.  The two recording implementations below are written
// against the reference's abstract classes (util/DrawInterface.h, util/HectorDebugInfoInterface.h).  Built by
// oracle/record.mk into oracle/_ref/libhsref_record.so where the reference headers are present.
#include <algorithm>
#include <cmath>

#include "ref_driver.cpp"

namespace {

struct HookLog {
  std::vector<float> arrows;    // 3 per drawArrow
  std::vector<float> hessians;  // 9 per addHessianMatrix, row-major
  long points = 0;
};

class LogDraw : public DrawInterface {
 public:
  explicit LogDraw(HookLog* log) : log_(log) {}
  void drawPoint(const Eigen::Vector2f&) override { ++log_->points; }
  void drawArrow(const Eigen::Vector3f& p) override {
    for (int i = 0; i < 3; ++i) log_->arrows.push_back(p[i]);
  }
  void drawCovariance(const Eigen::Vector2f&, const Eigen::Matrix2f&) override {}
  void setScale(double) override {}
  void setColor(double, double, double, double) override {}
  void sendAndResetData() override {}

 private:
  HookLog* log_;
};

class LogDebug : public HectorDebugInfoInterface {
 public:
  explicit LogDebug(HookLog* log) : log_(log) {}
  void sendAndResetData() override {}
  void addHessianMatrix(const Eigen::Matrix3f& H) override {
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) log_->hessians.push_back(H(r, c));
  }
  void addPoseLikelihood(float) override {}

 private:
  HookLog* log_;
};

}  // namespace

extern "C" {

// MapRepMultiMap::matchData (slam_main/MapRepMultiMap.h:116-132) — its level loop and setFrom scaling, restated so that
// the iteration count of each level can be chosen — on ScanMatchers built with the recording hooks above.
// iters (may be NULL = 5 / 3): maxIterations per level, level 0 first, as hsb_config::max_iterations (0 = the
// default, negative = 0).  out_hooks receives per level, COARSEST FIRST, 3 + 12 * maxIterations floats: the start arrow,
// then per reported evaluation i = 1 .. maxIterations the Hessian (9, row-major) and the arrow (3); zeros where an empty
// scan reported nothing.  out_points[level] = drawPoint calls of that level.
void hsref_match_record(void* hv, const float hint[3], const float* pts, int n, const float* origo, const int* iters,
                        float out_pose[3], float cov_inout[9], float* out_hooks, int* out_points) {
  Handle* h = static_cast<Handle*>(hv);
  hectorslam::DataContainer dc, scaled;
  fill(dc, pts, n, origo);
  Eigen::Matrix3f cov;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) cov(r, c) = cov_inout ? cov_inout[3 * r + c] : 0.0f;
  Eigen::Vector3f tmp(hint[0], hint[1], hint[2]);
  float* o = out_hooks;
  for (int index = h->levels - 1; index >= 0; --index) {
    int mi = iters ? iters[index] : 0;
    if (mi == 0) mi = index == 0 ? 5 : 3;
    if (mi < 0) mi = 0;
    HookLog log;
    LogDraw draw(&log);
    LogDebug debug(&log);
    hectorslam::GridMap& g = h->proc->grid(index);
    hectorslam::OccGridMapUtilConfig<hectorslam::GridMap> util(&g);
    hectorslam::ScanMatcher<hectorslam::OccGridMapUtilConfig<hectorslam::GridMap> > matcher(&draw, &debug);
    std::streambuf* saved = std::cout.rdbuf(&g_nullbuf);  // the clamp note, ScanMatcher.h:211,214
    if (index == 0) {
      tmp = matcher.matchData(tmp, util, dc, cov, mi);
    } else {
      scaled.setFrom(dc, static_cast<float>(1.0 / pow(2.0, static_cast<double>(index))));
      tmp = matcher.matchData(tmp, util, scaled, cov, mi);
    }
    std::cout.rdbuf(saved);
    const int m = static_cast<int>(log.hessians.size() / 9);
    std::fill(o, o + 3 + 12 * mi, 0.0f);
    std::copy(log.arrows.begin(), log.arrows.begin() + 3, o);
    for (int i = 0; i < m && i < mi; ++i) {
      std::copy(log.hessians.begin() + 9 * i, log.hessians.begin() + 9 * i + 9, o + 3 + 12 * i);
      std::copy(log.arrows.begin() + 3 * (i + 1), log.arrows.begin() + 3 * (i + 2), o + 3 + 12 * i + 9);
    }
    if (out_points) out_points[index] = static_cast<int>(log.points);
    o += 3 + 12 * mi;
  }
  put_pose(tmp, out_pose);
  if (cov_inout) put_mat(cov, cov_inout);
}

}  // extern "C"
