// oracle/dropin_hooks_check.cpp — TEST INFRASTRUCTURE.
//
// Runs the UNMODIFIED reference façade (HectorSlamProcessor::update, slam_main/HectorSlamProcessor.h:71) with a
// recording DrawInterface and HectorDebugInfoInterface twice over the same synthetic scan sequence: once on the
// reference's own CPU map representation (MapRepMultiMap, whose ScanMatchers call the hooks themselves) and once with
// hector_slam_b200/host/MapRepB200.h plugged in (which replays the matcher's calls from the device's per-evaluation
// record).  Both hook call sequences must agree: the same methods in the same order and numbers, setScale / setColor
// arguments exactly, arrows within 1e-4 m / rad, drawn points within the bound the pose difference of their scan
// implies (|dp| + r |dpsi|), and the largest relative difference of the forwarded Hessians is printed.
//
// Built by oracle/record.mk into oracle/_ref/dropin_hooks_check (needs the reference headers at build time); run by
// tests/test_gpu_dropin_hooks.py.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <iostream>
#include <random>
#include <streambuf>
#include <vector>

#include "MapRepB200.h"

namespace {

class NullBuf : public std::streambuf {
 protected:
  int overflow(int c) override { return c; }
};

enum Kind { POINT, ARROW, COVARIANCE, SCALE, COLOR, DRAW_SEND, HESSIAN, LIKELIHOOD, DEBUG_SEND };
const char* kKindName[] = {"drawPoint", "drawArrow", "drawCovariance", "setScale", "setColor",
                           "draw.sendAndResetData", "addHessianMatrix", "addPoseLikelihood", "debug.sendAndResetData"};

struct Call {
  Kind kind;
  double v[9];
};

// One log shared by both hooks, so that the interleaving of draw and debug calls is compared too.
struct Log {
  std::vector<Call> calls;
  void add(Kind k, std::initializer_list<double> vals) {
    Call c;
    c.kind = k;
    std::fill(c.v, c.v + 9, 0.0);
    int i = 0;
    for (double x : vals) c.v[i++] = x;
    calls.push_back(c);
  }
};

class RecordingDraw : public DrawInterface {
 public:
  explicit RecordingDraw(Log* log) : log_(log) {}
  virtual void drawPoint(const Eigen::Vector2f& p) { log_->add(POINT, {p[0], p[1]}); }
  virtual void drawArrow(const Eigen::Vector3f& p) { log_->add(ARROW, {p[0], p[1], p[2]}); }
  virtual void drawCovariance(const Eigen::Vector2f& m, const Eigen::Matrix2f& c) {
    log_->add(COVARIANCE, {m[0], m[1], c(0, 0), c(0, 1), c(1, 0), c(1, 1)});
  }
  virtual void setScale(double s) { log_->add(SCALE, {s}); }
  virtual void setColor(double r, double g, double b, double a = 1.0) { log_->add(COLOR, {r, g, b, a}); }
  virtual void sendAndResetData() { log_->add(DRAW_SEND, {}); }

 private:
  Log* log_;
};

class RecordingDebug : public HectorDebugInfoInterface {
 public:
  explicit RecordingDebug(Log* log) : log_(log) {}
  virtual void sendAndResetData() { log_->add(DEBUG_SEND, {}); }
  virtual void addHessianMatrix(const Eigen::Matrix3f& H) {
    log_->add(HESSIAN, {H(0, 0), H(0, 1), H(0, 2), H(1, 0), H(1, 1), H(1, 2), H(2, 0), H(2, 1), H(2, 2)});
  }
  virtual void addPoseLikelihood(float lh) { log_->add(LIKELIHOOD, {lh}); }

 private:
  Log* log_;
};

// 16 m x 10 m room with three pillars, analytic ray casting (the world of dropin_check.cpp).
struct World {
  double hx = 8.0, hy = 5.0;
  double pil[3][3] = {{-3.0, 1.5, 0.8}, {2.5, -2.0, 0.6}, {4.5, 2.5, 1.0}};
  double cast(double x, double y, double a) const {
    double dx = std::cos(a), dy = std::sin(a), t = 1e9;
    if (dx > 0) t = std::min(t, (hx - x) / dx);
    if (dx < 0) t = std::min(t, (-hx - x) / dx);
    if (dy > 0) t = std::min(t, (hy - y) / dy);
    if (dy < 0) t = std::min(t, (-hy - y) / dy);
    for (int k = 0; k < 3; ++k) {
      double ox = x - pil[k][0], oy = y - pil[k][1];
      double b = ox * dx + oy * dy, c = ox * ox + oy * oy - pil[k][2] * pil[k][2];
      double disc = b * b - c;
      if (disc >= 0) {
        double t0 = -b - std::sqrt(disc);
        if (t0 > 1e-9) t = std::min(t, t0);
      }
    }
    return t;
  }
};

void make_scan(const World& w, const double pose[3], std::mt19937& rng, float scale, hectorslam::DataContainer& dc) {
  std::normal_distribution<double> noise(0.0, 0.01);
  dc.clear();
  dc.setOrigo(Eigen::Vector2f(0.0f, 0.0f));
  float angle = -135.0f * 3.14159265f / 180.0f;
  const float inc = 0.25f * 3.14159265f / 180.0f;
  for (int i = 0; i < 1081; ++i) {
    float dist = static_cast<float>(w.cast(pose[0], pose[1], pose[2] + angle) + noise(rng));
    if (dist > 0.1f && dist < 29.9f) {  // HectorMappingRos.cpp:499
      dist *= scale;
      dc.add(Eigen::Vector2f(std::cos(angle) * dist, std::sin(angle) * dist));
    }
    angle += inc;
  }
}

double wrap(double a) { return std::fabs(std::remainder(a, 2.0 * 3.14159265358979323846)); }

}  // namespace

int main(int argc, char** argv) {
  const int steps = argc > 1 ? std::atoi(argv[1]) : 60;
  NullBuf nb;
  std::streambuf* saved = std::cout.rdbuf(&nb);  // the reference prints level banners / clamp notes

  const float res = 0.05f;
  const int size = 1024, levels = 3;
  Log log[2];
  RecordingDraw draw0(&log[0]), draw1(&log[1]);
  RecordingDebug debug0(&log[0]), debug1(&log[1]);
  hectorslam::HectorSlamProcessor cpu(res, size, size, Eigen::Vector2f(0.5f, 0.5f), levels, &draw0, &debug0);
  hectorslam::HectorSlamProcessorB200 gpu(res, size, size, Eigen::Vector2f(0.5f, 0.5f), levels, &draw1, &debug1);
  log[0].calls.clear();  // construction-time calls, if any, are not part of the comparison
  log[1].calls.clear();
  hectorslam::HectorSlamProcessor* procs[2] = {&cpu, &gpu};
  for (int k = 0; k < 2; ++k) {
    procs[k]->setUpdateFactorFree(0.4f);
    procs[k]->setUpdateFactorOccupied(0.9f);
    procs[k]->setMapUpdateMinDistDiff(0.2f);
    procs[k]->setMapUpdateMinAngleDiff(0.06f);
  }

  World world;
  std::mt19937 rng(7);
  double pose[3] = {-4.0, -2.5, 0.3};
  Eigen::Vector3f hint[2];
  hint[0] = hint[1] = Eigen::Vector3f(static_cast<float>(pose[0]), static_cast<float>(pose[1]), static_cast<float>(pose[2]));
  hectorslam::DataContainer dc;
  for (int s = 0; s < steps; ++s) {
    make_scan(world, pose, rng, cpu.getScaleToMap(), dc);
    for (int k = 0; k < 2; ++k) procs[k]->update(dc, hint[k]);
    hint[0] = cpu.getLastScanMatchPose();  // each side feeds its own estimate back (HectorMappingRos.cpp:314)
    hint[1] = gpu.getLastScanMatchPose();
    pose[0] += 0.09;
    pose[1] += 0.035;
    pose[2] += 0.015;
  }
  std::cout.rdbuf(saved);

  const std::vector<Call>& a = log[0].calls;
  const std::vector<Call>& b = log[1].calls;
  long counts[2][9] = {{0}};
  for (const Call& c : a) ++counts[0][c.kind];
  for (const Call& c : b) ++counts[1][c.kind];
  std::printf("calls: cpu=%zu gpu=%zu\n", a.size(), b.size());
  for (int k = 0; k < 9; ++k)
    if (counts[0][k] || counts[1][k]) std::printf("  %-24s cpu=%ld gpu=%ld\n", kKindName[k], counts[0][k], counts[1][k]);

  bool ok = a.size() == b.size() && !a.empty();
  long first_bad = -1;
  double max_arrow_pos = 0, max_arrow_ang = 0, max_point_excess = -1e300, max_point = 0, max_h_rel = 0;
  long points_checked = 0;
  // the arrow pair a scan is drawn at: ScanMatcher draws the start pose before its first drawScan and the last
  // estimate before its second one
  double ref_a[3] = {0, 0, 0}, dp = 0, dpsi = 0;
  for (size_t i = 0; ok && i < a.size(); ++i) {
    const Call &ca = a[i], &cb = b[i];
    bool same = ca.kind == cb.kind;
    if (same) {
      switch (ca.kind) {
        case SCALE:
        case COLOR:
          for (int j = 0; j < 4; ++j) same = same && ca.v[j] == cb.v[j];
          break;
        case ARROW: {
          const double ex = std::max(std::fabs(ca.v[0] - cb.v[0]), std::fabs(ca.v[1] - cb.v[1]));
          const double ea = wrap(ca.v[2] - cb.v[2]);
          max_arrow_pos = std::max(max_arrow_pos, ex);
          max_arrow_ang = std::max(max_arrow_ang, ea);
          same = ex <= 1e-4 && ea <= 1e-4;
          ref_a[0] = ca.v[0];
          ref_a[1] = ca.v[1];
          ref_a[2] = ca.v[2];
          dp = std::hypot(ca.v[0] - cb.v[0], ca.v[1] - cb.v[1]);
          dpsi = wrap(ca.v[2] - cb.v[2]);
          break;
        }
        case POINT: {
          const double r = std::hypot(ca.v[0] - ref_a[0], ca.v[1] - ref_a[1]);
          const double d = std::hypot(ca.v[0] - cb.v[0], ca.v[1] - cb.v[1]);
          // first order in the pose difference, plus the fp32 rounding of a world coordinate of a few metres
          const double bound = dp + r * dpsi + 2e-6 * (1.0 + r + std::fabs(ref_a[0]) + std::fabs(ref_a[1]));
          max_point = std::max(max_point, d);
          max_point_excess = std::max(max_point_excess, d - bound);
          ++points_checked;
          same = d <= bound;
          break;
        }
        case HESSIAN: {
          double scale = 1e-12, diff = 0;
          for (int j = 0; j < 9; ++j) {
            scale = std::max(scale, std::fabs(ca.v[j]));
            diff = std::max(diff, std::fabs(ca.v[j] - cb.v[j]));
          }
          max_h_rel = std::max(max_h_rel, diff / scale);
          break;
        }
        default:
          for (int j = 0; j < 9; ++j) same = same && ca.v[j] == cb.v[j];
      }
    }
    if (!same) {
      ok = false;
      first_bad = static_cast<long>(i);
    }
  }
  if (first_bad >= 0) {
    const Call &ca = a[first_bad], &cb = b[first_bad];
    std::printf("first mismatch at call %ld: cpu %s(%g, %g, %g) gpu %s(%g, %g, %g)\n", first_bad, kKindName[ca.kind], ca.v[0],
                ca.v[1], ca.v[2], kKindName[cb.kind], cb.v[0], cb.v[1], cb.v[2]);
  }
  std::printf("steps=%d max_arrow_dpos=%.3e max_arrow_dang=%.3e max_point_diff=%.3e max_point_excess_over_bound=%.3e "
              "points=%ld max_hessian_rel_diff=%.3e\n",
              steps, max_arrow_pos, max_arrow_ang, max_point, max_point_excess, points_checked, max_h_rel);
  std::printf("%s\n", ok ? "HOOKS OK" : "HOOKS MISMATCH");
  return ok ? 0 : 1;
}
