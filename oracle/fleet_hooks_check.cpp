// oracle/fleet_hooks_check.cpp — TEST INFRASTRUCTURE.
//
// A fleet of robots with the node's pub_drawings / pub_debug_output on, stepped two ways over the same synthetic scans:
// each robot by its own UNMODIFIED reference façade (HectorSlamProcessor::update on MapRepMultiMap, whose ScanMatchers
// call the recording hooks themselves), and all robots together by hsb200::SlamProcessor::updateMany /
// updateManyRanges (one heterogeneous group step per tick) with the step record on, the hooks replayed afterwards by
// replayMatchHooks (hector_slam_b200/host/MatchHooksB200.h) from each robot's step record and last-match container,
// followed by the façade's own calls (replayUpdateHooks).
// The robots differ in map size, resolution and level count, and have different hooks installed (draw only, debug
// only, both).  Even ticks step level-0 endpoints, odd ticks raw LaserScan ranges converted on the device.
//
// Per robot the two hook call sequences must agree under dropin_hooks_check.cpp's rules: the same methods in the same
// order and numbers, setScale / setColor arguments exactly, arrows within 1e-4 m / rad, drawn points within the bound
// the pose difference of their scan implies (|dp| + r |dpsi|); the largest relative difference of the forwarded
// Hessians is printed.
//
// Built by oracle/fleet_hooks.mk into oracle/_ref/fleet_hooks_check (needs the reference headers at build time); run by
// tests/test_gpu_step_record.py.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <iostream>
#include <memory>
#include <random>
#include <streambuf>
#include <vector>

#include "MatchHooksB200.h"
#include "SlamProcessorB200.hpp"

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

// One log shared by a robot's two hooks, so that the interleaving of draw and debug calls is compared too.
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

// the LaserScan: 1081 beams over 270 degrees, range window [0.1, 30] m
const int kBeams = 1081;
const float kAngleMin = -135.0f * 3.14159265f / 180.0f, kAngleInc = 0.25f * 3.14159265f / 180.0f;
const float kRangeMin = 0.1f, kRangeMax = 30.0f;

void make_ranges(const World& w, const double pose[3], std::mt19937& rng, std::vector<float>& ranges) {
  std::normal_distribution<double> noise(0.0, 0.01);
  ranges.resize(kBeams);
  float angle = kAngleMin;
  for (int i = 0; i < kBeams; ++i) {
    ranges[i] = static_cast<float>(w.cast(pose[0], pose[1], pose[2] + angle) + noise(rng));
    angle += kAngleInc;
  }
}

// HectorMappingRos::rosLaserScanToDataContainer (HectorMappingRos.cpp:483-507)
void ranges_to_container(const std::vector<float>& ranges, float scaleToMap, hectorslam::DataContainer& dc) {
  dc.clear();
  dc.setOrigo(Eigen::Vector2f(0.0f, 0.0f));
  float angle = kAngleMin;
  const float maxRangeForContainer = kRangeMax - 0.1f;
  for (int i = 0; i < kBeams; ++i) {
    float dist = ranges[i];
    if ((dist > kRangeMin) && (dist < maxRangeForContainer)) {
      dist *= scaleToMap;
      dc.add(Eigen::Vector2f(std::cos(angle) * dist, std::sin(angle) * dist));
    }
    angle += kAngleInc;
  }
}

double wrap(double a) { return std::fabs(std::remainder(a, 2.0 * 3.14159265358979323846)); }

// dropin_hooks_check.cpp's comparison of two hook call sequences; prints a summary, returns whether they agree
bool compare(const char* name, const std::vector<Call>& a, const std::vector<Call>& b) {
  long counts[2][9] = {{0}};
  for (const Call& c : a) ++counts[0][c.kind];
  for (const Call& c : b) ++counts[1][c.kind];
  std::printf("%s calls: cpu=%zu gpu=%zu\n", name, a.size(), b.size());
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
    std::printf("%s first mismatch at call %ld: cpu %s(%g, %g, %g) gpu %s(%g, %g, %g)\n", name, first_bad,
                kKindName[ca.kind], ca.v[0], ca.v[1], ca.v[2], kKindName[cb.kind], cb.v[0], cb.v[1], cb.v[2]);
  }
  std::printf("%s max_arrow_dpos=%.3e max_arrow_dang=%.3e max_point_diff=%.3e max_point_excess_over_bound=%.3e "
              "points=%ld max_hessian_rel_diff=%.3e\n",
              name, max_arrow_pos, max_arrow_ang, max_point, max_point_excess, points_checked, max_h_rel);
  return ok;
}

struct Robot {
  float res;
  int sx, sy, levels;
  bool draw, debug;
  double pose[3];
};

}  // namespace

int main(int argc, char** argv) {
  const int steps = argc > 1 ? std::atoi(argv[1]) : 40;
  NullBuf nb;
  std::streambuf* saved = std::cout.rdbuf(&nb);  // the reference prints level banners / clamp notes

  const Robot robots[] = {{0.05f, 1024, 1024, 3, true, true, {-4.0, -2.5, 0.3}},
                          {0.05f, 768, 640, 2, true, false, {-3.0, 0.5, -0.2}},
                          {0.1f, 512, 384, 1, false, true, {1.0, -3.5, 1.2}},
                          {0.025f, 1536, 1024, 4, true, true, {3.0, 0.0, 2.8}}};
  const int M = sizeof(robots) / sizeof(robots[0]);
  const Eigen::Vector2f start(0.5f, 0.5f);
  std::vector<Log> log(2 * M);
  std::vector<std::unique_ptr<RecordingDraw>> draws;
  std::vector<std::unique_ptr<RecordingDebug>> debugs;
  for (int k = 0; k < 2 * M; ++k) {
    draws.emplace_back(new RecordingDraw(&log[k]));
    debugs.emplace_back(new RecordingDebug(&log[k]));
  }
  // log[2k]: robot k on the CPU reference, log[2k + 1]: robot k on the device
  std::vector<std::unique_ptr<hectorslam::HectorSlamProcessor>> cpu;
  std::vector<std::unique_ptr<hsb200::SlamProcessor>> gpu;
  std::vector<std::unique_ptr<hectorslam::MatchHookFrames>> frames;
  std::vector<hsb200::SlamProcessor*> ps;
  for (int k = 0; k < M; ++k) {
    const Robot& r = robots[k];
    cpu.emplace_back(new hectorslam::HectorSlamProcessor(r.res, r.sx, r.sy, start, r.levels,
                                                         r.draw ? draws[2 * k].get() : 0,
                                                         r.debug ? debugs[2 * k].get() : 0));
    cpu[k]->setUpdateFactorFree(0.4f);
    cpu[k]->setUpdateFactorOccupied(0.9f);
    cpu[k]->setMapUpdateMinDistDiff(0.2f);
    cpu[k]->setMapUpdateMinAngleDiff(0.06f);
    gpu.emplace_back(new hsb200::SlamProcessor(r.res, r.sx, r.sy, start.x(), start.y(), r.levels));
    gpu[k]->setUpdateFactorFree(0.4f);
    gpu[k]->setUpdateFactorOccupied(0.9f);
    gpu[k]->setMapUpdateMinDistDiff(0.2f);
    gpu[k]->setMapUpdateMinAngleDiff(0.06f);
    hsb_scan_format fmt = {kBeams, kAngleMin, kAngleInc, kRangeMin, kRangeMax};
    gpu[k]->setScanFormat(fmt);
    gpu[k]->setStepRecord(true);   // every robot here publishes drawings or debug output
    frames.emplace_back(new hectorslam::MatchHookFrames(r.res, r.sx, r.sy, r.levels, start));
    ps.push_back(gpu[k].get());
  }
  ps[0]->setHeterogeneousGroups(true);   // the robots differ in map geometry and level count
  for (int k = 0; k < 2 * M; ++k) log[k].calls.clear();   // construction-time calls are not part of the comparison

  World world;
  std::mt19937 rng(11);
  std::vector<std::vector<double>> pose(M);
  std::vector<Eigen::Vector3f> hint_cpu(M);
  std::vector<hsb200::Pose> hint_gpu(M);
  for (int k = 0; k < M; ++k) {
    pose[k].assign(robots[k].pose, robots[k].pose + 3);
    hint_cpu[k] = Eigen::Vector3f(static_cast<float>(pose[k][0]), static_cast<float>(pose[k][1]),
                                  static_cast<float>(pose[k][2]));
    hint_gpu[k] = hsb200::Pose{hint_cpu[k][0], hint_cpu[k][1], hint_cpu[k][2]};
  }
  hectorslam::DataContainer dc, replay_dc, scaled;
  std::vector<float> ranges, all_ranges, all_pts, rec, last_pts;
  std::vector<int> offsets(M + 1);
  long replayed = 0;
  for (int s = 0; s < steps; ++s) {
    const bool as_ranges = (s & 1) != 0;
    all_ranges.clear();
    all_pts.clear();
    offsets[0] = 0;
    for (int k = 0; k < M; ++k) {
      make_ranges(world, pose[k].data(), rng, ranges);
      ranges_to_container(ranges, cpu[k]->getScaleToMap(), dc);
      cpu[k]->update(dc, hint_cpu[k]);
      hint_cpu[k] = cpu[k]->getLastScanMatchPose();  // each side feeds its own estimate back (HectorMappingRos.cpp:314)
      all_ranges.insert(all_ranges.end(), ranges.begin(), ranges.end());
      for (int i = 0; i < dc.getSize(); ++i) {
        all_pts.push_back(dc.getVecEntry(i)[0]);
        all_pts.push_back(dc.getVecEntry(i)[1]);
      }
      offsets[k + 1] = as_ranges ? offsets[k] + kBeams : offsets[k] + dc.getSize();
      pose[k][0] += 0.07;
      pose[k][1] += 0.03;
      pose[k][2] += 0.012;
    }
    if (as_ranges)
      hsb200::SlamProcessor::updateManyRanges(ps.data(), M, all_ranges.data(), offsets.data(), hint_gpu.data());
    else
      hsb200::SlamProcessor::updateMany(ps.data(), M, all_pts.data(), offsets.data(), 0, hint_gpu.data());
    for (int k = 0; k < M; ++k) {
      hint_gpu[k] = gpu[k]->getLastScanMatchPose();
      DrawInterface* draw = robots[k].draw ? draws[2 * k + 1].get() : 0;
      HectorDebugInfoInterface* debug = robots[k].debug ? debugs[2 * k + 1].get() : 0;
      if (!gpu[k]->stepRecord(rec)) {
        hectorslam::replayUpdateHooks(*frames[k], draw, debug);
        continue;
      }
      float origo[2];
      const int n = gpu[k]->lastMatchScan(last_pts, origo);
      replay_dc.clear();
      replay_dc.setOrigo(Eigen::Vector2f(origo[0], origo[1]));
      for (int i = 0; i < n; ++i) replay_dc.add(Eigen::Vector2f(last_pts[2 * i], last_pts[2 * i + 1]));
      hectorslam::replayMatchHooks(gpu[k]->handle(), rec.data(), replay_dc, frames[k]->levels(), draw, debug, scaled);
      hectorslam::replayUpdateHooks(*frames[k], draw, debug);
      ++replayed;
    }
  }
  std::cout.rdbuf(saved);

  bool ok = replayed == (long)steps * M;
  std::printf("robots=%d steps=%d replayed=%ld\n", M, steps, replayed);
  for (int k = 0; k < M; ++k) {
    char name[32];
    std::snprintf(name, sizeof(name), "robot%d", k);
    ok = compare(name, log[2 * k].calls, log[2 * k + 1].calls) && ok;
  }
  std::printf("%s\n", ok ? "FLEET HOOKS OK" : "FLEET HOOKS MISMATCH");
  return ok ? 0 : 1;
}
