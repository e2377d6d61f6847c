// MatchHooksB200.h — the matcher's draw and debug hooks replayed from a handle's per-evaluation match record.
//
// hector_mapping's pub_drawings / pub_debug_output (HectorMappingRos.cpp:59-60,110-119) hand every level's ScanMatcher
// a DrawInterface and a HectorDebugInfoInterface, which matchData (matcher/ScanMatcher.h:56-115) calls while it
// iterates.  On the device the match writes its record instead (include/hector_slam_b200.h: hsb_match_data_record, or
// hsb_set_step_record for the fused and group SLAM steps) and replayMatchHooks makes the same calls from it afterwards.
// MapRepB200 (MapRepB200.h) calls it after each matchData; a fleet server that steps hsb200::SlamProcessor's with
// updateMany* calls it for each robot that recorded, with that robot's MatchHookFrames.
//
// Like MapRepB200.h it is compiled against the reference's own headers: the hooks' interfaces, DataContainer and the
// GridMap transforms are the reference's.
#ifndef HECTOR_SLAM_B200_MATCHHOOKS_H
#define HECTOR_SLAM_B200_MATCHHOOKS_H

#include <cmath>
#include <vector>

#include "slam_main/HectorSlamProcessor.h"  // pulls map/, matcher/, scan/, util/ in the right order

#include "hector_slam_b200.h"

namespace hectorslam {

// MapRepMultiMap's level geometry (MapRepMultiMap.h:51-69): f(level, cell length, cells, top-left offset) per level.
template <class F>
void forEachMapLevel(float mapResolution, int mapSizeX, int mapSizeY, unsigned int numDepth,
                     const Eigen::Vector2f& startCoords, F f) {
  Eigen::Vector2i resolution(mapSizeX, mapSizeY);
  float totalMapSizeX = mapResolution * static_cast<float>(mapSizeX);
  float mid_offset_x = totalMapSizeX * startCoords.x();
  float totalMapSizeY = mapResolution * static_cast<float>(mapSizeY);
  float mid_offset_y = totalMapSizeY * startCoords.y();
  for (unsigned int i = 0; i < numDepth; ++i) {
    f(i, mapResolution, resolution, Eigen::Vector2f(mid_offset_x, mid_offset_y));
    resolution /= 2;
    mapResolution *= 2.0f;
  }
}

// One robot's level transforms for replayMatchHooks where no host mirror of its maps exists: per level a GridMap of a
// single cell built with the level's cell length and offset, whose getMapCoordsPose / getWorldCoordsPose /
// getWorldCoords are the reference's (only the transforms are read).  Arguments as MapRepMultiMap's.
class MatchHookFrames {
 public:
  MatchHookFrames(float mapResolution, int mapSizeX, int mapSizeY, unsigned int numDepth,
                  const Eigen::Vector2f& startCoords)
      : cells_(mapSizeX, mapSizeY) {
    forEachMapLevel(mapResolution, mapSizeX, mapSizeY, numDepth, startCoords,
                    [this](unsigned int, float cellLength, const Eigen::Vector2i&, const Eigen::Vector2f& offset) {
                      maps_.push_back(new GridMap(cellLength, Eigen::Vector2i(1, 1), offset));
                    });
  }
  ~MatchHookFrames() {
    for (size_t i = 0; i < maps_.size(); ++i) delete maps_[i];
  }
  MatchHookFrames(const MatchHookFrames&) = delete;
  MatchHookFrames& operator=(const MatchHookFrames&) = delete;
  const GridMap* const* levels() const { return maps_.data(); }
  const Eigen::Vector2i& levelZeroCells() const { return cells_; }

 private:
  std::vector<GridMap*> maps_;
  Eigen::Vector2i cells_;
};

// ScanMatcher::drawScan (ScanMatcher.h:228-239): OccGridMapUtil::getTransformForState (OccGridMapUtil.h:349-352) and
// getWorldCoordsPoint (:62) restated on `map`, which carries the level's geometry
template <class Map>
void drawMatchScan(DrawInterface* draw, const Eigen::Vector3f& pose, const Map& map, const DataContainer& dataContainer) {
  draw->setScale(0.02);
  Eigen::Affine2f transform(Eigen::Translation2f(pose[0], pose[1]) * Eigen::Rotation2Df(pose[2]));
  int size = dataContainer.getSize();
  for (int i = 0; i < size; ++i) {
    const Eigen::Vector2f& currPoint(dataContainer.getVecEntry(i));
    draw->drawPoint(map.getWorldCoords(transform * currPoint));
  }
}

// ScanMatcher::matchData's hook calls for every level of handle h, coarsest first, replayed from `record` (R floats,
// hsb_get_match_record_floats's layout) of a match of the level-0 container `scan`.  levelMaps[l] carries level l's
// transforms (the host mirrors, or MatchHookFrames::levels()); `scaled` is scratch for the coarse levels' containers,
// which are `scan` scaled as MapRepMultiMap.h:127 scales it.  The world conversions are the reference's own code on the
// device's estimates.  Either hook may be null.
template <class Map>
void replayMatchHooks(const hsb_handle* h, const float* record, const DataContainer& scan, const Map* const* levelMaps,
                      DrawInterface* draw, HectorDebugInfoInterface* debug, DataContainer& scaled) {
  const int levels = hsb_get_map_levels(h);
  const int n = scan.getSize();
  const float* r = record;
  for (int index = levels - 1; index >= 0; --index) {
    const int numIter = hsb_get_level_evals(h, index) - 1;  // the level's maxIterations (MapRepMultiMap.h:125,128)
    const Map& map = *levelMaps[index];
    const DataContainer* dc = &scan;
    if (index > 0) {
      scaled.setFrom(scan, static_cast<float>(1.0 / pow(2.0, static_cast<double>(index))));
      dc = &scaled;
    }
    const Eigen::Vector3f begin(r[0], r[1], r[2]);
    const float* ev = r + 3;  // 15 floats per evaluation: H (9), dTr (3), estimate after the step (3)
    if (draw) {
      draw->setScale(0.05f);
      draw->setColor(0.0f, 1.0f, 0.0f);
      draw->drawArrow(begin);
      drawMatchScan(draw, map.getMapCoordsPose(begin), map, *dc);
      draw->setColor(1.0, 0.0, 0.0);
    }
    if (n != 0) {
      for (int i = 0; i < numIter; ++i) {
        const float* e = ev + 15 * (i + 1);  // evaluation 0 (before the loop) is not reported
        if (draw) {
          float invNumIterf = 1.0f / static_cast<float>(numIter);
          draw->setColor(static_cast<float>(i) * invNumIterf, 0.0f, 0.0f);
          draw->drawArrow(map.getWorldCoordsPose(Eigen::Vector3f(e[12], e[13], e[14])));
        }
        if (debug) {
          Eigen::Matrix3f H;
          for (int a = 0; a < 3; ++a)
            for (int b = 0; b < 3; ++b) H(a, b) = e[3 * a + b];
          debug->addHessianMatrix(H);
        }
      }
      if (draw) {
        const float* e = ev + 15 * numIter;
        draw->setColor(0.0, 0.0, 1.0);
        drawMatchScan(draw, Eigen::Vector3f(e[12], e[13], e[14]), map, *dc);
      }
    }
    r += 3 + 15 * (numIter + 1);
  }
}

// HectorSlamProcessor::update's own hook calls, which follow the match and the map write of every step, matched or
// not (HectorSlamProcessor.h:98-113): level 0's first and last cell and (1, 1), then each hook's sendAndResetData.
// A server that steps hsb200::SlamProcessor's makes them after replayMatchHooks, where the reference façade would.
inline void replayUpdateHooks(const MatchHookFrames& frames, DrawInterface* draw, HectorDebugInfoInterface* debug) {
  if (draw) {
    const GridMap& gridMapRef(*frames.levels()[0]);
    draw->setColor(1.0, 0.0, 0.0);
    draw->setScale(0.15);

    draw->drawPoint(gridMapRef.getWorldCoords(Eigen::Vector2f::Zero()));
    draw->drawPoint(gridMapRef.getWorldCoords((frames.levelZeroCells().array() - 1).cast<float>()));
    draw->drawPoint(Eigen::Vector2f(1.0f, 1.0f));

    draw->sendAndResetData();
  }
  if (debug) debug->sendAndResetData();
}

}  // namespace hectorslam

#endif
