// MapRepB200.h — host-side adaptor: the reference's MapRepresentationInterface implemented on the
// B200 C-ABI (include/hector_slam_b200.h).
//
// This is the drop-in for hectorslam::MapRepMultiMap
// (hector_mapping/include/hector_slam_lib/slam_main/MapRepMultiMap.h:44-172): same constructor
// arguments, the same 11 virtuals (slam_main/MapRepresentationInterface.h:38-62), the same
// ownership rules (addMapMutex takes ownership, MapProcContainer.h:83-91), the same silent
// numerical edge-case behaviour.  The maps live in HBM; getGridMap() returns a host mirror that is
// refreshed lazily (only when a reader asks after a device-side write), so the map-publishing
// thread of the ROS node (src/HectorMappingRos.cpp:435-481) keeps working unchanged.
//
// It is compiled against the REFERENCE's own headers (it derives from the reference's abstract
// class and hands out the reference's GridMap type), so it needs hector_slam_lib and Eigen on the
// include path — exactly what hector_mapping already has.  See INTEGRATION.md.
//
// HectorSlamProcessorB200 below swaps the representation inside the unmodified façade:
// HectorSlamProcessor::mapRep is a protected member (slam_main/HectorSlamProcessor.h:143).
#ifndef HECTOR_SLAM_B200_MAPREP_H
#define HECTOR_SLAM_B200_MAPREP_H

#include <cmath>
#include <mutex>
#include <stdexcept>
#include <string>
#include <vector>

#include "slam_main/HectorSlamProcessor.h"  // pulls map/, matcher/, scan/, util/ in the right order

#include "MatchHooksB200.h"
#include "hector_slam_b200.h"

namespace hectorslam {

class MapRepB200 : public MapRepresentationInterface {
 public:
  // Arguments as MapRepMultiMap's (MapRepMultiMap.h:48); `device` selects the GPU.
  // The two hooks are what MapRepMultiMap hands every level's ScanMatcher (MapRepMultiMap.h:63); matchData replays the
  // matcher's calls on them from the device's per-evaluation record (replayMatchHooks, MatchHooksB200.h).
  MapRepB200(float mapResolution, int mapSizeX, int mapSizeY, unsigned int numDepth, const Eigen::Vector2f& startCoords,
             DrawInterface* drawInterfaceIn = 0, HectorDebugInfoInterface* debugInterfaceIn = 0, int device = 0)
      : handle_(0), draw_(drawInterfaceIn), debug_(debugInterfaceIn) {
    hsb_config cfg = hsb_config();
    cfg.map_resolution = mapResolution;
    cfg.map_size_x = mapSizeX;
    cfg.map_size_y = mapSizeY;
    cfg.start_x = startCoords.x();
    cfg.start_y = startCoords.y();
    cfg.levels = static_cast<int>(numDepth);
    cfg.device = device;
    // update factors: library defaults of the reference (0.4 / 0.6) until the setters are called
    int st = hsb_create(&cfg, &handle_);
    if (st != HSB_OK) {
      throw std::runtime_error(std::string("hsb_create failed: ") + hsb_last_error(0));
    }
    // host mirrors with the reference's own geometry (MapRepMultiMap.h:51-69)
    forEachMapLevel(mapResolution, mapSizeX, mapSizeY, numDepth, startCoords,
                    [this](unsigned int, float cellLength, const Eigen::Vector2i& cells, const Eigen::Vector2f& offset) {
                      mirrors_.push_back(new GridMap(cellLength, cells, offset));
                      stale_.push_back(false);
                      pending_updates_.push_back(0);
                      mutexes_.push_back(0);
                    });
  }

  virtual ~MapRepB200() {
    for (size_t i = 0; i < mirrors_.size(); ++i) {
      delete mirrors_[i];
      if (mutexes_[i]) delete mutexes_[i];  // MapProcContainer::cleanup, MapProcContainer.h:56-65
    }
    hsb_destroy(handle_);
  }

  virtual void reset() {
    std::lock_guard<std::mutex> g(api_);
    check(hsb_reset(handle_));
    for (size_t i = 0; i < mirrors_.size(); ++i) {
      mirrors_[i]->reset();
      int rect[4];
      check(hsb_get_mirror_dirty_rect(handle_, static_cast<int>(i), rect, 1));  // mirror and device are both empty now
      stale_[i] = false;
      pending_updates_[i] = 0;
    }
  }

  virtual float getScaleToMap() const { return hsb_get_scale_to_map(handle_); }
  virtual int getMapLevels() const { return hsb_get_map_levels(handle_); }

  // The mirror is synchronised here, i.e. inside whatever lock the caller holds for the level
  // (the node's publisher takes the level's MapLockerInterface first, HectorMappingRos.cpp:453).
  virtual const GridMap& getGridMap(int mapLevel) const {
    std::lock_guard<std::mutex> g(api_);
    if (stale_[mapLevel]) {
      // only what was written since the last look travels: the device keeps a dirty rectangle per level for the host
      // mirror (K2's apply phase folds each scan's bounding box into it), so the bytes copied under the level's
      // mutex are proportional to the touched area, not to the map (SURVEY.md N1; the reference's publisher walks
      // the whole grid under that mutex, HectorMappingRos.cpp:453-475)
      GridMap& m = *mirrors_[mapLevel];
      int rect[4];
      check(hsb_get_mirror_dirty_rect(handle_, mapLevel, rect, 1));
      if (rect[2] >= rect[0]) {
        const int w = rect[2] - rect[0] + 1, hgt = rect[3] - rect[1] + 1, sx = m.getSizeX();
        scratch_.resize(static_cast<size_t>(w) * static_cast<size_t>(hgt));
        check(hsb_download_level_rect(handle_, mapLevel, rect, scratch_.data()));
        for (int r = 0; r < hgt; ++r)
          for (int c = 0; c < w; ++c)
            m.getCell((rect[1] + r) * sx + rect[0] + c).logOddsVal = scratch_[static_cast<size_t>(r) * w + c];
      }
      for (int k = 0; k < pending_updates_[mapLevel]; ++k) m.setUpdated();  // GridMapBase.h:322
      pending_updates_[mapLevel] = 0;
      stale_[mapLevel] = false;
    }
    return *mirrors_[mapLevel];
  }

  virtual void addMapMutex(int i, MapLockerInterface* mapMutex) {
    if (mutexes_[i]) delete mutexes_[i];
    mutexes_[i] = mapMutex;
  }
  virtual MapLockerInterface* getMapMutex(int i) { return mutexes_[i]; }

  virtual void onMapUpdated() {
    std::lock_guard<std::mutex> g(api_);
    check(hsb_on_map_updated(handle_));
  }

  virtual Eigen::Vector3f matchData(const Eigen::Vector3f& beginEstimateWorld, const DataContainer& dataContainer,
                                    Eigen::Matrix3f& covMatrix) {
    std::lock_guard<std::mutex> g(api_);
    const int n = dataContainer.getSize();
    const float hint[3] = {beginEstimateWorld[0], beginEstimateWorld[1], beginEstimateWorld[2]};
    const Eigen::Vector2f origo = dataContainer.getOrigo();
    const float og[2] = {origo[0], origo[1]};
    float pose[3];
    float cov[9];
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) cov[3 * r + c] = covMatrix(r, c);
    const float* pts = n > 0 ? dataContainer.getVecEntry(0).data() : 0;
    if (draw_ || debug_) {
      record_.resize(static_cast<size_t>(hsb_get_match_record_floats(handle_)));
      check(hsb_match_data_record(handle_, hint, pts, n, og, pose, cov, record_.data()));
      replayMatchHooks(handle_, record_.data(), dataContainer, mirrors_.data(), draw_, debug_, scaled_);
    } else {
      check(hsb_match_data(handle_, hint, pts, n, og, pose, cov));
    }
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) covMatrix(r, c) = cov[3 * r + c];
    return Eigen::Vector3f(pose[0], pose[1], pose[2]);
  }

  virtual void updateByScan(const DataContainer& dataContainer, const Eigen::Vector3f& robotPoseWorld) {
    // the reference locks each level's mutex around that level's write (MapProcContainer.h:103-116);
    // all levels are written by one launch here, so every installed mutex is held for its duration
    for (size_t i = 0; i < mutexes_.size(); ++i)
      if (mutexes_[i]) mutexes_[i]->lockMap();
    {
      std::lock_guard<std::mutex> g(api_);
      const int n = dataContainer.getSize();
      const Eigen::Vector2f origo = dataContainer.getOrigo();
      const float og[2] = {origo[0], origo[1]};
      const float pose[3] = {robotPoseWorld[0], robotPoseWorld[1], robotPoseWorld[2]};
      check(hsb_update_by_scan(handle_, n > 0 ? dataContainer.getVecEntry(0).data() : 0, n, og, pose));
      for (size_t i = 0; i < stale_.size(); ++i) {
        stale_[i] = true;
        pending_updates_[i] += 1;
      }
    }
    for (size_t i = mutexes_.size(); i-- > 0;)
      if (mutexes_[i]) mutexes_[i]->unlockMap();
  }

  virtual void setUpdateFactorFree(float free_factor) {
    std::lock_guard<std::mutex> g(api_);
    check(hsb_set_update_factor_free(handle_, free_factor));
    for (size_t i = 0; i < mirrors_.size(); ++i) mirrors_[i]->setUpdateFreeFactor(free_factor);
  }
  virtual void setUpdateFactorOccupied(float occupied_factor) {
    std::lock_guard<std::mutex> g(api_);
    check(hsb_set_update_factor_occupied(handle_, occupied_factor));
    for (size_t i = 0; i < mirrors_.size(); ++i) mirrors_[i]->setUpdateOccupiedFactor(occupied_factor);
  }

  hsb_handle* handle() { return handle_; }

 private:
  // The reference has no error channel (no exceptions, no return codes) because nothing on its CPU
  // path can fail; a CUDA failure here is unrecoverable for the caller, so it is raised.
  void check(int st) const {
    if (st != HSB_OK) throw std::runtime_error(std::string("hector_slam_b200: ") + hsb_last_error(handle_));
  }

  hsb_handle* handle_;
  DrawInterface* draw_;
  HectorDebugInfoInterface* debug_;
  std::vector<float> record_;   // per-evaluation record of the last match (only with a hook installed)
  DataContainer scaled_;        // a coarse level's container (MapRepMultiMap::dataContainers)
  mutable std::mutex api_;  // the C-ABI handle is single-writer
  mutable std::vector<GridMap*> mirrors_;
  mutable std::vector<bool> stale_;
  mutable std::vector<int> pending_updates_;
  mutable std::vector<float> scratch_;
  std::vector<MapLockerInterface*> mutexes_;
};

// The unmodified façade with the B200 representation plugged in.
class HectorSlamProcessorB200 : public HectorSlamProcessor {
 public:
  HectorSlamProcessorB200(float mapResolution, int mapSizeX, int mapSizeY, const Eigen::Vector2f& startCoords,
                          int multi_res_size, DrawInterface* drawInterfaceIn = 0,
                          HectorDebugInfoInterface* debugInterfaceIn = 0, int device = 0)
      // the base class builds (tiny) CPU maps first; they are replaced right away
      : HectorSlamProcessor(mapResolution, 8 << (multi_res_size - 1), 8 << (multi_res_size - 1), startCoords,
                            multi_res_size, drawInterfaceIn, debugInterfaceIn) {
    delete mapRep;  // HectorSlamProcessor.h:143 (protected)
    mapRep = new MapRepB200(mapResolution, mapSizeX, mapSizeY, multi_res_size, startCoords, drawInterfaceIn,
                            debugInterfaceIn, device);
    this->reset();
  }
};

}  // namespace hectorslam

#endif
