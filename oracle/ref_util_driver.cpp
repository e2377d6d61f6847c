// oracle/ref_util_driver.cpp — TEST INFRASTRUCTURE, not product code.
//
// util::normalize_angle and util::poseDifferenceLargerThan (util/UtilFunctions.h:37-49, :73-92) of the UNMODIFIED
// reference header, compiled where it lies against oracle/shim (the shim's tf stub fixes which `abs` the gate calls).
// Built by oracle/Makefile into oracle/_ref/libhsref_util.so, a library of its own so that a libhsref.so built
// before these entry points existed never stands in for them.  tests/test_pose32_oracle.py ties oracle/pose32.py to it.
#include <Eigen/Core>

#include "util/UtilFunctions.h"

extern "C" {

void hsref_normalize_angle(const float* in, int n, float* out) {
  for (int i = 0; i < n; ++i) out[i] = util::normalize_angle(in[i]);
}

void hsref_pose_difference_larger_than(const float* p1, const float* p2, const float* dist, const float* ang, int n,
                                       int* out) {
  for (int i = 0; i < n; ++i)
    out[i] = util::poseDifferenceLargerThan(Eigen::Vector3f(p1[3 * i], p1[3 * i + 1], p1[3 * i + 2]),
                                            Eigen::Vector3f(p2[3 * i], p2[3 * i + 1], p2[3 * i + 2]), dist[i], ang[i]);
}

}  // extern "C"
