"""The per-scan fp32 pose arithmetic of the matcher — TEST INFRASTRUCTURE, not product code.

One restatement, every operation rounded to float32 (numpy scalars), of what lies between the Gauss-Newton sums and the
returned pose:

  * step: ScanMatcher::estimateTransformationLogLh's update (ScanMatcher.h:194-221) given one evaluation's H and dTr —
    the gate H(0,0) != 0 && H(1,1) != 0, Eigen's fixed-size inverse (cyclic cofactors, det from column 0, times 1/det;
    the order of hs_oracle.c inverse3_times and match_kernel.cuh solve3) times dTr, the +-0.2 rad clamp on the angle
    and the three additions;
  * normalize_angle: util::normalize_angle (UtilFunctions.h:37-49), double fmods (M_PI is a double) narrowed to float;
  * pose_difference_larger_than: util::poseDifferenceLargerThan (UtilFunctions.h:73-92), the map-update gate: fp32
    norm, the angle difference wrapped once with double pi, abs(float).

tests/test_pose32_oracle.py ties these to the C port's record and to the reference's own util:: functions
(oracle/ref_driver.cpp hsref_normalize_angle / hsref_pose_difference_larger_than).
"""
from __future__ import annotations

import math

import numpy as np

F32 = np.float32
CLAMP = F32(0.2)


def solve3(H, d):
    """inverse(H) * d in fp32: H (3, 3) row-major, d (3,) -> (3,) float32"""
    m = np.asarray(H, F32).reshape(3, 3)
    v = np.asarray(d, F32).reshape(3)

    def cof(i, j):
        i1, i2, j1, j2 = (i + 1) % 3, (i + 2) % 3, (j + 1) % 3, (j + 2) % 3
        return m[i1, j1] * m[i2, j2] - m[i1, j2] * m[i2, j1]

    with np.errstate(all="ignore"):
        c0, c1, c2 = cof(0, 0), cof(1, 0), cof(2, 0)
        det = c0 * m[0, 0] + (c1 * m[1, 0] + c2 * m[2, 0])
        invdet = F32(1.0) / det
        inv = [[cof(j, i) * invdet for j in range(3)] for i in range(3)]   # inv(i, j) = cof(j, i) / det
        return np.array([inv[r][0] * v[0] + (inv[r][1] * v[1] + inv[r][2] * v[2]) for r in range(3)], F32)


def step(est, H, dTr):
    """the estimate after one evaluation: est (3,) in the level's cells, H (3, 3), dTr (3,) -> (3,) float32"""
    e = np.asarray(est, F32).reshape(3).copy()
    m = np.asarray(H, F32).reshape(3, 3)
    if not (m[0, 0] != 0 and m[1, 1] != 0):   # ScanMatcher.h:201
        return e
    d = solve3(m, dTr)
    if d[2] > CLAMP:                          # :209-215 (NaN passes through)
        d[2] = CLAMP
    elif d[2] < -CLAMP:
        d[2] = -CLAMP
    with np.errstate(all="ignore"):
        return np.array([e[0] + d[0], e[1] + d[1], e[2] + d[2]], F32)   # :217


def normalize_angle(a) -> np.float32:
    """util::normalize_angle of one float"""
    two_pi = 2.0 * math.pi
    with np.errstate(invalid="ignore"):
        r = np.fmod(np.fmod(np.float64(F32(a)), two_pi) + two_pi, two_pi)   # fmod(+-inf) is NaN, not an error
    r = F32(r)
    if float(r) > math.pi:
        r = F32(float(r) - two_pi)
    return r


def pose_difference_larger_than(p1, p2, dist, ang) -> bool:
    """util::poseDifferenceLargerThan(p1, p2, dist, ang)"""
    a, b = np.asarray(p1, F32).reshape(3), np.asarray(p2, F32).reshape(3)
    with np.errstate(all="ignore"):
        dx, dy = a[0] - b[0], a[1] - b[1]
        if np.sqrt(dx * dx + dy * dy) > F32(dist):
            return True
        d = a[2] - b[2]
    if float(d) > math.pi:
        d = F32(float(d) - math.pi * 2.0)
    elif float(d) < -math.pi:
        d = F32(float(d) + math.pi * 2.0)
    return bool(abs(d) > F32(ang))
