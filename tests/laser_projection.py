"""laser_geometry's projection restated for the tests of the projected SLAM step (hsb_slam_update_projected).

ROS1 Melodic / Noetic laser_geometry, LaserProjection::projectLaser_ / getUnitVectors_ for the sensor_msgs/PointCloud
output, the call HectorMappingRos.cpp:273 makes (projectLaser(scan, cloud, 30.0)):
  * unit vectors, double: c_i = cos(angle_min + i * angle_increment), s_i = sin(...), libm (math.cos / math.sin here;
    numpy's SIMD cos need not equal libm);
  * beam i is kept iff (double)range < range_cutoff && range >= range_min (float compare), range_cutoff < 0 meaning
    range_max;
  * Point32 = ((float)(range * c_i), (float)(range * s_i), 0), one double product each, beam order kept.
The node then converts that cloud with rosPointCloudToDataContainer: oracle.pyoracle.cloud_to_points, the plain-C port
or (kind="reference") the node's own source compiled.  Both compose into the oracle container of a projected scan.

hector_slam_b200.synth.ranges_to_cloud is an input generator with different arithmetic (fp32 cos, `<=` windows); it is
not this oracle.
"""
import math

import numpy as np

F32 = np.float32


def unit_vectors(n_beams, angle_min, angle_increment):
    """(n, 2) float64 (cos, sin) of (double)angle_min + (double)i * (double)angle_increment."""
    a0, da = float(F32(angle_min)), float(F32(angle_increment))
    out = np.empty((n_beams, 2), np.float64)
    for i in range(n_beams):
        a = a0 + float(i) * da
        out[i, 0] = math.cos(a)
        out[i, 1] = math.sin(a)
    return out


def cutoff_of(proj):
    c = float(proj["range_cutoff"])
    return float(F32(proj["range_max"])) if c < 0 else c


def kept_beams(ranges, proj):
    r = np.asarray(ranges, F32).reshape(-1)
    with np.errstate(invalid="ignore"):
        return (r.astype(np.float64) < cutoff_of(proj)) & (r >= F32(proj["range_min"]))


def project(ranges, proj, unit=None):
    """The projected cloud: (m, 3) float32 Point32 triples in the laser frame."""
    r = np.asarray(ranges, F32).reshape(-1)
    assert r.size == proj["n_beams"], (r.size, proj["n_beams"])
    u = unit_vectors(proj["n_beams"], proj["angle_min"], proj["angle_increment"]) if unit is None else unit
    keep = kept_beams(r, proj)
    rk = r[keep].astype(np.float64)
    pts = np.zeros((int(keep.sum()), 3), F32)
    pts[:, 0] = (rk * u[keep, 0]).astype(F32)
    pts[:, 1] = (rk * u[keep, 1]).astype(F32)
    return pts


def container(ranges, proj, fmt, transform, scale_to_map, pyoracle, kind="port"):
    """The DataContainer a default node builds from this scan: (endpoints (k, 2) float32, origo (2,) float32)."""
    return pyoracle.cloud_to_points(project(ranges, proj), transform, fmt["sqr_laser_min_dist"], fmt["sqr_laser_max_dist"],
                                    fmt["laser_z_min_value"], fmt["laser_z_max_value"], scale_to_map, kind=kind)


def tilted_transform(pitch=0.3, z=0.4, yaw=0.2, xy=(0.1, -0.05)):
    """A laser mounted nose-down: its far returns leave the default +-1 m z window (rows of [R | t], float64)."""
    from hector_slam_b200 import synth

    return synth.laser_transform(xyz=(xy[0], xy[1], z), rpy=(0.01, pitch, yaw))


def edge_ranges(n, proj, seed, base=None, dropped_only=False):
    """Ranges with the projector's edge values at beams that move with the seed: NaN, +inf, -inf, a negative range, 0,
    r == range_min (kept) and the float below it (dropped), r == cutoff (dropped) and the float below it (kept), range_max
    and the float above it, plus short returns (0.45 .. 0.7 m) whose backward beams fall in the rear-close zone.
    dropped_only: only the values the projector drops, so that a scan of a real scene gains no phantom returns."""
    rng = np.random.default_rng(seed)
    r = (rng.uniform(0.3, 1.2 * cutoff_of(proj) + 1.0, n) if base is None else np.array(base, F32)).astype(F32)
    if n < 24:
        return r
    rmin = F32(proj["range_min"])
    cut = F32(cutoff_of(proj))
    rmax = F32(proj["range_max"])
    vals = [F32(np.nan), F32(np.inf), F32(-np.inf), F32(-1.5), F32(0.0), np.nextafter(rmin, F32(0)), cut]
    if not dropped_only:
        vals += [rmin, np.nextafter(cut, F32(0)), rmax, np.nextafter(rmax, F32(np.inf))]
    pos = rng.choice(n, size=len(vals) + 8, replace=False)
    for p, v in zip(pos, vals):
        r[p] = v
    if dropped_only:
        return r
    for p in pos[len(vals):]:
        r[p] = F32(rng.uniform(0.45, 0.7))
    r[n - 6:] = F32(0.55)   # the last beams of a scan reaching past +-90 degrees point backward: rear-close zone
    return r
