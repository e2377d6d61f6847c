"""ctypes front-end to the two CPU oracles — TEST INFRASTRUCTURE, not product code.

Only tests/, __graft_entry__.smoke() and bench.py's CPU-baseline / `--impl reference` legs may
import this module; nothing in hector_slam_b200/ does.

  * kind="reference": oracle/_ref/libhsref.so — the UNMODIFIED reference headers compiled against
    oracle/shim (built by oracle/Makefile where /root/reference exists; the .so travels to the
    GPU box prebuilt).
  * kind="port": oracle/_build/libhsoracle.so — the plain-C restatement oracle/hs_oracle.c.

Both libraries export the same entry points with prefixes `hsref_` / `hso_`.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_LIB = os.path.join(_HERE, "_ref", "libhsref.so")
PORT_LIB = os.path.join(_HERE, "_build", "libhsoracle.so")
REF_UTIL_LIB = os.path.join(_HERE, "_ref", "libhsref_util.so")   # the reference's util:: functions

_f32p = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
_i32p = np.ctypeslib.ndpointer(dtype=np.int32, flags="C_CONTIGUOUS")


def available(kind: str) -> bool:
    return os.path.exists(REF_LIB if kind == "reference" else PORT_LIB)


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


class Oracle:
    """One multi-level occupancy map + matcher on the CPU (reference or port)."""

    def __init__(self, kind: str, map_resolution: float, size: int, levels: int,
                 start=(0.5, 0.5), size_y: int | None = None, silent: bool = True):
        self.kind = kind
        path = REF_LIB if kind == "reference" else PORT_LIB
        if not os.path.exists(path):
            raise FileNotFoundError(f"oracle library missing: {path} (run `make -C oracle`)")
        self.lib = C.CDLL(path)
        self.p = "hsref_" if kind == "reference" else "hso_"
        self._bind()
        if silent and kind == "reference":
            self._fn("silence")(1)
        self.size_x = int(size)
        self.size_y = int(size if size_y is None else size_y)
        self.levels = int(levels)
        self.h = self._fn("create")(map_resolution, self.size_x, self.size_y, start[0], start[1], levels)

    def _fn(self, name):
        return getattr(self.lib, self.p + name)

    def _bind(self):
        L, p = self.lib, self.p
        vp, f, i = C.c_void_p, C.c_float, C.c_int

        def sig(name, res, *args):
            fn = getattr(L, p + name)
            fn.restype = res
            fn.argtypes = list(args)

        if p == "hsref_":
            sig("silence", None, i)
        sig("create", vp, f, i, i, f, f, i)
        sig("destroy", None, vp)
        sig("reset", None, vp)
        sig("set_update_factors", None, vp, f, f)
        sig("set_map_update_thresholds", None, vp, f, f)
        sig("levels", i, vp)
        sig("size_x", i, vp, i)
        sig("size_y", i, vp, i)
        sig("cell_length", f, vp, i)
        sig("scale_to_map", f, vp)
        sig("map_coords_pose", None, vp, i, _f32p, _f32p)
        sig("world_coords_pose", None, vp, i, _f32p, _f32p)
        sig("update", None, vp, _f32p, i, _f32p, _f32p, i, _f32p, _f32p)
        sig("match", None, vp, _f32p, _f32p, i, _f32p, _f32p, _f32p)
        sig("update_by_scan", None, vp, _f32p, i, _f32p, _f32p)
        sig("on_map_updated", None, vp)
        sig("get_logodds", None, vp, i, _f32p)
        sig("set_logodds", None, vp, i, _f32p)
        sig("get_prob", None, vp, i, _f32p)
        sig("get_logodds_increments", None, vp, _f32p)
        sig("hessian_derivs", None, vp, i, _f32p, _f32p, i, _f32p, _f32p)
        sig("match_level", None, vp, i, _f32p, _f32p, i, i, _f32p, _f32p)
        sig("update_level", None, vp, i, _f32p, i, _f32p, _f32p)
        sig("match_batch", C.c_double, vp, i, _f32p, _f32p, _i32p, _f32p, _f32p, i)
        sig("likelihood", f, vp, i, _f32p, _f32p, i)
        sig("covariance_for_pose", None, vp, i, _f32p, _f32p, i, _f32p, _f32p)

    def close(self):
        if getattr(self, "h", None):
            self._fn("destroy")(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # --- configuration -----------------------------------------------------------------
    def reset(self):
        self._fn("reset")(self.h)

    def set_update_factors(self, free: float, occ: float):
        self._fn("set_update_factors")(self.h, free, occ)

    def set_map_update_thresholds(self, dist: float, ang: float):
        self._fn("set_map_update_thresholds")(self.h, dist, ang)

    def level_size(self, level: int):
        return self._fn("size_x")(self.h, level), self._fn("size_y")(self.h, level)

    def cell_length(self, level: int) -> float:
        return float(self._fn("cell_length")(self.h, level))

    def scale_to_map(self) -> float:
        return float(self._fn("scale_to_map")(self.h))

    def map_coords_pose(self, level: int, world):
        out = np.zeros(3, np.float32)
        self._fn("map_coords_pose")(self.h, level, _f32(world), out)
        return out

    def world_coords_pose(self, level: int, mp):
        out = np.zeros(3, np.float32)
        self._fn("world_coords_pose")(self.h, level, _f32(mp), out)
        return out

    def logodds_increments(self):
        out = np.zeros(2, np.float32)
        self._fn("get_logodds_increments")(self.h, out)
        return out

    # --- the path ------------------------------------------------------------------------
    def update(self, pts, hint, map_without_matching=False, origo=(0.0, 0.0)):
        """HectorSlamProcessor::update — returns (pose, cov)."""
        pts = _f32(pts).reshape(-1, 2)
        pose, cov = np.zeros(3, np.float32), np.zeros(9, np.float32)
        self._fn("update")(self.h, pts, pts.shape[0], _f32(origo), _f32(hint), int(map_without_matching), pose, cov)
        return pose, cov.reshape(3, 3)

    def match(self, hint, pts, origo=(0.0, 0.0), cov_in=None):
        """MapRepMultiMap::matchData — returns (pose, cov)."""
        pts = _f32(pts).reshape(-1, 2)
        pose = np.zeros(3, np.float32)
        cov = np.zeros(9, np.float32) if cov_in is None else _f32(cov_in).reshape(9).copy()
        self._fn("match")(self.h, _f32(hint), pts, pts.shape[0], _f32(origo), pose, cov)
        return pose, cov.reshape(3, 3)

    def update_by_scan(self, pts, pose, origo=(0.0, 0.0)):
        pts = _f32(pts).reshape(-1, 2)
        self._fn("update_by_scan")(self.h, pts, pts.shape[0], _f32(origo), _f32(pose))

    def on_map_updated(self):
        self._fn("on_map_updated")(self.h)

    def get_logodds(self, level: int) -> np.ndarray:
        sx, sy = self.level_size(level)
        out = np.zeros((sy, sx), np.float32)
        self._fn("get_logodds")(self.h, level, out.reshape(-1))
        return out

    def set_logodds(self, level: int, plane):
        sx, sy = self.level_size(level)
        a = _f32(plane).reshape(-1)
        assert a.size == sx * sy
        self._fn("set_logodds")(self.h, level, a)

    def get_prob(self, level: int) -> np.ndarray:
        sx, sy = self.level_size(level)
        out = np.zeros((sy, sx), np.float32)
        self._fn("get_prob")(self.h, level, out.reshape(-1))
        return out

    def hessian_derivs(self, level: int, pose_map, pts_level):
        """getCompleteHessianDerivs on one level; pts in that level's cell units. -> (H 3x3, dTr 3)."""
        pts = _f32(pts_level).reshape(-1, 2)
        H, d = np.zeros(9, np.float32), np.zeros(3, np.float32)
        self._fn("hessian_derivs")(self.h, level, _f32(pose_map), pts, pts.shape[0], H, d)
        return H.reshape(3, 3), d

    def raycast(self, level: int, begin, end):
        """checkOccupancyBresenhami (port only). -> (dist, (hx, hy))"""
        fn = self.lib.hso_raycast
        fn.restype = C.c_float
        fn.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int)]
        hit = (C.c_int * 2)()
        d = fn(self.h, level, int(begin[0]), int(begin[1]), int(end[0]), int(end[1]), hit)
        return float(d), (int(hit[0]), int(hit[1]))

    def map_origin(self, level: int) -> np.ndarray:
        """nav_msgs/OccupancyGrid origin of the level (setServiceGetMapData; port only)."""
        fn = self.lib.hso_map_origin
        fn.restype = None
        fn.argtypes = [C.c_void_p, C.c_int, _f32p]
        out = np.zeros(2, np.float32)
        fn(self.h, level, out)
        return out

    def get_dist(self, level: int, begin_world, end_world):
        """DistanceMeasurementProvider::getDist (port only). -> (dist [m], hit_world (2,), found)"""
        fn = self.lib.hso_get_dist
        fn.restype = C.c_float
        fn.argtypes = [C.c_void_p, C.c_int, _f32p, _f32p, _f32p, C.POINTER(C.c_int)]
        hw, found = np.zeros(2, np.float32), C.c_int(0)
        d = fn(self.h, level, _f32(begin_world), _f32(end_world), hw, C.byref(found))
        return float(d), hw, bool(found.value)

    def likelihood(self, level: int, pose_map, pts_level) -> float:
        """OccGridMapUtil::getLikelihoodForState (state and points in the level's cell units)."""
        pts = _f32(pts_level).reshape(-1, 2)
        return float(self._fn("likelihood")(self.h, level, _f32(pose_map), pts, pts.shape[0]))

    def covariance_for_pose(self, level: int, pose_map, pts_level):
        """OccGridMapUtil::getCovarianceForPose + getCovMatrixWorldCoords. -> (cov_map 3x3, cov_world 3x3)"""
        pts = _f32(pts_level).reshape(-1, 2)
        cm, cw = np.zeros(9, np.float32), np.zeros(9, np.float32)
        self._fn("covariance_for_pose")(self.h, level, _f32(pose_map), pts, pts.shape[0], cm, cw)
        return cm.reshape(3, 3), cw.reshape(3, 3)

    def match_level(self, level: int, hint_world, pts_level, max_iterations: int):
        """ScanMatcher::matchData on one level (1 + max_iterations evaluations)."""
        pts = _f32(pts_level).reshape(-1, 2)
        pose, cov = np.zeros(3, np.float32), np.zeros(9, np.float32)
        self._fn("match_level")(self.h, level, _f32(hint_world), pts, pts.shape[0], int(max_iterations), pose, cov)
        return pose, cov.reshape(3, 3)

    def update_level(self, level: int, pts_level, pose_world, origo_level=(0.0, 0.0)):
        pts = _f32(pts_level).reshape(-1, 2)
        self._fn("update_level")(self.h, level, pts, pts.shape[0], _f32(origo_level), _f32(pose_world))

    def match_batch(self, hints, pts, offsets, nthreads: int = 1, want_cov: bool = True):
        """B independent matchData calls against the frozen map. -> (poses, covs, seconds)."""
        hints = _f32(hints).reshape(-1, 3)
        B = hints.shape[0]
        pts = _f32(pts).reshape(-1, 2)
        offsets = np.ascontiguousarray(offsets, dtype=np.int32)
        poses = np.zeros((B, 3), np.float32)
        covs = np.zeros((B, 9), np.float32)
        secs = self._fn("match_batch")(self.h, B, hints, pts, offsets, poses, covs, int(nthreads))
        return poses, covs.reshape(B, 3, 3), float(secs)


class RefMapTools:
    """hector_map_tools' DistanceMeasurementProvider compiled from the UNMODIFIED HectorMapTools.h
    (oracle/maptools_driver.cpp, reference kind only) over an occupancy grid (int8: 0 / 100 / -1)."""

    def __init__(self, occupancy: np.ndarray, resolution: float, origin_xy):
        self.lib = C.CDLL(REF_LIB)
        L = self.lib
        L.hsref_maptools_create.restype = C.c_void_p
        L.hsref_maptools_create.argtypes = [C.c_int, C.c_int, C.c_float, C.c_double, C.c_double, C.c_void_p]
        L.hsref_maptools_destroy.argtypes = [C.c_void_p]
        L.hsref_maptools_raycast.restype = C.c_float
        L.hsref_maptools_raycast.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int)]
        L.hsref_maptools_get_dist.restype = C.c_float
        L.hsref_maptools_get_dist.argtypes = [C.c_void_p, _f32p, _f32p, _f32p, C.POINTER(C.c_int)]
        occ = np.ascontiguousarray(occupancy, dtype=np.int8)
        self.h = L.hsref_maptools_create(occ.shape[1], occ.shape[0], resolution, float(origin_xy[0]), float(origin_xy[1]),
                                         occ.ctypes.data)

    def raycast(self, begin, end):
        hit = (C.c_int * 2)()
        d = self.lib.hsref_maptools_raycast(self.h, int(begin[0]), int(begin[1]), int(end[0]), int(end[1]), hit)
        return float(d), (int(hit[0]), int(hit[1]))

    def get_dist(self, begin_world, end_world):
        hw, found = np.zeros(2, np.float32), C.c_int(0)
        d = self.lib.hsref_maptools_get_dist(self.h, _f32(begin_world), _f32(end_world), hw, C.byref(found))
        return float(d), hw, bool(found.value)

    def close(self):
        if self.h:
            self.lib.hsref_maptools_destroy(self.h)
            self.h = None


def _conv_lib(kind: str):
    if kind == "reference":
        return C.CDLL(REF_LIB), "hsref_"
    return C.CDLL(PORT_LIB), "hso_"


def _util_lib(kind: str):
    if kind == "reference":
        return C.CDLL(REF_UTIL_LIB), "hsref_"
    return C.CDLL(PORT_LIB), "hso_"


def util_available(kind: str) -> bool:
    """the library behind normalize_angle / pose_difference_larger_than of `kind` is built"""
    return os.path.exists(REF_UTIL_LIB if kind == "reference" else PORT_LIB)


def normalize_angle(angles, kind: str = "port") -> np.ndarray:
    """util::normalize_angle of each float of `angles` (the reference's own, or the C port's) -> float32 array"""
    lib, p = _util_lib(kind)
    fn = getattr(lib, p + "normalize_angle")
    fn.restype = None
    fn.argtypes = [_f32p, C.c_int, _f32p]
    a = _f32(angles).reshape(-1)
    out = np.zeros_like(a)
    fn(a, a.size, out)
    return out


def pose_difference_larger_than(p1, p2, dist, ang, kind: str = "port") -> np.ndarray:
    """util::poseDifferenceLargerThan of each row pair of p1 / p2 (n, 3) with per-row thresholds -> bool array"""
    lib, p = _util_lib(kind)
    fn = getattr(lib, p + "pose_difference_larger_than")
    fn.restype = None
    fn.argtypes = [_f32p, _f32p, _f32p, _f32p, C.c_int, _i32p]
    a, b = _f32(p1).reshape(-1, 3), _f32(p2).reshape(-1, 3)
    n = a.shape[0]
    d, g = np.broadcast_to(_f32(dist), (n,)).copy(), np.broadcast_to(_f32(ang), (n,)).copy()
    out = np.zeros(n, np.int32)
    fn(a, b, d, g, n, out)
    return out != 0


def scan_to_points(ranges, angle_min, angle_increment, range_min, range_max, scale_to_map, kind: str = "port"):
    """rosLaserScanToDataContainer (HectorMappingRos.cpp:483-507): the C port, or (kind="reference") the node's own
    source text compiled by oracle/ros_conv_driver.cpp. -> (n, 2) float32"""
    lib, p = _conv_lib(kind)
    fn = getattr(lib, p + "scan_to_points")
    fn.restype = C.c_int
    fn.argtypes = [_f32p, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, _f32p]
    r = _f32(ranges).reshape(-1)
    out = np.zeros(2 * r.size, np.float32)
    n = fn(r, r.size, angle_min, angle_increment, range_min, range_max, scale_to_map, out)
    return out[: 2 * n].reshape(n, 2).copy()


def cloud_to_points(xyz, transform, sqr_min_dist, sqr_max_dist, z_min, z_max, scale_to_map, kind: str = "port"):
    """rosPointCloudToDataContainer (HectorMappingRos.cpp:509-542). xyz: (n, 3) float32 points in the laser frame
    (sensor_msgs/PointCloud.points), transform: 12 float64, rows of [R | t] base <- laser.
    -> (endpoints (k, 2) float32 in map cells, origo (2,) float32)"""
    lib, p = _conv_lib(kind)
    fn = getattr(lib, p + "cloud_to_points")
    fn.restype = C.c_int
    fn.argtypes = [_f32p, C.c_int, np.ctypeslib.ndpointer(dtype=np.float64, flags="C_CONTIGUOUS"), C.c_float, C.c_float,
                   C.c_float, C.c_float, C.c_float, _f32p, _f32p]
    pts = _f32(xyz).reshape(-1, 3)
    T = np.ascontiguousarray(transform, dtype=np.float64).reshape(12)
    out = np.zeros(2 * max(1, pts.shape[0]), np.float32)
    origo = np.zeros(2, np.float32)
    n = fn(pts.reshape(-1), pts.shape[0], T, sqr_min_dist, sqr_max_dist, z_min, z_max, scale_to_map, out, origo)
    return out[: 2 * n].reshape(n, 2).copy(), origo


def build_map_by_slam(orc: Oracle, world, scale_to_map: float = 20.0, noise_seed: int = 11, sigma: float = 0.01):
    """SLAM-mode map building, exactly what the reference node does: HectorSlamProcessor::update
    along the world's mapping poses, hint = ground truth, thresholds 0 so every scan writes.
    Only meaningful for single-room worlds (the matcher may slide along a shared wall when it
    enters an unmapped room)."""
    from hector_slam_b200 import synth

    rng = np.random.default_rng(noise_seed)
    orc.set_map_update_thresholds(0.0, 0.0)
    poses = world.mapping_poses()
    est = []
    for p in poses:
        scan = synth.make_scan(world, p, rng, scale_to_map, sigma)
        pose, _ = orc.update(scan, p.astype(np.float32))
        est.append(pose)
    return poses, np.asarray(est)


def build_map_known_poses(orc: Oracle, world, scale_to_map: float = 20.0, noise_seed: int = 11, sigma: float = 0.01):
    """Mapping with known poses through the MapRepresentationInterface calls: matchData (its result
    is discarded; the call is what fills the coarse levels' scaled containers, MapRepMultiMap.h:127,
    which updateByScan then reuses, :143) followed by updateByScan at the TRUE pose and
    onMapUpdated.  Gives a map registered to the synthetic world for any number of rooms."""
    from hector_slam_b200 import synth

    rng = np.random.default_rng(noise_seed)
    poses = world.mapping_poses()
    for p in poses:
        scan = synth.make_scan(world, p, rng, scale_to_map, sigma)
        p32 = p.astype(np.float32)
        orc.match(p32, scan)
        orc.update_by_scan(scan, p32)
        orc.on_map_updated()
    return poses
