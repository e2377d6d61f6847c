"""ctypes binding of the C-ABI in include/hector_slam_b200.h (lib/libhsb200.so).

Python here is plumbing only (tests, bench.py, multi-GPU launcher): device memory and streams may
come from torch, everything that computes goes through the C-ABI into the CUDA kernels.  There is
no CPU fallback — if the library is missing or no GPU is visible, calls raise.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("HSB_LIB_PATH") or os.path.join(_PKG, "lib", "libhsb200.so")
HSB_MAX_LEVELS = 8

GATHER_AUTO, GATHER_LDG, GATHER_TEX = 0, 1, 2

# every symbol include/hector_slam_b200.h declares (tests check the .so exports them all)
EXPORTED = [
    "hsb_create", "hsb_destroy", "hsb_reset", "hsb_set_update_factor_free", "hsb_set_update_factor_occupied",
    "hsb_get_logodds_increments", "hsb_get_scale_to_map", "hsb_get_map_levels", "hsb_get_level_info",
    "hsb_map_coords_pose", "hsb_world_coords_pose", "hsb_match_data", "hsb_match_batch", "hsb_match_batch_device",
    "hsb_hessian_derivs", "hsb_update_by_scan", "hsb_update_level_by_scan", "hsb_on_map_updated",
    "hsb_set_map_update_min_dist_diff", "hsb_set_map_update_min_angle_diff", "hsb_slam_update",
    "hsb_slam_update_nowait", "hsb_slam_update_cloud", "hsb_get_last_map_update_pose", "hsb_set_last_map_update_pose",
    "hsb_upload_level", "hsb_download_level", "hsb_download_prob", "hsb_level_logodds_device_ptr",
    "hsb_refresh_level", "hsb_last_error", "hsb_status_string", "hsb_get_launch_count", "hsb_get_gather_mode",
    "hsb_set_tuning", "hsb_version", "hsb_set_scan_format", "hsb_scan_to_points", "hsb_match_batch_ranges",
    "hsb_match_batch_ranges_device", "hsb_download_occupancy", "hsb_likelihood_batch", "hsb_likelihood_batch_device", "hsb_best_hypothesis_device",
    "hsb_get_dirty_rect", "hsb_pack_rect_device", "hsb_unpack_rect_device", "hsb_raycast_batch",
    "hsb_read_trace", "hsb_get_last_launch_shape", "hsb_get_last_update_device_ms",
    "hsb_match_batch_submit", "hsb_match_batch_ranges_submit", "hsb_match_batch_cloud_submit", "hsb_match_batch_wait",
    "hsb_alloc_pinned", "hsb_free_pinned", "hsb_measure_h2d_gbs", "hsb_get_dirty_rects", "hsb_pack_dirty_device", "hsb_unpack_dirty_device", "hsb_get_replication_overflows", "hsb_get_mirror_dirty_rect", "hsb_download_level_rect", "hsb_download_occupancy_rect",
    "hsb_get_d2h_bytes", "hsb_covariance_batch", "hsb_get_map_origin", "hsb_get_dist_batch", "hsb_set_cloud_format", "hsb_cloud_to_points", "hsb_match_batch_cloud", "hsb_match_batch_cloud_device",
    "hsb_get_match_record_floats", "hsb_match_data_record", "hsb_match_batch_record_device",
    "hsb_group_create", "hsb_group_destroy", "hsb_group_slam_update", "hsb_group_slam_update_cloud",
    "hsb_slam_update_ranges", "hsb_group_slam_update_ranges",
    "hsb_set_laser_projection", "hsb_projected_scan_to_points", "hsb_slam_update_projected",
    "hsb_group_slam_update_projected", "hsb_match_batch_projected", "hsb_match_batch_projected_submit",
    "hsb_match_batch_projected_device",
    "hsb_group_slam_update_subset", "hsb_group_slam_update_cloud_subset", "hsb_group_slam_update_ranges_subset",
    "hsb_group_slam_update_projected_subset", "hsb_group_sync_occupancy", "hsb_group_sync_occupancy_subset",
    "hsb_group_get_dist", "hsb_group_get_dist_subset", "hsb_group_raycast", "hsb_group_raycast_subset",
    "hsb_group_likelihood", "hsb_group_likelihood_subset", "hsb_group_covariance", "hsb_group_covariance_subset",
    "hsb_group_best_hypothesis", "hsb_group_best_hypothesis_subset",
    "hsb_group_match_batch", "hsb_group_match_batch_subset",
    "hsb_group_pack_dirty_device", "hsb_group_pack_dirty_device_subset", "hsb_group_unpack_dirty_device",
    "hsb_group_create_mixed", "hsb_group_create_heterogeneous", "hsb_group_reset", "hsb_group_reset_subset",
    "hsb_get_level_evals", "hsb_set_step_record", "hsb_get_step_record", "hsb_get_last_match_scan",
]


class HsbConfig(C.Structure):
    _fields_ = [
        ("map_resolution", C.c_float),
        ("map_size_x", C.c_int),
        ("map_size_y", C.c_int),
        ("start_x", C.c_float),
        ("start_y", C.c_float),
        ("levels", C.c_int),
        ("device", C.c_int),
        ("max_iterations", C.c_int * HSB_MAX_LEVELS),
        ("update_factor_free", C.c_float),
        ("update_factor_occupied", C.c_float),
        ("gather_mode", C.c_int),
        ("reserved", C.c_int * 7),
    ]


class HsbScanFormat(C.Structure):
    _fields_ = [("n_beams", C.c_int), ("angle_min", C.c_float), ("angle_increment", C.c_float),
                ("range_min", C.c_float), ("range_max", C.c_float)]


class HsbCloudFormat(C.Structure):
    _fields_ = [("laser_transform", C.c_double * 12), ("sqr_laser_min_dist", C.c_float), ("sqr_laser_max_dist", C.c_float),
                ("laser_z_min_value", C.c_float), ("laser_z_max_value", C.c_float)]


class HsbLaserProjection(C.Structure):
    _fields_ = [("n_beams", C.c_int), ("angle_min", C.c_float), ("angle_increment", C.c_float),
                ("range_min", C.c_float), ("range_max", C.c_float), ("range_cutoff", C.c_double)]


class HsbError(RuntimeError):
    def __init__(self, status: int, msg: str):
        super().__init__(f"hsb status {status}: {msg}")
        self.status = status


_lib = None


def load_library() -> C.CDLL:
    """Load lib/libhsb200.so (built in-tree by hector_slam_b200.build). Raises if it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise FileNotFoundError(
            f"{LIB_PATH} not found — build it with `python -m hector_slam_b200.build` (nvcc, sm_90a). "
            "There is no CPU fallback.")
    L = C.CDLL(LIB_PATH)
    vp, f, i, fp, ip = C.c_void_p, C.c_float, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_int)

    def sig(name, res, *args):
        fn = getattr(L, name)
        fn.restype = res
        fn.argtypes = list(args)

    sig("hsb_create", i, C.POINTER(HsbConfig), C.POINTER(vp))
    sig("hsb_destroy", i, vp)
    sig("hsb_reset", i, vp)
    sig("hsb_set_update_factor_free", i, vp, f)
    sig("hsb_set_update_factor_occupied", i, vp, f)
    sig("hsb_get_logodds_increments", i, vp, vp)
    sig("hsb_get_scale_to_map", f, vp)
    sig("hsb_get_map_levels", i, vp)
    sig("hsb_get_level_info", i, vp, i, ip, ip, fp)
    sig("hsb_map_coords_pose", i, vp, i, vp, vp)
    sig("hsb_world_coords_pose", i, vp, i, vp, vp)
    sig("hsb_match_data", i, vp, vp, vp, i, vp, vp, vp)
    sig("hsb_match_batch", i, vp, i, vp, vp, vp, i, vp, vp)
    sig("hsb_match_batch_device", i, vp, i, vp, vp, vp, i, i, vp, vp, vp)
    sig("hsb_get_match_record_floats", i, vp)
    sig("hsb_match_data_record", i, vp, vp, vp, i, vp, vp, vp, vp)
    sig("hsb_match_batch_record_device", i, vp, i, vp, vp, vp, i, i, vp, vp, vp, vp)
    sig("hsb_hessian_derivs", i, vp, i, vp, vp, i, vp, vp)
    sig("hsb_update_by_scan", i, vp, vp, i, vp, vp)
    sig("hsb_update_level_by_scan", i, vp, i, vp, i, vp, vp)
    sig("hsb_on_map_updated", i, vp)
    sig("hsb_set_map_update_min_dist_diff", i, vp, f)
    sig("hsb_set_map_update_min_angle_diff", i, vp, f)
    sig("hsb_slam_update", i, vp, vp, vp, i, vp, i, vp, vp, vp)
    sig("hsb_slam_update_nowait", i, vp, vp, vp, i, vp, i, vp, vp, vp)
    sig("hsb_slam_update_cloud", i, vp, vp, vp, i, vp, i, i, vp, vp, vp, vp)
    sig("hsb_slam_update_ranges", i, vp, vp, vp, i, i, i, vp, vp, vp, vp)
    sig("hsb_set_laser_projection", i, vp, C.POINTER(HsbLaserProjection))
    sig("hsb_projected_scan_to_points", i, vp, vp, i, vp, vp, ip, vp)
    sig("hsb_slam_update_projected", i, vp, vp, vp, i, vp, i, i, vp, vp, vp, vp)
    sig("hsb_match_batch_projected", i, vp, i, vp, vp, vp, vp, vp, vp)
    sig("hsb_match_batch_projected_submit", i, vp, i, vp, vp, vp, vp, vp, vp, ip)
    sig("hsb_match_batch_projected_device", i, vp, i, vp, vp, vp, vp, vp, vp, vp)
    sig("hsb_get_last_map_update_pose", i, vp, vp)
    sig("hsb_set_last_map_update_pose", i, vp, vp)
    sig("hsb_upload_level", i, vp, i, vp)
    sig("hsb_download_level", i, vp, i, vp)
    sig("hsb_download_prob", i, vp, i, vp)
    sig("hsb_level_logodds_device_ptr", vp, vp, i)
    sig("hsb_refresh_level", i, vp, i, vp)
    sig("hsb_last_error", C.c_char_p, vp)
    sig("hsb_status_string", C.c_char_p, i)
    sig("hsb_get_launch_count", C.c_uint64, vp)
    sig("hsb_get_gather_mode", i, vp)
    sig("hsb_set_tuning", i, vp, C.c_char_p, i)
    sig("hsb_version", C.c_char_p)
    sig("hsb_set_scan_format", i, vp, C.POINTER(HsbScanFormat))
    sig("hsb_scan_to_points", i, vp, vp, vp, ip)
    sig("hsb_match_batch_ranges", i, vp, i, vp, vp, vp, vp)
    sig("hsb_match_batch_ranges_device", i, vp, i, vp, vp, vp, vp, vp)
    sig("hsb_download_occupancy", i, vp, i, vp)
    sig("hsb_likelihood_batch", i, vp, i, i, vp, vp, vp, i, vp)
    sig("hsb_likelihood_batch_device", i, vp, i, i, vp, vp, vp, i, vp, vp)
    sig("hsb_best_hypothesis_device", i, vp, i, i, vp, vp, vp, i, vp, vp, vp)
    sig("hsb_covariance_batch", i, vp, i, i, vp, vp, vp, i, vp, vp)
    sig("hsb_get_map_origin", i, vp, i, vp)
    sig("hsb_get_dist_batch", i, vp, i, i, vp, vp, vp, vp, vp)
    sig("hsb_get_dirty_rect", i, vp, i, vp, i)
    sig("hsb_get_dirty_rects", i, vp, vp, i)
    sig("hsb_pack_dirty_device", i, vp, vp, C.c_size_t, i, vp)
    sig("hsb_unpack_dirty_device", i, vp, vp, C.c_size_t, vp)
    sig("hsb_get_replication_overflows", i, vp, ip, i)
    sig("hsb_get_mirror_dirty_rect", i, vp, i, vp, i)
    sig("hsb_download_level_rect", i, vp, i, vp, vp)
    sig("hsb_download_occupancy_rect", i, vp, i, vp, vp)
    sig("hsb_get_d2h_bytes", C.c_uint64, vp)
    sig("hsb_raycast_batch", i, vp, i, i, vp, vp, vp, vp)
    sig("hsb_set_cloud_format", i, vp, C.POINTER(HsbCloudFormat))
    sig("hsb_cloud_to_points", i, vp, vp, i, vp, ip, vp)
    sig("hsb_match_batch_cloud", i, vp, i, vp, vp, vp, vp, vp, vp, vp)
    sig("hsb_match_batch_cloud_device", i, vp, i, vp, vp, vp, i, vp, vp, vp, vp, vp)
    sig("hsb_match_batch_submit", i, vp, i, vp, vp, vp, i, vp, vp, ip)
    sig("hsb_match_batch_ranges_submit", i, vp, i, vp, vp, vp, vp, ip)
    sig("hsb_match_batch_cloud_submit", i, vp, i, vp, vp, vp, vp, vp, vp, vp, ip)
    sig("hsb_match_batch_wait", i, vp, i)
    sig("hsb_alloc_pinned", vp, C.c_size_t)
    sig("hsb_free_pinned", i, vp)
    sig("hsb_measure_h2d_gbs", i, vp, vp, C.c_size_t, i, fp)
    sig("hsb_get_last_update_device_ms", i, vp, fp)
    sig("hsb_read_trace", i, vp, vp, i)
    sig("hsb_get_last_launch_shape", i, vp, vp)
    sig("hsb_pack_rect_device", i, vp, i, vp, vp, vp)
    sig("hsb_unpack_rect_device", i, vp, i, vp, vp, vp)
    sig("hsb_group_create", i, vp, i, C.POINTER(vp))
    sig("hsb_group_create_mixed", i, vp, i, C.POINTER(vp))
    sig("hsb_group_create_heterogeneous", i, vp, i, C.POINTER(vp))
    sig("hsb_group_destroy", i, vp)
    sig("hsb_group_slam_update", i, vp, vp, vp, vp, vp, vp, i, vp, vp, vp)
    sig("hsb_group_slam_update_cloud", i, vp, vp, vp, vp, vp, vp, i, vp, vp, vp, vp)
    sig("hsb_group_slam_update_ranges", i, vp, vp, vp, vp, vp, i, vp, vp, vp, vp)
    sig("hsb_group_slam_update_projected", i, vp, vp, vp, vp, vp, vp, i, vp, vp, vp, vp)
    sig("hsb_group_slam_update_subset", i, vp, i, vp, vp, vp, vp, vp, vp, i, vp, vp, vp)
    sig("hsb_group_slam_update_cloud_subset", i, vp, i, vp, vp, vp, vp, vp, vp, i, vp, vp, vp, vp)
    sig("hsb_group_slam_update_ranges_subset", i, vp, i, vp, vp, vp, vp, vp, i, vp, vp, vp, vp)
    sig("hsb_group_slam_update_projected_subset", i, vp, i, vp, vp, vp, vp, vp, vp, i, vp, vp, vp, vp)
    sig("hsb_group_sync_occupancy", i, vp, i, vp, vp, i)
    sig("hsb_group_sync_occupancy_subset", i, vp, i, vp, i, vp, vp, i)
    sig("hsb_group_get_dist", i, vp, i, vp, vp, vp, vp, vp, vp)
    sig("hsb_group_get_dist_subset", i, vp, i, vp, i, vp, vp, vp, vp, vp, vp)
    sig("hsb_group_raycast", i, vp, i, vp, vp, vp, vp, vp)
    sig("hsb_group_raycast_subset", i, vp, i, vp, i, vp, vp, vp, vp, vp)
    sig("hsb_group_likelihood", i, vp, i, vp, vp, vp, vp, vp)
    sig("hsb_group_likelihood_subset", i, vp, i, vp, i, vp, vp, vp, vp, vp)
    sig("hsb_group_covariance", i, vp, i, vp, vp, vp, vp, vp, vp)
    sig("hsb_group_covariance_subset", i, vp, i, vp, i, vp, vp, vp, vp, vp, vp)
    sig("hsb_group_best_hypothesis", i, vp, i, vp, vp, vp, vp, vp, vp, vp)
    sig("hsb_group_best_hypothesis_subset", i, vp, i, vp, i, vp, vp, vp, vp, vp, vp, vp)
    sig("hsb_group_match_batch", i, vp, vp, vp, vp, vp, vp, vp)
    sig("hsb_group_match_batch_subset", i, vp, i, vp, vp, vp, vp, vp, vp, vp)
    sig("hsb_group_pack_dirty_device", i, vp, vp, C.c_size_t, i, vp)
    sig("hsb_group_pack_dirty_device_subset", i, vp, i, vp, vp, C.c_size_t, i, vp)
    sig("hsb_group_unpack_dirty_device", i, vp, vp, C.c_size_t, vp)
    sig("hsb_group_reset", i, vp)
    sig("hsb_group_reset_subset", i, vp, i, vp)
    sig("hsb_get_level_evals", i, vp, i)
    sig("hsb_set_step_record", i, vp, i)
    sig("hsb_get_step_record", i, vp, vp, vp)
    sig("hsb_get_last_match_scan", i, vp, vp, i, vp, vp)
    _lib = L
    return L


def _ptr(a):
    """Host pointer of a contiguous numpy array / torch CPU tensor, or None."""
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data
    if hasattr(a, "data_ptr"):
        return a.data_ptr()
    raise TypeError(type(a))


def _f32(a, shape=None):
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a if shape is None else a.reshape(shape)


class PinnedArray:
    """A numpy view of page-locked host memory from hsb_alloc_pinned (cudaHostAlloc by the calling thread)."""

    def __init__(self, shape, dtype=np.float32):
        self.lib = load_library()
        self.shape = tuple(int(x) for x in (shape if isinstance(shape, (tuple, list)) else (shape,)))
        self.dtype = np.dtype(dtype)
        nbytes = int(np.prod(self.shape)) * self.dtype.itemsize
        self.ptr = self.lib.hsb_alloc_pinned(max(1, nbytes))
        if not self.ptr:
            raise MemoryError(f"hsb_alloc_pinned({nbytes}) failed")
        buf = (C.c_char * max(1, nbytes)).from_address(self.ptr)
        self.array = np.frombuffer(buf, dtype=self.dtype, count=int(np.prod(self.shape))).reshape(self.shape)

    def free(self):
        if getattr(self, "ptr", None):
            self.array = None
            self.lib.hsb_free_pinned(self.ptr)
            self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def pinned_copy(a: np.ndarray) -> PinnedArray:
    p = PinnedArray(a.shape, a.dtype)
    p.array[...] = a
    return p


class MapRepB200:
    """The C-ABI handle with MapRepresentationInterface's method names
    (slam_main/MapRepresentationInterface.h:38-62), numpy in / numpy out."""

    def __init__(self, map_resolution: float, map_size_x: int, map_size_y: int | None = None, levels: int = 3,
                 start=(0.5, 0.5), device: int = 0, max_iterations=None, update_factor_free: float = 0.0,
                 update_factor_occupied: float = 0.0, gather_mode: int = GATHER_AUTO):
        self.lib = load_library()
        cfg = HsbConfig()
        cfg.map_resolution = map_resolution
        cfg.map_size_x = int(map_size_x)
        cfg.map_size_y = int(map_size_x if map_size_y is None else map_size_y)
        cfg.start_x, cfg.start_y = float(start[0]), float(start[1])
        cfg.levels = int(levels)
        cfg.device = int(device)
        if max_iterations is not None:
            for k, v in enumerate(max_iterations):
                cfg.max_iterations[k] = int(v)
        cfg.update_factor_free = update_factor_free
        cfg.update_factor_occupied = update_factor_occupied
        cfg.gather_mode = gather_mode
        self.cfg = cfg
        h = C.c_void_p()
        st = self.lib.hsb_create(C.byref(cfg), C.byref(h))
        if st != 0:
            raise HsbError(st, (self.lib.hsb_last_error(None) or b"").decode())
        self.h = h
        self.levels = int(levels)
        self.device = int(device)

    # -- plumbing --------------------------------------------------------------------------------
    def _check(self, st: int):
        if st != 0:
            raise HsbError(st, (self.lib.hsb_last_error(self.h) or b"").decode())

    def close(self):
        if getattr(self, "h", None):
            self.lib.hsb_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_tuning(self, **kw):
        for k, v in kw.items():
            self._check(self.lib.hsb_set_tuning(self.h, k.encode(), int(v)))

    def last_launch_shape(self) -> dict:
        out = (C.c_int * 6)()
        self._check(self.lib.hsb_get_last_launch_shape(self.h, out))
        return dict(zip(("warps_per_scan", "scans_per_block", "unroll", "staged_points", "grid", "resident_ctas"),
                        (int(v) for v in out)))

    def last_update_device_ms(self) -> float:
        ms = C.c_float()
        self._check(self.lib.hsb_get_last_update_device_ms(self.h, C.byref(ms)))
        return float(ms.value)

    def read_trace(self, max_scans: int) -> np.ndarray:
        out = np.zeros((max_scans, 8), np.uint64)
        n = self.lib.hsb_read_trace(self.h, out.ctypes.data, max_scans)
        if n < 0:
            self._check(n)
        return out[:n]

    @property
    def launch_count(self) -> int:
        return int(self.lib.hsb_get_launch_count(self.h))

    @property
    def gather_mode(self) -> int:
        return int(self.lib.hsb_get_gather_mode(self.h))

    # -- MapRepresentationInterface ------------------------------------------------------------------
    def reset(self):
        self._check(self.lib.hsb_reset(self.h))

    def getScaleToMap(self) -> float:
        return float(self.lib.hsb_get_scale_to_map(self.h))

    def getMapLevels(self) -> int:
        return int(self.lib.hsb_get_map_levels(self.h))

    def level_info(self, level: int):
        sx, sy, cl = C.c_int(), C.c_int(), C.c_float()
        self._check(self.lib.hsb_get_level_info(self.h, level, C.byref(sx), C.byref(sy), C.byref(cl)))
        return sx.value, sy.value, cl.value

    def setUpdateFactorFree(self, f: float):
        self._check(self.lib.hsb_set_update_factor_free(self.h, f))

    def setUpdateFactorOccupied(self, f: float):
        self._check(self.lib.hsb_set_update_factor_occupied(self.h, f))

    def logodds_increments(self):
        out = np.zeros(2, np.float32)
        self._check(self.lib.hsb_get_logodds_increments(self.h, out.ctypes.data))
        return out

    def map_coords_pose(self, level: int, world):
        w, out = _f32(world, 3), np.zeros(3, np.float32)
        self._check(self.lib.hsb_map_coords_pose(self.h, level, w.ctypes.data, out.ctypes.data))
        return out

    def world_coords_pose(self, level: int, mp):
        m, out = _f32(mp, 3), np.zeros(3, np.float32)
        self._check(self.lib.hsb_world_coords_pose(self.h, level, m.ctypes.data, out.ctypes.data))
        return out

    def matchData(self, begin_estimate_world, points_xy, cov_inout=None, origo=None, record: bool = False):
        """-> (pose (3,), cov (3,3)), or with record=True (pose, cov, record) where record is split_record() of the
        scan's per-evaluation record.  cov_inout is returned untouched for an empty scan."""
        hint = _f32(begin_estimate_world, 3)
        pts = _f32(points_xy).reshape(-1, 2)
        pose = np.zeros(3, np.float32)
        cov = np.zeros(9, np.float32) if cov_inout is None else _f32(cov_inout).reshape(9).copy()
        og = None if origo is None else _f32(origo, 2)
        args = (self.h, hint.ctypes.data, pts.ctypes.data if pts.size else None, pts.shape[0], _ptr(og), pose.ctypes.data,
                cov.ctypes.data)
        if not record:
            self._check(self.lib.hsb_match_data(*args))
            return pose, cov.reshape(3, 3)
        rec = np.zeros(self.record_floats, np.float32)
        self._check(self.lib.hsb_match_data_record(*args, rec.ctypes.data))
        return pose, cov.reshape(3, 3), self.split_record(rec)

    match_data = matchData

    # -- per-evaluation record (include/hector_slam_b200.h, hsb_get_match_record_floats) -------------
    @property
    def record_floats(self) -> int:
        """R: floats of one scan's record"""
        r = int(self.lib.hsb_get_match_record_floats(self.h))
        if r < 0:
            self._check(r)
        return r

    def level_evals(self) -> list[int]:
        """Gauss-Newton evaluations per level, level 0 first (maxIterations + 1, the defaults 5 / 3 for a zero entry)"""
        out = []
        for l in range(self.levels):
            e = int(self.lib.hsb_get_level_evals(self.h, l))
            if e < 0:
                self._check(e)
            out.append(e)
        return out

    # -- the fused steps' record (hsb_set_step_record) ---------------------------------------------
    def set_step_record(self, on: bool = True):
        """Every matched fused SLAM step of this handle (single or group) records its match from now on."""
        self._check(self.lib.hsb_set_step_record(self.h, int(bool(on))))

    def step_record(self, raw: bool = False):
        """The record of the handle's last fused step: split_record() of it (raw=True: the (R,) float32 array), or None
        when that step ran no match (map_without_matching, or no step since recording was turned on)."""
        rec = np.zeros(self.record_floats, np.float32)
        matched = C.c_int(0)
        self._check(self.lib.hsb_get_step_record(self.h, rec.ctypes.data, C.byref(matched)))
        if not matched.value:
            return None
        return rec if raw else self.split_record(rec)

    def last_match_scan(self):
        """-> (endpoints (n, 2) in level-0 cells, origo (2,)): the container of the handle's last matched scan."""
        n, origo = C.c_int(0), np.zeros(2, np.float32)
        st = self.lib.hsb_get_last_match_scan(self.h, None, 0, C.byref(n), origo.ctypes.data)
        if st != 0 and n.value == 0:
            self._check(st)
        pts = np.zeros((max(n.value, 1), 2), np.float32)
        self._check(self.lib.hsb_get_last_match_scan(self.h, pts.ctypes.data, pts.shape[0], C.byref(n), origo.ctypes.data))
        return pts[:n.value].copy(), origo

    def split_record(self, rec) -> list[dict]:
        """(..., R) float32 records -> one dict per level, INDEXED BY LEVEL (0 = finest):
        start (..., 3) world pose the level starts from, H (..., E, 3, 3), dTr (..., E, 3), est (..., E, 3) the
        estimate after each evaluation's step in the level's map cells."""
        rec = np.asarray(rec, np.float32)
        assert rec.shape[-1] == self.record_floats, (rec.shape, self.record_floats)
        lead = rec.shape[:-1]
        evals = self.level_evals()
        out = [None] * self.levels
        off = 0
        for l in range(self.levels - 1, -1, -1):
            E = evals[l]
            start = rec[..., off:off + 3]
            ev = rec[..., off + 3:off + 3 + 15 * E].reshape(lead + (E, 15))
            out[l] = dict(start=start.copy(), H=ev[..., :9].reshape(lead + (E, 3, 3)).copy(), dTr=ev[..., 9:12].copy(),
                          est=ev[..., 12:15].copy())
            off += 3 + 15 * E
        return out

    def match_batch_record_device(self, B: int, d_hints: int, d_points: int, d_offsets: int | None, n_shared: int,
                                  max_points_per_scan: int, d_out_poses: int, d_out_cov: int | None, d_record: int,
                                  stream: int = 0):
        """match_batch_device plus the records: d_record holds B x record_floats float32 (device); asynchronous."""
        self._check(self.lib.hsb_match_batch_record_device(self.h, int(B), d_hints, d_points, d_offsets, int(n_shared),
                                                           int(max_points_per_scan), d_out_poses, d_out_cov, d_record,
                                                           stream))

    def match_batch_record(self, hints, points_xy, offsets=None):
        """A batch with records through the device entry point (torch allocates the device buffers).
        -> (poses (B, 3), cov (B, 3, 3), records: split_record() of the (B, R) array, raw (B, R) array)"""
        import torch

        hints = _f32(hints).reshape(-1, 3)
        pts = _f32(points_xy).reshape(-1, 2)
        B = hints.shape[0]
        dev = torch.device("cuda", self.device)
        d_h = torch.from_numpy(hints).to(dev)
        d_p = torch.from_numpy(pts if pts.size else np.zeros((1, 2), np.float32)).to(dev)
        if offsets is None:
            d_o, n_shared, max_n = None, pts.shape[0], pts.shape[0]
        else:
            offsets = np.ascontiguousarray(offsets, dtype=np.int32)
            d_o = torch.from_numpy(offsets).to(dev)
            n_shared, max_n = 0, int(np.diff(offsets).max()) if B else 0
        poses = torch.zeros((B, 3), dtype=torch.float32, device=dev)
        cov = torch.zeros((B, 9), dtype=torch.float32, device=dev)
        rec = torch.zeros((B, self.record_floats), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream().cuda_stream
            self.match_batch_record_device(B, d_h.data_ptr(), d_p.data_ptr(), None if d_o is None else d_o.data_ptr(),
                                           n_shared, max_n, poses.data_ptr(), cov.data_ptr(), rec.data_ptr(), stream)
            torch.cuda.current_stream().synchronize()
        raw = rec.cpu().numpy()
        return poses.cpu().numpy(), cov.cpu().numpy().reshape(B, 3, 3), self.split_record(raw), raw

    def updateByScan(self, points_xy, robot_pose_world, origo=None):
        pts = _f32(points_xy).reshape(-1, 2)
        pose = _f32(robot_pose_world, 3)
        og = None if origo is None else _f32(origo, 2)
        self._check(self.lib.hsb_update_by_scan(self.h, pts.ctypes.data if pts.size else None, pts.shape[0], _ptr(og),
                                                pose.ctypes.data))

    def onMapUpdated(self):
        self._check(self.lib.hsb_on_map_updated(self.h))

    # -- one SLAM step (HectorSlamProcessor::update, HectorSlamProcessor.h:71-113) ------------------
    def setMapUpdateMinDistDiff(self, d: float):
        self._check(self.lib.hsb_set_map_update_min_dist_diff(self.h, float(d)))

    def setMapUpdateMinAngleDiff(self, a: float):
        self._check(self.lib.hsb_set_map_update_min_angle_diff(self.h, float(a)))

    def slam_update(self, pose_hint_world, points_xy, map_without_matching: bool = False, cov_inout=None, origo=None,
                    nowait: bool = False):
        """match -> gate -> updateByScan -> onMapUpdated in one stream-ordered call (nowait: return when the pose has
        arrived, the map write continues on the handle's stream).  -> (pose (3,), cov (3,3), map_updated: bool)"""
        hint = _f32(pose_hint_world, 3)
        pts = _f32(points_xy).reshape(-1, 2)
        pose = np.zeros(3, np.float32)
        cov = np.zeros(9, np.float32) if cov_inout is None else _f32(cov_inout).reshape(9).copy()
        og = None if origo is None else _f32(origo, 2)
        upd = C.c_int(0)
        fn = self.lib.hsb_slam_update_nowait if nowait else self.lib.hsb_slam_update
        self._check(fn(self.h, hint.ctypes.data, pts.ctypes.data if pts.size else None,
                       pts.shape[0], _ptr(og), int(bool(map_without_matching)),
                       pose.ctypes.data, cov.ctypes.data, C.addressof(upd)))
        return pose, cov.reshape(3, 3), bool(upd.value)

    def slam_update_cloud(self, pose_hint_world, points_xyz, transform=None, map_without_matching: bool = False,
                          nowait: bool = False, cov_inout=None):
        """scanCallback's default branch in one call: cloud -> endpoints (fused), match, gate, map write.
        -> (pose (3,), cov (3,3), map_updated: bool, kept endpoints: int)"""
        hint = _f32(pose_hint_world, 3)
        pts = _f32(points_xyz).reshape(-1, 3)
        T = None if transform is None else np.ascontiguousarray(transform, dtype=np.float64).reshape(12)
        pose = np.zeros(3, np.float32)
        cov = np.zeros(9, np.float32) if cov_inout is None else _f32(cov_inout).reshape(9).copy()
        upd, kept = C.c_int(0), C.c_int(0)
        self._check(self.lib.hsb_slam_update_cloud(self.h, hint.ctypes.data, pts.ctypes.data if pts.size else None,
                                                   pts.shape[0], _ptr(T), int(bool(map_without_matching)), int(bool(nowait)),
                                                   pose.ctypes.data, cov.ctypes.data, C.addressof(upd), C.addressof(kept)))
        return pose, cov.reshape(3, 3), bool(upd.value), int(kept.value)

    def slam_update_ranges(self, pose_hint_world, ranges, map_without_matching: bool = False, nowait: bool = False,
                           cov_inout=None):
        """scanCallback's branch without the laser tf in one call: raw ranges in the scan format (set_scan_format) ->
        endpoints (fused), match, gate, map write.  -> (pose (3,), cov (3,3), map_updated: bool, kept endpoints: int)"""
        hint = _f32(pose_hint_world, 3)
        r = _f32(ranges).reshape(-1)
        pose = np.zeros(3, np.float32)
        cov = np.zeros(9, np.float32) if cov_inout is None else _f32(cov_inout).reshape(9).copy()
        upd, kept = C.c_int(0), C.c_int(0)
        self._check(self.lib.hsb_slam_update_ranges(self.h, hint.ctypes.data, r.ctypes.data, r.size,
                                                    int(bool(map_without_matching)), int(bool(nowait)), pose.ctypes.data,
                                                    cov.ctypes.data, C.addressof(upd), C.addressof(kept)))
        return pose, cov.reshape(3, 3), bool(upd.value), int(kept.value)

    def slam_update_projected(self, pose_hint_world, ranges, transform=None, map_without_matching: bool = False,
                              nowait: bool = False, cov_inout=None):
        """scanCallback's default branch from the LaserScan itself: raw ranges -> laser_geometry's projection (the
        handle's set_laser_projection) -> cloud rule (set_cloud_format) -> match, gate, map write, all fused.
        transform: 12 float64 (None = the cloud format's).  -> (pose (3,), cov (3,3), map_updated: bool, kept: int)"""
        hint = _f32(pose_hint_world, 3)
        r = _f32(ranges).reshape(-1)
        T = None if transform is None else np.ascontiguousarray(transform, dtype=np.float64).reshape(12)
        pose = np.zeros(3, np.float32)
        cov = np.zeros(9, np.float32) if cov_inout is None else _f32(cov_inout).reshape(9).copy()
        upd, kept = C.c_int(0), C.c_int(0)
        self._check(self.lib.hsb_slam_update_projected(self.h, hint.ctypes.data, r.ctypes.data, r.size, _ptr(T),
                                                       int(bool(map_without_matching)), int(bool(nowait)),
                                                       pose.ctypes.data, cov.ctypes.data, C.addressof(upd),
                                                       C.addressof(kept)))
        return pose, cov.reshape(3, 3), bool(upd.value), int(kept.value)

    def last_map_update_pose(self) -> np.ndarray:
        out = np.zeros(3, np.float32)
        self._check(self.lib.hsb_get_last_map_update_pose(self.h, out.ctypes.data))
        return out

    # -- finer seams -----------------------------------------------------------------------------
    def update_level_by_scan(self, level: int, points_level_xy, robot_pose_world, origo_level=None):
        pts = _f32(points_level_xy).reshape(-1, 2)
        pose = _f32(robot_pose_world, 3)
        og = None if origo_level is None else _f32(origo_level, 2)
        self._check(self.lib.hsb_update_level_by_scan(self.h, level, pts.ctypes.data if pts.size else None,
                                                      pts.shape[0], _ptr(og), pose.ctypes.data))

    def hessian_derivs(self, level: int, pose_map, points_level_xy):
        pts = _f32(points_level_xy).reshape(-1, 2)
        pm = _f32(pose_map, 3)
        H, d = np.zeros(9, np.float32), np.zeros(3, np.float32)
        self._check(self.lib.hsb_hessian_derivs(self.h, level, pm.ctypes.data, pts.ctypes.data if pts.size else None,
                                                pts.shape[0], H.ctypes.data, d.ctypes.data))
        return H.reshape(3, 3), d

    def match_batch(self, hints, points_xy, offsets=None, want_cov: bool = True, out_poses=None, out_cov=None):
        """Host-buffer batch (numpy arrays or pinned torch CPU tensors). offsets=None -> every hint
        uses the one scan `points_xy` (pose-hypothesis mode). -> (poses (B,3), cov (B,3,3) | None)"""
        B = int(hints.shape[0])
        if isinstance(hints, np.ndarray):
            hints = _f32(hints).reshape(-1, 3)
        if isinstance(points_xy, np.ndarray):
            points_xy = _f32(points_xy).reshape(-1, 2)
        n_shared = 0
        if offsets is None:
            n_shared = int(points_xy.shape[0])
        elif isinstance(offsets, np.ndarray):
            offsets = np.ascontiguousarray(offsets, dtype=np.int32)
        if out_poses is None:
            out_poses = np.zeros((B, 3), np.float32)
        if want_cov and out_cov is None:
            out_cov = np.zeros((B, 9), np.float32)
        self._check(self.lib.hsb_match_batch(self.h, B, _ptr(hints), _ptr(points_xy), _ptr(offsets), n_shared,
                                             _ptr(out_poses), _ptr(out_cov) if want_cov else None))
        cov = None
        if want_cov:
            cov = out_cov.reshape(B, 3, 3) if isinstance(out_cov, np.ndarray) else out_cov
        return out_poses, cov

    def match_batch_device(self, B: int, d_hints: int, d_points: int, d_offsets: int | None, n_shared: int,
                           max_points_per_scan: int, d_out_poses: int, d_out_cov: int | None, stream: int = 0):
        """Raw device pointers (ints, e.g. tensor.data_ptr()) and a CUDA stream handle; asynchronous."""
        self._check(self.lib.hsb_match_batch_device(self.h, int(B), d_hints, d_points, d_offsets, int(n_shared),
                                                    int(max_points_per_scan), d_out_poses, d_out_cov, stream))

    # -- raw ranges in (rosLaserScanToDataContainer fused into the match kernel) -----------------
    def set_scan_format(self, n_beams: int, angle_min: float, angle_increment: float, range_min: float,
                        range_max: float):
        fmt = HsbScanFormat(int(n_beams), float(angle_min), float(angle_increment), float(range_min), float(range_max))
        self._check(self.lib.hsb_set_scan_format(self.h, C.byref(fmt)))
        self.n_beams = int(n_beams)

    def scan_to_points(self, ranges) -> np.ndarray:
        r = _f32(ranges).reshape(-1)
        assert r.size == self.n_beams
        out = np.zeros((self.n_beams, 2), np.float32)
        n = C.c_int()
        self._check(self.lib.hsb_scan_to_points(self.h, r.ctypes.data, out.ctypes.data, C.byref(n)))
        return out[: n.value].copy()

    def match_batch_ranges(self, hints, ranges, want_cov: bool = True, out_poses=None, out_cov=None):
        """ranges: (B, n_beams) float32 host array / pinned tensor."""
        B = int(hints.shape[0])
        if isinstance(hints, np.ndarray):
            hints = _f32(hints).reshape(-1, 3)
        if isinstance(ranges, np.ndarray):
            ranges = _f32(ranges).reshape(B, self.n_beams)
        if out_poses is None:
            out_poses = np.zeros((B, 3), np.float32)
        if want_cov and out_cov is None:
            out_cov = np.zeros((B, 9), np.float32)
        self._check(self.lib.hsb_match_batch_ranges(self.h, B, _ptr(hints), _ptr(ranges), _ptr(out_poses),
                                                    _ptr(out_cov) if want_cov else None))
        cov = None
        if want_cov:
            cov = out_cov.reshape(B, 3, 3) if isinstance(out_cov, np.ndarray) else out_cov
        return out_poses, cov

    # -- submit / wait (streams of batches; buffers must stay alive and untouched until wait) --------
    def match_batch_ranges_submit(self, hints, ranges, out_poses, out_cov=None) -> int:
        t = C.c_int(-1)
        self._check(self.lib.hsb_match_batch_ranges_submit(self.h, int(hints.shape[0]), _ptr(hints), _ptr(ranges),
                                                           _ptr(out_poses), _ptr(out_cov), C.byref(t)))
        return t.value

    def match_batch_submit(self, hints, points_xy, offsets, out_poses, out_cov=None) -> int:
        t = C.c_int(-1)
        n_shared = 0 if offsets is not None else int(points_xy.shape[0])
        self._check(self.lib.hsb_match_batch_submit(self.h, int(hints.shape[0]), _ptr(hints), _ptr(points_xy),
                                                    _ptr(offsets), n_shared, _ptr(out_poses), _ptr(out_cov), C.byref(t)))
        return t.value

    def match_batch_cloud_submit(self, hints, points_xyz, offsets, out_poses, out_cov=None, out_origo=None,
                                 transforms=None) -> int:
        t = C.c_int(-1)
        self._check(self.lib.hsb_match_batch_cloud_submit(self.h, int(hints.shape[0]), _ptr(hints), _ptr(points_xyz),
                                                          _ptr(offsets), _ptr(transforms), _ptr(out_poses), _ptr(out_cov),
                                                          _ptr(out_origo), C.byref(t)))
        return t.value

    def measure_h2d_gbs(self, host_ptr: int, nbytes: int, reps: int = 5) -> float:
        out = C.c_float()
        self._check(self.lib.hsb_measure_h2d_gbs(self.h, host_ptr, nbytes, reps, C.byref(out)))
        return float(out.value)

    def match_batch_wait(self, ticket: int):
        self._check(self.lib.hsb_match_batch_wait(self.h, int(ticket)))

    def match_batch_ranges_device(self, B: int, d_hints: int, d_ranges: int, d_out_poses: int, d_out_cov: int | None,
                                  stream: int = 0):
        self._check(self.lib.hsb_match_batch_ranges_device(self.h, int(B), d_hints, d_ranges, d_out_poses, d_out_cov,
                                                           stream))

    # -- point clouds in (rosPointCloudToDataContainer fused into the match kernel) -----------------
    def set_cloud_format(self, laser_transform, sqr_laser_min_dist: float, sqr_laser_max_dist: float,
                         laser_z_min_value: float, laser_z_max_value: float):
        fmt = HsbCloudFormat()
        for k, v in enumerate(np.asarray(laser_transform, np.float64).reshape(12)):
            fmt.laser_transform[k] = float(v)
        fmt.sqr_laser_min_dist, fmt.sqr_laser_max_dist = float(sqr_laser_min_dist), float(sqr_laser_max_dist)
        fmt.laser_z_min_value, fmt.laser_z_max_value = float(laser_z_min_value), float(laser_z_max_value)
        self._check(self.lib.hsb_set_cloud_format(self.h, C.byref(fmt)))

    def cloud_to_points(self, points_xyz):
        """-> (endpoints (k, 2) float32, origo (2,) float32)"""
        p = _f32(points_xyz).reshape(-1, 3)
        out = np.zeros((max(1, p.shape[0]), 2), np.float32)
        origo = np.zeros(2, np.float32)
        n = C.c_int()
        self._check(self.lib.hsb_cloud_to_points(self.h, p.ctypes.data if p.size else None, p.shape[0], out.ctypes.data,
                                                 C.byref(n), origo.ctypes.data))
        return out[: n.value].copy(), origo

    # -- LaserScan ranges through laser_geometry's projection, then the cloud rule ------------------
    def set_laser_projection(self, n_beams: int, angle_min: float, angle_increment: float, range_min: float,
                             range_max: float, range_cutoff: float = 30.0):
        """range_cutoff: projectLaser's third argument (the node passes 30.0); < 0 means range_max."""
        proj = HsbLaserProjection(int(n_beams), float(angle_min), float(angle_increment), float(range_min),
                                  float(range_max), float(range_cutoff))
        self._check(self.lib.hsb_set_laser_projection(self.h, C.byref(proj)))

    def projected_scan_to_points(self, ranges, transform=None):
        """-> (endpoints (k, 2) float32, origo (2,) float32)"""
        r = _f32(ranges).reshape(-1)
        T = None if transform is None else np.ascontiguousarray(transform, dtype=np.float64).reshape(12)
        out = np.zeros((max(1, r.size), 2), np.float32)
        origo = np.zeros(2, np.float32)
        n = C.c_int()
        self._check(self.lib.hsb_projected_scan_to_points(self.h, r.ctypes.data, r.size, _ptr(T), out.ctypes.data,
                                                          C.byref(n), origo.ctypes.data))
        return out[: n.value].copy(), origo

    def match_batch_projected(self, hints, ranges, transforms=None, want_cov: bool = True):
        """A default node's LaserScans matched in one batch: ranges (B, n_beams) float32, n_beams = the projection's;
        transforms (B, 12) float64 or None (the cloud format's).  -> (poses (B, 3), cov (B, 3, 3) | None, origo (B, 2))"""
        B = int(hints.shape[0])
        if isinstance(hints, np.ndarray):
            hints = _f32(hints).reshape(-1, 3)
        if isinstance(ranges, np.ndarray):
            ranges = _f32(ranges).reshape(B, -1) if B else _f32(ranges)
        if transforms is not None:
            transforms = np.ascontiguousarray(transforms, dtype=np.float64).reshape(B, 12)
        poses = np.zeros((B, 3), np.float32)
        cov = np.zeros((B, 9), np.float32) if want_cov else None
        origo = np.zeros((B, 2), np.float32)
        self._check(self.lib.hsb_match_batch_projected(self.h, B, _ptr(hints), _ptr(ranges), _ptr(transforms),
                                                       poses.ctypes.data, _ptr(cov), origo.ctypes.data))
        return poses, (cov.reshape(B, 3, 3) if want_cov else None), origo

    def match_batch_projected_submit(self, hints, ranges, out_poses, out_cov=None, out_origo=None,
                                     transforms=None) -> int:
        t = C.c_int(-1)
        self._check(self.lib.hsb_match_batch_projected_submit(self.h, int(hints.shape[0]), _ptr(hints), _ptr(ranges),
                                                              _ptr(transforms), _ptr(out_poses), _ptr(out_cov),
                                                              _ptr(out_origo), C.byref(t)))
        return t.value

    def match_batch_projected_device(self, B: int, d_hints: int, d_ranges: int, d_transforms: int | None,
                                     d_out_poses: int, d_out_cov: int | None, d_out_origo: int | None, stream: int = 0):
        self._check(self.lib.hsb_match_batch_projected_device(self.h, int(B), d_hints, d_ranges, d_transforms,
                                                              d_out_poses, d_out_cov, d_out_origo, stream))

    def match_batch_cloud(self, hints, points_xyz, offsets, transforms=None, want_cov: bool = True):
        """-> (poses (B, 3), cov (B, 3, 3) | None, origo (B, 2))"""
        B = int(hints.shape[0])
        if isinstance(hints, np.ndarray):
            hints = _f32(hints).reshape(-1, 3)
        if isinstance(points_xyz, np.ndarray):
            points_xyz = _f32(points_xyz).reshape(-1, 3)
        offsets = np.ascontiguousarray(offsets, dtype=np.int32)
        if transforms is not None:
            transforms = np.ascontiguousarray(transforms, dtype=np.float64).reshape(B, 12)
        poses = np.zeros((B, 3), np.float32)
        cov = np.zeros((B, 9), np.float32) if want_cov else None
        origo = np.zeros((B, 2), np.float32)
        self._check(self.lib.hsb_match_batch_cloud(self.h, B, _ptr(hints), _ptr(points_xyz), offsets.ctypes.data,
                                                   _ptr(transforms), poses.ctypes.data, _ptr(cov), origo.ctypes.data))
        return poses, (cov.reshape(B, 3, 3) if want_cov else None), origo

    def match_batch_cloud_device(self, B: int, d_hints: int, d_points_xyz: int, d_offsets: int, max_points_per_scan: int,
                                 d_transforms: int | None, d_out_poses: int, d_out_cov: int | None,
                                 d_out_origo: int | None, stream: int = 0):
        self._check(self.lib.hsb_match_batch_cloud_device(self.h, int(B), d_hints, d_points_xyz, d_offsets,
                                                          int(max_points_per_scan), d_transforms, d_out_poses, d_out_cov,
                                                          d_out_origo, stream))

    # -- planes ----------------------------------------------------------------------------------
    def upload_level(self, level: int, logodds):
        sx, sy, _ = self.level_info(level)
        a = _f32(logodds).reshape(-1)
        assert a.size == sx * sy, (a.size, sx, sy)
        self._check(self.lib.hsb_upload_level(self.h, level, a.ctypes.data))

    def download_level(self, level: int) -> np.ndarray:
        sx, sy, _ = self.level_info(level)
        out = np.zeros((sy, sx), np.float32)
        self._check(self.lib.hsb_download_level(self.h, level, out.ctypes.data))
        return out

    def download_prob(self, level: int) -> np.ndarray:
        sx, sy, _ = self.level_info(level)
        out = np.zeros((sy, sx), np.float32)
        self._check(self.lib.hsb_download_prob(self.h, level, out.ctypes.data))
        return out

    def download_occupancy(self, level: int) -> np.ndarray:
        """nav_msgs/OccupancyGrid data of one level: 0 free, 100 occupied, -1 unknown."""
        sx, sy, _ = self.level_info(level)
        out = np.zeros((sy, sx), np.int8)
        self._check(self.lib.hsb_download_occupancy(self.h, level, out.ctypes.data))
        return out

    def likelihood_batch(self, level: int, poses_world, points_xy, offsets=None) -> np.ndarray:
        """getLikelihoodForState for B world poses (scan layout as match_batch)."""
        poses = _f32(poses_world).reshape(-1, 3)
        pts = _f32(points_xy).reshape(-1, 2)
        B = poses.shape[0]
        n_shared = 0
        offp = None
        if offsets is None:
            n_shared = pts.shape[0]
        else:
            offsets = np.ascontiguousarray(offsets, dtype=np.int32)
            offp = offsets.ctypes.data
        out = np.zeros(B, np.float32)
        self._check(self.lib.hsb_likelihood_batch(self.h, level, B, poses.ctypes.data, pts.ctypes.data if pts.size else None,
                                                  offp, n_shared, out.ctypes.data))
        return out

    def likelihood_batch_device(self, level: int, B: int, d_poses_world: int, d_points_xy: int, d_offsets, n_shared: int,
                                d_out: int, stream: int = 0) -> None:
        """getLikelihoodForState on device pointers, enqueued on `stream` (no synchronisation)."""
        self._check(self.lib.hsb_likelihood_batch_device(self.h, level, B, d_poses_world, d_points_xy, d_offsets, n_shared,
                                                         d_out, stream))

    def best_hypothesis_device(self, level: int, B: int, d_poses_world: int, d_points_xy: int, d_offsets, n_shared: int,
                               d_best4: int, d_out=None, stream: int = 0) -> None:
        """likelihood of B poses + arg-max on the device: d_best4 <- {likelihood, x, y, psi} of the best one."""
        self._check(self.lib.hsb_best_hypothesis_device(self.h, level, B, d_poses_world, d_points_xy, d_offsets, n_shared,
                                                        d_out, d_best4, stream))

    def covariance_batch(self, level: int, poses_world, points_xy, offsets=None):
        """getCovarianceForPose (+ getCovMatrixWorldCoords) for B world poses. -> (cov_map (B,3,3), cov_world (B,3,3))"""
        poses = _f32(poses_world).reshape(-1, 3)
        pts = _f32(points_xy).reshape(-1, 2)
        B = poses.shape[0]
        n_shared, offp = 0, None
        if offsets is None:
            n_shared = pts.shape[0]
        else:
            offsets = np.ascontiguousarray(offsets, dtype=np.int32)
            offp = offsets.ctypes.data
        cm, cw = np.zeros((B, 9), np.float32), np.zeros((B, 9), np.float32)
        self._check(self.lib.hsb_covariance_batch(self.h, level, B, poses.ctypes.data, pts.ctypes.data if pts.size else None,
                                                  offp, n_shared, cm.ctypes.data, cw.ctypes.data))
        return cm.reshape(B, 3, 3), cw.reshape(B, 3, 3)

    def raycast_batch(self, level: int, begin_cells, end_cells):
        """checkOccupancyBresenhami for B rays. -> (dist (B,) float32 [-1 = no hit], hit (B,2) int32)"""
        b = np.ascontiguousarray(begin_cells, dtype=np.int32).reshape(-1, 2)
        e = np.ascontiguousarray(end_cells, dtype=np.int32).reshape(-1, 2)
        B = b.shape[0]
        dist = np.zeros(B, np.float32)
        hit = np.zeros((B, 2), np.int32)
        self._check(self.lib.hsb_raycast_batch(self.h, level, B, b.ctypes.data, e.ctypes.data, dist.ctypes.data,
                                               hit.ctypes.data))
        return dist, hit

    def map_origin(self, level: int) -> np.ndarray:
        out = np.zeros(2, np.float32)
        self._check(self.lib.hsb_get_map_origin(self.h, level, out.ctypes.data))
        return out

    def get_dist_batch(self, level: int, begin_world, end_world):
        """DistanceMeasurementProvider::getDist for B world-frame rays.
        -> (dist [m] (B,), hit_world (B, 2), found (B,) bool)"""
        b = _f32(begin_world).reshape(-1, 2)
        e = _f32(end_world).reshape(-1, 2)
        B = b.shape[0]
        dist, hit, found = np.zeros(B, np.float32), np.zeros((B, 2), np.float32), np.zeros(B, np.int32)
        self._check(self.lib.hsb_get_dist_batch(self.h, level, B, b.ctypes.data, e.ctypes.data, dist.ctypes.data,
                                                hit.ctypes.data, found.ctypes.data))
        return dist, hit, found.astype(bool)

    def get_dirty_rect(self, level: int, reset: bool = False):
        """(x0, y0, x1, y1) inclusive of the cells written since the last reset, or None."""
        r = (C.c_int * 4)()
        self._check(self.lib.hsb_get_dirty_rect(self.h, level, r, int(reset)))
        rect = tuple(int(v) for v in r)
        return None if rect[2] < rect[0] else rect

    def get_dirty_rects(self, reset: bool = False):
        """All levels' replication rectangles with one copy: list of (x0, y0, x1, y1) or None."""
        r = (C.c_int * (4 * self.levels))()
        self._check(self.lib.hsb_get_dirty_rects(self.h, r, int(reset)))
        out = []
        for l in range(self.levels):
            rect = tuple(int(v) for v in r[4 * l:4 * l + 4])
            out.append(None if rect[2] < rect[0] else rect)
        return out

    def get_mirror_dirty_rect(self, level: int, reset: bool = False):
        r = (C.c_int * 4)()
        self._check(self.lib.hsb_get_mirror_dirty_rect(self.h, level, r, int(reset)))
        rect = tuple(int(v) for v in r)
        return None if rect[2] < rect[0] else rect

    def download_level_rect(self, level: int, rect) -> np.ndarray:
        w, hgt = rect[2] - rect[0] + 1, rect[3] - rect[1] + 1
        out = np.zeros((hgt, w), np.float32)
        self._check(self.lib.hsb_download_level_rect(self.h, level, (C.c_int * 4)(*rect), out.ctypes.data))
        return out

    def download_occupancy_rect(self, level: int, rect) -> np.ndarray:
        w, hgt = rect[2] - rect[0] + 1, rect[3] - rect[1] + 1
        out = np.zeros((hgt, w), np.int8)
        self._check(self.lib.hsb_download_occupancy_rect(self.h, level, (C.c_int * 4)(*rect), out.ctypes.data))
        return out

    @property
    def d2h_bytes(self) -> int:
        return int(self.lib.hsb_get_d2h_bytes(self.h))

    def pack_dirty_device(self, d_buf: int, capacity_bytes: int, reset: bool = True, stream: int = 0):
        self._check(self.lib.hsb_pack_dirty_device(self.h, d_buf, int(capacity_bytes), int(reset), stream))

    def unpack_dirty_device(self, d_buf: int, capacity_bytes: int, stream: int = 0):
        self._check(self.lib.hsb_unpack_dirty_device(self.h, d_buf, int(capacity_bytes), stream))

    def replication_overflows(self, reset: bool = False) -> int:
        n = C.c_int(0)
        self._check(self.lib.hsb_get_replication_overflows(self.h, C.byref(n), int(reset)))
        return int(n.value)

    def pack_rect_device(self, level: int, rect, d_buf: int, stream: int = 0):
        r = (C.c_int * 4)(*rect)
        self._check(self.lib.hsb_pack_rect_device(self.h, level, r, d_buf, stream))

    def unpack_rect_device(self, level: int, rect, d_buf: int, stream: int = 0):
        r = (C.c_int * 4)(*rect)
        self._check(self.lib.hsb_unpack_rect_device(self.h, level, r, d_buf, stream))

    def level_logodds_device_ptr(self, level: int) -> int:
        return int(self.lib.hsb_level_logodds_device_ptr(self.h, level) or 0)

    def refresh_level(self, level: int, stream: int = 0):
        self._check(self.lib.hsb_refresh_level(self.h, level, stream))


class SlamGroup:
    """HectorSlamProcessor::update for several MapRepB200 handles — one SLAM session, one map each — in one device pass
    (hsb_group_slam_update).  Each session's results and its handle's state equal a slam_update() on that handle bit for
    bit.  The group does not own the handles: close() it before closing any of them.
    mixed=True (hsb_group_create_mixed): the handles may differ in map size, resolution and start; every call then takes
    each member's own sizes (grids, cell units, world-to-map transforms).
    heterogeneous=True (hsb_group_create_heterogeneous): the handles may also differ in level count, per-level
    max_iterations and gather mode; every call runs each member's own levels, and a call at a `level` rejects a listed
    member that does not have it."""

    def __init__(self, reps, mixed: bool = False, heterogeneous: bool = False):
        self.lib = load_library()
        self.reps = list(reps)
        self.M = len(self.reps)
        arr = (C.c_void_p * max(1, self.M))(*[None if r is None else r.h for r in self.reps])
        g = C.c_void_p()
        create = (self.lib.hsb_group_create_heterogeneous if heterogeneous
                  else self.lib.hsb_group_create_mixed if mixed else self.lib.hsb_group_create)
        st = create(C.cast(arr, C.c_void_p), self.M, C.byref(g))
        if st != 0:
            raise HsbError(st, (self.lib.hsb_last_error(None) or b"").decode())
        self.g = g

    def _check(self, st: int):
        if st != 0:
            raise HsbError(st, (self.lib.hsb_last_error(self.reps[0].h) or b"").decode())

    def slam_update(self, hints, scans, origo=None, map_without_matching=None, nowait: bool = False, cov_inout=None,
                    members=None):
        """scans: M (n_s, 2) endpoint arrays, or a tuple (points (N, 2), offsets (M + 1,)).  hints (M, 3), origo (M, 2),
        map_without_matching (M,) bools.  -> (poses (M, 3), covs (M, 3, 3), updated (M,) bool); a cov entry keeps its
        cov_inout value (zeros if None) where the session matched nothing.
        members: step only these members (indices into the group's handles, in session order,
        hsb_group_slam_update_subset); every per-session argument and result then has len(members) entries."""
        K, mem = self._sessions(members)
        h = _f32(hints).reshape(K, 3)
        pts, offsets = self._pack(scans, 2, K)
        og = None if origo is None else _f32(origo).reshape(K, 2)
        mwm = None if map_without_matching is None else np.ascontiguousarray(map_without_matching, np.int32).reshape(K)
        poses = np.zeros((K, 3), np.float32)
        cov = np.zeros((K, 9), np.float32) if cov_inout is None else _f32(cov_inout).reshape(K, 9).copy()
        upd = np.zeros(K, np.int32)
        args = (h.ctypes.data, pts.ctypes.data if pts.size else None, offsets.ctypes.data, _ptr(og), _ptr(mwm),
                int(bool(nowait)), poses.ctypes.data, cov.ctypes.data, upd.ctypes.data)
        if mem is None:
            self._check(self.lib.hsb_group_slam_update(self.g, *args))
        else:
            self._check(self.lib.hsb_group_slam_update_subset(self.g, K, _ptr(mem), *args))
        return poses, cov.reshape(K, 3, 3), upd.astype(bool)

    def slam_update_cloud(self, hints, clouds, transforms=None, map_without_matching=None, nowait: bool = False,
                          cov_inout=None, members=None):
        """The same step from the node's default input (hsb_group_slam_update_cloud): clouds are M (n_s, 3) Point32
        arrays in the laser frame, or a tuple (points (N, 3), offsets (M + 1,)); transforms (M, 12) float64 laser
        transforms, None = each member's cloud format.  Each member converts with its own cloud format's thresholds.
        members as in slam_update (hsb_group_slam_update_cloud_subset).
        -> (poses (M, 3), covs (M, 3, 3), updated (M,) bool, kept (M,) int: endpoints each conversion kept)"""
        K, mem = self._sessions(members)
        h = _f32(hints).reshape(K, 3)
        pts, offsets = self._pack(clouds, 3, K)
        T = None if transforms is None else np.ascontiguousarray(transforms, dtype=np.float64).reshape(K, 12)
        mwm = None if map_without_matching is None else np.ascontiguousarray(map_without_matching, np.int32).reshape(K)
        poses = np.zeros((K, 3), np.float32)
        cov = np.zeros((K, 9), np.float32) if cov_inout is None else _f32(cov_inout).reshape(K, 9).copy()
        upd = np.zeros(K, np.int32)
        kept = np.zeros(K, np.int32)
        args = (h.ctypes.data, pts.ctypes.data if pts.size else None, offsets.ctypes.data, _ptr(T), _ptr(mwm),
                int(bool(nowait)), poses.ctypes.data, cov.ctypes.data, upd.ctypes.data, kept.ctypes.data)
        if mem is None:
            self._check(self.lib.hsb_group_slam_update_cloud(self.g, *args))
        else:
            self._check(self.lib.hsb_group_slam_update_cloud_subset(self.g, K, _ptr(mem), *args))
        return poses, cov.reshape(K, 3, 3), upd.astype(bool), kept.astype(int)

    def slam_update_ranges(self, hints, ranges_list, map_without_matching=None, nowait: bool = False, cov_inout=None,
                           members=None):
        """The same step from raw LaserScan ranges (hsb_group_slam_update_ranges): ranges_list is M (n_beams_s,) arrays,
        or a tuple (ranges (N,), offsets (M + 1,)).  Each member converts with its own scan format.  members as in
        slam_update (hsb_group_slam_update_ranges_subset).
        -> (poses (M, 3), covs (M, 3, 3), updated (M,) bool, kept (M,) int: endpoints each conversion kept)"""
        K, mem = self._sessions(members)
        h = _f32(hints).reshape(K, 3)
        r, offsets = self._pack(ranges_list, 1, K)
        mwm = None if map_without_matching is None else np.ascontiguousarray(map_without_matching, np.int32).reshape(K)
        poses = np.zeros((K, 3), np.float32)
        cov = np.zeros((K, 9), np.float32) if cov_inout is None else _f32(cov_inout).reshape(K, 9).copy()
        upd = np.zeros(K, np.int32)
        kept = np.zeros(K, np.int32)
        args = (h.ctypes.data, r.ctypes.data if r.size else None, offsets.ctypes.data, _ptr(mwm), int(bool(nowait)),
                poses.ctypes.data, cov.ctypes.data, upd.ctypes.data, kept.ctypes.data)
        if mem is None:
            self._check(self.lib.hsb_group_slam_update_ranges(self.g, *args))
        else:
            self._check(self.lib.hsb_group_slam_update_ranges_subset(self.g, K, _ptr(mem), *args))
        return poses, cov.reshape(K, 3, 3), upd.astype(bool), kept.astype(int)

    def slam_update_projected(self, hints, ranges_list, transforms=None, map_without_matching=None, nowait: bool = False,
                              cov_inout=None, members=None):
        """The same step from the LaserScans of default-configured nodes (hsb_group_slam_update_projected): ranges_list
        is M (n_beams_s,) arrays, or a tuple (ranges (N,), offsets (M + 1,)); transforms (M, 12) float64, None = each
        member's cloud format.  Each member projects with its own laser projection and converts with its own cloud
        format.  members as in slam_update (hsb_group_slam_update_projected_subset).
        -> (poses (M, 3), covs (M, 3, 3), updated (M,) bool, kept (M,) int: endpoints each conversion kept)"""
        K, mem = self._sessions(members)
        h = _f32(hints).reshape(K, 3)
        r, offsets = self._pack(ranges_list, 1, K)
        T = None if transforms is None else np.ascontiguousarray(transforms, dtype=np.float64).reshape(K, 12)
        mwm = None if map_without_matching is None else np.ascontiguousarray(map_without_matching, np.int32).reshape(K)
        poses = np.zeros((K, 3), np.float32)
        cov = np.zeros((K, 9), np.float32) if cov_inout is None else _f32(cov_inout).reshape(K, 9).copy()
        upd = np.zeros(K, np.int32)
        kept = np.zeros(K, np.int32)
        args = (h.ctypes.data, r.ctypes.data if r.size else None, offsets.ctypes.data, _ptr(T), _ptr(mwm),
                int(bool(nowait)), poses.ctypes.data, cov.ctypes.data, upd.ctypes.data, kept.ctypes.data)
        if mem is None:
            self._check(self.lib.hsb_group_slam_update_projected(self.g, *args))
        else:
            self._check(self.lib.hsb_group_slam_update_projected_subset(self.g, K, _ptr(mem), *args))
        return poses, cov.reshape(K, 3, 3), upd.astype(bool), kept.astype(int)

    def sync_occupancy(self, level: int, grids, members=None, reset: bool = True):
        """publishMap for the members in one pass (hsb_group_sync_occupancy): grids are one C-contiguous int8
        (size_y, size_x) array per session, its member's own level size, kept by the caller between calls; the cells of
        each member's mirror rectangle are rewritten in place, no other byte is touched.  members as in slam_update
        (hsb_group_sync_occupancy_subset).  -> one (x0, y0, x1, y1) per session, or None where the map did not change."""
        K, mem = self._sessions(members)
        assert len(grids) == K, (len(grids), K)
        sel = range(K) if mem is None else mem
        for k, (m, a) in enumerate(zip(sel, grids)):
            assert isinstance(a, np.ndarray) and a.dtype == np.int8 and a.flags.c_contiguous, "grids: C-contiguous int8"
            rep = self.reps[m] if 0 <= m < self.M else None   # (a bad member or level is the C call's rejection)
            if rep is not None and 0 <= level < rep.levels:
                sx, sy, _ = rep.level_info(level)
                assert a.shape == (sy, sx), (k, a.shape, (sy, sx))
        arr = (C.c_void_p * max(1, K))(*[a.ctypes.data for a in grids])
        rects = np.zeros((max(1, K), 4), np.int32)
        if mem is None:
            self._check(self.lib.hsb_group_sync_occupancy(self.g, int(level), C.cast(arr, C.c_void_p), rects.ctypes.data,
                                                          int(bool(reset))))
        else:
            self._check(self.lib.hsb_group_sync_occupancy_subset(self.g, K, _ptr(mem), int(level), C.cast(arr, C.c_void_p),
                                                                 rects.ctypes.data, int(bool(reset))))
        return [None if r[2] < r[0] else tuple(int(v) for v in r) for r in rects[:K]]

    def pack_dirty_device(self, d_buf: int, capacity: int, reset: bool = True, stream: int = 0, members=None):
        """Every member's dirty tiles into one device buffer of `capacity` bytes (hsb_group_pack_dirty_device): a group
        header, then per session the buffer MapRepB200.pack_dirty_device writes for that member alone; rows placed
        first-fit in session order, a block that does not fit is deferred and keeps its rectangles.  members as in
        slam_update (hsb_group_pack_dirty_device_subset).  Asynchronous on `stream`."""
        K, mem = self._sessions(members)
        if mem is None:
            self._check(self.lib.hsb_group_pack_dirty_device(self.g, d_buf, int(capacity), int(bool(reset)), stream))
        else:
            self._check(self.lib.hsb_group_pack_dirty_device_subset(self.g, K, _ptr(mem), d_buf, int(capacity),
                                                                    int(bool(reset)), stream))

    def unpack_dirty_device(self, d_buf: int, capacity: int, stream: int = 0):
        """Apply a buffer pack_dirty_device wrote on an owner group listing its handles in this group's order
        (hsb_group_unpack_dirty_device).  Deferred blocks count on their member's replication_overflows(), a buffer that
        does not fit this group on reps[0]'s.  Asynchronous on `stream`."""
        self._check(self.lib.hsb_group_unpack_dirty_device(self.g, d_buf, int(capacity), stream))

    def reset(self, members=None):
        """MapRepB200.reset() for the members in one launch (hsb_group_reset): each is left as reset() leaves it, except
        that its replication rectangles are clean with the cleared flags set, so the next pack ships a clear record and
        the cells written since instead of whole levels.  members as in slam_update (hsb_group_reset_subset).  Returns
        once queued; every later call on a reset member runs after it."""
        K, mem = self._sessions(members)
        if mem is None:
            self._check(self.lib.hsb_group_reset(self.g))
        else:
            self._check(self.lib.hsb_group_reset_subset(self.g, K, _ptr(mem)))

    def get_dist(self, level: int, begin_world, end_world, members=None):
        """DistanceMeasurementProvider::getDist for the members' rays in one pass (hsb_group_get_dist): begin_world and
        end_world are one (n_s, 2) array of world points per session, or a tuple (points (Q, 2), offsets (K + 1,)).
        members as in slam_update (hsb_group_get_dist_subset).  Each ray equals get_dist_batch on its member.
        -> (dist [m] (Q,), hit_world (Q, 2), found (Q,) bool), in ray order"""
        K, mem = self._sessions(members)
        b, offsets = self._pack(begin_world, 2, K)
        e, e_off = self._pack(end_world, 2, K)
        assert np.array_equal(offsets, e_off), "begin_world and end_world hold different numbers of rays"
        Q = b.shape[0]
        dist, hit, found = np.zeros(Q, np.float32), np.zeros((Q, 2), np.float32), np.zeros(Q, np.int32)
        args = (int(level), offsets.ctypes.data, _ptr(b if Q else None), _ptr(e if Q else None), dist.ctypes.data,
                hit.ctypes.data, found.ctypes.data)
        if mem is None:
            self._check(self.lib.hsb_group_get_dist(self.g, *args))
        else:
            self._check(self.lib.hsb_group_get_dist_subset(self.g, K, _ptr(mem), *args))
        return dist, hit, found.astype(bool)

    def raycast(self, level: int, begin_cells, end_cells, members=None):
        """checkOccupancyBresenhami for the members' rays in one pass (hsb_group_raycast): begin_cells and end_cells
        are one (n_s, 2) int32 array of cells per session, or a tuple (cells (Q, 2), offsets (K + 1,)).  members as in
        slam_update (hsb_group_raycast_subset).  Each ray equals raycast_batch on its member.
        -> (dist (Q,) float32 [-1 = no hit], hit (Q, 2) int32), in ray order"""
        K, mem = self._sessions(members)
        b, offsets = self._pack(begin_cells, 2, K, np.int32)
        e, e_off = self._pack(end_cells, 2, K, np.int32)
        assert np.array_equal(offsets, e_off), "begin_cells and end_cells hold different numbers of rays"
        Q = b.shape[0]
        dist, hit = np.zeros(Q, np.float32), np.zeros((Q, 2), np.int32)
        args = (int(level), offsets.ctypes.data, _ptr(b if Q else None), _ptr(e if Q else None), dist.ctypes.data,
                hit.ctypes.data)
        if mem is None:
            self._check(self.lib.hsb_group_raycast(self.g, *args))
        else:
            self._check(self.lib.hsb_group_raycast_subset(self.g, K, _ptr(mem), *args))
        return dist, hit

    def _score_args(self, level, poses_world, points, members):
        """the arguments the three pose-scoring calls share -> (K, mem, Q, args, arrays kept alive)"""
        K, mem = self._sessions(members)
        poses, pose_off = self._pack(poses_world, 3, K)
        if points is None:
            pts, scan_off, pp, op = None, None, None, None
        else:
            pts, scan_off = self._pack(points, 2, K)
            if pts.shape[0] == 0:
                pts = np.zeros((1, 2), np.float32)   # (a pointer for the C call: points and offsets come together)
            pp, op = pts.ctypes.data, scan_off.ctypes.data
        Q = poses.shape[0]
        return K, mem, Q, (int(level), pose_off.ctypes.data, _ptr(poses if Q else None), pp, op), (poses, pose_off, pts, scan_off)

    def likelihood(self, level: int, poses_world, points=None, members=None) -> np.ndarray:
        """getLikelihoodForState of the members' poses in one pass (hsb_group_likelihood): poses_world is one (q_s, 3)
        array of world poses per session, or a tuple (poses (Q, 3), offsets (K + 1,)); every pose of a session is
        scored against that session's one scan on its member's map.  points: one (n_s, 2) endpoint array per session
        (level-0 cells), or a tuple (points, offsets); None = each member's last matched scan as it is on the device.
        members as in slam_update (hsb_group_likelihood_subset).  Each value equals likelihood_batch on its member.
        -> likelihood (Q,), in pose order"""
        K, mem, Q, args, keep = self._score_args(level, poses_world, points, members)
        out = np.zeros(Q, np.float32)
        if mem is None:
            self._check(self.lib.hsb_group_likelihood(self.g, *args, out.ctypes.data))
        else:
            self._check(self.lib.hsb_group_likelihood_subset(self.g, K, _ptr(mem), *args, out.ctypes.data))
        return out

    def covariance(self, level: int, poses_world, points=None, members=None):
        """getCovarianceForPose (+ getCovMatrixWorldCoords) of the members' poses in one pass (hsb_group_covariance);
        arguments as in likelihood (hsb_group_covariance_subset with members).  Each matrix equals covariance_batch on
        its member.  -> (cov_map (Q, 3, 3), cov_world (Q, 3, 3)), in pose order"""
        K, mem, Q, args, keep = self._score_args(level, poses_world, points, members)
        cm, cw = np.zeros((Q, 9), np.float32), np.zeros((Q, 9), np.float32)
        if mem is None:
            self._check(self.lib.hsb_group_covariance(self.g, *args, cm.ctypes.data, cw.ctypes.data))
        else:
            self._check(self.lib.hsb_group_covariance_subset(self.g, K, _ptr(mem), *args, cm.ctypes.data, cw.ctypes.data))
        return cm.reshape(Q, 3, 3), cw.reshape(Q, 3, 3)

    def best_hypothesis(self, level: int, poses_world, points=None, members=None):
        """The most likely of each session's poses in one pass (hsb_group_best_hypothesis): relocalisation of several
        robots at once; arguments as in likelihood (hsb_group_best_hypothesis_subset with members).  Each session's
        winner equals best_hypothesis_device on its member: the highest likelihood, the lowest index among equals.
        -> (likelihood (Q,), best4 (K, 4) {likelihood, x, y, psi}, index (K,) within the session, -1 where it is empty)"""
        K, mem, Q, args, keep = self._score_args(level, poses_world, points, members)
        out, best4, index = np.zeros(Q, np.float32), np.zeros((K, 4), np.float32), np.zeros(K, np.int32)
        tail = (out.ctypes.data, best4.ctypes.data if K else None, index.ctypes.data if K else None)
        if mem is None:
            self._check(self.lib.hsb_group_best_hypothesis(self.g, *args, *tail))
        else:
            self._check(self.lib.hsb_group_best_hypothesis_subset(self.g, K, _ptr(mem), *args, *tail))
        return out, best4, index

    def match_batch(self, hints, points=None, members=None, want_cov: bool = True):
        """matchData from many start poses for the members in one pass (hsb_group_match_batch): hints is one (q_s, 3)
        array of world hints per session, or a tuple (hints (Q, 3), offsets (K + 1,)); every hint of a session is matched
        over all levels with that session's one scan on its member's map.  points as in likelihood: one (n_s, 2) endpoint
        array per session (level-0 cells), or a tuple (points, offsets); None = each member's last matched scan as it is
        on the device.  members as in slam_update (hsb_group_match_batch_subset).  Each pose equals match_batch on its
        member in shared-scan mode with the warps per scan the group call reports (handles[0]'s last_launch_shape).
        -> (poses (Q, 3), cov (Q, 3, 3) | None), in hint order"""
        K, mem = self._sessions(members)
        h, hint_off = self._pack(hints, 3, K)
        if points is None:
            pp, op, keep = None, None, None
        else:
            pts, scan_off = self._pack(points, 2, K)
            if pts.shape[0] == 0:
                pts = np.zeros((1, 2), np.float32)   # (a pointer for the C call: points and offsets come together)
            pp, op, keep = pts.ctypes.data, scan_off.ctypes.data, (pts, scan_off)
        Q = h.shape[0]
        poses = np.zeros((Q, 3), np.float32)
        cov = np.zeros((Q, 9), np.float32) if want_cov else None
        args = (hint_off.ctypes.data, _ptr(h if Q else None), pp, op, _ptr(poses if Q else None), _ptr(cov if Q else None))
        if mem is None:
            self._check(self.lib.hsb_group_match_batch(self.g, *args))
        else:
            self._check(self.lib.hsb_group_match_batch_subset(self.g, K, _ptr(mem), *args))
        del keep
        return poses, None if cov is None else cov.reshape(Q, 3, 3)

    def _sessions(self, members):
        """-> (sessions of the step, the member list as int32, or None for a step of every member)"""
        if members is None:
            return self.M, None
        mem = np.ascontiguousarray(members, dtype=np.int32).reshape(-1)
        return mem.shape[0], mem

    def _pack(self, scans, width, n, dtype=np.float32):
        """n per-session arrays (n_s, width), or a tuple (points (N, width), offsets (n + 1,)) -> (points, offsets)."""
        def arr(a):
            return np.ascontiguousarray(a, dtype=dtype).reshape(-1, width)
        if isinstance(scans, tuple):
            return arr(scans[0]), np.ascontiguousarray(scans[1], dtype=np.int32)
        scans = [arr(s) for s in scans]
        assert len(scans) == n, (len(scans), n)
        offsets = np.zeros(n + 1, np.int32)
        offsets[1:] = np.cumsum([s.shape[0] for s in scans])
        return (np.concatenate(scans) if offsets[-1] else np.zeros((0, width), dtype)), offsets

    def close(self):
        if getattr(self, "g", None):
            self.lib.hsb_group_destroy(self.g)
            self.g = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
