"""The per-evaluation match record on the two CPU oracles — TEST INFRASTRUCTURE, not product code.

  * kind="port": oracle/_build/libhsoracle_record.so (port_record.c): the C port's matchData with the record in the
    layout of include/hector_slam_b200.h (hsb_match_data_record), R floats.
  * kind="reference": oracle/_ref/libhsref_record.so (ref_record_driver.cpp): what the reference's ScanMatcher reports to
    recording DrawInterface / HectorDebugInfoInterface hooks — per level, coarsest first, 3 + 12 * maxIterations floats:
    the start arrow, then per reported evaluation the Hessian (9) and the arrow (3).

Both libraries also export every entry point of the plain oracle libraries, so RecordOracle is a pyoracle.Oracle.
Built by `make -C oracle -f record.mk`.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from oracle import pyoracle

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_LIB = os.path.join(_HERE, "_ref", "libhsref_record.so")
PORT_LIB = os.path.join(_HERE, "_build", "libhsoracle_record.so")
_f32p, _i32p = pyoracle._f32p, pyoracle._i32p


def available(kind: str) -> bool:
    return os.path.exists(REF_LIB if kind == "reference" else PORT_LIB)


def level_iterations(levels: int, iters=None) -> list[int]:
    """maxIterations per level, level 0 first (hsb_config::max_iterations: 0 = the reference's 5 / 3, < 0 = 0)"""
    out = []
    for l in range(levels):
        mi = int(iters[l]) if iters is not None else 0
        out.append(0 if mi < 0 else (mi or (5 if l == 0 else 3)))
    return out


class RecordOracle(pyoracle.Oracle):
    def __init__(self, kind: str, map_resolution: float, size: int, levels: int, start=(0.5, 0.5), silent: bool = True,
                 *, size_y: int | None = None):
        path = REF_LIB if kind == "reference" else PORT_LIB
        if not os.path.exists(path):
            raise FileNotFoundError(f"record oracle missing: {path} (run `make -C oracle -f record.mk`)")
        self.kind = kind
        self.lib = C.CDLL(path)
        self.p = "hsref_" if kind == "reference" else "hso_"
        self._bind()
        fn = self._fn("match_record")
        fn.restype = None
        vp, i = C.c_void_p, C.c_int
        fn.argtypes = [vp, _f32p, _f32p, i, _f32p, vp, _f32p, _f32p, _f32p] + ([_i32p] if kind == "reference" else [])
        if silent and kind == "reference":
            self._fn("silence")(1)
        self.size_x = int(size)
        self.size_y = int(size if size_y is None else size_y)
        self.levels = int(levels)
        self.h = self._fn("create")(map_resolution, self.size_x, self.size_y, start[0], start[1], levels)

    def level_iterations(self, iters=None) -> list[int]:
        return level_iterations(self.levels, iters)

    def match_record(self, hint, pts, iters=None, origo=(0.0, 0.0)):
        """matchData with the record.  -> (pose, cov, record) for the port, (pose, cov, hooks, drawPoint calls per
        level) for the reference"""
        pts = np.ascontiguousarray(pts, dtype=np.float32).reshape(-1, 2)
        mis = self.level_iterations(iters)
        it = None if iters is None else np.ascontiguousarray(
            [int(iters[l]) for l in range(self.levels)] + [0] * (8 - self.levels), dtype=np.int32)
        itp = None if it is None else it.ctypes.data
        pose, cov = np.zeros(3, np.float32), np.zeros(9, np.float32)
        hint = np.ascontiguousarray(hint, dtype=np.float32)
        origo = np.ascontiguousarray(origo, dtype=np.float32)
        if self.kind == "reference":
            rec = np.zeros(sum(3 + 12 * m for m in mis), np.float32)
            npts = np.zeros(self.levels, np.int32)
            self._fn("match_record")(self.h, hint, pts, pts.shape[0], origo, itp, pose, cov, rec, npts)
            return pose, cov.reshape(3, 3), rec, npts
        rec = np.zeros(sum(3 + 15 * (m + 1) for m in mis), np.float32)
        self._fn("match_record")(self.h, hint, pts, pts.shape[0], origo, itp, pose, cov, rec)
        return pose, cov.reshape(3, 3), rec


def port_hooks(orc, rec, n, iters=None):
    """A record in the layout of include/hector_slam_b200.h reduced to what ScanMatcher::matchData reports to its hooks:
    per level, coarsest first, the start arrow, then for evaluations 1 .. maxIterations the Hessian and
    getWorldCoordsPose of the estimate after the step (zeros for an empty scan)."""
    out, off = [], 0
    mis = level_iterations(orc.levels, iters)
    for l in range(orc.levels - 1, -1, -1):
        mi = mis[l]
        out.append(rec[off:off + 3])
        ev = rec[off + 3:off + 3 + 15 * (mi + 1)].reshape(mi + 1, 15)
        for e in range(1, mi + 1):
            if n:
                out += [ev[e, :9], orc.world_coords_pose(l, ev[e, 12:15])]
            else:
                out.append(np.zeros(12, np.float32))
        off += 3 + 15 * (mi + 1)
    return np.concatenate(out).astype(np.float32)
