"""float64 reference of ONE Gauss-Newton evaluation — TEST INFRASTRUCTURE, not product code.

OccGridMapUtil::getCompleteHessianDerivs (OccGridMapUtil.h:64-104, restated by hs_oracle.c
complete_hessian_derivs) for a batch of scans, split where the kernel and the reference necessarily
agree bit for bit and where they may not:

  * fp32, in the reference's operation order — the data every implementation sees:
    sinf / cosf of psi (libm, what the reference calls; the kernel's sincosf_glibc.h is tied to them by
    tests/test_sincosf_glibc.py), the level's point scale, the map coordinate q = c*px + ((-s)*py + x)
    and qy = s*px + (c*py + y) with every operation rounded separately, the inclusive [0, S-2] bounds
    test (NaN is out of the map), the cell (trunc), fx = qx - ix, fy = qy - iy and the four fetched
    probabilities.
  * float64: the bilinear value, the reference's gradient blend (SURVEY.md Q1: the row differences
    blended with the x weights, the column differences with the y weights), 1 - M, rotDeriv, the nine
    products and their sums.

Besides H64 / dTr64 it returns, per scan and per entry, A = sum |products| (the scale of a summation
error bound) and E = sum of first-order bounds on how far the kernel's fp32 evaluation of ONE endpoint's
product (match_kernel.cuh point_accumulate, HSB_FP_VARIANT 2, and the paired path) can be from the
exact product of the same fp32 data; and the per-endpoint contributions (to show that a test can see
one endpoint).  Entry order everywhere: ENTRIES.
"""
from __future__ import annotations

import ctypes as C
import ctypes.util

import numpy as np

# H00 H11 H22 H01 H02 H12 dTr0 dTr1 dTr2 — the kernel's accumulator order (match_kernel.cuh Acc)
ENTRIES = ("h00", "h11", "h22", "h01", "h02", "h12", "d0", "d1", "d2")
U32 = 2.0 ** -24   # unit roundoff of fp32 (round to nearest)

_libm = C.CDLL(ctypes.util.find_library("m") or "libm.so.6")
_libm.sinf.restype = C.c_float
_libm.sinf.argtypes = [C.c_float]
_libm.cosf.restype = C.c_float
_libm.cosf.argtypes = [C.c_float]


def sinf(x) -> np.float32:
    return np.float32(_libm.sinf(float(np.float32(x))))


def cosf(x) -> np.float32:
    return np.float32(_libm.cosf(float(np.float32(x))))


def h_matrix(v9) -> np.ndarray:
    """(..., 9) in ENTRIES order -> (..., 3, 3) symmetric H."""
    v = np.asarray(v9)
    return np.stack([v[..., 0], v[..., 3], v[..., 4],
                     v[..., 3], v[..., 1], v[..., 5],
                     v[..., 4], v[..., 5], v[..., 2]], axis=-1).reshape(v.shape[:-1] + (3, 3))


class Eval64:
    """One scan's evaluation.  H (3, 3), dTr (3,), A (9,), E (9,) in ENTRIES order, contrib (n, 9), inside (n,)."""

    def __init__(self, H, dTr, A, E, contrib, inside):
        self.H, self.dTr, self.A, self.E, self.contrib, self.inside = H, dTr, A, E, contrib, inside

    @property
    def sums(self) -> np.ndarray:
        """(9,) in ENTRIES order"""
        return np.array([self.H[0, 0], self.H[1, 1], self.H[2, 2], self.H[0, 1], self.H[0, 2], self.H[1, 2],
                         self.dTr[0], self.dTr[1], self.dTr[2]])


def evaluate(prob, pts, pose_map, pt_scale=1.0, cs=None) -> Eval64:
    """getCompleteHessianDerivs of one scan.  prob: (S_y, S_x) float32 probability plane of the level; pts: (n, 2)
    float32 endpoints in level-0 cells (the container's units); pose_map: (3,) float32 in the level's cells;
    pt_scale: the level's 2^-k (MapRepMultiMap.h:127)."""
    prob = np.ascontiguousarray(prob, dtype=np.float32)
    sy, sx = prob.shape
    pts = np.ascontiguousarray(pts, dtype=np.float32).reshape(-1, 2)
    n = pts.shape[0]
    pose = np.asarray(pose_map, np.float32).reshape(3)
    f32 = np.float32
    s, c = (sinf(pose[2]), cosf(pose[2])) if cs is None else (np.float32(cs[1]), np.float32(cs[0]))   # cs: (c, s) in place of libm's
    x, y = pose[0], pose[1]
    with np.errstate(invalid="ignore", over="ignore"):
        px = pts[:, 0] * f32(pt_scale)                      # DataPointContainer setFrom: exact (power of two)
        py = pts[:, 1] * f32(pt_scale)
        qx = c * px + ((-s) * py + x)                       # Eigen Affine2f * Vector2f, every op rounded (fp32)
        qy = s * px + (c * py + y)
        lim_x, lim_y = f32(sx) - f32(2.0), f32(sy) - f32(2.0)
        inside = (qx >= 0) & (qx <= lim_x) & (qy >= 0) & (qy <= lim_y)   # NaN compares false: out of the map
    qx_in = np.where(inside, qx, f32(0))
    qy_in = np.where(inside, qy, f32(0))
    ix, iy = qx_in.astype(np.int64), qy_in.astype(np.int64)   # trunc == floor on [0, S-2]
    fx = (qx_in - ix.astype(np.float32)).astype(np.float64)   # exact in fp32 (q >= 0, same binade or below)
    fy = (qy_in - iy.astype(np.float32)).astype(np.float64)
    flat = prob.reshape(-1)
    idx = iy * sx + ix
    i0 = flat[idx].astype(np.float64)
    i1 = flat[idx + 1].astype(np.float64)
    i2 = flat[idx + sx].astype(np.float64)
    i3 = flat[idx + sx + 1].astype(np.float64)

    # ---- float64: the reference's formulas (OccGridMapUtil.h:342-345, :82, :87) ----------------------------
    with np.errstate(invalid="ignore", over="ignore"):   # non-finite endpoints: masked below
        xi, yi = 1.0 - fx, 1.0 - fy
        M = (i0 * xi + i1 * fx) * yi + (i2 * xi + i3 * fx) * fy
        gx = -((i0 - i1) * xi + (i2 - i3) * fx)
        gy = -((i0 - i2) * yi + (i1 - i3) * fy)
        F = 1.0 - M
        s64, c64 = float(s), float(c)
        px64, py64 = px.astype(np.float64), py.astype(np.float64)
        rx = c64 * px64 - s64 * py64
        ry = s64 * px64 + c64 * py64
        R = (-ry) * gx + rx * gy
        prods = np.stack([gx * gx, gy * gy, R * R, gx * gy, gx * R, gy * R, gx * F, gy * F, R * F], axis=1)
        prods[~inside] = 0.0

        # ---- first-order bounds on the kernel's fp32 rounding of one endpoint (fp32 data in, exact products out) ----
        # regrouped bilinear form: d01 = i1-i0, d02 = i2-i0, t = i3-i2, dd = t-d01, gx = fma(fx,dd,d01),
        # gy = fma(fy,dd,d02), M = fma(fy, fma(fx,dd,d02), fma(fx,d01,i0)), f = 1-M, r = fma(rx,gy,-(ry*gx)) with
        # rx = cs*px - ss*py, ry = ss*px + cs*py (products rounded); e(.) is |computed - exact| to first order in u.
        u = U32
        d01, d02, t = i1 - i0, i2 - i0, i3 - i2
        dd = t - d01
        e_d01, e_d02, e_t = u * np.abs(d01), u * np.abs(d02), u * np.abs(t)
        e_dd = u * np.abs(dd) + e_t + e_d01
        e_gx = u * np.abs(gx) + fx * e_dd + e_d01
        e_gy = u * np.abs(gy) + fy * e_dd + e_d02
        in1, in2 = fx * dd + d02, fx * d01 + i0
        e_in1 = u * np.abs(in1) + fx * e_dd + e_d02
        e_in2 = u * np.abs(in2) + fx * e_d01
        e_M = u * np.abs(M) + fy * e_in1 + e_in2
        e_F = u * np.abs(F) + e_M
        cpx, spy, spx, cpy = np.abs(c64 * px64), np.abs(s64 * py64), np.abs(s64 * px64), np.abs(c64 * py64)
        e_rx = u * (cpx + spy + np.abs(rx))
        e_ry = u * (spx + cpy + np.abs(ry))
        e_R = (u * np.abs(R) + u * np.abs(ry * gx) + np.abs(gy) * e_rx + np.abs(rx) * e_gy + np.abs(gx) * e_ry
               + np.abs(ry) * e_gx)
        ag, bg, ar, af = np.abs(gx), np.abs(gy), np.abs(R), np.abs(F)

        def e_prod(a, ea, b, eb):
            return a * eb + b * ea + ea * eb

        errs = np.stack([e_prod(ag, e_gx, ag, e_gx), e_prod(bg, e_gy, bg, e_gy), e_prod(ar, e_R, ar, e_R),
                         e_prod(ag, e_gx, bg, e_gy), e_prod(ag, e_gx, ar, e_R), e_prod(bg, e_gy, ar, e_R),
                         e_prod(ag, e_gx, af, e_F), e_prod(bg, e_gy, af, e_F), e_prod(ar, e_R, af, e_F)], axis=1)
        errs[~inside] = 0.0
    sums = prods.sum(axis=0) if n else np.zeros(9)
    H = h_matrix(sums)
    dTr = sums[6:9].copy()
    A = np.abs(prods).sum(axis=0) if n else np.zeros(9)
    E = errs.sum(axis=0) if n else np.zeros(9)
    return Eval64(H, dTr, A, E, prods, inside)


def evaluate_batch(prob, pts, offsets, poses_map, pt_scale=1.0) -> list[Eval64]:
    """A batch in the C-ABI's layout: pts (N, 2), offsets (B + 1,) or None (every pose uses all of pts)."""
    poses_map = np.asarray(poses_map, np.float32).reshape(-1, 3)
    out = []
    for b in range(poses_map.shape[0]):
        scan = pts if offsets is None else pts[int(offsets[b]):int(offsets[b + 1])]
        out.append(evaluate(prob, scan, poses_map[b], pt_scale))
    return out
