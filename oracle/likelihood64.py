"""float64 reference of the pose likelihood and the sigma-point covariance — TEST INFRASTRUCTURE, not product code.

OccGridMapUtil::getLikelihoodForState = getLikelihoodForResidual(getResidualForState) with interpMapValue
(OccGridMapUtil.h:189-285, restated by hs_oracle.c hso_likelihood / interp_value), split the way oracle/hessian64.py
splits getCompleteHessianDerivs:

  * fp32, in the reference's operation order — the data every implementation shares: sinf / cosf of psi (libm), the
    level's 2^-k point scale, q = c*px + ((-s)*py + x) and qy = s*px + (c*py + y) with every operation rounded
    separately, the inclusive [0, S-2] bounds test (NaN is out of the map), the cell (trunc), fx, fy, the four fetched
    probabilities and each endpoint's funval = 1 - interp with the bilinear form exactly as :278-284 writes it
    (((i0*xi + i1*fx)*yi) + ((i2*xi + i3*fx)*fy), xi = 1 - fx, yi = 1 - fy), and 1 for an endpoint out of the map.
    The kernel evaluates funval with the same rounded operations (the library is built with -fmad=false), so these
    values are bit for bit what every implementation adds up.
  * float64: R64 = sum funval_i and lh64 = 1 - R64 / n (NaN for an empty scan, the reference's 0/0).

getCovarianceForPose + getCovMatrixWorldCoords (:106-187) is restated as an fp32 function of the seven likelihoods at
the sigma points, in the order the shim fixes for the fixed-size Eigen operations (hs_oracle.c hso_covariance_for_pose,
covariance_kernel): likelihoods.sum() by recursive halving, mean += sp*lh, mean *= 1/sum, cov += (lh*inv) * (d*d^T),
then the world-coordinate scaling — every operation rounded separately.
"""
from __future__ import annotations

import numpy as np

from oracle.hessian64 import U32, cosf, sinf

F32 = np.float32
DT, DA = F32(1.5), F32(0.05)   # OccGridMapUtil.h:109-111: sigma-point offsets (cells, rad)


class Lh64:
    """One pose's likelihood.  funval (n,) float32 per endpoint, inside (n,), R64 = sum funval, lh64 = 1 - R64/n."""

    def __init__(self, funval, inside):
        self.funval, self.inside = funval, inside
        self.n = int(funval.shape[0])
        self.R64 = float(funval.astype(np.float64).sum())
        with np.errstate(invalid="ignore", divide="ignore"):
            self.lh64 = 1.0 - self.R64 / self.n if self.n else float("nan")

    def tol(self, k: int) -> float:
        """Bound on an fp32 evaluation whose every funval passes through at most k additions, followed by one division by
        (float)n and one subtraction: funval >= 0, so each partial sum is <= R64 and
        |lh32 - lh64| <= 1.01 ((k + 1) u R64 / n + u |lh64|)."""
        return 1.01 * ((k + 1) * U32 * self.R64 / self.n + U32 * abs(self.lh64)) if self.n else 0.0


def endpoint_funval(prob, pts, pose_map, pt_scale=1.0):
    """-> (funval (n,) float32, inside (n,) bool).  prob: (S_y, S_x) float32 probability plane of the level; pts: (n, 2)
    float32 endpoints in level-0 cells; pose_map: (3,) float32 state in the level's cells; pt_scale: the level's 2^-k."""
    prob = np.ascontiguousarray(prob, dtype=F32)
    sy, sx = prob.shape
    pts = np.ascontiguousarray(pts, dtype=F32).reshape(-1, 2)
    pose = np.asarray(pose_map, F32).reshape(3)
    s, c = sinf(pose[2]), cosf(pose[2])
    x, y = pose[0], pose[1]
    with np.errstate(invalid="ignore", over="ignore"):
        px = pts[:, 0] * F32(pt_scale)                      # exact (power of two)
        py = pts[:, 1] * F32(pt_scale)
        qx = c * px + ((-s) * py + x)                       # OccGridMapUtil.h:214, every op rounded (fp32)
        qy = s * px + (c * py + y)
        lim_x, lim_y = F32(sx) - F32(2.0), F32(sy) - F32(2.0)
        inside = (qx >= 0) & (qx <= lim_x) & (qy >= 0) & (qy <= lim_y)   # :289-291; NaN compares false: out
    qx_in = np.where(inside, qx, F32(0))
    qy_in = np.where(inside, qy, F32(0))
    ix, iy = qx_in.astype(np.int64), qy_in.astype(np.int64)   # :295 trunc
    fx = qx_in - ix.astype(F32)                               # :298 (exact)
    fy = qy_in - iy.astype(F32)
    flat = prob.reshape(-1)
    idx = iy * sx + ix
    i0, i1, i2, i3 = flat[idx], flat[idx + 1], flat[idx + sx], flat[idx + sx + 1]
    xi, yi = F32(1.0) - fx, F32(1.0) - fy                     # :278-279
    m = ((i0 * xi + i1 * fx) * yi) + ((i2 * xi + i3 * fx) * fy)   # :282-284
    funval = np.where(inside, F32(1.0) - m, F32(1.0)).astype(F32)   # :216; interpMapValue is 0 out of the map
    return funval, inside


def evaluate(prob, pts, pose_map, pt_scale=1.0) -> Lh64:
    return Lh64(*endpoint_funval(prob, pts, pose_map, pt_scale))


def sequential_fp32(funval) -> np.float32:
    """The reference's own fp32 evaluation from the per-endpoint data: residual += funval in endpoint order, then
    1 - residual / (float)n (:203-209)."""
    f = np.asarray(funval, F32)
    r = np.add.accumulate(f, dtype=F32)[-1] if f.size else F32(0.0)
    with np.errstate(invalid="ignore", divide="ignore"):
        return F32(1.0) - r / F32(f.size)


def sigma_points(pose_map) -> np.ndarray:
    """(7, 3) float32: the sigma points of getCovarianceForPose (:119-125) in the level's cells, fp32 as the reference
    forms them: +-1.5 cells in x, in y, +-0.05 rad, the pose itself."""
    x, y, a = (F32(v) for v in np.asarray(pose_map, F32).reshape(3))
    return np.array([[x + DT, y, a], [x - DT, y, a], [x, y + DT, a], [x, y - DT, a],
                     [x, y, a + DA], [x, y, a - DA], [x, y, a]], F32)


def covariance_fp32(lhs, pose_map, cell_length):
    """getCovarianceForPose (:106-160) + getCovMatrixWorldCoords (:162-187) from the seven likelihoods at
    sigma_points(pose_map), every fp32 operation rounded separately in the shim's order.  -> (cov_map, cov_world), each
    (3, 3) float32 row-major."""
    lh = [F32(v) for v in np.asarray(lhs, F32).reshape(7)]
    sp = sigma_points(pose_map)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        total = (lh[0] + (lh[1] + lh[2])) + ((lh[3] + lh[4]) + (lh[5] + lh[6]))   # likelihoods.sum(): recursive halving
        inv = F32(1.0) / total                                                    # :137
        mean = [F32(0.0)] * 3
        for i in range(7):
            for k in range(3):
                mean[k] = mean[k] + sp[i, k] * lh[i]                                # :144
        mean = [mk * inv for mk in mean]                                          # :147
        cov = [F32(0.0)] * 9
        for i in range(7):                                                        # :151-154
            d = [sp[i, 0] - mean[0], sp[i, 1] - mean[1], sp[i, 2] - mean[2]]
            wgt = lh[i] * inv
            for r in range(3):
                for c in range(3):
                    cov[3 * r + c] = cov[3 * r + c] + wgt * (d[r] * d[c])
        st = F32(cell_length)
        st2 = st * st                                                             # :169-170
        w = [F32(0.0)] * 9
        w[0] = cov[0] * st2                                                       # :172
        w[4] = cov[4] * st2
        w[3] = cov[3] * st2                                                       # (1,0) :175
        w[1] = w[3]
        w[6] = cov[6] * st                                                        # (2,0) :178
        w[2] = w[6]
        w[7] = cov[7] * st                                                        # (2,1) :181
        w[5] = w[7]
        w[8] = cov[8]                                                             # :184
    return np.array(cov, F32).reshape(3, 3), np.array(w, F32).reshape(3, 3)


def same_bits_or_nan(a, b) -> bool:
    """a and b equal bit for bit, except that a NaN matches any NaN (numpy's and the device's canonical NaNs differ)"""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))
