"""CPU: the float64 reference of the pose likelihood and the fp32 restatement of the sigma-point covariance
(oracle/likelihood64.py) against Oracle.likelihood / Oracle.covariance_for_pose — the C port always, the compiled
reference where oracle/_ref exists — on seeded planes with endpoints on the edges of the map's domain, on every level
of a 3-level map.

Bars:
  * the module's per-endpoint fp32 funval, summed sequentially and finished with 1 - R / (float)n in fp32, is the
    oracle's likelihood bit for bit: the per-endpoint data are the reference's own;
  * the oracle's fp32 likelihood is within 1.01 ((n + 1) u R64 / n + u |lh64|) of lh64 (the sequential sum's own bound);
  * covariance_fp32 applied to the oracle's seven likelihoods at sigma_points(pose) is the oracle's covariance, map and
    world matrices, bit for bit."""
import numpy as np
import pytest

from oracle import likelihood64

F32 = np.float32


def _edge_scan(rng, sx, sy, pose):
    """Endpoints for a state with psi = 0 and integer position: q = p + pose exactly, so the domain's edges are hit
    exactly — q on 0, on S-2, one ulp above S-2, one ulp below 0, at integers — plus -0.0 coordinates and bulk points
    inside and around the map.  (No non-finite endpoints: the reference lets NaN through its bounds test and indexes
    memory with it, SURVEY.md Q4; test_nonfinite_endpoints_count_one covers them.)"""
    lx, ly = F32(sx - 2), F32(sy - 2)
    x, y = pose[0], pose[1]
    up = np.float32(1e9)
    edge = [(0.0 - x, 0.0 - y), (lx - x, ly - y), (0.0 - x, ly - y), (lx - x, 0.0 - y),
            (np.nextafter(lx, up) - x, 5.0), (5.0, np.nextafter(ly, up) - y),
            (np.nextafter(F32(-x), -up), 3.0), (3.0, np.nextafter(F32(-y), -up)), (-x - 1.0, 2.0), (7.0, -y - 0.5),
            (-0.0, 2.0), (2.0, -0.0), (-0.0, -0.0)]
    ints = (rng.integers(0, min(sx, sy) - 2, (40, 2)).astype(F32) - F32([x, y])).astype(F32)
    bulk = np.stack([rng.uniform(-x - 3.0, sx - x + 3.0, 300), rng.uniform(-y - 3.0, sy - y + 3.0, 300)], axis=1)
    return np.concatenate([np.float32(edge), ints, bulk.astype(F32)]).astype(F32)


def _plane(rng, sx, sy):
    lo = rng.uniform(-4.0, 4.0, (sy, sx)).astype(F32)
    lo[: sy // 4, : sx // 4] = 0.0                       # flat patch: p = 0.5
    lo[sy // 2: sy // 2 + 3, :4] = 60.0                  # saturated: p = 1
    return lo


@pytest.mark.parametrize("size", [64, 96])
def test_likelihood_and_covariance_against_oracle(pyoracle, oracle_kinds, size):
    rng = np.random.default_rng(100 + size)
    planes = [_plane(rng, size >> l, size >> l) for l in range(3)]
    worst = 0.0
    for kind in oracle_kinds:
        orc = pyoracle.Oracle(kind, 0.05, size, 3)
        for l, p in enumerate(planes):
            orc.set_logodds(l, p)
        for l in range(3):
            s = size >> l
            prob = orc.get_prob(l)
            poses = [F32([3.0, 4.0, 0.0]), F32([1.0, 2.0, 0.0]), F32([-0.0, 5.0, 0.0]),
                     F32([s / 3.0, s / 2.0, 0.3]), F32([s / 2.0, s / 3.0, -2.9])]
            scans = []
            for k, pose in enumerate(poses):
                if pose[2] == 0.0:
                    pts = _edge_scan(rng, s, s, pose)
                else:
                    pts = rng.uniform(-s, s, (500, 2)).astype(F32)
                    pts[:3] = [[1e30, 2.0], [-3e38, 1.0], [2.0, 1e20]]     # far out of the map
                scans.append((pose, pts))
            scans += [(poses[3], np.zeros((0, 2), F32)), (poses[4], scans[3][1][:1]), (poses[0], scans[0][1][:33])]
            for k, (pose, pts) in enumerate(scans):
                what = f"{kind} size {size} level {l} pose {k} n {pts.shape[0]}"
                ev = likelihood64.evaluate(prob, pts, pose)
                got = F32(orc.likelihood(l, pose, pts))
                assert likelihood64.same_bits_or_nan(likelihood64.sequential_fp32(ev.funval), got), (what, got)
                if ev.n == 0:
                    assert np.isnan(got) and np.isnan(ev.lh64), what
                else:
                    tol = ev.tol(ev.n)
                    err = abs(float(got) - ev.lh64)
                    assert err <= tol, (what, err, tol)
                    worst = max(worst, err / tol if tol else 0.0)
                if pose[2] == 0.0 and pts.shape[0] > 16:
                    # q == 0 and q == S-2 are in (inclusive bounds), one ulp past them is out, -0.0 is in (q == -0.0
                    # itself for the state at x = -0.0)
                    assert ev.inside[:4].all() and not ev.inside[4:10].any() and ev.inside[10:13].all(), (what, ev.inside[:13])
                # the covariance from the oracle's own seven likelihoods at the sigma points
                sp = likelihood64.sigma_points(pose)
                lhs = [orc.likelihood(l, sp[i], pts) for i in range(7)]
                wm, ww = likelihood64.covariance_fp32(lhs, pose, orc.cell_length(l))
                cm, cw = orc.covariance_for_pose(l, pose, pts)
                assert likelihood64.same_bits_or_nan(wm, cm), (what, wm, cm)
                assert likelihood64.same_bits_or_nan(ww, cw), (what, ww, cw)
        orc.close()
    print(f"fp64 likelihood vs fp32 oracles: worst err / tol = {worst:.3f}")


def test_out_of_map_sigma_points_give_the_formula_nan_pattern(pyoracle):
    """A pose whose seven sigma points are all out of the map: every likelihood is 0, the sum is 0 and the covariance
    carries the formula's NaNs — the port agrees entry by entry."""
    orc = pyoracle.Oracle("port", 0.05, 64, 1)
    orc.set_logodds(0, np.zeros((64, 64), F32))
    pose = F32([500.0, 500.0, 0.1])
    pts = np.float32([[1.0, 2.0], [3.0, -1.0], [0.5, 0.5]])
    lhs = [orc.likelihood(0, p, pts) for p in likelihood64.sigma_points(pose)]
    assert lhs == [0.0] * 7
    wm, ww = likelihood64.covariance_fp32(lhs, pose, orc.cell_length(0))
    cm, cw = orc.covariance_for_pose(0, pose, pts)
    assert np.isnan(wm).any() and likelihood64.same_bits_or_nan(wm, cm) and likelihood64.same_bits_or_nan(ww, cw)
    orc.close()


def test_one_endpoint_is_visible():
    """The per-endpoint funval are kept so that a test can show its bound would see one endpoint lost: on a 2049-point
    scan with out-of-map endpoints at the lane boundaries, each of them moves lh64 by far more than the warp bound."""
    rng = np.random.default_rng(5)
    prob = rng.uniform(0.05, 0.95, (48, 48)).astype(F32)
    n = 2049
    pts = rng.uniform(1.0, 40.0, (n, 2)).astype(F32)
    idx = np.arange(n)
    heavy = (idx % 32 == 0) | (idx % 32 == 31) | (idx < 2) | (idx >= n - 2)
    pts[heavy] = (500.0, 500.0)
    ev = likelihood64.evaluate(prob, pts, F32([2.0, 3.0, 0.2]))
    assert np.all(ev.funval[heavy] == 1.0) and not ev.inside[heavy].any()
    tol = ev.tol(-(-n // 32) + 5)
    assert ev.funval[heavy].min() / n > 4 * tol


def test_nonfinite_endpoints_count_one():
    """NaN and +-inf endpoints are out of the map (the kernel's rule): funval 1 each, so the likelihood is the one of
    the finite endpoints with one residual of 1 per non-finite endpoint."""
    rng = np.random.default_rng(4)
    prob = rng.uniform(0.05, 0.95, (48, 40)).astype(F32)
    pts = rng.uniform(-5, 45, (200, 2)).astype(F32)
    pts[::7] = np.nan
    pts[3::11, 0] = np.inf
    pts[5::13, 1] = -np.inf
    bad = ~np.all(np.isfinite(pts), axis=1)
    ev = likelihood64.evaluate(prob, pts, F32([1.5, 2.25, 0.1]))
    ok = likelihood64.evaluate(prob, pts[~bad], F32([1.5, 2.25, 0.1]))
    assert not ev.inside[bad].any() and np.all(ev.funval[bad] == 1.0)
    assert np.array_equal(ev.funval[~bad], ok.funval)
    assert abs(ev.R64 - (ok.R64 + bad.sum())) <= 1e-12 * ev.R64
    # a non-finite or absurd state puts every endpoint out of the map: likelihood exactly 0
    for pose in ([np.nan, 2.0, 0.1], [np.inf, 2.0, 0.1], [1.0, -np.inf, 0.1], [1e30, 2.0, 0.1], [1.0, 2.0, np.nan]):
        ev = likelihood64.evaluate(prob, pts, F32(pose))
        assert not ev.inside.any() and ev.lh64 == 0.0 and likelihood64.sequential_fp32(ev.funval) == 0.0
