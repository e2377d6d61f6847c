"""GPU: the per-scan scalar pose arithmetic bit for bit, at every angle, in both gather modes.

  1. sin / cos of the pose angle at every call site for |psi| from 120 up (glibc's large-argument reduction,
     sincosf_glibc.h): the likelihood of one-endpoint scans equals likelihood64.sequential_fp32 of the endpoint's funval
     bit for bit through the host and device entry points and hsb_best_hypothesis_device's d_out_likelihood; the
     covariance equals likelihood64.covariance_fp32 of the seven sigma-point likelihoods; every coarsest-level
     evaluation of a match from a hint psi + 2 pi k lies within test_gpu_match_record.tol of the float64 evaluation at
     the device's input pose; the map writer's planes equal oracle/mapwrite.py's `dev` plane on every cell.  The
     likelihood, record and map-writer sections have a power check: at the chosen angles libm's sinf or cosf differs
     from the correctly rounded value, and with the correctly rounded pair at least one compared value would change.
     (The covariance is held to the formula on the device's own likelihoods, so its angle power is the likelihood's.)
  2. normalize_angle: a scan entirely out of the map (H = 0, no step) leaves each level's normalisation and conversion
     alone on the pose; outputs equal oracle/pose32.py's chain and the C port's match, NaN as NaN.
  3. The Gauss-Newton step: every recorded estimate equals pose32.step(previous estimate, H, dTr) bit for bit.
  4. The map-update gate (slam_gate) on empty-scan steps, whose pose is the hint: threshold boundaries, wrapped and
     unwrappable angle differences, zero and negative thresholds, the FLT_MAX state after reset, NaN hints and a NaN
     stored by a forced write, through slam_update (sync / nowait, inline_scan 0 / 1) and SlamGroup (full and subset).
"""
import math

import numpy as np
import pytest

from conftest import angle_diff, golden_planes, load_golden, report
from oracle import hessian64, likelihood64, mapwrite, pose32, record_oracle
from oracle.hessian64 import cosf, sinf

pytestmark = pytest.mark.gpu

F32 = np.float32
FMAX = np.finfo(F32).max
MODES = (1, 2)   # LDG, TEX
same = likelihood64.same_bits_or_nan


def bits(a):
    return np.ascontiguousarray(a, F32).view(np.uint32)


def cr(a):
    """the correctly rounded (cos, sin) of a float"""
    return F32(math.cos(float(F32(a)))), F32(math.sin(float(F32(a))))


def libm_differs(a):
    c, s = cr(a)
    return bits(cosf(a)) != bits(c) or bits(sinf(a)) != bits(s)


def step_ulps(x, k):
    x = F32(x)
    for _ in range(abs(k)):
        x = np.nextafter(x, F32(np.inf) if k > 0 else F32(-np.inf))
    return x


def large_angles(seed, n_diff=24):
    """(angles, chosen): large angles of both signs — n_diff where libm differs from the correctly rounded pair (the
    chosen ones), the floats around 120 and 2 pi k +- a few ulp"""
    rng = np.random.default_rng(seed)
    chosen = []
    while len(chosen) < n_diff:
        a = F32(math.copysign(10.0 ** rng.uniform(math.log10(120.0), 38.5), rng.uniform(-1, 1)))
        if np.isfinite(a) and abs(a) >= 120 and libm_differs(a):
            chosen.append(a)
    extra = [step_ulps(120.0, k) for k in (-2, -1, 0, 1, 2)] + [-F32(120.0), -step_ulps(120.0, 1)]
    for k in (20, 81, 1000, 159155):
        m = F32(2 * math.pi * k)
        extra += [step_ulps(m, d) for d in (-2, 0, 2)]
    return np.array(chosen + extra, F32), np.array(chosen, F32)


# ---- 1a. likelihood and covariance at large angles -------------------------------------------------------------------
RES, SIZE = 0.25, 1024   # start (0, 0): world <-> map is exact (a power-of-two scale, no offset)


@pytest.fixture(scope="module")
def plane_reps(hsb_lib):
    from hector_slam_b200 import capi

    rng = np.random.default_rng(21)
    lo = rng.uniform(-3.0, 3.0, (SIZE, SIZE)).astype(F32)
    reps = {}
    for mode in MODES:
        rep = capi.MapRepB200(RES, SIZE, levels=1, start=(0.0, 0.0), gather_mode=mode)
        rep.upload_level(0, lo)
        reps[mode] = rep
    yield reps
    for r in reps.values():
        r.close()


@pytest.mark.parametrize("mode", MODES)
def test_likelihood_large_angles(plane_reps, mode):
    import torch

    rep = plane_reps[mode]
    prob = rep.download_prob(0)
    angles, chosen = large_angles(3)
    rng = np.random.default_rng(4)
    pts = rng.uniform(-400.0, 400.0, (64, 2)).astype(F32)
    want, powered = [], 0
    poses = []
    for a in angles:
        pw = F32([128.0, 128.0, a])
        pm = rep.map_coords_pose(0, pw)
        assert np.array_equal(bits(pm), bits(F32([512.0, 512.0, a])))
        f, _ = likelihood64.endpoint_funval(prob, pts, pm)
        want.append([likelihood64.sequential_fp32([v]) for v in f])
        if a in chosen:
            g, _ = likelihood64.endpoint_funval(prob, pts, pm, cs=cr(a))
            assert np.any(bits(f) != bits(g)), (float(a), "a one-ulp sin / cos would go unseen")
            powered += 1
        poses.append(np.repeat(pw[None], 64, axis=0))
    want = np.array(want, F32).reshape(-1)
    poses = np.concatenate(poses).astype(F32)
    allpts = np.tile(pts, (len(angles), 1)).astype(F32)
    offs = np.arange(len(poses) + 1, dtype=np.int32)
    got = rep.likelihood_batch(0, poses, allpts, offs)
    bad = np.flatnonzero(bits(got) != bits(want))
    assert bad.size == 0, [(float(poses[i, 2]), float(got[i]), float(want[i])) for i in bad[:6]]
    dev = torch.device("cuda", 0)
    d_poses, d_pts, d_offs = (torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in (poses, allpts, offs))
    d_out = torch.full((len(poses),), -7.0, dtype=torch.float32, device=dev)
    rep.likelihood_batch_device(0, len(poses), d_poses.data_ptr(), d_pts.data_ptr(), d_offs.data_ptr(), 0,
                                d_out.data_ptr(), 0)
    torch.cuda.synchronize()
    assert np.array_equal(bits(d_out.cpu().numpy()), bits(want))
    d_best = torch.zeros(4, dtype=torch.float32, device=dev)
    d_out2 = torch.full((len(poses),), -7.0, dtype=torch.float32, device=dev)
    rep.best_hypothesis_device(0, len(poses), d_poses.data_ptr(), d_pts.data_ptr(), d_offs.data_ptr(), 0,
                               d_best.data_ptr(), d_out2.data_ptr(), 0)
    torch.cuda.synchronize()
    assert np.array_equal(bits(d_out2.cpu().numpy()), bits(want))
    assert powered == len(chosen)
    report(f"pose angles: likelihood mode{mode}: {len(poses)} one-endpoint poses at {len(angles)} angles bit for bit, "
           f"{powered} with a power check")


@pytest.mark.parametrize("mode", MODES)
def test_covariance_large_angles(plane_reps, mode):
    rep = plane_reps[mode]
    angles, _ = large_angles(5, n_diff=8)
    pts = np.random.default_rng(6).uniform(-300.0, 300.0, (96, 2)).astype(F32)
    poses = np.stack([F32([128.0, 128.0, a]) for a in angles]).astype(F32)
    cm, cw = rep.covariance_batch(0, poses, pts, None)
    for b, a in enumerate(angles):
        pm = F32([512.0, 512.0, a])
        sp = likelihood64.sigma_points(pm)
        lhs = rep.likelihood_batch(0, (sp * F32([RES, RES, 1.0])).astype(F32), pts, None)
        wm, ww = likelihood64.covariance_fp32(lhs, pm, RES)
        assert same(cm[b], wm) and same(cw[b], ww), (mode, float(a), cm[b], wm)


# ---- 1b. the map writer at large angles ------------------------------------------------------------------------------
def boundary_points(L, pose, rng, n=3000):
    """endpoints whose end cells lie on a cell boundary (q + 0.5 an integer, up to rounding), all around the pose"""
    mx, my = (float(v) for v in mapwrite._affine(L.mtw, pose[0], pose[1]))
    r = rng.uniform(20.0, 250.0, n)
    t = rng.uniform(0.0, 2 * math.pi, n)
    tx, ty = np.floor(mx + r * np.cos(t)) - 0.5, np.floor(my + r * np.sin(t)) - 0.5
    sel = rng.random(n) < 0.5   # half on an x boundary, half on a y boundary
    tx = np.where(sel, tx, tx + 0.3)
    ty = np.where(sel, ty + 0.3, ty)
    return mapwrite.points_for_targets(L, pose, np.stack([tx, ty], axis=1))


@pytest.mark.parametrize("mode", MODES)
def test_map_writer_large_angles(hsb_lib, mode):
    from hector_slam_b200 import capi

    rng = np.random.default_rng(8)
    angles, chosen = large_angles(9, n_diff=6)
    res, size = 0.05, 512
    L = mapwrite.geometry(res, size, size, 1)[0]
    flips = 0
    for k, a in enumerate(list(chosen) + [angles[-1], angles[-4]]):
        pose = mapwrite.pose_for_cell(L, 256.3, 255.7, a)
        pts = boundary_points(L, pose, rng)
        b_lib, b_cr = mapwrite.beams(L, pts, pose), mapwrite.beams(L, pts, pose, cs=cr(pose[2]))
        moved = int(np.sum(b_lib.kept & ((b_lib.x1 != b_cr.x1) | (b_lib.y1 != b_cr.y1))))
        if a in chosen:
            assert moved > 0, (float(a), "no end cell moves under the correctly rounded sin / cos")
        flips += moved
        for path in ("level", "slam"):
            rep = capi.MapRepB200(res, size, levels=1, gather_mode=mode, update_factor_free=0.4,
                                  update_factor_occupied=0.9)
            lf, lo = rep.logodds_increments()
            m = mapwrite.MultiMap(res, size, size, 1, lf, lo)
            want = m.update_level(0, pts, pose).dev
            if path == "level":
                rep.update_level_by_scan(0, pts, pose)
            else:
                p, _, upd = rep.slam_update(pose, pts, map_without_matching=True)
                assert upd and np.array_equal(bits(p), bits(pose))
            got = rep.download_level(0)
            rep.close()
            diff = int(np.sum(bits(got) != bits(want)))
            assert diff == 0, (mode, path, float(a), diff)
    report(f"pose angles: map writer mode{mode}: {flips} end cells that a one-ulp sin / cos moves, planes bit for bit")


# ---- 1c / 2 / 3. matches: records at large angles, normalisation, the step ------------------------------------------------
class Golden:
    def __init__(self, capi, name):
        g = load_golden(name + ".npz")
        self.g = g
        self.size, self.levels, self.res = int(g["size"]), int(g["levels"]), float(g["res"])
        planes = golden_planes(g)
        self.reps = {}
        for mode in MODES:
            rep = capi.MapRepB200(self.res, self.size, levels=self.levels, gather_mode=mode)
            for l in range(self.levels):
                rep.upload_level(l, planes[l])
            self.reps[mode] = rep
        self.port = record_oracle.RecordOracle("port", self.res, self.size, self.levels)
        for l in range(self.levels):
            self.port.set_logodds(l, planes[l])
        self.prob = [self.reps[1].download_prob(l) for l in range(self.levels)]

    def close(self):
        for r in self.reps.values():
            r.close()
        self.port.close()


@pytest.fixture(scope="module")
def G3(hsb_lib):
    import subprocess

    from conftest import ROOT
    from hector_slam_b200 import capi

    if not record_oracle.available("port"):
        subprocess.run(["make", "-C", f"{ROOT}/oracle", "-f", "record.mk", "port"], check=True, capture_output=True)
    s = Golden(capi, "match3")
    yield s
    s.close()


RESET = dict(warps_per_scan=0, scans_per_block=0, unroll=0, stage_smem=1, partial=1, packed=0, seq=0, inline_scan=0,
             host_out=1)
TURNS = (0, 20, 81, 1000, 159155, -37)


def large_hints(S):
    """the golden scans with their hints turned by 2 pi k"""
    scans, hints = [], []
    for k in range(S.g["scans"].shape[0]):
        for t in TURNS:
            scans.append(S.g["scans"][k])
            h = S.g["hints"][k].astype(np.float64)
            hints.append(F32([h[0], h[1], h[2] + 2 * math.pi * t]))
    return scans, np.stack(hints).astype(F32)


def records(S, rep, hints, scans, W):
    """-> list of (hint, scan, split record) for the batch entry point at W warps per scan (W = None: the single-scan
    entry point)"""
    out = []
    if W is None:
        rep.set_tuning(**RESET)
        for h, s in zip(hints, scans):
            _, _, rec = rep.matchData(h, s, record=True)
            out.append((h, s, [dict(start=r["start"], H=r["H"], dTr=r["dTr"], est=r["est"]) for r in rec]))
        return out
    rep.set_tuning(**{**RESET, "warps_per_scan": W, "scans_per_block": 1})
    pts = np.concatenate(scans).astype(F32) if scans else np.zeros((0, 2), F32)
    offs = np.concatenate([[0], np.cumsum([s.shape[0] for s in scans])]).astype(np.int32)
    P, C, recs, _ = rep.match_batch_record(hints, pts, offs)
    rep.set_tuning(**RESET)
    for b in range(len(scans)):
        out.append((hints[b], scans[b], [{k: v[b] for k, v in recs[l].items()} for l in range(S.levels)], P[b]))
    return out


@pytest.mark.parametrize("mode", MODES)
def test_k1_records_large_angles(G3, mode):
    """coarsest-level evaluations within test_gpu_match_record.tol around hessian64 at the device's input pose; the
    record is self-consistent; estimates within 1e-4 of the port's where |psi| < 512"""
    from test_gpu_match_record import tol

    S = G3
    rep = S.reps[mode]
    scans, hints = large_hints(S)
    top = S.levels - 1
    checked, powered = 0, 0
    for W in (1, 8, None):
        for item in records(S, rep, hints, scans, W):
            hint, scan, rec = item[:3]
            n = scan.shape[0]
            r = rec[top]
            pin = rep.map_coords_pose(top, r["start"])
            for e in range(r["H"].shape[0]):
                ev = hessian64.evaluate(S.prob[top], scan, pin, 2.0 ** -top)
                H, d = r["H"][e], r["dTr"][e]
                got = np.array([H[0, 0], H[1, 1], H[2, 2], H[0, 1], H[0, 2], H[1, 2], d[0], d[1], d[2]], np.float64)
                t = tol(ev, n, W or 8)
                assert np.all(np.abs(got - ev.sums) <= t), (W, float(hint[2]), e, np.abs(got - ev.sums), t)
                if abs(float(pin[2])) >= 120 and libm_differs(pin[2]):
                    ev_cr = hessian64.evaluate(S.prob[top], scan, pin, 2.0 ** -top, cs=cr(pin[2]))
                    powered += int(np.any(np.abs(ev_cr.sums - ev.sums) > t))
                checked += 1
                pin = r["est"][e]
            # self-consistency: normalised and converted, the last estimate is the next level's start / the pose
            nxt = hint
            for l in range(top, -1, -1):
                assert np.array_equal(bits(rec[l]["start"]), bits(nxt)), (W, float(hint[2]), l)
                last = rec[l]["est"][-1]
                nxt = rep.world_coords_pose(l, F32([last[0], last[1], pose32.normalize_angle(last[2])]))
            if W is not None:
                assert np.array_equal(bits(item[3]), bits(nxt)), (W, float(hint[2]))
            if abs(float(hint[2])) < 512:
                _, _, prec = S.port.match_record(hint, scan)
                port = rep.split_record(prec)
                for l in range(top, -1, -1):
                    cl = S.port.cell_length(l)
                    for e in range(rec[l]["est"].shape[0]):
                        a, p = rec[l]["est"][e], port[l]["est"][e]
                        dxy = float(np.abs(a[:2].astype(np.float64) - p[:2]).max()) * cl
                        assert dxy <= 1e-4 and float(angle_diff(a[2], p[2])) <= 1e-4, (W, float(hint[2]), l, e, a, p)
    report(f"pose angles: K1 mode{mode}: {checked} coarsest-level evaluations at hints psi + 2 pi k within the float64 "
           f"bound; {powered} of them would leave it with the correctly rounded sin / cos")
    assert powered > 0


EDGE_ANGLES = F32([0.0, -0.0, math.pi, -math.pi, 3.1415925, -3.1415925, 3.1415929, -3.1415929, 6.2831855, -6.2831855,
                   6.283185, 6.2831860, -6.2831860, 12.566371, -12.566371, 1e3, -1e3, 1e6, -1e6, 3.4e38, -3.4e38, FMAX,
                   1e-40, -1e-40, 1e-45, -1e-30, np.inf, -np.inf, np.nan])


@pytest.mark.parametrize("mode", MODES)
def test_normalisation_chain(G3, mode):
    S = G3
    rep = S.reps[mode]
    far = (S.g["scans"][0] + F32(1e5)).astype(F32)   # every endpoint out of the map: H = 0, no step
    hints = np.stack([F32([S.g["hints"][0][0], S.g["hints"][0][1], a]) for a in EDGE_ANGLES]).astype(F32)
    P, _ = rep.match_batch(hints, np.tile(far, (len(hints), 1)),
                           (np.arange(len(hints) + 1) * far.shape[0]).astype(np.int32))
    for b, h in enumerate(hints):
        w = h.copy()
        for l in range(S.levels - 1, -1, -1):
            est = S.port.map_coords_pose(l, w)
            est[2] = pose32.normalize_angle(est[2])
            w = S.port.world_coords_pose(l, est)
        port, _ = S.port.match(h, far)
        assert same(P[b], w) and same(port, w), (mode, float(h[2]), P[b], w, port)
    # the single-scan entry point on the same inputs
    for b, h in enumerate(hints[::3]):
        p, _ = rep.matchData(h, far)
        assert same(p, P[3 * b]), (mode, float(h[2]))


def step_inputs(S):
    """the goldens, their hints 0.3 rad off, scans of 1 / 2 / 3 endpoints, NaN / inf endpoints, all out of the map, and
    hints turned by 2 pi k"""
    scans, hints = [], []
    g = S.g
    for k in range(g["scans"].shape[0]):
        s, h = g["scans"][k], g["hints"][k]
        bad = s[:40].copy()
        bad[3], bad[7] = [np.nan, 1.0], [np.inf, -np.inf]
        for hh, ss in ((h, s), (h + F32([0, 0, 0.3]), s), (h - F32([0, 0, 0.3]), s), (h, s[:1]), (h, s[:2]),
                       (h, s[:3]), (h, bad), (h, (s + F32(1e5)).astype(F32))):
            scans.append(np.ascontiguousarray(ss, F32))
            hints.append(F32(hh))
    ls, lh = large_hints(S)
    return scans + ls, np.concatenate([np.stack(hints), lh]).astype(F32)


@pytest.mark.parametrize("mode", MODES)
def test_step_every_evaluation(G3, mode):
    S = G3
    rep = S.reps[mode]
    scans, hints = step_inputs(S)
    n_steps, n_nan = 0, 0
    for W in (1, 2, 8, 16, None):
        for item in records(S, rep, hints, scans, W):
            hint, scan, rec = item[:3]
            if scan.shape[0] == 0:
                continue
            for l in range(S.levels - 1, -1, -1):
                r = rec[l]
                prev = rep.map_coords_pose(l, r["start"])
                for e in range(r["H"].shape[0]):
                    want = pose32.step(prev, r["H"][e], r["dTr"][e])
                    assert same(r["est"][e], want), (W, mode, float(hint[2]), l, e, prev, r["H"][e], r["dTr"][e],
                                                     r["est"][e], want)
                    n_steps += 1
                    n_nan += int(np.isnan(want).any())
                    prev = r["est"][e]
    report(f"pose angles: step mode{mode}: {n_steps} recorded evaluations equal pose32.step ({n_nan} NaN)")
    assert n_nan > 0


# ---- 4. the map-update gate ------------------------------------------------------------------------------------------
def gate_cases():
    """(first hint, second hint, dist, ang, force first): the second step's gate runs against the first step's state"""
    pi = F32(math.pi)
    up = lambda x: np.nextafter(F32(x), F32(np.inf))      # noqa: E731
    dn = lambda x: np.nextafter(F32(x), F32(-np.inf))     # noqa: E731
    base = F32([1.5, -2.0, 0.25])
    out = []
    for k in (0, 3, 7, 12, 20):
        s = F32(2.0 ** -k)
        p1 = (base + F32([3 * s, 4 * s, 0.0])).astype(F32)
        out += [(base, p1, 5 * s, 1.0, False), (base, p1, dn(5 * s), 1.0, False)]
        out += [(F32([0, 0, 0]), F32([3 * s, 4 * s, 0]), 5 * s, 1.0, False),
                (F32([0, 0, 0]), F32([3 * s, 4 * s, 0]), dn(5 * s), 1.0, False)]
    for a, b in ((pi, -pi), (-pi, pi), (3.1, -3.1), (10.0, 0.0), (-10.0, 0.0), (0.0, 10.0), (up(pi), 0.0),
                 (0.0, up(pi)), (1e6, 0.0)):
        for ang in (0.05, 0.9, 3.0, 4.0):
            out.append((F32([1, 1, b]), F32([1, 1, a]), 0.4, ang, False))
    for t in (F32(0.25), F32(0.05)):
        for a in (t, -t):
            out += [(F32([0, 0, 0]), F32([0, 0, a]), 0.4, t, False), (F32([0, 0, 0]), F32([0, 0, a]), 0.4, dn(t), False),
                    (F32([0, 0, 0]), F32([0, 0, a]), 0.4, up(t), False), (F32([0, 0, 0]), F32([0, 0, up(a)]), 0.4, t, False)]
    z = F32([0.5, -0.5, 0.1])
    out += [(z, z, 0.0, 0.0, False), (z, z, -1.0, 0.0, False), (z, z, 0.0, -1.0, False),
            (z, F32([0.5, -0.5, up(0.1)]), 0.0, 0.0, False),
            (F32([np.nan, 0, 0]), z, 0.4, 0.9, False),        # a NaN hint after reset: no write, state stays FLT_MAX
            (F32([np.nan, 0, 0]), z, 0.4, 0.9, True),         # a NaN stored by a forced write: nothing writes after
            (F32([0, 0, np.nan]), z, -1.0, -1.0, True),
            (z, F32([0.5, -0.5, np.nan]), 0.4, 0.9, False)]
    return out


def expect_gate(state, pose, dist, ang, force):
    upd = pose32.pose_difference_larger_than(pose, state, dist, ang) or force
    return upd, (F32(pose).copy() if upd else state)


def expected_run(case):
    first, second, dist, ang, force = case
    state = np.full(3, FMAX, F32)
    u1, state = expect_gate(state, first, dist, ang, force)
    u2, state2 = expect_gate(state, second, dist, ang, False)
    u3, state3 = expect_gate(state2, first, dist, ang, False)
    return [(u1, state), (u2, state2), (u3, state3)]


def test_gate_single(hsb_lib):
    from hector_slam_b200 import capi

    empty = np.zeros((0, 2), F32)
    cases = gate_cases()
    fired = 0
    rep = capi.MapRepB200(0.05, 256, levels=2)
    for inline in (0, 1):
        rep.set_tuning(inline_scan=inline)
        for nowait in (False, True):
            for i, case in enumerate(cases):
                first, second, dist, ang, force = case
                rep.reset()
                assert np.all(rep.last_map_update_pose() == FMAX)
                rep.setMapUpdateMinDistDiff(float(dist))
                rep.setMapUpdateMinAngleDiff(float(ang))
                want = expected_run(case)
                for j, (hint, f) in enumerate(((first, force), (second, False), (first, False))):
                    p, _, upd = rep.slam_update(hint, empty, map_without_matching=f, nowait=nowait)
                    assert same(p, hint), (i, j, p, hint)
                    assert upd == want[j][0], (inline, nowait, i, j, case, upd, want[j][0])
                    assert same(rep.last_map_update_pose(), want[j][1]), (inline, nowait, i, j, case)
                    fired += int(upd)
    rep.close()
    assert 0 < fired < 12 * len(cases)


@pytest.mark.parametrize("subset", [False, True])
def test_gate_group(hsb_lib, subset):
    """every case a member of one group with its own thresholds; the subset form steps every other member, and the
    members left out keep their state"""
    from hector_slam_b200 import capi

    cases = gate_cases()
    reps = [capi.MapRepB200(0.05, 128, levels=2) for _ in cases]
    for rep, case in zip(reps, cases):
        rep.setMapUpdateMinDistDiff(float(case[2]))
        rep.setMapUpdateMinAngleDiff(float(case[3]))
    group = capi.SlamGroup(reps)
    M = len(cases)
    members = np.arange(0, M, 2, dtype=np.int32) if subset else np.arange(M, dtype=np.int32)
    want = [expected_run(c) for c in cases]
    for j in range(3):
        hints = np.stack([cases[i][0] if j != 1 else cases[i][1] for i in members]).astype(F32)
        force = [bool(cases[i][4]) and j == 0 for i in members]
        before = [reps[i].last_map_update_pose() for i in range(M)]
        P, _, U = group.slam_update(hints, [np.zeros((0, 2), F32)] * len(members), map_without_matching=force,
                                    members=members if subset else None)
        for k, i in enumerate(members):
            assert same(P[k], hints[k]), (j, i)
            assert U[k] == want[i][j][0], (subset, j, i, cases[i], U[k])
            assert same(reps[i].last_map_update_pose(), want[i][j][1]), (subset, j, i, cases[i])
        for i in set(range(M)) - set(members.tolist()):
            assert same(reps[i].last_map_update_pose(), before[i]), (j, i)
    group.close()
    for r in reps:
        r.close()
