"""GPU: every Gauss-Newton evaluation of the match kernel on non-square, odd-sized and off-centre multi-level maps
(tests/match_cases.py: 404 x 300 x 3, 150 x 404 x 2 at start (0.3, 0.7), 243 x 200 x 2, 257 x 131 x 3, 404 x 300 x 3
at 0.025 m and start (0.3, 0.7), 6000 x 100, 7 x 4; each with a 1-level companion whose origin is world (-0, -0)),
through the per-evaluation record (match_batch_record, matchData(record=True)), in both gather modes, with the default
iteration schedule and [-1, 2, 4].

  1. Sums: every recorded H / dTr on every level lies within tests/test_gpu_match_record.py's bound (tol) around
     oracle/hessian64.py at the device's own input pose, for W = 1, 2, 4, 8, 16, the single-scan entry and the
     shared-scan (hypothesis) mode.
  2. Power: every endpoint at a lane, warp-group, staging or CTA boundary moves some H entry by more than 4 tol at the
     coarsest level's first evaluation, at the hint the scan is designed for (the finer levels start where the
     coarser one hands over, and a scan unrelated to the map lets Gauss-Newton wander there), and so does every edge
     endpoint built to be inside, at its level's first evaluation: losing or doubling any of them fails 1.  (40 000
     endpoints on one or two warps: the bound exceeds one endpoint's share; held to the bound only.)
  3. Edges, built exactly (match_cases.build_edge_scan, coarsest level first, at the input pose the coarser levels
     hand over, on handles with one evaluation per coarse level; adding a level's edges leaves the coarser levels'
     records unchanged bit for bit): at the recorded input pose hessian64 classifies each as designed.  Which assertion sees which mistake in the bounds test:
       * lim_x and lim_y swapped, or one limit applied to both axes: the endpoints whose long-axis q lies between the
         two limits are inside, so 1 fails (by 2, each moves H by > 4 tol); with the short-axis limit on the long axis
         the q == lim_x (or lim_y) endpoints are lost as well;
       * `<` for `<=` on either axis: the q == lim_x / q == lim_y endpoints are lost: 1 fails, by 2;
       * a dropped -0 (a sign test in place of `>= 0`): the companions' q == -0 endpoints are lost: 1 fails, by 2.
     The first q past each edge and below 0 are asserted to be outside by the same classification.
  4. Bitwise classes: the record has the same bits in every HSB_CASE shape with the same W (stage_smem 0 / 1 / 2, with
     and without partial, seq 1 / 2 / 3) and in TEX and LDG, and turning it on changes no pose or covariance bit.
  5. Hand-offs: each level starts at the port's world_coords_pose(l + 1, .) of the coarser level's last estimate (angle
     by pose32.normalize_angle) and the result is the same conversion at level 0, bit for bit; hsb_map_coords_pose /
     hsb_world_coords_pose equal the port's (GridMapBase) on every level.  A scan wholly in level 0's strip beyond the
     coarse levels records H = 0 and est == start on every coarse level; a scan wholly outside does so everywhere.
  6. Estimates: every recorded estimate within 1e-4 m / rad of the C port's record, for the finite scans (the port,
     like the reference, indexes the map with a NaN endpoint) from hints settled where the port's match ends, where H
     is well conditioned (scaled cond < 1e3; the others are reported).  Not the edge scan: its endpoints lie exactly on
     the limits, so poses an ulp apart classify them differently; its sums are held to the bound at the device's poses.
  7. hsb_hessian_derivs on every level at the recorded input pose, with the edge endpoints, within the bound.
  8. The group step on 404 x 300 x 3 (0.025 m, start (0.3, 0.7)) and 243 x 200 x 2 equals the members stepped one by
     one, poses, covariances and planes bit for bit.
"""
import math

import numpy as np
import pytest

import match_cases as mcs
from conftest import report
from oracle import hessian64, pose32, record_oracle
from test_gpu_match_record import CASES, compare_with_port, port_record, tol  # noqa: F401 (port_record: a fixture)
from test_gpu_match_sums import boundary_indices

pytestmark = pytest.mark.gpu

f32 = np.float32
MODES = (1, 2)   # LDG, TEX
RESET = dict(warps_per_scan=0, scans_per_block=0, unroll=0, stage_smem=1, partial=1, packed=0, seq=0, inline_scan=0,
             host_out=1)
ALL = mcs.GEOMS + [mcs.companion(g) for g in mcs.GEOMS]
IDS = [mcs.geom_id(g) + ("-corner" if g[3] is mcs.CORNER else "") for g in ALL]
_SETUPS = {}
_WORST, _POWER, _EDGE = {}, {}, {}


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


class Setup:
    def __init__(self, capi, gi, sched):
        g = ALL[gi]
        sx, sy, L, start, res = g
        self.g, self.levels, self.iters = g, L, mcs.schedule(sched, L)
        self.corner = start is mcs.CORNER
        self.reps, self.edge_reps = {}, {}
        for reps, iters in ((self.reps, self.iters), (self.edge_reps, mcs.edge_iterations(L))):
            for mode in MODES:
                rep = capi.MapRepB200(res, sx, sy, levels=L, start=start, gather_mode=mode, max_iterations=iters)
                assert rep.gather_mode == mode
                for l, (a, b) in enumerate(mcs.level_sizes(g)):
                    assert rep.level_info(l)[:2] == (a, b)
                    rep.upload_level(l, mcs.field(a, b, l))
                reps[mode] = rep
        self.prob = [self.reps[1].download_prob(l) for l in range(L)]
        for l in range(L):
            assert np.array_equal(bits(self.prob[l]), bits(self.reps[2].download_prob(l))), l
        self.port = record_oracle.RecordOracle("port", res, sx, L, start=start, size_y=sy)
        for l, (a, b) in enumerate(mcs.level_sizes(g)):
            self.port.set_logodds(l, mcs.field(a, b, l))
        cases = mcs.Cases(g, self.prob, self.port, seed=100 + gi)
        self.cases = cases
        scans = []            # (hint, pts, tag, port: the port can match it)
        for k, n in enumerate(mcs.LENGTHS):
            h = cases.hint(k)
            scans.append((h, cases.scan(n, h), f"n{n}", False))
        for k, n in ((1, 1081), (2, 2049)):
            h = cases.hint(k)
            scans.append((h, cases.scan(n, h, nonfinite=False), f"finite{n}", True))
        if L > 1:
            h = cases.hint(5)
            scans.append((h, cases.strip_scan(700, h), "strip", True))
        h = cases.hint(6)
        scans.append((h, cases.outside_scan(300, h), "outside", True))
        rep = self.edge_reps[1]

        def runner(hint, pts):
            rep.set_tuning(**RESET)
            return rep.matchData(hint, pts, record=True)[2]

        h = cases.hint(3)
        base = cases.scan(1081, h, nonfinite=False, slots=mcs.SLOTS)
        h, pts, self.designed, _ = mcs.build_edge_scan(cases, runner, h, base, cases.slots)
        self.edge_index = len(scans)
        scans.append((h, pts, "edges", True))
        self.zero = []        # (scan index, endpoint index, axis): q == -0 endpoints
        if self.corner:
            for axis in (0, 1):
                h = f32([-0.0, -0.0, 0.0 if axis == 0 else -0.0])
                pose = self.port.map_coords_pose(0, h)
                assert np.array_equal(bits(pose), bits(rep.map_coords_pose(0, h))), (pose, rep.map_coords_pose(0, h))
                pts = cases.scan(1081, h, nonfinite=False, slots=1)
                ev = hessian64.evaluate(self.prob[0], pts, pose)
                pts[cases.slots[0]] = cases.zero_points(pose, ev.A[:6] / max(1, int(ev.inside.sum())), axis)
                self.zero.append((len(scans), int(cases.slots[0]), axis))
                scans.append((h, pts, f"minus-zero-{'xy'[axis]}", True))
        self.scans = scans
        self.hints = np.stack([s[0] for s in scans]).astype(np.float32)
        self.pts = np.concatenate([s[1] for s in scans]).astype(np.float32)
        self.offs = np.concatenate([[0], np.cumsum([s[1].shape[0] for s in scans])]).astype(np.int32)
        self.family = IDS[gi] + ("" if sched == "default" else "-" + sched)

    def close(self):
        for r in list(self.reps.values()) + list(self.edge_reps.values()):
            r.close()
        self.port.close()


@pytest.fixture(scope="module")
def setups(hsb_lib, port_record):
    from hector_slam_b200 import capi

    def get(gi, sched="default"):
        if (gi, sched) not in _SETUPS:
            _SETUPS[(gi, sched)] = Setup(capi, gi, sched)
        return _SETUPS[(gi, sched)]

    yield get
    for s in _SETUPS.values():
        s.close()
    for fam in sorted(_WORST):
        edge = f", min edge power {_EDGE[fam]:.1f}" if fam in _EDGE else ""
        report(f"match geometry [{fam}]: sums max err / tol = {_WORST[fam]:.3f}, min boundary power "
               f"{_POWER.get(fam, math.inf):.1f}{edge}")


def batch_record(rep, S, **tuning):
    rep.set_tuning(**{**RESET, **tuning})
    P, C, recs, raw = rep.match_batch_record(S.hints, S.pts, S.offs)
    shape = rep.last_launch_shape()
    rep.set_tuning(**RESET)
    return P, C, recs, raw, shape


def rec_batch(rec):
    """one scan's split record as a batch of one"""
    return [{k: np.asarray(v)[None] for k, v in r.items()} for r in rec]


def inside_power(ev, i, t):
    return float((np.abs(ev.contrib[i, :6]) / np.maximum(t[:6], 1e-300)).max())


def check_sums(S, recs, W, ns, label, scans=None, edges=False, power=True):
    """every level's every evaluation within tol(W) of hessian64 at the recorded input pose; the power of the boundary
    endpoints at the coarsest level's first evaluation and (edges) of the inside edge and -0 endpoints at their
    level's first evaluation"""
    scans = S.scans if scans is None else scans
    fam = S.family
    worst, pmin, emin = 0.0, math.inf, math.inf
    for b, (_, pts, tag, _) in enumerate(scans):
        n = pts.shape[0]
        if n == 0:
            for l in range(S.levels):
                assert np.all(recs[l]["H"][b] == 0) and np.all(recs[l]["est"][b] == 0), (label, tag, l)
            continue
        for l in range(S.levels):
            r = recs[l]
            pin = S.reps[1].map_coords_pose(l, r["start"][b])
            for e in range(r["H"].shape[1]):
                ev = hessian64.evaluate(S.prob[l], pts, pin, 2.0 ** -l)
                H, d = r["H"][b, e], r["dTr"][b, e]
                got = np.array([H[0, 0], H[1, 1], H[2, 2], H[0, 1], H[0, 2], H[1, 2], d[0], d[1], d[2]], np.float64)
                t = tol(ev, n, W)
                err = np.abs(got - ev.sums)
                assert np.all(err <= t), (label, tag, l, e, err, t)
                worst = max(worst, float((err / np.maximum(t, 1e-300)).max()))
                if e == 0 and ev.inside.any():
                    # the boundary endpoints at the pose the scan was designed for: the coarsest level's first
                    # evaluation, at the hint (the shared scan's other hints, and a multi-level edge scan's settled
                    # one, see it elsewhere)
                    settled = tag == "edges" and S.levels > 1
                    if power and l == S.levels - 1 and not settled and not (W <= 2 and n >= mcs.LONG):
                        idx = boundary_indices(n, W, ns)
                        if len(idx):
                            c = np.abs(ev.contrib[idx, :6]) / np.maximum(t[:6], 1e-300)
                            p = float(c.max(axis=1).min())
                            assert p > 4.0, (label, tag, l, "a lost / doubled boundary endpoint would go unseen", p)
                            pmin = min(pmin, p)
                    if edges and tag.startswith("minus-zero"):
                        for sb, i, axis in S.zero:
                            if sb == b:
                                p = inside_power(ev, i, t)
                                assert p > 4.0, (label, tag, "the -0 endpoint would go unseen", p)
                                emin = min(emin, p)
                pin = r["est"][b, e]
    _WORST[fam] = max(_WORST.get(fam, 0.0), worst)
    _POWER[fam] = min(_POWER.get(fam, math.inf), pmin)
    if emin < math.inf:
        _EDGE[fam] = min(_EDGE.get(fam, math.inf), emin)


GS = [(gi, sched) for gi in range(len(ALL)) for sched in ("default", "random")
      if sched == "default" or ALL[gi][2] > 1]
GS_IDS = [IDS[gi] + ("" if s == "default" else "-" + s) for gi, s in GS]


# ---- 1, 2, 3: sums, power, edges --------------------------------------------------------------------------------------
@pytest.mark.parametrize("gi,sched", GS, ids=GS_IDS)
def test_sums_every_w(setups, gi, sched):
    S = setups(gi, sched)
    for W in (1, 2, 4, 8, 16):
        P1, C1, recs, raw1, shape = batch_record(S.reps[1], S, warps_per_scan=W, scans_per_block=1)
        assert shape["warps_per_scan"] == W
        P2, C2, _, raw2, _ = batch_record(S.reps[2], S, warps_per_scan=W, scans_per_block=1)
        assert np.array_equal(bits(raw1), bits(raw2)), W          # TEX == LDG
        assert np.array_equal(bits(P1), bits(P2)) and np.array_equal(bits(C1), bits(C2)), W
        check_sums(S, recs, W, shape["staged_points"], f"{S.family} W{W}", edges=(W == 8))
        if W == 8:
            # the single-scan entry: the same record as the batch entry in its shape, in both gather modes
            for mode in MODES:
                rep = S.reps[mode]
                rep.set_tuning(**RESET)
                for b, (h, pts, tag, _) in enumerate(S.scans):
                    p, c, rec = rep.matchData(h, pts, record=True)
                    flat = np.concatenate([np.concatenate([rec[l]["start"], np.concatenate(
                        [rec[l]["H"].reshape(-1, 9), rec[l]["dTr"], rec[l]["est"]], axis=1).reshape(-1)])
                        for l in range(S.levels - 1, -1, -1)])
                    assert np.array_equal(bits(flat), bits(raw1[b])), (mode, tag)
                    assert np.array_equal(bits(p), bits(P1[b])), (mode, tag)


@pytest.mark.parametrize("gi,sched", GS, ids=GS_IDS)
def test_shared_scan_mode(setups, gi, sched):
    """offsets = None: every hint matches the same scan (pose hypotheses), hints in every quadrant and past +-pi"""
    S = setups(gi, sched)
    pts = S.scans[[s[2] for s in S.scans].index("finite1081")][1]
    hints = np.stack([S.cases.hint(k) for k in range(9)]).astype(np.float32)
    scans = [(h, pts, "shared", True) for h in hints]
    for mode in MODES:
        rep = S.reps[mode]
        rep.set_tuning(**RESET)
        _, _, recs, raw = rep.match_batch_record(hints, pts, None)
        shape = rep.last_launch_shape()
        if mode == 1:
            raw1 = raw
            check_sums(S, recs, shape["warps_per_scan"], shape["staged_points"], f"{S.family} shared", scans=scans,
                       power=False)
        else:
            assert np.array_equal(bits(raw), bits(raw1))


@pytest.mark.parametrize("gi", range(len(ALL)), ids=IDS)
def test_edges(setups, gi):
    """The edge scan, rebuilt nowhere: at the input pose each level records, every designed endpoint is classified as
    designed (q exactly its target), in both gather modes; the companions' q == -0 endpoints are inside."""
    S = setups(gi)
    h, pts, _, _ = S.scans[S.edge_index]
    for mode in MODES:
        rep = S.edge_reps[mode]
        rep.set_tuning(**RESET)
        _, _, rec = rep.matchData(h, pts, record=True)
        evs = mcs.check_edges(S.cases, rec, pts, S.designed)
        for l, i, axis, q, inside in S.designed:
            if inside:
                ev = evs[l][1]
                p = inside_power(ev, i, tol(ev, len(pts), 8))
                assert p > 4.0, (mode, l, i, axis, q, "an edge endpoint would go unseen", p)
                _EDGE[S.family] = min(_EDGE.get(S.family, math.inf), p)
        if mode == 1:   # the sums of every evaluation, and the boundary endpoints' power at the hint
            check_sums(S, rec_batch(rec), 8, rep.last_launch_shape()["staged_points"], f"{S.family} edges",
                       scans=[S.scans[S.edge_index]])
        kinds = {(a, t is None, inside) for _, _, a, t, inside in S.designed}
        assert {(0, False, True), (0, False, False), (1, False, True), (1, False, False)} <= kinds
        for b, i, axis in S.zero:
            hb, pb = S.scans[b][0], S.scans[b][1]
            _, _, rz = S.reps[mode].matchData(hb, pb, record=True)
            pin = rep.map_coords_pose(0, rz[0]["start"])
            q = mcs.q_map(pb[i], pin, 0)[axis][0]
            assert q == 0 and np.signbit(q), (axis, q, pin)
            assert hessian64.evaluate(S.prob[0], pb, pin).inside[i], axis
    if S.corner:
        assert len(S.zero) == 2


# ---- 4. bitwise classes -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gi", range(len(mcs.GEOMS)), ids=IDS[:len(mcs.GEOMS)])
def test_record_bitwise_classes(setups, gi):
    S = setups(gi)
    by_w = {}
    for mode in MODES:
        rep = S.reps[mode]
        for W, G, U in CASES:
            for stage, partial in ((0, 0), (1, 0), (1, 1), (2, 0), (2, 1)):
                for seq in (1, 2, 3):
                    tune = dict(warps_per_scan=W, scans_per_block=G, unroll=U, stage_smem=stage, partial=partial,
                                seq=seq)
                    rep.set_tuning(**{**RESET, **tune})
                    P0, C0 = rep.match_batch(S.hints, S.pts, S.offs)
                    P1, C1, _, raw, _ = batch_record(rep, S, **tune)
                    case = f"mode{mode} {tune}"
                    assert np.array_equal(bits(P0), bits(P1)) and np.array_equal(bits(C0), bits(C1)), case
                    if W not in by_w:
                        by_w[W] = (raw, case)
                    else:
                        assert np.array_equal(bits(raw), bits(by_w[W][0])), (case, "record differs from", by_w[W][1])
    rep.set_tuning(**RESET)


# ---- 5. hand-offs, strip, outside -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("gi,sched", GS, ids=GS_IDS)
def test_level_handoffs(setups, gi, sched):
    S = setups(gi, sched)
    rep, port = S.reps[1], S.port
    P, _, recs, _, _ = batch_record(rep, S)
    poses = []
    for b, (h, pts, tag, _) in enumerate(S.scans):
        nxt = h
        for l in range(S.levels - 1, -1, -1):
            r = recs[l]
            assert np.array_equal(bits(r["start"][b]), bits(nxt)), (tag, l, r["start"][b], nxt)
            poses += [r["start"][b]] + list(r["est"][b])
            if pts.shape[0] == 0:
                continue
            last = r["est"][b, -1]
            nxt = port.world_coords_pose(l, f32([last[0], last[1], pose32.normalize_angle(last[2])]))
        assert np.array_equal(bits(P[b]), bits(nxt)), (tag, P[b], nxt)
        sx_strip = tag == "strip" or tag == "outside"
        if sx_strip and pts.shape[0]:
            coarse = range(1, S.levels) if tag == "strip" else range(S.levels)
            for l in coarse:
                start_map = rep.map_coords_pose(l, recs[l]["start"][b])
                assert np.all(recs[l]["H"][b] == 0) and np.all(recs[l]["dTr"][b] == 0), (tag, l)
                for e in range(recs[l]["est"].shape[1]):
                    assert np.array_equal(bits(recs[l]["est"][b, e]), bits(start_map)), (tag, l, e)
            if tag == "strip":
                assert np.any(recs[0]["H"][b] != 0), "the strip scan must match on level 0"
    # the host's affine maps against GridMapBase's on every level, odd / off-centre / non-power-of-two included
    rng = np.random.default_rng(gi)
    sx, sy = S.g[0], S.g[1]
    extra = np.stack([rng.uniform(-0.2, 1.2, 64) * sx * S.g[4], rng.uniform(-0.2, 1.2, 64) * sy * S.g[4],
                      rng.uniform(-4, 4, 64)], axis=1).astype(np.float32)
    for p in list(S.hints) + poses + list(extra):
        for l in range(S.levels):
            assert np.array_equal(bits(rep.map_coords_pose(l, p)), bits(port.map_coords_pose(l, p))), (l, p)
            assert np.array_equal(bits(rep.world_coords_pose(l, p)), bits(port.world_coords_pose(l, p))), (l, p)


def scaled_cond(h):
    """condition number of H with its diagonal scaled to 1 (translation and angle have different units); 0 for H = 0"""
    h = np.asarray(h, np.float64)
    d = np.sqrt(np.abs(np.diag(h)))
    if not np.all(d > 0):
        return 0.0 if not np.any(h) else math.inf
    return float(np.linalg.cond(h / np.outer(d, d)))


# ---- 6. estimates against the C port -------------------------------------------------------------------------------------
@pytest.mark.parametrize("gi,sched", GS, ids=GS_IDS)
def test_estimates_vs_port(setups, gi, sched):
    S = setups(gi, sched)
    keep = []

    def port_runner(hint, pts):
        return mcs.split_record(S.port.match_record(hint, pts, S.iters)[2], S.levels, S.iters)

    for s in S.scans:
        if not s[3] or s[2] == "edges":   # (endpoints exactly on an edge flip as the pose moves by an ulp)
            continue
        # from a hint where the port's match ends: a scan unrelated to the map otherwise keeps Gauss-Newton moving,
        # and over five steps the last-bit differences the sums' bound allows grow past the bar
        hint = mcs.settle(S.cases, port_runner, s[0], s[1])
        # where some evaluation's H is ill-conditioned the fp32 solve amplifies them at once: reported, not compared
        H = np.concatenate([r["H"].reshape(-1, 3, 3) for r in port_runner(hint, s[1])])
        cond = max(scaled_cond(h) for h in H)
        if cond < 1e3:
            keep.append((hint, s[1], s[2]))
        else:
            report(f"match geometry [{S.family}] {s[2]}: cond(H) {cond:.1e} on the port's path, estimates not compared")
    assert len(keep) >= 2, (S.family, [s[2] for s in keep])
    for mode in MODES:
        rep = S.reps[mode]
        rep.set_tuning(**RESET)
        compare_with_port(S, rep, np.stack([s[0] for s in keep]).astype(np.float32), [s[1] for s in keep],
                          f"{S.family} mode{mode}")


# ---- 7. the one-evaluation seam ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gi", range(len(ALL)), ids=IDS)
def test_hessian_derivs_seam(setups, gi):
    S = setups(gi)
    rep = S.edge_reps[1]
    rep.set_tuning(**RESET)
    for b in [S.edge_index] + [z[0] for z in S.zero]:
        h, pts = S.scans[b][0], S.scans[b][1]
        _, _, rec = rep.matchData(h, pts, record=True)
        for l in range(S.levels):
            pin = rep.map_coords_pose(l, rec[l]["start"])
            pl = (pts * f32(2.0 ** -l)).astype(np.float32)
            ev = hessian64.evaluate(S.prob[l], pts, pin, 2.0 ** -l)
            t = np.max([tol(ev, len(pts), W) for W in (1, 2, 4, 8, 16)], axis=0)
            for mode in MODES:
                H, d = S.reps[mode].hessian_derivs(l, pin, pl)
                got = np.array([H[0, 0], H[1, 1], H[2, 2], H[0, 1], H[0, 2], H[1, 2], d[0], d[1], d[2]], np.float64)
                assert np.all(np.abs(got - ev.sums) <= t), (mode, l, got, ev.sums, t)


# ---- 8. the group step ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gi", [4, 2], ids=[IDS[4], IDS[2]])
def test_group_step_equals_single_steps(setups, gi):
    from hector_slam_b200 import capi

    S = setups(gi)
    sx, sy, L, start, res = S.g
    M, steps = 4, 5

    def make():
        rep = capi.MapRepB200(res, sx, sy, levels=L, start=start)
        rep.setMapUpdateMinDistDiff(0.0)
        rep.setMapUpdateMinAngleDiff(0.0)
        for l, (a, b) in enumerate(mcs.level_sizes(S.g)):
            rep.upload_level(l, mcs.field(a, b, l))
        return rep

    grp, one = [make() for _ in range(M)], [make() for _ in range(M)]
    group = capi.SlamGroup(grp)
    rng = np.random.default_rng(5)
    for k in range(steps):
        hints = np.stack([S.cases.hint(k * M + s) for s in range(M)]).astype(np.float32)
        scans = [S.cases.scan(int(rng.integers(300, 1500)), hints[s], nonfinite=False) for s in range(M)]
        mwm = [(s + k) % 3 == 2 for s in range(M)]
        P, Cv, U = group.slam_update(hints, scans, map_without_matching=mwm)
        for s in range(M):
            p, c, u = one[s].slam_update(hints[s], scans[s], map_without_matching=mwm[s])
            assert np.array_equal(bits(P[s]), bits(p)) and np.array_equal(bits(Cv[s]), bits(c)), (k, s)
            assert U[s] == u, (k, s)
    for s in range(M):
        for l in range(L):
            assert np.array_equal(bits(grp[s].download_level(l)), bits(one[s].download_level(l))), (s, l)
            assert np.array_equal(bits(grp[s].download_prob(l)), bits(one[s].download_prob(l))), (s, l)
    group.close()
    for r in grp + one:
        r.close()
