"""Scoring poses for a group's members in one pass (hsb_group_likelihood, hsb_group_covariance,
hsb_group_best_hypothesis and their _subset forms): every session's poses scored against that session's one scan on its
member's map by one launch, with one copy each way; the scan either sent with the call or the member's last matched scan
as it lies on the device.

Every likelihood, both covariance matrices and every session's best hypothesis are compared in bits with the single
calls (hsb_likelihood_batch, hsb_covariance_batch, hsb_best_hypothesis_device) on maps written by mixed full, subset,
nowait and map_without_matching group steps, on three non-square geometries, every level, ragged and empty sessions,
permuted member lists; with the float64 bound of oracle/likelihood64.py and the fp32 covariance formula on the group's
own seven sigma-point likelihoods; in last-match mode after steps of every input kind (conversions that drop beams
included); right after nowait steps of this group, of a member alone and of a second group.  Also: no member state
changes (a twin fleet stepped without queries ends byte-identical), edges, launch accounting, rejections and the C++
façade.  Every group case runs on a TEX and an LDG group."""
import ctypes as C
import os

import numpy as np
import pytest

import maptools_cases as mc
from conftest import ROOT
from oracle import likelihood64
from test_gpu_group_subset import geometry, group_step, member_cloud, member_transform, scan_of, session_data

pytestmark = pytest.mark.gpu

F32 = np.float32
MODES = pytest.mark.parametrize("mode", [2, 1], ids=["tex", "ldg"])   # capi.GATHER_TEX, capi.GATHER_LDG
# (sx, sy, levels, start)
GEOMS = [(404, 300, 3, (0.5, 0.5)), (150, 404, 2, (0.3, 0.7)), (257, 131, 2, (0.5, 0.5))]
GEOM = GEOMS[0]
KINDS = ("endpoints", "cloud", "ranges", "projected")
COUNTS = (0, 1, 7, 33, 700)
SENTINEL = 77


def bits(a):
    return np.ascontiguousarray(a, F32).view(np.uint32)


def make_rep(geom, s, mode):
    """Member s's handle: its own update factors, gate thresholds, beam geometry, laser mount and cloud thresholds"""
    from hector_slam_b200 import capi

    sx, sy, levels, start = geom
    rep = capi.MapRepB200(mc.RES, sx, sy, levels=levels, start=start, update_factor_free=0.4 + 0.02 * (s % 3),
                          update_factor_occupied=0.6 + 0.1 * (s % 4), gather_mode=mode)
    dist, ang = ((0.0, 0.0), (0.15, 0.1), (0.3, 0.5))[s % 3]
    rep.setMapUpdateMinDistDiff(dist)
    rep.setMapUpdateMinAngleDiff(ang)
    g = geometry(s)
    rep.set_scan_format(**g)
    rep.set_laser_projection(**g, range_cutoff=30.0)
    rep.set_cloud_format(member_transform(s), **member_cloud(s))
    assert rep.gather_mode == mode
    return rep


def fleet(geom, M, mode):
    from hector_slam_b200 import capi

    reps = [make_rep(geom, s, mode) for s in range(M)]
    return reps, capi.SlamGroup(reps)


def thinned(kind, scan):
    """the scan with every 7th beam (cloud: point) made one the conversion drops, so that the kept count is well below
    the input length"""
    if kind == "endpoints":
        return scan
    out = scan.copy()
    out[::7] = 0.0     # a range below range_min / a point nearer than the minimum distance
    return out


class Tracker:
    """What each member's last matched scan is (the input as given, and its kind) and the pose its last step returned."""

    def __init__(self, geom, M, mode):
        self.conv = [make_rep(geom, s, mode) for s in range(M)]   # never stepped: they only convert
        self.last = [None] * M      # (kind, input)
        self.pose = [np.zeros(3, F32) for _ in range(M)]

    def note(self, j, kind, scan, without, pose):
        if not without:
            self.last[j] = (kind, scan)
        self.pose[j] = np.asarray(pose, F32).copy()

    def scan(self, j):
        """the endpoints the matching *_to_points call returns for member j's last matched input (none: never matched)"""
        if self.last[j] is None:
            return np.zeros((0, 2), F32)
        kind, x = self.last[j]
        c = self.conv[j]
        if kind == "endpoints":
            return np.ascontiguousarray(x, F32)
        if kind == "ranges":
            return c.scan_to_points(x)
        return (c.cloud_to_points(x) if kind == "cloud" else c.projected_scan_to_points(x))[0]

    def close(self):
        for c in self.conv:
            c.close()


def step(groups, data, at, kind, members, rng, nowait, track=None, p_without=0.2):
    """one group step of `kind` over `members` (None: all) on every group of `groups`, the same inputs
    -> the results of each group"""
    M = len(data)
    sel = list(range(M)) if members is None else members
    without = [bool(rng.random() < p_without) and at[j] > 0 for j in sel]
    hints = np.asarray([data[j]["truth" if w else "hints"][at[j]] for j, w in zip(sel, without)], F32).reshape(len(sel), 3)
    scans = [thinned(kind, scan_of(kind, data[j], at[j])) for j in sel]
    out = [group_step(g, kind, hints, scans, without, members=members, nowait=nowait) for g in groups]
    for k, j in enumerate(sel):
        at[j] += 1
        if track is not None:
            track.note(j, kind, scans[k], without[k], out[0][0][k])
    return out


def hypotheses(rng, centre, q, specials=True):
    """q world poses around `centre`; with specials (q >= 7) a NaN and an infinite one, angles of 120 rad and beyond,
    and a tie: the last pose repeats an earlier one"""
    p = (np.asarray(centre, F32)[None] + rng.normal(0.0, 1.0, (q, 3)) * np.array([0.15, 0.15, 0.05])).astype(F32)
    if specials and q >= 7:
        p[1, 0] = np.nan
        p[2, 2] = np.inf
        p[3, 2] += F32(120.0)
        p[4, 2] = F32(-1000.5)
        p[q - 1] = p[5]
    return p


def single_best(rep, level, poses, pts):
    """hsb_best_hypothesis_device on device copies of one session -> (best4, likelihoods)"""
    import torch

    B = poses.shape[0]
    d_poses = torch.from_numpy(np.ascontiguousarray(poses, F32).reshape(-1)).cuda() if B else torch.zeros(3, device="cuda")
    d_pts = torch.from_numpy(np.ascontiguousarray(pts, F32).reshape(-1)).cuda() if pts.size else torch.zeros(2, device="cuda")
    d_best = torch.full((4,), 7.0, dtype=torch.float32, device="cuda")
    d_out = torch.full((max(B, 1),), 7.0, dtype=torch.float32, device="cuda")
    rep.best_hypothesis_device(level, B, d_poses.data_ptr(), d_pts.data_ptr(), None, pts.shape[0], d_best.data_ptr(),
                               d_out.data_ptr(), 0)
    torch.cuda.synchronize()
    return d_best.cpu().numpy(), d_out.cpu().numpy()[:B]


def expected_index(scores, poses):
    """the lowest index of the highest score, a non-finite pose and a NaN likelihood ranked -1 (no poses: -1)"""
    if not len(scores):
        return -1
    rank = np.where(np.all(np.isfinite(poses), axis=1) & ~np.isnan(scores), scores, F32(-1.0)).astype(F32)
    return int(np.argmax(rank))


def assert_sessions(g, reps, level, members, poses, scans, points, tag, cov_stride=1):
    """The three group calls over `members` (None: all) against the single calls on each member, in bits.  scans: the
    scan each session is scored against; points: what the group calls are given (the scans, or None for the members'
    last matched scans).  -> the group's likelihoods"""
    sel = list(range(len(reps))) if members is None else members
    lh = g.likelihood(level, poses, points, members=members)
    cm, cw = g.covariance(level, [p[::cov_stride] for p in poses], points, members=members)
    out, best4, index = g.best_hypothesis(level, poses, points, members=members)
    assert np.array_equal(bits(out), bits(lh)), tag
    q = c = 0
    for k, j in enumerate(sel):
        n, t = poses[k].shape[0], tag + (level, k, j)
        if n:
            want = reps[j].likelihood_batch(level, poses[k], scans[k])
            assert np.array_equal(bits(lh[q:q + n]), bits(want)), t
            pc = poses[k][::cov_stride]
            wm, ww = reps[j].covariance_batch(level, pc, scans[k])
            assert np.array_equal(bits(cm[c:c + len(pc)]), bits(wm)), t
            assert np.array_equal(bits(cw[c:c + len(pc)]), bits(ww)), t
            c += len(pc)
        b4, _ = single_best(reps[j], level, poses[k], scans[k])
        assert np.array_equal(bits(best4[k]), bits(b4)), (t, best4[k], b4)
        assert index[k] == expected_index(lh[q:q + n], poses[k]), (t, index[k])
        q += n
    assert q == lh.shape[0] and c == cm.shape[0]
    return lh


def close_all(*xs):
    for x in xs:
        for y in (x if isinstance(x, (list, tuple)) else [x]):
            y.close()


# ---- 1: against the single calls ----------------------------------------------------------------------------------

@MODES
@pytest.mark.parametrize("geom", GEOMS, ids=mc.geom_id)
def test_against_single_calls(hsb_lib, geom, mode):
    """Fleets of 3 to 6 members, 10 ticks of full and subset, sync and nowait group steps of every input kind (some
    sessions map_without_matching); after every tick a round at one level over a permuted subset with ragged sessions
    (0, 1, 7, 33, 700 poses: non-finite poses, angles past 120 rad and a tie among them), the scans sent with the call;
    at the end a full round at every level.  Everything equals the single calls on the members in bits."""
    M, ticks = 3 + GEOMS.index(geom) + (1 if mode == 1 else 0), 10
    reps, g = fleet(geom, M, mode)
    track = Tracker(geom, M, mode)
    data = [session_data(3100 + s, ticks, geometry(s)) for s in range(M)]
    rng = np.random.default_rng(41)
    at = [0] * M
    levels = geom[2]
    seen = []
    for t in range(ticks):
        members = None if t % 4 == 0 else [int(j) for j in rng.permutation(M)[:int(rng.integers(1, M + 1))]]
        step([g], data, at, KINDS[t % 4], members, rng, nowait=(t % 3 != 0), track=track)
        sel = [int(j) for j in rng.permutation(M)[:int(rng.integers(1, M + 1))]]
        counts = [int(c) for c in rng.permutation(np.resize(COUNTS, len(sel)))] if t % 2 else [int(rng.choice(COUNTS[:4])) for _ in sel]
        poses = [hypotheses(rng, track.pose[j], c) for j, c in zip(sel, counts)]
        scans = [track.scan(j)[::1 + k % 3] for k, j in enumerate(sel)]
        seen.append(assert_sessions(g, reps, t % levels, sel, poses, scans, scans, ("tick", t), cov_stride=9))
    for l in range(levels):
        poses = [hypotheses(rng, track.pose[j], int(c)) for j, c in zip(range(M), rng.permutation(COUNTS).tolist() + [5])]
        scans = [track.scan(j) for j in range(M)]
        seen.append(assert_sessions(g, reps, l, None, poses, scans, scans, ("final",), cov_stride=9))
    lh = np.concatenate(seen)
    assert (lh[~np.isnan(lh)] > 0.2).sum() > 50    # the poses sit on the written maps
    close_all(g, reps, track)


# ---- 2: against the float64 bound ---------------------------------------------------------------------------------

def field(sx, sy, j):
    yy, xx = np.mgrid[0:sy, 0:sx].astype(np.float64)
    lo = (1.5 * np.sin(2 * np.pi * (xx + 5 * j) / 37.0) + 1.5 * np.sin(2 * np.pi * yy / (29.0 + j))
          + 0.8 * np.sin(2 * np.pi * (xx + 0.6 * yy) / 53.0)).astype(F32)
    lo[sy // 3: sy // 3 + 4, sx // 2: sx // 2 + 6] = 60.0      # saturated: p == 1
    return lo


@MODES
def test_against_float64(hsb_lib, mode):
    """Three members with their own uploaded planes (404 x 300 x 3, resolution 0.25 and start (0, 0): world = cells x
    cell length exactly).  Every group likelihood lies within 1.01 ((ceil(n/32) + 6) u R64/n + u |lh64|) of the float64
    evaluation on its member's plane; every covariance equals the fp32 formula on the group's own likelihoods at the
    seven sigma points.  One scan runs along the [0, S-2] bounds (psi = 0, integer pose); one is empty."""
    from hector_slam_b200 import capi

    sx, sy, levels, res = 404, 300, 3, 0.25
    M = 3
    reps = [capi.MapRepB200(res, sx, sy, levels=levels, start=(0.0, 0.0), gather_mode=mode) for _ in range(M)]
    for j, rep in enumerate(reps):
        for l in range(levels):
            rep.upload_level(l, field(sx >> l, sy >> l, j))
    g = capi.SlamGroup(reps)
    rng = np.random.default_rng(43)
    members = [2, 0, 1]
    worst = 0.0
    for l in range(levels):
        lx, ly, cell = reps[0].level_info(l)
        scale = F32([cell, cell, 1.0])
        pt_scale = F32(2.0 ** -l)
        maps, scans = [], []
        for k, j in enumerate(members):
            n = (1081, 0, 300)[k]
            q = int(rng.integers(3, 9))
            pm = np.stack([rng.uniform(lx / 4, 3 * lx / 4, q), rng.uniform(ly / 4, 3 * ly / 4, q),
                           rng.uniform(-3.1, 3.1, q)], axis=1).astype(F32)
            pts = (np.stack([rng.uniform(-lx / 3, lx / 3, n), rng.uniform(-ly / 3, ly / 3, n)], axis=1) / pt_scale).astype(F32)
            if k == 2:    # endpoints on 0 and S-2, one ulp past each, for an integer pose without rotation
                pm[0] = F32([5.0, 7.0, 0.0])
                up = F32(1e9)
                edge = F32([(0 - 5.0, 0 - 7.0), (lx - 2 - 5.0, ly - 2 - 7.0), (np.nextafter(F32(lx - 2), up) - F32(5.0), 3.0),
                            (3.0, np.nextafter(F32(ly - 2), up) - F32(7.0)), (np.nextafter(F32(-5.0), -up), 2.0)])
                pts[:len(edge)] = edge / pt_scale
            maps.append(pm)
            scans.append(pts)
        world = [(pm * scale).astype(F32) for pm in maps]
        lh = g.likelihood(l, world, scans, members=members)
        cm, cw = g.covariance(l, world, scans, members=members)
        i = 0
        for k, j in enumerate(members):
            prob = reps[j].download_prob(l)
            n = scans[k].shape[0]
            sig = [likelihood64.sigma_points(p) for p in maps[k]]
            lhs = g.likelihood(l, [(np.concatenate(sig) * scale).astype(F32)], [scans[k]], members=[j]).reshape(-1, 7)
            for b, p in enumerate(maps[k]):
                ev = likelihood64.evaluate(prob, scans[k], p, pt_scale)
                if n == 0:
                    assert np.isnan(lh[i]) and np.isnan(lhs[b]).all(), (l, k, b)
                else:
                    tol = ev.tol(-(-n // 32) + 5)
                    err = abs(float(lh[i]) - ev.lh64)
                    assert err <= tol, (l, k, b, float(lh[i]), ev.lh64, err, tol)
                    worst = max(worst, err / tol if tol else 0.0)
                    assert bits(lhs[b, 6]) == bits(lh[i]), (l, k, b)   # the pose itself is the seventh sigma point
                wm, ww = likelihood64.covariance_fp32(lhs[b], p, cell)
                assert likelihood64.same_bits_or_nan(cm[i], wm), (l, k, b, cm[i], wm)
                assert likelihood64.same_bits_or_nan(cw[i], ww), (l, k, b, cw[i], ww)
                i += 1
            if k == 2:
                ev = likelihood64.evaluate(prob, scans[k], maps[k][0], pt_scale)
                assert ev.inside[:2].all() and not ev.inside[2:5].any(), (l, ev.inside[:5])
        assert i == lh.shape[0]
    assert worst > 0.0
    close_all(g, reps)


# ---- 3: the last matched scan --------------------------------------------------------------------------------------

@MODES
def test_last_match_mode(hsb_lib, mode):
    """M = 5, 16 ticks of group steps of every input kind (full and subset, sync and nowait, some sessions
    map_without_matching; every 7th beam of a converted scan is one its conversion drops).  After every tick the group
    calls without points over a permuted subset equal the single calls given the endpoints the matching *_to_points
    call returns for each member's last MATCHED input.  Before its first step a member gives NaN and best -1."""
    M, ticks = 5, 16
    reps, g = fleet(GEOM, M, mode)
    track = Tracker(GEOM, M, mode)
    data = [session_data(3200 + s, ticks, geometry(s)) for s in range(M)]
    rng = np.random.default_rng(47)
    at = [0] * M
    poses = [hypotheses(rng, (0, 0, 0), 4, specials=False) for _ in range(M)]
    lh = g.likelihood(0, poses)
    out, best4, index = g.best_hypothesis(0, poses)
    assert np.isnan(lh).all() and np.isnan(out).all()
    assert np.array_equal(best4[:, 0], np.full(M, -1, F32)) and (index == 0).all()   # every pose ranks -1: the first wins
    kept_below = 0
    stale_seen = 0
    for t in range(ticks):
        # the first two ticks step only some members: the others have still never matched
        members = ([0, 3], [3, 1])[t] if t < 2 else None if t % 4 == 0 else \
            [int(j) for j in rng.permutation(M)[:int(rng.integers(1, M + 1))]]
        kind = KINDS[(t + t // 4) % 4]
        before = [x for x in track.last]
        res = step([g], data, at, kind, members, rng, nowait=(t % 2 == 0), track=track, p_without=0.3)[0]
        sel = list(range(M)) if members is None else members
        if res[3] is not None:
            kept_below += sum(int(res[3][k]) < len(track.last[j][1]) for k, j in enumerate(sel) if track.last[j] is not None
                              and track.last[j] is not before[j])
        stale_seen += sum(track.last[j] is before[j] and before[j] is not None for j in sel)
        ask = [int(j) for j in rng.permutation(M)[:int(rng.integers(1, M + 1))]]
        poses = [hypotheses(rng, track.pose[j], int(rng.choice((1, 7, 33)))) for j in ask]
        poses = [np.concatenate([track.pose[j][None], p]) for j, p in zip(ask, poses)]   # the pose the step returned first
        assert_sessions(g, reps, t % GEOM[2], ask, poses, [track.scan(j) for j in ask], None, ("last", t), cov_stride=5)
    assert kept_below > 5      # conversions dropped beams: a stale upper bound would have shown
    assert stale_seen > 3      # map_without_matching steps left the previous matched scan in force
    close_all(g, reps, track)


# ---- 4: ordering --------------------------------------------------------------------------------------------------

@MODES
def test_ordering(hsb_lib, mode):
    """A group call issued straight after (1) a nowait step of this group, (2) a member's own nowait single step, (3) a
    nowait step of a second group that shares a member sees that step's map and last matched scan: it equals the call
    on a twin fleet stepped synchronously and settled with hsb_on_map_updated."""
    from hector_slam_b200 import capi

    M, ticks = 4, 5
    a, ga = fleet(GEOM, M, mode)
    b, gb = fleet(GEOM, M, mode)
    solo_a, solo_b = capi.SlamGroup([a[3]]), capi.SlamGroup([b[3]])
    data = [session_data(3300 + s, 3 * ticks + 1, geometry(s)) for s in range(M)]
    rng = np.random.default_rng(53)
    at = [0] * M

    def compare(members, poses, tag):
        got = ga.likelihood(0, poses, members=members), ga.covariance(1, poses, members=members)[1], \
            ga.best_hypothesis(0, poses, members=members)[1]
        for j in members:
            b[j].onMapUpdated()
        want = gb.likelihood(0, poses, members=members), gb.covariance(1, poses, members=members)[1], \
            gb.best_hypothesis(0, poses, members=members)[1]
        for x, y in zip(got, want):
            assert np.array_equal(bits(x), bits(y)), tag
        assert not np.isnan(got[0]).any(), tag

    for t in range(ticks):
        kind = KINDS[t % 4]                                                                       # (1)
        hints = np.asarray([data[j]["hints"][at[j]] for j in range(M)], F32)
        scans = [thinned(kind, scan_of(kind, data[j], at[j])) for j in range(M)]
        pa = group_step(ga, kind, hints, scans, None, nowait=True)[0]
        group_step(gb, kind, hints, scans, None, nowait=False)
        at = [k + 1 for k in at]
        members = [int(j) for j in rng.permutation(M)]
        compare(members, [hypotheses(rng, pa[j], 9, specials=False) for j in members], ("group", t))
        j = t % M                                                                                 # (2)
        pj = a[j].slam_update(data[j]["hints"][at[j]], data[j]["scans"][at[j]], nowait=True)[0]
        b[j].slam_update(data[j]["hints"][at[j]], data[j]["scans"][at[j]])
        at[j] += 1
        compare([j, (j + 1) % M], [hypotheses(rng, pj, 9, specials=False), hypotheses(rng, pa[(j + 1) % M], 5, specials=False)],
                ("single", t))
        k = at[3]                                                                                 # (3)
        ps = solo_a.slam_update(data[3]["hints"][k][None], [data[3]["scans"][k]], nowait=True)[0]
        solo_b.slam_update(data[3]["hints"][k][None], [data[3]["scans"][k]])
        at[3] += 1
        compare([3, 0], [hypotheses(rng, ps[0], 9, specials=False), hypotheses(rng, pa[0], 5, specials=False)],
                ("other group", t))
    close_all(solo_a, solo_b, ga, gb, a, b)


# ---- 5: no state change -------------------------------------------------------------------------------------------

def state(rep):
    """every level's log-odds, probability and stamps' effect (the occupancy grid), both dirty rectangles (read without
    reset), gate pose"""
    lv = [(bits(rep.download_level(l)).copy(), bits(rep.download_prob(l)).copy(), rep.download_occupancy(l),
           rep.get_mirror_dirty_rect(l)) for l in range(rep.levels)]
    return lv, rep.get_dirty_rects(), bits(rep.last_map_update_pose()).copy()


@MODES
def test_no_state_change(hsb_lib, mode):
    """Twin fleets take the same 10 ticks of group steps; fleet A answers all three calls, in both scan modes, over a
    subset after most of them.  Poses, covariances and gate decisions of every step are equal in bits, and at the end
    every member's planes, grids, both dirty rectangles, gate pose and last matched scan (its size and, through a
    following map write whose coarse levels read it, its points) are byte-identical to its twin's."""
    M, ticks = 5, 10
    a, ga = fleet(GEOM, M, mode)
    b, gb = fleet(GEOM, M, mode)
    track = Tracker(GEOM, M, mode)
    data = [session_data(3400 + s, ticks, geometry(s)) for s in range(M)]
    rng = np.random.default_rng(59)
    at = [0] * M
    for t in range(ticks):
        members = None if t % 3 == 0 else [int(j) for j in rng.permutation(M)[:int(rng.integers(1, M + 1))]]
        ra, rb = step([ga, gb], data, at, KINDS[t % 4], members, rng, nowait=(t % 2 == 0), track=track)
        for x, y in zip(ra[:3], rb[:3]):
            assert np.array_equal(bits(x) if x.dtype != bool else x, bits(y) if y.dtype != bool else y), t
        if t % 4 != 3:
            sel = [int(j) for j in rng.permutation(M)[:int(rng.integers(1, M))]]
            left = [j for j in range(M) if j not in sel]
            before = {j: ([a[j].get_mirror_dirty_rect(l) for l in range(GEOM[2])], a[j].get_dirty_rects()) for j in left}
            poses = [hypotheses(rng, track.pose[j], 12) for j in sel]
            for l in range(GEOM[2]):
                for points in (None, [track.scan(j) for j in sel]):
                    ga.likelihood(l, poses, points, members=sel)
                    ga.covariance(l, poses, points, members=sel)
                    ga.best_hypothesis(l, poses, points, members=sel)
            for j in left:
                assert ([a[j].get_mirror_dirty_rect(l) for l in range(GEOM[2])], a[j].get_dirty_rects()) == before[j]
    poses = [hypotheses(rng, track.pose[j], 6, specials=False) for j in range(M)]
    la, lb = ga.likelihood(0, poses), gb.likelihood(0, poses)     # the last matched scans: the same points, the same size
    assert np.array_equal(bits(la), bits(lb)) and not np.isnan(la).any()
    assert np.array_equal(bits(la), bits(np.concatenate([a[j].likelihood_batch(0, poses[j], track.scan(j)) for j in range(M)])))
    for j in range(M):
        sa, sb = state(a[j]), state(b[j])
        for l, (x, y) in enumerate(zip(sa[0], sb[0])):
            assert all(np.array_equal(u, v) for u, v in zip(x[:3], y[:3])) and x[3] == y[3], (j, l)
        assert sa[1] == sb[1] and np.array_equal(sa[2], sb[2]), j
        pts = data[j]["scans"][0][::3]
        a[j].updateByScan(pts, track.pose[j])
        b[j].updateByScan(pts, track.pose[j])
        for l in range(1, GEOM[2]):
            assert np.array_equal(bits(a[j].download_level(l)), bits(b[j].download_level(l))), (j, l)
    close_all(ga, gb, a, b, track)


# ---- 6: edges -----------------------------------------------------------------------------------------------------

@MODES
def test_empty_sessions_and_ties(hsb_lib, mode):
    """Empty sessions first, in the middle and last (their best hypothesis is {-1, 0, 0, 0}, index -1, and the poses
    of the others keep their places); empty scans (NaN, best -1 at index 0); a session whose poses are all the same
    (the lowest index wins)."""
    M = 5
    reps, g = fleet(GEOM, M, mode)
    track = Tracker(GEOM, M, mode)
    data = [session_data(3500 + s, 2, geometry(s)) for s in range(M)]
    rng = np.random.default_rng(61)
    step([g], data, [0] * M, "endpoints", None, rng, nowait=True, track=track, p_without=0.0)
    same = np.repeat(track.pose[2][None], 40, axis=0)
    for counts in ((0, 5, 0, 40, 0), (3, 0, 0, 40, 2), (0, 0, 0, 0, 1)):
        members = [4, 0, 3, 2, 1]
        poses = [same[:c] if j == 2 else hypotheses(rng, track.pose[j], c, specials=False) for j, c in zip(members, counts)]
        scans = [track.scan(j) if j != 0 else np.zeros((0, 2), F32) for j in members]
        assert_sessions(g, reps, 0, members, poses, scans, scans, ("empty", counts))
        out, best4, index = g.best_hypothesis(0, poses, scans, members=members)
        for k, (j, c) in enumerate(zip(members, counts)):
            if c == 0:
                assert np.array_equal(best4[k], F32([-1, 0, 0, 0])) and index[k] == -1, (counts, k)
            elif j == 0:
                assert best4[k, 0] == -1 and index[k] == 0, (counts, k)
            elif j == 2:
                assert index[k] == 0 and best4[k, 0] > 0, (counts, k, best4[k])
    close_all(g, reps, track)


@MODES
def test_past_the_grid_caps(hsb_lib, mode):
    """More poses than either launch covers in one pass (sm_count x 64 for the likelihood, sm_count x 8 for the
    covariance), in two sessions of two members: the grid-stride loops give what the single calls give."""
    import torch

    sm = torch.cuda.get_device_properties(0).multi_processor_count
    M = 3
    reps, g = fleet(GEOM, M, mode)
    track = Tracker(GEOM, M, mode)
    data = [session_data(3600 + s, 2, geometry(s)) for s in range(M)]
    rng = np.random.default_rng(67)
    step([g], data, [0] * M, "ranges", None, rng, nowait=False, track=track, p_without=0.0)
    members = [2, 0]
    counts = [sm * 64 + 37, 500]
    poses = [hypotheses(rng, track.pose[j], c) for j, c in zip(members, counts)]
    scans = [track.scan(j)[::8] for j in members]
    lh = g.likelihood(0, poses, scans, members=members)
    out, best4, index = g.best_hypothesis(0, poses, scans, members=members)
    q = 0
    for k, j in enumerate(members):
        want = reps[j].likelihood_batch(0, poses[k], scans[k])
        assert np.array_equal(bits(lh[q:q + counts[k]]), bits(want)) and np.array_equal(bits(out[q:q + counts[k]]), bits(want))
        assert np.array_equal(bits(best4[k]), bits(single_best(reps[j], 0, poses[k], scans[k])[0])), k
        assert index[k] == expected_index(want, poses[k])
        q += counts[k]
    counts = [sm * 8 + 11, 60]
    pc = [p[:c] for p, c in zip(poses, counts)]
    cm, cw = g.covariance(1, pc, scans, members=members)
    q = 0
    for k, j in enumerate(members):
        wm, ww = reps[j].covariance_batch(1, pc[k], scans[k])
        assert np.array_equal(bits(cm[q:q + counts[k]]), bits(wm)) and np.array_equal(bits(cw[q:q + counts[k]]), bits(ww)), k
        q += counts[k]
    close_all(g, reps, track)


# ---- 7: accounting and rejections ---------------------------------------------------------------------------------

@MODES
def test_launches_and_rejections(hsb_lib, mode):
    """A likelihood or covariance call is one launch on handles[0], a best-hypothesis call two, whichever members they
    list; the other members' counts do not move.  Every rejection returns -1 with its message, launches nothing and
    writes no output byte; K = 0 and Q = 0 queue nothing; the group answers a following call as before."""
    M = 4
    reps, g = fleet(GEOM, M, mode)
    track = Tracker(GEOM, M, mode)
    data = [session_data(3700 + s, 1, geometry(s)) for s in range(M)]
    rng = np.random.default_rng(71)
    step([g], data, [0] * M, "endpoints", None, rng, nowait=True, track=track, p_without=0.0)
    lib = g.lib
    hyp = [hypotheses(rng, track.pose[j], 10) for j in range(M)]
    scans = [track.scan(j) for j in range(M)]
    for members in (None, [2], [3, 1], [1, 0, 3, 2]):
        sel = list(range(M)) if members is None else members
        for points in (None, [scans[j] for j in sel]):
            counts = [r.launch_count for r in reps]
            g.likelihood(0, [hyp[j] for j in sel], points, members=members)
            assert [r.launch_count for r in reps] == [counts[0] + 1] + counts[1:], members
            g.covariance(0, [hyp[j] for j in sel], points, members=members)
            assert [r.launch_count for r in reps] == [counts[0] + 2] + counts[1:], members
            g.best_hypothesis(0, [hyp[j] for j in sel], points, members=members)
            assert [r.launch_count for r in reps] == [counts[0] + 4] + counts[1:], members
    valid_members = [3, 0, 2]
    valid = [hyp[j] for j in valid_members]
    before = assert_sessions(g, reps, 0, valid_members, valid, [scans[j] for j in valid_members], None, ("before",))

    Q, N = 12, 30
    poses = np.tile(track.pose[0], (Q, 1)).astype(F32)
    pts = np.ones((N, 2), F32)
    lh, c1, c2 = np.full(Q, SENTINEL, F32), np.full((Q, 9), SENTINEL, F32), np.full((Q, 9), SENTINEL, F32)
    best4, index = np.full((3, 4), SENTINEL, F32), np.full(3, SENTINEL, np.int32)

    def p(x, dt=np.int32):
        if x is None:
            return None, None
        a = np.ascontiguousarray(x, dt)
        return a, a.ctypes.data

    def call(kind, K, members, level=0, po=(0, 4, 4, 12), ps=poses, xy=pts, so=(0, 10, 10, 30), out=True):
        m, mp = p(members)
        o, op = p(po)
        s, sp = p(so)
        head = (g.g, K, mp, level, op, None if ps is None else ps.ctypes.data, None if xy is None else xy.ctypes.data, sp)
        if kind == "lh":
            return lib.hsb_group_likelihood_subset(*head, lh.ctypes.data if out else None)
        if kind == "cov":
            return lib.hsb_group_covariance_subset(*head, c1.ctypes.data if out else None, c2.ctypes.data if out else None)
        return lib.hsb_group_best_hypothesis_subset(*head, lh.ctypes.data, best4.ctypes.data if out else None, index.ctypes.data)

    def err():
        return (lib.hsb_last_error(reps[0].h) or b"").decode()

    cases = []
    for kind in ("lh", "cov", "best"):
        def c(**kw):
            K = kw.pop("K", 3)
            members = kw.pop("members", [0, 1, 2])
            return lambda kind=kind, K=K, members=members, kw=kw: call(kind, K, members, **kw)
        cases += [(c(K=-1, members=[0]), "K is -1"), (c(K=M + 1, members=[0, 1, 2, 3, 0]), "K is 5"),
                  (c(members=None), "members is NULL"), (c(members=[0, 1, M]), "session 2: member 4"),
                  (c(members=[-1, 0, 1]), "session 0: member -1"), (c(members=[1, 3, 1]), "session 2: member 1 is listed twice"),
                  (c(level=-1), "level -1"), (c(level=GEOM[2]), "level 3"),
                  (c(po=None), "pose_offsets is NULL"), (c(po=(1, 4, 4, 12)), "pose_offsets[0] is 1"),
                  (c(po=(0, 4, 3, 12)), "pose_offsets decrease at session 1"),
                  (c(xy=None), "both be given or both be NULL"), (c(so=None), "both be given or both be NULL"),
                  (c(so=(2, 10, 10, 30)), "scan_offsets[0] is 2"), (c(so=(0, 10, 30, 20)), "scan_offsets decrease at session 2"),
                  (c(ps=None), "poses_world is NULL"),
                  (c(out=False), {"lh": "out_likelihood is NULL", "cov": "both NULL", "best": "out_best4 is NULL"}[kind])]
    full_po, fp = p((0, 3, 3, 3, 12))
    cases += [(lambda: lib.hsb_group_likelihood(g.g, GEOM[2], fp, poses.ctypes.data, None, None, lh.ctypes.data), "level 3"),
              (lambda: lib.hsb_group_covariance(g.g, 0, None, poses.ctypes.data, None, None, c1.ctypes.data, None),
               "pose_offsets is NULL"),
              (lambda: lib.hsb_group_best_hypothesis(g.g, 0, fp, poses.ctypes.data, pts.ctypes.data, None, None,
                                                     best4.ctypes.data, None), "both be given or both be NULL")]
    counts = [r.launch_count for r in reps]
    for fn, text in cases:
        assert fn() == -1, text
        assert text in err(), (text, err())
    # K = 0 reads nothing else; Q = 0 (every session empty) needs no poses and no outputs
    for kind in ("lh", "cov", "best"):
        assert call(kind, 0, None, level=-5, po=None, ps=None, xy=None, so=None, out=False) == 0
        assert call(kind, 3, [0, 1, 2], po=(0, 0, 0, 0), ps=None, out=False) == 0
        assert call(kind, 3, [0, 1, 2], po=(0, 0, 0, 0), ps=None, xy=None, so=None, out=False) == 0
    assert [r.launch_count for r in reps] == counts
    assert (lh == SENTINEL).all() and (c1 == SENTINEL).all() and (c2 == SENTINEL).all()
    assert (best4 == SENTINEL).all() and (index == SENTINEL).all()
    assert call("best", 3, [0, 1, 2], po=(0, 0, 0, 0), ps=None) == 0    # given outputs: every session is empty
    assert np.array_equal(best4, np.tile(F32([-1, 0, 0, 0]), (3, 1))) and (index == -1).all()
    assert [r.launch_count for r in reps] == counts
    after = assert_sessions(g, reps, 0, valid_members, valid, [scans[j] for j in valid_members], None, ("after",))
    assert np.array_equal(bits(before), bits(after))
    close_all(g, reps, track)


# ---- 8: the C++ façade --------------------------------------------------------------------------------------------

def test_facade(hsb_lib):
    """hsb200::SlamProcessor::likelihoodMany, covarianceMany and bestHypothesisMany (both overloads each), through their
    shims, against the C-ABI group calls on a second set of processors stepped with the same scans: the same bits, with
    the scans given and with each processor's last matched scan."""
    L = C.CDLL(os.path.join(ROOT, "hector_slam_b200", "lib", "libhsb200_host.so"))
    vp, i, f = C.c_void_p, C.c_int, C.c_float
    L.hsbp_create.restype = vp
    L.hsbp_create.argtypes = [f, i, i, f, f, i, i]
    L.hsbp_destroy.argtypes = [vp]
    L.hsbp_handle.restype = vp
    L.hsbp_handle.argtypes = [vp]
    L.hsbp_update.argtypes = [vp, vp, i, vp, vp, i, vp, vp]
    L.hsbp_likelihood_many.argtypes = [vp, i, i, vp, vp, vp, vp, vp]
    L.hsbp_likelihood_many_subset.argtypes = [vp, i, vp, i, i, vp, vp, vp, vp, vp]
    L.hsbp_covariance_many.argtypes = [vp, i, i, vp, vp, vp, vp, vp, vp]
    L.hsbp_covariance_many_subset.argtypes = [vp, i, vp, i, i, vp, vp, vp, vp, vp, vp]
    L.hsbp_best_hypothesis_many.argtypes = [vp, i, i, vp, vp, vp, vp, vp, vp, vp]
    L.hsbp_best_hypothesis_many_subset.argtypes = [vp, i, vp, i, i, vp, vp, vp, vp, vp, vp, vp]
    lib = hsb_lib

    sx0, sy0, levels, start = GEOM
    M, ticks = 4, 6
    data = [session_data(3800 + s, ticks, geometry(s)) for s in range(M)]
    sets = [[L.hsbp_create(mc.RES, sx0, sy0, start[0], start[1], levels, 0) for _ in range(M)] for _ in range(2)]
    assert all(q for s in sets for q in s)
    many, capi_set = sets
    hs = (C.c_void_p * M)(*[L.hsbp_handle(q) for q in capi_set])
    g = C.c_void_p()
    assert lib.hsb_group_create(C.cast(hs, vp), M, C.byref(g)) == 0
    arr = C.cast((C.c_void_p * M)(*many), vp)
    rng = np.random.default_rng(73)
    good = 0
    for t in range(ticks):
        last = np.zeros((M, 3), F32)
        for s in range(M):
            x = data[s]["scans"][t]
            for st in sets:
                pose, cov = np.zeros(3, F32), np.zeros(9, F32)
                assert L.hsbp_update(st[s], x.ctypes.data, x.shape[0], None, data[s]["hints"][t].ctypes.data, 0,
                                     pose.ctypes.data, cov.ctypes.data) == 0
            last[s] = pose
        level = t % levels
        members = None if t % 2 == 0 else np.ascontiguousarray(rng.permutation(M)[:int(rng.integers(1, M + 1))], np.int32)
        sel = list(range(M)) if members is None else [int(j) for j in members]
        K = len(sel)
        po = np.zeros(K + 1, np.int32)
        po[1:] = np.cumsum(rng.integers(0, 12, K))
        Q = int(po[-1])
        poses = np.concatenate([hypotheses(rng, last[j], int(po[k + 1] - po[k]), specials=False) for k, j in enumerate(sel)]
                               + [np.zeros((1, 3), F32)]).astype(F32)
        given = t % 3 != 2     # otherwise: the last matched scans
        scans = [data[j]["scans"][t][::2] for j in sel]
        so = np.zeros(K + 1, np.int32)
        so[1:] = np.cumsum([s.shape[0] for s in scans])
        pts = np.ascontiguousarray(np.concatenate(scans), F32)
        pp, sp = (pts.ctypes.data, so.ctypes.data) if given else (None, None)
        outs = [[np.zeros(Q + 1, F32), np.zeros((Q + 1, 9), F32), np.zeros((Q + 1, 9), F32), np.zeros(Q + 1, F32),
                 np.zeros((K, 4), F32), np.zeros(K, np.int32)] for _ in range(2)]
        (lh, cm, cw, bl, b4, bi), (lh2, cm2, cw2, bl2, b42, bi2) = [[o.ctypes.data for o in out] for out in outs]
        common = (level, po.ctypes.data, poses.ctypes.data, pp, sp)
        if members is None:
            assert L.hsbp_likelihood_many(arr, M, *common, lh) == 0
            assert L.hsbp_covariance_many(arr, M, *common, cm, cw) == 0
            assert L.hsbp_best_hypothesis_many(arr, M, *common, b4, bi, bl) == 0
            assert lib.hsb_group_likelihood(g, *common, lh2) == 0
            assert lib.hsb_group_covariance(g, *common, cm2, cw2) == 0
            assert lib.hsb_group_best_hypothesis(g, *common, bl2, b42, bi2) == 0
        else:
            mp = members.ctypes.data
            assert L.hsbp_likelihood_many_subset(arr, M, mp, K, *common, lh) == 0
            assert L.hsbp_covariance_many_subset(arr, M, mp, K, *common, cm, cw) == 0
            assert L.hsbp_best_hypothesis_many_subset(arr, M, mp, K, *common, b4, bi, bl) == 0
            assert lib.hsb_group_likelihood_subset(g, K, mp, *common, lh2) == 0
            assert lib.hsb_group_covariance_subset(g, K, mp, *common, cm2, cw2) == 0
            assert lib.hsb_group_best_hypothesis_subset(g, K, mp, *common, bl2, b42, bi2) == 0
        for x, y in zip(*outs):
            assert np.array_equal(x if x.dtype == np.int32 else bits(x), y if y.dtype == np.int32 else bits(y)), t
        assert np.array_equal(bits(outs[0][0]), bits(outs[0][3])), t
        good += int((outs[0][0][:Q] > 0.2).sum())
    assert good > 20
    lib.hsb_group_destroy(g)
    for q in many + capi_set:
        L.hsbp_destroy(q)
