"""Re-matching a group's robots from their new raw scans in one pass (hsb_group_match_batch_ranges / _cloud / _projected
and their _subset forms): each session's LaserScan ranges, Point32 cloud or ranges to project are converted on the
device with its member's formats, every hint runs matchData with the converted scan, and the matched poses are scored
and picked, with one copy each way.

Twins, in bits: the kept counts against the single conversion calls on each member; every pose and Hessian against
hsb_group_match_batch(_subset) on the same hints with those endpoints (same launch shape); every likelihood, best4 and
index against hsb_group_best_hypothesis(_subset) at level 0 on the returned poses.  On same-geometry TEX and LDG groups,
a mixed group and a heterogeneous one (level counts 1 to 8, TEX and LDG, different resolutions), with ragged permuted
sessions, non-finite hints, angles past 120 rad, sessions without hints, scans whose every input is dropped and a member
that never matched; the launch shapes W = 8, 4, 2, 1 by Q and by tuning; a 300-member fleet; raw scans past the pinned
staging chunk; no state change, ordering behind a nowait step, launch accounting, rejections; the CPU oracle."""
import numpy as np
import pytest

import laser_projection as lp
import maptools_cases as mc
from test_gpu_group_match import auto_w, ragged, sm_count
from test_gpu_group_score import (GEOM, SENTINEL, Tracker, bits, close_all, fleet, hypotheses, make_rep, state, step,
                                  thinned)
from test_gpu_group_subset import (beam_angles, geometry, group_step, member_cloud, member_transform, scan_of,
                                   session_data)

pytestmark = pytest.mark.gpu

F32 = np.float32
RAW = ("ranges", "cloud", "projected")
MODES = pytest.mark.parametrize("mode", [2, 1], ids=["tex", "ldg"])   # capi.GATHER_TEX, capi.GATHER_LDG


def call(g, kind, hints, scans, transforms=None, members=None, want_cov=True, score=True):
    fn = {"ranges": g.match_batch_ranges, "cloud": g.match_batch_cloud, "projected": g.match_batch_projected}[kind]
    return fn(hints, scans, transforms, members=members, want_cov=want_cov, score=score)


def convert(rep, kind, x, T=None, fmt=None):
    """the single conversion call on rep (cloud with an explicit transform: rep's cloud format set to it, fmt its
    thresholds, for the call) -> endpoints"""
    if kind == "ranges":
        return rep.scan_to_points(x)
    if kind == "projected":
        return rep.projected_scan_to_points(x, T)[0]
    if T is None:
        return rep.cloud_to_points(x)[0]
    rep.set_cloud_format(T, **fmt)
    return rep.cloud_to_points(x)[0]


def dropped(kind, x):
    """every input of the scan dropped by its conversion: NaN ranges, projected ranges past the cutoff, cloud points
    outside the z window"""
    out = np.array(x, F32, copy=True)
    if kind == "ranges":
        out[:] = np.nan
    elif kind == "projected":
        out[:] = F32(100.0)
    else:
        out[:, 2] = F32(5.0)
    return out


def check(g, reps, convs, kind, members, hints, scans, transforms=None, fmts=None, tag=()):
    """The call over `members` (None: all) against its twins in bits; convs[j] converts as member j does.
    -> (poses, cov (Q, 9), kept, W)"""
    sel = list(range(len(reps))) if members is None else members
    before = [r.launch_count for r in reps]
    poses, cov, kept, lh, best4, index = call(g, kind, hints, scans, transforms, members)
    W = reps[0].last_launch_shape()["warps_per_scan"]
    Q = sum(h.shape[0] for h in hints)
    assert [r.launch_count for r in reps] == [before[0] + (4 if Q else 0)] + before[1:], tag
    if Q == 0:   # nothing queued: every session's pick is the empty one's, kept is not written
        assert best4.tolist() == [[-1.0, 0.0, 0.0, 0.0]] * len(sel) and (index == -1).all(), tag
        return poses, cov.reshape(-1, 9), kept, W
    pts = [convert(convs[j], kind, scans[k], None if transforms is None else transforms[k],
                   None if fmts is None else fmts[j]) for k, j in enumerate(sel)]
    assert list(kept) == [p.shape[0] for p in pts], tag
    wp, wc = g.match_batch(hints, pts, members=members)
    assert reps[0].last_launch_shape()["warps_per_scan"] == W, tag
    assert np.array_equal(bits(poses), bits(wp)) and np.array_equal(bits(cov), bits(wc)), tag
    off = np.zeros(len(sel) + 1, np.int32)
    off[1:] = np.cumsum([h.shape[0] for h in hints])
    wl, wb, wi = g.best_hypothesis(0, (poses, off), pts, members=members)
    assert np.array_equal(bits(lh), bits(wl)), tag
    assert np.array_equal(bits(best4), bits(wb)) and np.array_equal(index, wi), tag
    for k in range(len(sel)):
        q0, q1 = off[k], off[k + 1]
        if q0 == q1:
            assert list(best4[k]) == [-1.0, 0.0, 0.0, 0.0] and index[k] == -1, tag
        if kept[k] == 0 and q1 > q0:   # every input dropped: the hints and zero Hessians
            assert np.array_equal(bits(poses[q0:q1]), bits(hints[k])) and not cov[q0:q1].any(), tag
    return poses, cov.reshape(-1, 9), kept, W


# ---- 1: same-geometry groups, the launch shapes ------------------------------------------------------------------

@MODES
@pytest.mark.parametrize("kind", RAW)
def test_against_twins(hsb_lib, kind, mode):
    """M = 5 on one geometry (members differ in beam geometry, laser mount and cloud thresholds); member 4 is never
    stepped.  8 ticks of group steps of every input kind; after each a call over a permuted subset (all members on every
    third tick) with ragged sessions, a session without hints and, every other tick, one whose scan is dropped whole;
    cloud and projected ticks alternate between explicit transforms and the members' own.  The first four ticks size Q
    so that the default rule takes W = 8, 4, 2 and 1; the last four force each through handles[0]'s tuning."""
    M, ticks = 5, 8
    reps, g = fleet(GEOM, M, mode)
    track = Tracker(GEOM, M, mode)
    data = [session_data(6100 + s, ticks + 1, geometry(s)) for s in range(M)]
    fmts = [member_cloud(s) for s in range(M)]
    rng = np.random.default_rng(161)
    at = [0] * M
    sm = sm_count()
    seen = set()
    for t in range(ticks):
        stepped = [int(j) for j in rng.permutation(M - 1)[:int(rng.integers(1, M))]]
        step([g], data, at, ("endpoints", "cloud", "ranges", "projected")[t % 4], stepped, rng, nowait=(t % 2 == 0),
             track=track)
        sel = list(range(M)) if t % 3 == 0 else [int(j) for j in rng.permutation(M)[:int(rng.integers(2, M + 1))]]
        members = None if t % 3 == 0 else sel
        forced = (0, 0, 0, 0, 8, 4, 2, 1)[t]
        target = (2 * sm, 5 * sm, 10 * sm, 14 * sm)[t % 4] if not forced else int(rng.integers(40, 3 * sm))
        counts = ragged(rng, len(sel), target)
        hints = [hypotheses(rng, data[j]["truth"][at[j]], c) for j, c in zip(sel, counts)]
        scans = [scan_of(kind, data[j], at[j]) for j in sel]
        if t % 2 == 1:
            k = int(np.argmax(counts))
            scans[k] = dropped(kind, scans[k])
        T = None
        if kind != "ranges" and t % 2 == 0:
            T = np.stack([member_transform(j + 7) for j in sel])
        reps[0].set_tuning(warps_per_scan=forced)
        try:
            _, _, kept, W = check(g, reps, track.conv, kind, members, hints, scans, T, fmts, ("tick", t, kind))
        finally:
            reps[0].set_tuning(warps_per_scan=0)
            for j in range(M):
                track.conv[j].set_cloud_format(member_transform(j), **fmts[j])
        assert W == (forced or auto_w(sum(counts))), (t, W, sum(counts))
        seen.add(W)
        if t % 2 == 1:
            assert kept[int(np.argmax(counts))] == 0
    assert seen == {1, 2, 4, 8}
    close_all(g, reps, track)


# ---- 2: mixed and heterogeneous groups ---------------------------------------------------------------------------

def hetero_fleet():
    """The heterogeneous group of test_gpu_group_heterogeneous (levels 1 to 8, TEX and LDG, resolutions 0.025 to
    0.1 m), its never-stepped converters, and its trajectories, after 6 group ticks of every input kind"""
    from hector_slam_b200 import capi
    from test_gpu_group_heterogeneous import M, make_rep as hetero_rep, member_data

    reps = [hetero_rep(s) for s in range(M)]
    convs = [hetero_rep(s) for s in range(M)]
    g = capi.SlamGroup(reps, heterogeneous=True)
    data = [member_data(s) for s in range(M)]
    rng = np.random.default_rng(163)
    for t in range(6):
        kind = ("endpoints", "cloud", "ranges", "projected")[t % 4]
        hints = np.stack([data[j]["hints"][t] for j in range(M)]).astype(F32)
        group_step(g, kind, hints, [thinned(kind, scan_of(kind, data[j], t)) for j in range(M)], None,
                   nowait=bool(rng.random() < 0.5))
    return reps, convs, g, data


def mixed_fleet():
    """Four members of different map size, resolution and start, one level count and gather mode, after 6 ticks"""
    from hector_slam_b200 import capi, synth

    specs = [(400, 300, 0.05, (0.5, 0.5)), (256, 512, 0.1, (0.3, 0.6)), (640, 480, 0.025, (0.5, 0.5)),
             (300, 300, 0.075, (0.6, 0.4))]

    def make(s):
        sx, sy, res, start = specs[s]
        rep = capi.MapRepB200(res, sx, sy, levels=3, start=start, gather_mode=2)
        g = geometry(s)
        rep.set_scan_format(**g)
        rep.set_laser_projection(**g, range_cutoff=30.0)
        rep.set_cloud_format(member_transform(s), **member_cloud(s))
        return rep

    M = len(specs)
    reps, convs = [make(s) for s in range(M)], [make(s) for s in range(M)]
    g = capi.SlamGroup(reps, mixed=True)
    data = [session_data(6300 + s, 8, geometry(s)) for s in range(M)]
    for s in range(M):   # endpoints in each member's own cells
        data[s]["scans"] = [np.ascontiguousarray(synth.ranges_to_points(r, 1.0 / specs[s][2], beam_angles(geometry(s))),
                                                 F32) for r in data[s]["ranges"]]
    for t in range(6):
        kind = ("endpoints", "cloud", "ranges", "projected")[t % 4]
        hints = np.stack([data[j]["hints"][t] for j in range(M)]).astype(F32)
        group_step(g, kind, hints, [thinned(kind, scan_of(kind, data[j], t)) for j in range(M)], None)
    return reps, convs, g, data


@pytest.mark.parametrize("which", ["mixed", "heterogeneous"])
def test_mixed_and_heterogeneous(hsb_lib, which):
    """Every raw kind, full and over a permuted subset, each member's next scan, with W forced to 1, 2, 4 and 8 and by
    the default rule: every member converts with its own formats and matches on its own geometry and pyramid."""
    reps, convs, g, data = mixed_fleet() if which == "mixed" else hetero_fleet()
    M = len(reps)
    rng = np.random.default_rng(165)
    fmts = [member_cloud(s) for s in range(M)]
    for i, kind in enumerate(RAW):
        for W in (0, 1, 2, 4, 8):
            members = None if W % 2 == 0 else [int(j) for j in rng.permutation(M)[:int(rng.integers(2, M + 1))]]
            sel = list(range(M)) if members is None else members
            hints = [hypotheses(rng, data[j]["truth"][6], int(rng.choice((0, 1, 9, 40)))) for j in sel]
            scans = [scan_of(kind, data[j], 6) for j in sel]
            T = np.stack([member_transform(j + 3) for j in sel]) if kind != "ranges" and W in (1, 4) else None
            reps[0].set_tuning(warps_per_scan=W)
            try:
                check(g, reps, convs, kind, members, hints, scans, T, fmts, (which, kind, W))
            finally:
                reps[0].set_tuning(warps_per_scan=0)
                for j in range(M):
                    convs[j].set_cloud_format(member_transform(j), **fmts[j])
    close_all(g, reps, convs)


# ---- 3: a 300-member fleet ---------------------------------------------------------------------------------------

def test_300_member_fleet(hsb_lib):
    """A 300-member heterogeneous group of small maps (levels 1 to 4, TEX and LDG, three resolutions), written by two
    group steps; a call over K = 129 members whose sessions cross the 32- and 128-session boundaries, per kind."""
    from hector_slam_b200 import capi

    specs = [(128, 128, 0.1, (0.5, 0.5)), (136, 104, 0.1, (0.3, 0.6)), (96, 160, 0.05, (0.5, 0.5))]

    def make(s):
        sx, sy, res, start = specs[s % 3]
        rep = capi.MapRepB200(res, sx, sy, levels=1 + s % 4, start=start, gather_mode=(2, 1)[(s // 4) % 2])
        g = geometry(s // 3)
        rep.set_scan_format(**g)
        rep.set_laser_projection(**g, range_cutoff=30.0)
        rep.set_cloud_format(member_transform(s), **member_cloud(s))
        return rep

    M = 300
    reps = [make(s) for s in range(M)]
    g = capi.SlamGroup(reps, heterogeneous=True)
    cache = {}
    for s in range(M):   # (a dozen trajectories in each of the three beam geometries)
        cache.setdefault((s % 12, s // 3 % 3), session_data(7000 + s % 12, 3, geometry(s // 3)))
    data = [cache[(s % 12, s // 3 % 3)] for s in range(M)]
    for t in range(2):
        hints = np.stack([data[j]["truth"][t] for j in range(M)]).astype(F32)
        group_step(g, "ranges", hints, [data[j]["ranges"][t] for j in range(M)], None)
    rng = np.random.default_rng(167)
    members = [int(j) for j in rng.permutation(M)[:129]]
    convs = {j: make(j) for j in members}
    fmts = {j: member_cloud(j) for j in members}
    for kind in RAW:
        hints = [hypotheses(rng, data[j]["truth"][2], (0, 1, 3, 7)[k % 4]) for k, j in enumerate(members)]
        scans = [scan_of(kind, data[j], 2) for j in members]
        check(g, reps, convs, kind, members, hints, scans, None, fmts, ("fleet", kind))
    close_all(g, reps, list(convs.values()))


# ---- 4: raw scans past the staging chunk -------------------------------------------------------------------------

def test_long_scans(hsb_lib):
    """Three members whose raw scans together exceed the 1 MB the call stages in pinned memory, per kind: 300 000-beam
    scan formats and laser projections, 100 000-point clouds.  The long projected scans' twin is hsb_cloud_to_points on
    the cloud laser_projection.py projects (the single projected conversion stops at the fused step's staging)."""
    from hector_slam_b200 import capi, synth

    M, N = 3, 300_000
    fmts = [member_cloud(s) for s in range(M)]

    def long_geom(s):
        return dict(n_beams=N, angle_min=float(F32(-2.3 + 0.1 * s)), angle_increment=float(F32(4.6 / N)),
                    range_min=float(F32(0.1)), range_max=float(F32(25.0)))

    def make(s):
        rep = capi.MapRepB200(0.05, 512, levels=3)
        rep.set_scan_format(**long_geom(s))
        rep.set_laser_projection(**long_geom(s), range_cutoff=30.0)
        rep.set_cloud_format(member_transform(s), **fmts[s])
        return rep

    reps, convs = [make(s) for s in range(M)], [make(s) for s in range(M)]
    g = capi.SlamGroup(reps)
    data = [session_data(7100 + s, 3, geometry(s)) for s in range(M)]
    group_step(g, "endpoints", np.stack([data[j]["truth"][0] for j in range(M)]).astype(F32),
               [data[j]["scans"][0] for j in range(M)], None)
    world = synth.World(1, seed=1000 + 7100)
    rng = np.random.default_rng(169)

    ranges = [(world.cast(data[j]["truth"][1], beam_angles(long_geom(j))) + rng.normal(0, 0.01, N)).astype(F32)
              for j in range(M)]
    clouds = [np.resize(data[j]["clouds"][1], (100_000, 3)) for j in range(M)]
    hints = [hypotheses(rng, data[j]["truth"][1], (5, 0, 9)[j]) for j in range(M)]
    assert sum(r.nbytes for r in ranges) > 1 << 20 and sum(c.nbytes for c in clouds) > 1 << 20
    check(g, reps, convs, "ranges", None, hints, ranges, tag=("long ranges",))
    check(g, reps, convs, "cloud", [2, 0, 1], [hints[j] for j in (2, 0, 1)], [clouds[j] for j in (2, 0, 1)],
          tag=("long cloud",))
    # projected: the twin conversion is the cloud conversion of the projected cloud
    proj = [dict(long_geom(s), range_cutoff=30.0) for s in range(M)]
    projected = [lp.project(ranges[j], proj[j]) for j in range(M)]
    poses, cov, kept, lh, best4, index = call(g, "projected", hints, ranges)
    pts = [convs[j].cloud_to_points(projected[j])[0] for j in range(M)]
    assert list(kept) == [p.shape[0] for p in pts]
    wp, wc = g.match_batch(hints, pts)
    assert np.array_equal(bits(poses), bits(wp)) and np.array_equal(bits(cov), bits(wc))
    off = np.cumsum([0] + [h.shape[0] for h in hints]).astype(np.int32)
    wl, wb, wi = g.best_hypothesis(0, (poses, off), pts)
    assert np.array_equal(bits(lh), bits(wl)) and np.array_equal(bits(best4), bits(wb)) and np.array_equal(index, wi)
    close_all(g, reps, convs)


# ---- 5: no state change, ordering --------------------------------------------------------------------------------

@MODES
def test_no_state_change_and_ordering(hsb_lib, mode):
    """Twin fleets take the same 8 ticks of group steps (nowait on most); fleet A calls every raw kind over a subset
    straight after each step, which the call's results must already see (they equal the twins computed after it).  At
    the end every member of fleet A, listed or not, has the planes, occupancy, dirty rectangles, gate pose and last-match
    container of its twin, and the next group step gives the same bits on both fleets."""
    M, ticks = 5, 8
    a, ga = fleet(GEOM, M, mode)
    b, gb = fleet(GEOM, M, mode)
    track = Tracker(GEOM, M, mode)
    data = [session_data(6500 + s, ticks + 2, geometry(s)) for s in range(M)]
    rng = np.random.default_rng(171)
    at = [0] * M
    for t in range(ticks):
        members = None if t % 3 == 0 else [int(j) for j in rng.permutation(M)[:int(rng.integers(1, M + 1))]]
        ra, rb = step([ga, gb], data, at, ("endpoints", "cloud", "ranges", "projected")[t % 4], members, rng,
                      nowait=(t % 4 != 3), track=track)
        sel = [int(j) for j in rng.permutation(M)[:int(rng.integers(1, M))]]
        kind = RAW[t % 3]
        hints = [hypotheses(rng, track.pose[j], 12) for j in sel]
        scans = [scan_of(kind, data[j], at[j]) for j in sel]
        check(ga, a, track.conv, kind, sel, hints, scans, tag=("tick", t))
        for x, y in zip(ra[:3], rb[:3]):
            assert np.array_equal(bits(x) if x.dtype != bool else x, bits(y) if y.dtype != bool else y), t
    for j in range(M):
        sa, sb = state(a[j]), state(b[j])
        for l, (x, y) in enumerate(zip(sa[0], sb[0])):
            assert all(np.array_equal(u, v) for u, v in zip(x[:3], y[:3])) and x[3] == y[3], (j, l)
        assert sa[1] == sb[1] and np.array_equal(sa[2], sb[2]), j
        if track.last[j] is not None:
            pa, oa = a[j].last_match_scan()
            pb, ob = b[j].last_match_scan()
            assert np.array_equal(bits(pa), bits(pb)) and np.array_equal(bits(oa), bits(ob)), j
    ra, rb = step([ga, gb], data, at, "ranges", None, rng, nowait=False, p_without=0.3)
    for x, y in zip(ra[:3], rb[:3]):
        assert np.array_equal(bits(x) if x.dtype != bool else x, bits(y) if y.dtype != bool else y)
    assert np.array_equal(ra[3], rb[3])
    close_all(ga, gb, a, b, track)


# ---- 6: accounting and rejections --------------------------------------------------------------------------------

@MODES
def test_launches_and_rejections(hsb_lib, mode):
    """2, 3 or 4 launches on handles[0] by the scoring outputs asked for, none on the other members.  Every rejection
    returns its code with its message, launches nothing and writes no output byte; K = 0 reads nothing; Q = 0 queues
    nothing and writes only the empty session's pick; a tuning without a group match kernel gives HSB_ERR_UNSUPPORTED."""
    M = 4
    reps, g = fleet(GEOM, M, mode)
    track = Tracker(GEOM, M, mode)
    data = [session_data(6700 + s, 2, geometry(s)) for s in range(M)]
    rng = np.random.default_rng(173)
    step([g], data, [0] * M, "ranges", None, rng, nowait=True, track=track, p_without=0.0)
    lib = g.lib
    sel = [2, 0]
    hints = [hypotheses(rng, track.pose[j], 6) for j in sel]
    for kind in RAW:
        scans = [scan_of(kind, data[j], 1) for j in sel]
        for score, want in ((False, 2), (True, 4)):
            n0 = [r.launch_count for r in reps]
            call(g, kind, hints, scans, members=sel, score=score)
            assert [r.launch_count for r in reps] == [n0[0] + want] + n0[1:], (kind, score)

    h = np.concatenate(hints)
    big = np.zeros(4000, F32)   # room for either kind's scans below
    outs = dict(poses=np.full((12, 3), SENTINEL, F32), cov=np.full((12, 9), SENTINEL, F32),
                lh=np.full(12, SENTINEL, F32), best4=np.full((4, 4), SENTINEL, F32),
                index=np.full(4, SENTINEL, np.int32), kept=np.full(4, SENTINEL, np.int32))
    keep = []

    def arr(a):
        if a is None:
            return None
        a = np.ascontiguousarray(a, np.int32)
        keep.append(a)
        return a.ctypes.data

    def raw(kind, K=2, members=(2, 0), ho=(0, 6, 12), hw=h, x=big, so="valid", out=True, lh=True, best=True):
        """the _subset call of `kind`; so="valid": the members' beam counts (ranges, projected) or 500 points each"""
        if so == "valid":
            so = (0, 500, 1000) if kind == "cloud" else (0, 360, 1441)   # members 2 and 0: 360 and 1081 beams
        args = [arr(ho), None if hw is None else hw.ctypes.data, None if x is None else x.ctypes.data, arr(so)]
        if kind != "ranges":
            args.append(None)
        args += [outs["poses"].ctypes.data if out else None, outs["cov"].ctypes.data,
                 outs["lh"].ctypes.data if lh else None, outs["best4"].ctypes.data if best else None,
                 outs["index"].ctypes.data if best else None, outs["kept"].ctypes.data]
        return getattr(lib, f"hsb_group_match_batch_{kind}_subset")(g.g, K, arr(members), *args)

    def err():
        return (lib.hsb_last_error(reps[0].h) or b"").decode()

    # the likelihoods alone: three launches, the values the pick reports with them
    n0 = reps[0].launch_count
    assert raw("ranges", best=False) == 0
    assert reps[0].launch_count == n0 + 3
    lh3 = outs["lh"].copy()
    assert raw("ranges") == 0 and reps[0].launch_count == n0 + 7
    assert np.array_equal(bits(lh3), bits(outs["lh"]))
    for v in outs.values():
        v[:] = SENTINEL

    cases = []
    for kind in RAW:
        cases += [(kind, dict(K=-1, members=[0]), "K is -1"), (kind, dict(members=None), "members is NULL"),
                  (kind, dict(members=(1, 1)), "session 1: member 1 is listed twice"),
                  (kind, dict(ho=None), "hint_offsets is NULL"),
                  (kind, dict(ho=(0, 7, 6)), "hint_offsets decrease at session 1"),
                  (kind, dict(so=None), "scan_offsets is NULL"), (kind, dict(so=(1, 2, 3)), "scan_offsets[0] is 1"),
                  (kind, dict(so=(0, 9, 3)), "scan_offsets decrease at session 1"),
                  (kind, dict(x=None), "points_xyz is NULL" if kind == "cloud" else "ranges is NULL"),
                  (kind, dict(hw=None), "hints_world is NULL"), (kind, dict(out=False), "out_poses_world is NULL")]
        if kind != "cloud":
            cases.append((kind, dict(so=(0, 360, 1000)), "session 1 has 640 ranges"))
    counts = [r.launch_count for r in reps]
    for kind, kw, text in cases:
        assert raw(kind, **kw) == -1, (kind, text)
        assert text in err(), (kind, text, err())
    for kw in (dict(warps_per_scan=16), dict(scans_per_block=2), dict(unroll=8)):
        reps[0].set_tuning(**kw)
        assert raw("projected") == -5, kw
        assert "no group match kernel" in err(), (kw, err())
        reps[0].set_tuning(**{k: 0 for k in kw})
    assert [r.launch_count for r in reps] == counts
    for v in outs.values():
        assert (v == SENTINEL).all()
    # K = 0 reads nothing else; Q = 0 writes the empty session's pick and nothing else
    assert raw("ranges", K=0, members=None, ho=None, hw=None, x=None, so=None, out=False) == 0
    assert raw("cloud", ho=(0, 0, 0), hw=None, out=False) == 0
    assert outs["index"][:2].tolist() == [-1, -1] and outs["best4"][:2].tolist() == [[-1, 0, 0, 0]] * 2
    assert (outs["index"][2:] == SENTINEL).all() and (outs["best4"][2:] == SENTINEL).all()
    for name in ("poses", "cov", "lh", "kept"):
        assert (outs[name] == SENTINEL).all(), name
    assert [r.launch_count for r in reps] == counts
    close_all(g, reps, track)


@MODES
def test_member_without_format(hsb_lib, mode):
    """A listed member without the scan format, laser projection or cloud format its kind needs is rejected with the
    session named, before anything is queued; a member that is not listed is not checked."""
    from hector_slam_b200 import capi

    good = make_rep(GEOM, 0, mode)
    sx, sy, levels, start = GEOM
    bare = capi.MapRepB200(mc.RES, sx, sy, levels=levels, start=start, gather_mode=mode)
    g = capi.SlamGroup([good, bare])
    d = session_data(6900, 1, geometry(0))
    rng = np.random.default_rng(175)
    hints = [hypotheses(rng, d["truth"][0], 3), hypotheses(rng, d["truth"][0], 2)]
    needs = {"ranges": "hsb_set_scan_format", "cloud": "hsb_set_cloud_format", "projected": "hsb_set_laser_projection"}
    for kind in RAW:
        x = scan_of(kind, d, 0)
        n0 = good.launch_count
        with pytest.raises(Exception):
            call(g, kind, hints, [x, x])
        err = (g.lib.hsb_last_error(good.h) or b"").decode()
        assert "session 1" in err and needs[kind] in err, (kind, err)
        assert good.launch_count == n0
        call(g, kind, hints[:1], [x], members=[0])   # the bare member is not listed
    close_all(g, good, bare)


# ---- 7: the CPU oracle -------------------------------------------------------------------------------------------

def test_against_oracle(hsb_lib, pyoracle, oracle_kinds):
    """The 3-level 2048^2 map the CPU oracle builds from known poses, uploaded into three members; one session per raw
    kind, 24 hints around its own pose: the oracle's conversion, then its matchData, within 1e-4 m / rad."""
    from hector_slam_b200 import capi, synth

    kind = "reference" if "reference" in oracle_kinds else "port"
    world = synth.World.for_map_size(2048)
    orc = pyoracle.Oracle(kind, 0.05, 2048, 3)
    orc.set_update_factors(0.4, 0.9)
    pyoracle.build_map_known_poses(orc, world)
    M, H = 3, 24
    geo = dict(n_beams=1081, angle_min=float(F32(np.radians(-135.0))), angle_increment=float(F32(np.radians(0.25))),
               range_min=float(F32(0.1)), range_max=float(F32(30.0)))
    fmt = dict(sqr_laser_min_dist=float(F32(0.16)), sqr_laser_max_dist=float(F32(900.0)), laser_z_min_value=-1.0,
               laser_z_max_value=1.0)
    T = synth.laser_transform(xyz=(0.0, 0.0, 0.2), rpy=(0.0, 0.0, 0.0))
    reps = [capi.MapRepB200(0.05, 2048, levels=3, update_factor_free=0.4, update_factor_occupied=0.9) for _ in range(M)]
    for rep in reps:
        for l in range(3):
            rep.upload_level(l, orc.get_logodds(l))
        rep.set_scan_format(**geo)
        rep.set_laser_projection(**geo, range_cutoff=30.0)
        rep.set_cloud_format(T, **fmt)
    g = capi.SlamGroup(reps)
    rng = np.random.default_rng(177)
    truth = world.sample_free_poses(M, rng)
    ang = beam_angles(geo)
    proj = dict(geo, range_cutoff=30.0)
    checked = 0
    for j, raw_kind in enumerate(RAW):
        r = (world.cast(truth[j], ang) + rng.normal(0.0, 0.01, ang.size)).astype(F32)
        if raw_kind == "ranges":
            x, want_pts = r, pyoracle.scan_to_points(r, geo["angle_min"], geo["angle_increment"], geo["range_min"],
                                                     geo["range_max"], 20.0, kind=kind)
        elif raw_kind == "cloud":
            x = lp.project(r, proj)
            want_pts = pyoracle.cloud_to_points(x, T, fmt["sqr_laser_min_dist"], fmt["sqr_laser_max_dist"],
                                                fmt["laser_z_min_value"], fmt["laser_z_max_value"], 20.0, kind=kind)[0]
        else:
            x = r
            want_pts = lp.container(r, proj, fmt, T, 20.0, pyoracle, kind=kind)[0]
        hints = (truth[j][None] + rng.uniform(-1, 1, (H, 3)) * np.array([0.1, 0.1, 0.05])).astype(F32)
        poses, _, kept, _, best4, _ = call(g, raw_kind, [hints], [x], members=[j])
        assert kept[0] == want_pts.shape[0], raw_kind
        n = want_pts.shape[0]
        want, _, _ = orc.match_batch(hints, np.tile(want_pts, (H, 1)), np.arange(H + 1, dtype=np.int32) * n)
        ok = np.abs(want[:, :2] - hints[:, :2]).max(axis=1) < 0.5
        assert ok.mean() > 0.9, raw_kind
        d = np.abs(poses[ok].astype(np.float64) - want[ok].astype(np.float64))
        d[:, 2] = np.abs((d[:, 2] + np.pi) % (2 * np.pi) - np.pi)
        assert d[:, :2].max() <= 1e-4 and d[:, 2].max() <= 1e-4, (raw_kind, d.max(axis=0))
        assert np.abs(best4[0, 1:3] - truth[j][:2]).max() < 0.05, raw_kind
        checked += int(ok.sum())
    assert checked >= 0.9 * M * H
    orc.close()
    close_all(g, reps)


# ---- 8: the C++ façade -------------------------------------------------------------------------------------------

def test_facade(hsb_lib):
    """hsb200::SlamProcessor::matchManyRanges / matchManyCloud / matchManyProjected, both overloads each, through their
    shim, against the C-ABI group calls on a second set of processors stepped with the same scans: the same bits in
    every output."""
    import ctypes as C
    import os

    from conftest import ROOT
    from hector_slam_b200 import capi

    L = C.CDLL(os.path.join(ROOT, "hector_slam_b200", "lib", "libhsb200_host.so"))
    vp, i, f = C.c_void_p, C.c_int, C.c_float
    L.hsbp_create.restype = vp
    L.hsbp_create.argtypes = [f, i, i, f, f, i, i]
    L.hsbp_destroy.argtypes = [vp]
    L.hsbp_handle.restype = vp
    L.hsbp_handle.argtypes = [vp]
    L.hsbp_update.argtypes = [vp, vp, i, vp, vp, i, vp, vp]
    L.hsbp_match_many_scans.argtypes = [vp, i, i, vp, i] + [vp] * 11
    lib = hsb_lib

    sx0, sy0, levels, start = GEOM
    M = 4
    data = [session_data(6800 + s, 3, geometry(s)) for s in range(M)]
    sets = [[L.hsbp_create(mc.RES, sx0, sy0, start[0], start[1], levels, 0) for _ in range(M)] for _ in range(2)]
    assert all(q for s in sets for q in s)
    for st in sets:
        for s, q in enumerate(st):
            h = L.hsbp_handle(q)
            g = geometry(s)
            sf = capi.HsbScanFormat(g["n_beams"], g["angle_min"], g["angle_increment"], g["range_min"], g["range_max"])
            lp_ = capi.HsbLaserProjection(g["n_beams"], g["angle_min"], g["angle_increment"], g["range_min"],
                                          g["range_max"], 30.0)
            cf = capi.HsbCloudFormat()
            for k, v in enumerate(np.asarray(member_transform(s), np.float64).reshape(12)):
                cf.laser_transform[k] = float(v)
            c = member_cloud(s)
            cf.sqr_laser_min_dist, cf.sqr_laser_max_dist = c["sqr_laser_min_dist"], c["sqr_laser_max_dist"]
            cf.laser_z_min_value, cf.laser_z_max_value = c["laser_z_min_value"], c["laser_z_max_value"]
            assert lib.hsb_set_scan_format(h, C.byref(sf)) == 0
            assert lib.hsb_set_laser_projection(h, C.byref(lp_)) == 0
            assert lib.hsb_set_cloud_format(h, C.byref(cf)) == 0
    many, capi_set = sets
    hs = (C.c_void_p * M)(*[L.hsbp_handle(q) for q in capi_set])
    g = C.c_void_p()
    assert lib.hsb_group_create(C.cast(hs, vp), M, C.byref(g)) == 0
    arr = C.cast((C.c_void_p * M)(*many), vp)
    rng = np.random.default_rng(179)
    for t in range(2):
        for s in range(M):
            x = data[s]["scans"][t]
            for st in sets:
                pose, cov = np.zeros(3, F32), np.zeros(9, F32)
                assert L.hsbp_update(st[s], x.ctypes.data, x.shape[0], None, data[s]["hints"][t].ctypes.data, 0,
                                     pose.ctypes.data, cov.ctypes.data) == 0
    for n, kind in enumerate(RAW):
        for members in (None, np.array([3, 1, 2], np.int32)):
            sel = list(range(M)) if members is None else [int(j) for j in members]
            K = len(sel)
            ho = np.zeros(K + 1, np.int32)
            ho[1:] = np.cumsum(rng.integers(0, 12, K))
            Q = int(ho[-1])
            hints = np.concatenate([hypotheses(rng, data[j]["truth"][2], int(ho[k + 1] - ho[k]))
                                    for k, j in enumerate(sel)] + [np.zeros((1, 3), F32)]).astype(F32)
            scans = [scan_of(kind, data[j], 2) for j in sel]
            so = np.zeros(K + 1, np.int32)
            so[1:] = np.cumsum([x.shape[0] for x in scans])
            x = np.ascontiguousarray(np.concatenate(scans), F32)
            T = np.stack([member_transform(j + 5) for j in sel]) if kind != "ranges" else None
            outs = [[np.zeros((Q + 1, 3), F32), np.zeros((Q + 1, 9), F32), np.zeros(Q + 1, F32),
                     np.zeros((K, 4), F32), np.zeros(K, np.int32), np.zeros(K, np.int32)] for _ in range(2)]
            a, b = [[o.ctypes.data for o in out] for out in outs]
            mp = None if members is None else members.ctypes.data
            common = (ho.ctypes.data, hints.ctypes.data, x.ctypes.data, so.ctypes.data)
            tp = None if T is None else T.ctypes.data
            assert L.hsbp_match_many_scans(arr, M, n, mp, K, *common, tp, *a) == 0, kind
            fn = f"hsb_group_match_batch_{kind}" + ("" if members is None else "_subset")
            head = (g,) if members is None else (g, K, mp)
            tail = (common + ((tp,) if kind != "ranges" else ()))
            assert getattr(lib, fn)(*head, *tail, *b) == 0, kind
            for u, v in zip(*outs):
                assert np.array_equal(u.view(np.uint32), v.view(np.uint32)), (kind, members)
            assert (outs[0][5] > 0).all(), kind
    lib.hsb_group_destroy(g)
    for q in many + capi_set:
        L.hsbp_destroy(q)
