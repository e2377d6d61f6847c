"""hsb_slam_update_ranges and hsb_group_slam_update_ranges — the SLAM step from raw LaserScan ranges, converted in the
match kernel (the node's branch without the laser tf) — for one session and for a group.

The single step is checked against the two-call path it replaces (hsb_scan_to_points + hsb_slam_update with origo 0) and
against the node's compiled converter; the group step against single steps on twin handles.  Every comparison is
bitwise: poses, covariances, gate decisions, kept counts, every level's log-odds and probability planes, the gate pose
and both dirty rectangles.  Every member has its own scan format (beam count, angles, range window), update factors and
gate thresholds, so a session that read another member's settings would differ."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from conftest import ROOT

pytestmark = pytest.mark.gpu

RES, SIZE, LEVELS = 0.05, 512, 3
SCALE = 1.0 / RES

# n_beams, angle_min (deg), angle_increment (deg), range_min, range_max of the four basic members
FORMATS = [(1081, -135.0, 0.25, 0.1, 30.0), (720, -180.0, 0.5, 0.3, 12.0), (360, -120.0, 0.75, 0.5, 20.0),
           (1440, -180.0, 0.25, 0.2, 8.0)]


def member_format(s):
    """Member s's scan format; members s and s + 4 share a beam count but not their angles or range window."""
    n, a0, da, rmin, rmax = FORMATS[s % 4]
    j = s // 4
    return dict(n_beams=n, angle_min=float(np.float32(math.radians(a0 + 2.0 * j))),
                angle_increment=float(np.float32(math.radians(da))), range_min=float(np.float32(rmin + 0.05 * j)),
                range_max=float(np.float32(rmax - 1.0 * j)))


def beam_angles(fmt):
    """The beam angles the node accumulates in fp32 (HectorMappingRos.cpp:487, 505)."""
    out = np.empty(fmt["n_beams"], np.float32)
    a, inc = np.float32(fmt["angle_min"]), np.float32(fmt["angle_increment"])
    for i in range(fmt["n_beams"]):
        out[i] = a
        a = np.float32(a + inc)
    return out


def with_edges(r, fmt, k):
    """Ranges exactly at range_min and at the container's bound range_max - 0.1 (both dropped), just inside both
    (kept), and 0, NaN, +inf and -inf, at beams that move with the step."""
    n = r.shape[0]
    if n < 16:
        return r
    rmin = np.float32(fmt["range_min"])
    rmaxc = np.float32(np.float32(fmt["range_max"]) - np.float32(0.1))
    vals = [rmin, rmaxc, np.nextafter(rmin, np.float32(np.inf)), np.nextafter(rmaxc, np.float32(0)), np.float32(0),
            np.float32(np.nan), np.float32(np.inf), np.float32(-np.inf)]
    for i, v in enumerate(vals):
        r[(7 * k + 13 * i + 3) % n] = v
    return r


def session_data(seed, steps, fmt):
    """A trajectory through its own synthetic room: per step the ranges in `fmt`'s beam geometry (with edge values),
    the true pose and a noisy hint."""
    from hector_slam_b200 import synth

    rng = np.random.default_rng(seed)
    world = synth.World(1, seed=1000 + seed)
    angles = beam_angles(fmt)
    x, y, a = rng.uniform(-2, 2), rng.uniform(-1.5, 1.5), rng.uniform(-3, 3)
    truth, ranges = [], []
    for k in range(steps):
        p = np.array([x, y, a], np.float32)
        truth.append(p)
        r = (world.cast(p, angles) + rng.normal(0.0, 0.01, angles.shape[0])).astype(np.float32)
        ranges.append(np.ascontiguousarray(with_edges(r, fmt, k)))
        a += rng.uniform(-0.08, 0.08)
        step = rng.uniform(0.03, 0.12)
        x = float(np.clip(x + step * np.cos(a), -6.0, 6.0))
        y = float(np.clip(y + step * np.sin(a), -4.0, 4.0))
    truth = np.asarray(truth, np.float32)
    hints = truth + rng.uniform(-1, 1, truth.shape).astype(np.float32) * np.array([0.04, 0.04, 0.02], np.float32)
    return dict(truth=truth, ranges=ranges, hints=hints.astype(np.float32), angles=angles)


def make_rep(s, fmt=None, scan_format=True, **kw):
    """Handle of member s: update factors, gate thresholds and scan format differ between members."""
    from hector_slam_b200 import capi

    rep = capi.MapRepB200(RES, SIZE, levels=LEVELS, update_factor_free=0.4 + 0.02 * (s % 3),
                          update_factor_occupied=0.6 + 0.1 * (s % 4), **kw)
    dist, ang = ((0.0, 0.0), (0.15, 0.1), (0.3, 0.5))[s % 3]
    rep.setMapUpdateMinDistDiff(dist)
    rep.setMapUpdateMinAngleDiff(ang)
    if scan_format:
        rep.set_scan_format(**(fmt or member_format(s)))
    return rep


def same(a, b):
    """Bitwise equality of float32 arrays (a NaN pose equals the same NaN: a one-beam scan's rank-1 Hessian gives one)."""
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


def assert_same_state(a, b, tag):
    """Planes, probability planes, gate pose and both dirty rectangles of every level."""
    for l in range(LEVELS):
        assert np.array_equal(a.download_level(l), b.download_level(l)), (tag, l)
        assert np.array_equal(a.download_prob(l), b.download_prob(l)), (tag, l)
        assert a.get_mirror_dirty_rect(l) == b.get_mirror_dirty_rect(l), (tag, l)
    assert a.get_dirty_rects() == b.get_dirty_rects(), tag
    assert same(a.last_map_update_pose(), b.last_map_update_pose()), tag


def assert_same_step(group_out, single_outs, tag):
    P, Cv, U, K = group_out
    for i, (p, c, u, kept) in enumerate(single_outs):
        assert same(P[i], p), (tag, i, P[i], p)
        assert same(Cv[i], c), (tag, i)
        assert U[i] == u, (tag, i)
        assert K[i] == kept, (tag, i, K[i], kept)


def two_call(rep, hint, ranges, map_without_matching=False, nowait=False, cov_inout=None):
    """The path hsb_slam_update_ranges replaces: hsb_scan_to_points, then hsb_slam_update with origo (0, 0)."""
    pts = rep.scan_to_points(ranges)
    p, c, u = rep.slam_update(hint, pts, map_without_matching=map_without_matching, cov_inout=cov_inout,
                              origo=np.zeros(2, np.float32), nowait=nowait)
    return p, c, u, pts.shape[0]


def close_all(*groups):
    for g in groups:
        for x in (g if isinstance(g, (list, tuple)) else [g]):
            x.close()


@pytest.mark.parametrize("nowait", [False, True])
def test_single_ranges_step_bitwise_equals_scan_to_points_plus_slam_update(hsb_lib, nowait):
    """40 steps on four members with different formats: pose, covariance, gate flag and kept count of every step, and
    planes, gate pose and dirty rectangles at the end, equal the two-call path on a twin handle.  map_without_matching
    steps, also straight after a match, write the coarse levels from the last-match container the fused step left."""
    M, steps = 4, 40
    data = [session_data(s, steps, member_format(s)) for s in range(M)]
    fused = [make_rep(s) for s in range(M)]
    twins = [make_rep(s) for s in range(M)]
    covs = {s: np.full((3, 3), 5.0, np.float32) for s in range(M)}
    covs_two = {s: c.copy() for s, c in covs.items()}
    fired = np.zeros(2, int)
    seen_without_after_match = False
    for k in range(steps):
        for s in range(M):
            without = (k % 7 == 3) or (k % 11 == 5 and s % 2 == 0)
            hint = data[s]["truth" if without else "hints"][k]
            p, c, u, kept = fused[s].slam_update_ranges(hint, data[s]["ranges"][k], map_without_matching=without,
                                                        nowait=nowait, cov_inout=covs[s])
            q, d, v, n = two_call(twins[s], hint, data[s]["ranges"][k], map_without_matching=without, nowait=nowait,
                                  cov_inout=covs_two[s])
            assert same(p, q) and same(c, d) and u == v and kept == n, (k, s, p, q, kept, n)
            assert 0 < kept < data[s]["ranges"][k].shape[0], (k, s, kept)
            if not without:
                shape = fused[s].last_launch_shape()
                assert (shape["warps_per_scan"], shape["scans_per_block"], shape["unroll"]) == (8, 1, 4), shape
            elif k > 0 and not ((k - 1) % 7 == 3 or ((k - 1) % 11 == 5 and s % 2 == 0)):
                seen_without_after_match = True
            covs[s], covs_two[s] = c, d
            fired[int(u)] += 1
        if k % 10 == 9:
            for s in range(M):
                assert_same_state(fused[s], twins[s], (k, s))
    assert fired[0] > 0 and fired[1] > 0, fired   # the gate both fires and holds back
    assert seen_without_after_match
    close_all(fused, twins)


def test_kept_counts_and_planes_against_the_node_converter(hsb_lib, pyoracle, oracle_kinds):
    """Kept counts equal the node's compiled rosLaserScanToDataContainer (pyoracle.scan_to_points, kind="reference"
    where it is built); a twin driven by those endpoints through hsb_slam_update ends with identical planes.  Every scan
    carries ranges exactly at range_min and range_max - 0.1, just inside both, 0, NaN and +-inf."""
    kind = "reference" if "reference" in oracle_kinds else "port"
    M, steps = 4, 12
    data = [session_data(130 + s, steps, member_format(s)) for s in range(M)]
    fused = [make_rep(s) for s in range(M)]
    twins = [make_rep(s) for s in range(M)]
    scale = fused[0].getScaleToMap()
    for k in range(steps):
        for s in range(M):
            f = member_format(s)
            r = data[s]["ranges"][k]
            pts = pyoracle.scan_to_points(r, f["angle_min"], f["angle_increment"], f["range_min"], f["range_max"], scale,
                                          kind=kind)
            without = k % 5 == 4
            p, _, u, kept = fused[s].slam_update_ranges(data[s]["hints"][k], r, map_without_matching=without)
            assert kept == pts.shape[0], (k, s, kept, pts.shape[0])
            q, _, v = twins[s].slam_update(data[s]["hints"][k], pts, map_without_matching=without,
                                           origo=np.zeros(2, np.float32))
            assert same(p, q) and u == v, (k, s)
    for s in range(M):
        assert_same_state(fused[s], twins[s], s)
    close_all(fused, twins)


def test_group_ranges_step_bitwise_equals_single_ranges_steps(hsb_lib):
    """12 members (beam counts 1081, 720, 360 and 1440 with differing angles and range windows), 40 steps: every pose,
    covariance, gate decision and kept count and the final handle state equal twin handles stepped with
    hsb_slam_update_ranges."""
    from hector_slam_b200 import capi

    M, steps = 12, 40
    data = [session_data(s, steps, member_format(s)) for s in range(M)]
    grp_reps = [make_rep(s) for s in range(M)]
    one_reps = [make_rep(s) for s in range(M)]
    group = capi.SlamGroup(grp_reps)
    fired = np.zeros(2, int)
    for k in range(steps):
        hints = np.stack([d["hints"][k] for d in data])
        out = group.slam_update_ranges(hints, [d["ranges"][k] for d in data], nowait=(k % 3 == 1))
        single = [one_reps[s].slam_update_ranges(hints[s], data[s]["ranges"][k]) for s in range(M)]
        assert_same_step(out, single, k)
        for s in range(M):
            fired[int(out[2][s])] += 1
    assert fired[0] > 0 and fired[1] > 0, fired
    for s in range(M):
        assert_same_state(grp_reps[s], one_reps[s], s)
    group.close()
    close_all(grp_reps, one_reps)


def test_edge_sessions_in_permuted_groups(hsb_lib):
    """Scans whose every range is filtered out (kept 0: pose = hint, covariance untouched), a member with n_beams = 1
    (its one endpoint gives a rank-1 Hessian and, as in the reference, a non-finite pose, which the map writer drops),
    and map_without_matching sessions (also straight after a matched step) over three groups of the same handles in
    different session orders."""
    from hector_slam_b200 import capi

    M, steps = 6, 18
    fmts = [member_format(s) for s in range(M - 1)] + [dict(n_beams=1, angle_min=0.3, angle_increment=0.01,
                                                          range_min=0.1, range_max=30.0)]
    data = [session_data(20 + s, steps, fmts[s]) for s in range(M)]
    grp_reps = [make_rep(s, fmts[s]) for s in range(M)]
    one_reps = [make_rep(s, fmts[s]) for s in range(M)]
    rng = np.random.default_rng(4)
    orders = [list(range(M)), list(range(M))[::-1], [int(x) for x in rng.permutation(M)]]
    groups = [capi.SlamGroup([grp_reps[s] for s in o]) for o in orders]
    covs = {s: np.full((3, 3), 7.0, np.float32) for s in range(M)}
    covs_one = {s: c.copy() for s, c in covs.items()}
    kinds_seen = set()
    prev_matched = np.zeros(M, bool)
    for k in range(steps):
        kind = rng.choice(["match", "match", "filtered", "without"], M)
        if k == 0:
            kind[:] = "match"
        if k == 1:
            kind[0] = "without"   # straight after a matched step
        order = orders[k % 3]
        hints, ranges, mwm, cin = [], [], [], []
        for s in order:
            r = data[s]["ranges"][k].copy()
            if kind[s] == "filtered":
                r[:] = np.float32(fmts[s]["range_min"]) * np.float32(0.5)   # every beam below range_min
            hints.append(data[s]["truth"][k] if kind[s] == "without" else data[s]["hints"][k])
            ranges.append(r)
            mwm.append(kind[s] == "without")
            cin.append(covs[s])
            if kind[s] == "without" and prev_matched[s]:
                kinds_seen.add("without-after-match")
            kinds_seen.add(str(kind[s]))
        P, Cv, U, K = groups[k % 3].slam_update_ranges(np.stack(hints), ranges, map_without_matching=mwm,
                                                        cov_inout=np.stack(cin))
        single = []
        for i, s in enumerate(order):
            single.append(one_reps[s].slam_update_ranges(hints[i], ranges[i], map_without_matching=mwm[i],
                                                         cov_inout=covs_one[s]))
            if kind[s] == "filtered":
                assert K[i] == 0, (k, s)
                assert same(P[i], hints[i]) and same(Cv[i], covs[s]), (k, s)
            if s == M - 1 and kind[s] != "filtered":
                assert K[i] == 1, (k, K[i])   # the one-beam member's beam hits a wall
        assert_same_step((P, Cv, U, K), single, k)
        for i, s in enumerate(order):
            covs[s], covs_one[s] = Cv[i], single[i][1]
            prev_matched[s] = kind[s] == "match"
    assert {"match", "filtered", "without", "without-after-match"} <= kinds_seen, kinds_seen
    for s in range(M):
        assert_same_state(grp_reps[s], one_reps[s], s)
    close_all(groups, grp_reps, one_reps)


def test_mixing_with_other_calls_without_synchronisation(hsb_lib):
    """Between nowait group ranges steps the same members take group cloud and group endpoint steps, single steps of
    every input kind, a reset, a scan-format change between two nowait steps, torch-stream hsb_match_batch_ranges_device
    calls and downloads, with no synchronisation by the caller.  Everything equals the same sequence driven only by
    single calls."""
    import torch

    from hector_slam_b200 import capi, synth

    M, steps = 4, 16
    fmts = [member_format(s) for s in range(M)]
    data = [session_data(60 + s, steps, fmts[s]) for s in range(M)]
    grp_reps = [make_rep(s) for s in range(M)]
    one_reps = [make_rep(s) for s in range(M)]
    for r in grp_reps + one_reps:
        r.set_cloud_format(synth.laser_transform(), **synth.CLOUD_FORMAT)
    group = capi.SlamGroup(grp_reps)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)

    def cloud(s, k):
        return np.ascontiguousarray(synth.ranges_to_cloud(data[s]["ranges"][k], data[s]["angles"]), np.float32)

    def endpoints(s, k):
        return np.ascontiguousarray(synth.ranges_to_points(data[s]["ranges"][k], SCALE, data[s]["angles"]), np.float32)

    def batch(rep, hint, ranges):
        d_h = torch.from_numpy(np.repeat(hint[None], 8, axis=0)).to(dev)
        d_r = torch.from_numpy(np.repeat(ranges[None], 8, axis=0)).to(dev)
        poses = torch.zeros((8, 3), dtype=torch.float32, device=dev)
        torch.cuda.current_stream(dev).synchronize()   # the inputs are on the device
        rep.match_batch_ranges_device(8, d_h.data_ptr(), d_r.data_ptr(), poses.data_ptr(), None, stream.cuda_stream)
        with torch.cuda.stream(stream):
            return poses.cpu().numpy()   # reads the results: waits for this stream only

    for k in range(steps):
        hints = np.stack([d["hints"][k] for d in data])
        if k % 4 == 1:   # a group step of the other two input kinds on the same members
            if k % 8 == 1:
                P, Cv, U = group.slam_update(hints, [endpoints(s, k) for s in range(M)], nowait=True)
                for s in range(M):
                    p, c, u = one_reps[s].slam_update(hints[s], endpoints(s, k))
                    assert same(P[s], p) and same(Cv[s], c) and U[s] == u, (k, s)
            else:
                out = group.slam_update_cloud(hints, [cloud(s, k) for s in range(M)], nowait=True)
                assert_same_step(out, [one_reps[s].slam_update_cloud(hints[s], cloud(s, k)) for s in range(M)], k)
        else:
            out = group.slam_update_ranges(hints, [d["ranges"][k] for d in data], nowait=True)
            assert_same_step(out, [one_reps[s].slam_update_ranges(hints[s], data[s]["ranges"][k]) for s in range(M)], k)
        if k % 4 == 2:   # single steps of every kind on members right after the group step
            x = grp_reps[0].slam_update_ranges(data[0]["truth"][k], data[0]["ranges"][k], nowait=True)
            y = one_reps[0].slam_update_ranges(data[0]["truth"][k], data[0]["ranges"][k])
            assert all(same(u, v) for u, v in zip(x, y)), k
            x = grp_reps[1].slam_update(data[1]["truth"][k], endpoints(1, k), nowait=True)
            y = one_reps[1].slam_update(data[1]["truth"][k], endpoints(1, k))
            assert all(same(u, v) for u, v in zip(x, y)), k
            x = grp_reps[2].slam_update_cloud(data[2]["truth"][k], cloud(2, k), nowait=True)
            y = one_reps[2].slam_update_cloud(data[2]["truth"][k], cloud(2, k))
            assert all(same(u, v) for u, v in zip(x, y)), k
        if k == 6:
            grp_reps[2].reset()
            one_reps[2].reset()
        if k == 8:   # between two nowait group ranges steps: read at the next step's conversion
            new = dict(fmts[3], angle_min=fmts[3]["angle_min"] + 0.01, range_max=10.0)
            for r in (grp_reps[3], one_reps[3]):
                r.set_scan_format(**new)
        if k % 3 == 2:
            assert np.array_equal(batch(grp_reps[2], data[2]["hints"][k], data[2]["ranges"][k]),
                                  batch(one_reps[2], data[2]["hints"][k], data[2]["ranges"][k])), k
        if k % 4 == 3:
            assert np.array_equal(grp_reps[3].download_occupancy(0), one_reps[3].download_occupancy(0)), k
    for s in range(M):
        assert_same_state(grp_reps[s], one_reps[s], s)
    group.close()
    close_all(grp_reps, one_reps)


def test_single_member_group_and_nowait(hsb_lib):
    """M = 1 equals hsb_slam_update_ranges bit for bit; nowait = 1 equals nowait = 0 for a 5-member group, with
    hsb_on_map_updated of each member as the completion point before the planes are read."""
    from hector_slam_b200 import capi

    steps = 14
    d = session_data(77, steps, member_format(1))
    a, b = make_rep(1), make_rep(1)
    ga = capi.SlamGroup([a])
    for k in range(steps):
        out = ga.slam_update_ranges(d["hints"][k][None], [d["ranges"][k]], map_without_matching=[k == 5])
        assert_same_step(out, [b.slam_update_ranges(d["hints"][k], d["ranges"][k], map_without_matching=(k == 5))], k)
    assert_same_state(a, b, "M=1")
    ga.close()
    close_all([a, b])

    M = 5
    data = [session_data(40 + s, steps, member_format(s)) for s in range(M)]

    def run(nowait):
        reps = [make_rep(s) for s in range(M)]
        grp = capi.SlamGroup(reps)
        out = []
        for k in range(steps):
            out.append(grp.slam_update_ranges(np.stack([x["hints"][k] for x in data]), [x["ranges"][k] for x in data],
                                              map_without_matching=[k % 6 == 5] * M, nowait=nowait))
        for r in reps:
            r.onMapUpdated()
        planes = [[r.download_level(l) for l in range(LEVELS)] for r in reps]
        grp.close()
        return out, planes, reps

    (oa, pa, ra), (ob, pb, rb) = run(False), run(True)
    for k in range(steps):
        for x, y in zip(oa[k], ob[k]):
            assert same(x, y), k
    for s in range(M):
        for l in range(LEVELS):
            assert np.array_equal(pa[s][l], pb[s][l]), (s, l)
        assert_same_state(ra[s], rb[s], s)
    close_all(ra, rb)


def test_validation_leaves_every_member_unchanged(hsb_lib):
    """A member without a scan format, offsets that disagree with the members' n_beams, n != n_beams on the single
    call and an oversize format are rejected before any member changes.  The step after each rejection is
    map_without_matching everywhere, so its coarse levels write the last-match container the members hold: it still
    equals the single-call twins, and the group keeps working."""
    from hector_slam_b200 import capi

    M, steps = 3, 10
    data = [session_data(150 + s, steps, member_format(s)) for s in range(M)]
    grp_reps = [make_rep(s, scan_format=(s != 1)) for s in range(M)]
    one_reps = [make_rep(s) for s in range(M)]
    group = capi.SlamGroup(grp_reps)
    step_no = [0]

    def valid_step(without):
        k = step_no[0]
        step_no[0] += 1
        hints = np.stack([d["truth" if without else "hints"][k] for d in data])
        out = group.slam_update_ranges(hints, [d["ranges"][k] for d in data], map_without_matching=[without] * M,
                                       nowait=(k % 2 == 1))
        single = [one_reps[s].slam_update_ranges(hints[s], data[s]["ranges"][k], map_without_matching=without)
                  for s in range(M)]
        assert_same_step(out, single, k)

    def rejected(status, text, ranges):
        hints = np.stack([d["hints"][step_no[0]] for d in data])
        with pytest.raises(capi.HsbError) as e:
            group.slam_update_ranges(hints, ranges)
        assert e.value.status == status and text in str(e.value), str(e.value)
        return str(e.value)

    ranges = [d["ranges"][0] for d in data]
    rejected(-1, "session 1", ranges)   # member 1 has no scan format
    grp_reps[1].set_scan_format(**member_format(1))
    valid_step(False)
    valid_step(False)

    n = [r.shape[0] for r in ranges]
    flat = np.concatenate(ranges)
    for offs in ([1, n[0], n[0] + n[1], flat.shape[0]], [0, n[0], n[0] - 1, flat.shape[0]],
                 [0, n[0] + 1, n[0] + n[1], flat.shape[0]], [0, n[0], n[0] + n[1], flat.shape[0] - 1]):
        rejected(-1, "offsets" if offs[0] or offs[2] < offs[1] else "beams", (flat, np.array(offs, np.int32)))
    valid_step(True)
    valid_step(False)

    for bad in (ranges[0][:-1], np.concatenate([ranges[0], ranges[0][:1]])):   # the single call: n != n_beams
        with pytest.raises(capi.HsbError) as e:
            grp_reps[0].slam_update_ranges(data[0]["hints"][0], bad)
        assert e.value.status == -1 and "beams" in str(e.value), str(e.value)
    valid_step(True)
    valid_step(False)

    big_fmt = dict(member_format(0), n_beams=30000, angle_increment=float(np.float32(1e-4)))
    grp_reps[0].set_scan_format(**big_fmt)
    big = np.full(30000, 3.0, np.float32)
    msg = rejected(-5, "scan too long for the fused conversion (30000 points)", [big, ranges[1], ranges[2]])
    probe = make_rep(0, big_fmt)   # the single call's limit and wording (on a handle of its own: its state is not compared)
    with pytest.raises(capi.HsbError) as e:
        probe.slam_update_ranges(data[0]["hints"][0], big)
    assert e.value.status == -5 and str(e.value) == msg
    probe.close()
    grp_reps[0].set_scan_format(**member_format(0))
    valid_step(True)
    valid_step(False)
    for s in range(M):
        assert_same_state(grp_reps[s], one_reps[s], s)
    group.close()
    close_all(grp_reps, one_reps)


@pytest.mark.parametrize("M", [1, 16])
def test_launch_count(hsb_lib, M):
    """A matched single ranges step is three launches; a group ranges step is three launches, counted on handles[0],
    also with map_without_matching sessions, and the other members' counts do not move."""
    from hector_slam_b200 import capi

    reps = [make_rep(s) for s in range(M)]
    data = [session_data(90 + s, 4, member_format(s)) for s in range(M)]
    before = reps[0].launch_count
    reps[0].slam_update_ranges(data[0]["hints"][0], data[0]["ranges"][0])
    reps[0].slam_update_ranges(data[0]["hints"][0], data[0]["ranges"][0], nowait=True)
    assert reps[0].launch_count - before == 6
    group = capi.SlamGroup(reps)
    for k in range(1, 4):
        before = [r.launch_count for r in reps]
        group.slam_update_ranges(np.stack([d["hints"][k] for d in data]), [d["ranges"][k] for d in data],
                                 map_without_matching=[k == 3 and s % 2 == 0 for s in range(M)], nowait=(k == 2))
        after = [r.launch_count for r in reps]
        assert after[0] - before[0] == 3, (k, before[0], after[0])
        assert after[1:] == before[1:], k
    group.close()
    close_all(reps)


def test_facade_update_ranges_and_update_many_ranges(hsb_lib):
    """hsb200::SlamProcessor::updateManyRanges and updateRanges (C++ façade, through its shim) equal each other and
    hsb_slam_update_ranges on a third processor's handle — poses, covariances, kept counts and maps — with per-processor
    scan formats and gate thresholds."""
    L = C.CDLL(os.path.join(ROOT, "hector_slam_b200", "lib", "libhsb200_host.so"))
    lib = hsb_lib
    vp, i, f = C.c_void_p, C.c_int, C.c_float
    L.hsbp_create.restype = vp
    L.hsbp_create.argtypes = [f, i, i, f, f, i, i]
    L.hsbp_destroy.argtypes = [vp]
    L.hsbp_handle.restype = vp
    L.hsbp_handle.argtypes = [vp]
    L.hsbp_set_scan_format.argtypes = [vp, i, f, f, f, f]
    L.hsbp_set_map_update_thresholds.argtypes = [vp, f, f]
    L.hsbp_update_ranges.argtypes = [vp, vp, i, vp, i, vp]
    L.hsbp_update_many_ranges.argtypes = [vp, i, vp, vp, vp, vp, vp]
    L.hsbp_get_pose_and_cov.argtypes = [vp, vp, vp]
    L.hsbp_get_grid_map.argtypes = [vp, i, vp]
    M, steps = 3, 8
    fmts = [member_format(s) for s in range(M)]
    data = [session_data(110 + s, steps, fmts[s]) for s in range(M)]
    sets = [[L.hsbp_create(RES, SIZE, SIZE, 0.5, 0.5, LEVELS, 0) for _ in range(M)] for _ in range(3)]
    many, one, capi_ps = sets
    assert all(all(x) for x in sets)
    for s in range(M):
        fm = fmts[s]
        for p in (many[s], one[s], capi_ps[s]):
            assert L.hsbp_set_scan_format(p, fm["n_beams"], fm["angle_min"], fm["angle_increment"], fm["range_min"],
                                          fm["range_max"]) == 0
            L.hsbp_set_map_update_thresholds(p, (0.0, 0.15, 0.3)[s], (0.0, 0.1, 0.5)[s])
    arr = (C.c_void_p * M)(*many)
    cov3 = {s: np.zeros(9, np.float32) for s in range(M)}
    for k in range(steps):
        rs = [d["ranges"][k] for d in data]
        flat = np.ascontiguousarray(np.concatenate(rs), np.float32)
        offs = np.zeros(M + 1, np.int32)
        offs[1:] = np.cumsum([x.shape[0] for x in rs])
        hints = np.ascontiguousarray(np.stack([d["hints"][k] for d in data]), np.float32)
        mwm = np.array([0, int(k % 3 == 2), 0], np.int32)
        kept = np.zeros(M, np.int32)
        assert L.hsbp_update_many_ranges(C.cast(arr, C.c_void_p), M, flat.ctypes.data, offs.ctypes.data,
                                         hints.ctypes.data, mwm.ctypes.data, kept.ctypes.data) == 0
        for s in range(M):
            p1, c1, p2, c2 = (np.zeros(3, np.float32), np.zeros(9, np.float32), np.zeros(3, np.float32),
                              np.zeros(9, np.float32))
            k1 = C.c_int(-1)
            assert L.hsbp_update_ranges(one[s], rs[s].ctypes.data, rs[s].shape[0], hints[s].ctypes.data, int(mwm[s]),
                                        C.byref(k1)) == 0
            p3, upd, k3 = np.zeros(3, np.float32), C.c_int(0), C.c_int(-1)
            assert lib.hsb_slam_update_ranges(L.hsbp_handle(capi_ps[s]), hints[s].ctypes.data, rs[s].ctypes.data,
                                              rs[s].shape[0], int(mwm[s]), 0, p3.ctypes.data, cov3[s].ctypes.data,
                                              C.addressof(upd), C.addressof(k3)) == 0
            L.hsbp_get_pose_and_cov(many[s], p1.ctypes.data, c1.ctypes.data)
            L.hsbp_get_pose_and_cov(one[s], p2.ctypes.data, c2.ctypes.data)
            assert same(p1, p2) and same(c1, c2) and kept[s] == k1.value, (k, s)
            assert same(p1, p3) and same(c1, cov3[s]) and k3.value == k1.value, (k, s)
    for s in range(M):
        for l in range(LEVELS):
            sz = SIZE >> l
            x, y, z = (np.zeros((sz, sz), np.float32) for _ in range(3))
            assert L.hsbp_get_grid_map(many[s], l, x.ctypes.data) == 0
            assert L.hsbp_get_grid_map(one[s], l, y.ctypes.data) == 0
            assert L.hsbp_get_grid_map(capi_ps[s], l, z.ctypes.data) == 0
            assert np.array_equal(x, y) and np.array_equal(x, z), (s, l)
    for p in many + one + capi_ps:   # any member first: its cached group goes with it
        L.hsbp_destroy(p)
