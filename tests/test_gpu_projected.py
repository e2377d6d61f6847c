"""hsb_slam_update_projected and hsb_group_slam_update_projected — the node's default SLAM step from the LaserScan it
receives: laser_geometry's projection, the cloud conversion, match, gate and map write in one device pass — for one
session and for a group.

The conversion is checked against the oracle (tests/laser_projection.py + the node's cloud converter) and against
hsb_cloud_to_points on the projected cloud; the single step against hsb_slam_update_cloud on the numpy-projected cloud
on a twin handle; the group step against single projected steps.  Every comparison is bitwise: poses, covariances, gate
decisions, kept counts, every level's log-odds and probability planes, the gate pose and both dirty rectangles.  Members
differ in beam count, angles, cutoff, range window, laser mount, cloud thresholds, update factors and gate thresholds."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from conftest import ROOT, pose_err, report
from laser_projection import cutoff_of, edge_ranges, project, tilted_transform

pytestmark = pytest.mark.gpu

RES, SIZE, LEVELS = 0.05, 512, 3
SCALE = 1.0 / RES
F32 = np.float32
# the staging limit of the fused conversion (8-warp shape): 2448 B of header + whole_scan_slots(n) * 8 B <= 227 KB
LIMIT = 28749

# n_beams, angle_min (deg), angle_increment (deg), range_min, range_max, range_cutoff of the four basic members
PROJ = [(1081, -135.0, 0.25, 0.1, 30.0, 30.0), (720, -180.0, 0.5, 0.3, 12.0, 30.0), (360, -120.0, 0.75, 0.5, 20.0, -1.0),
        (1440, -180.0, 0.25, 0.2, 8.0, 6.5)]


def member_proj(s):
    n, a0, da, rmin, rmax, cut = PROJ[s % 4]
    j = s // 4
    return dict(n_beams=n, angle_min=float(F32(math.radians(a0 + 2.0 * j))), angle_increment=float(F32(math.radians(da))),
                range_min=float(F32(rmin + 0.05 * j)), range_max=float(F32(rmax - 1.0 * j)),
                range_cutoff=cut if cut < 0 else cut - 0.5 * j)


def member_transform(s):
    from hector_slam_b200 import synth

    if s % 5 == 4:
        return tilted_transform(pitch=0.05 + 0.01 * s)
    return synth.laser_transform(xyz=(0.1 + 0.01 * s, -0.03 + 0.005 * s, 0.3), rpy=(0.02, -0.01 * (s % 3), 0.03 * s))


def member_cloud(s):
    from hector_slam_b200 import synth

    fmt = dict(synth.CLOUD_FORMAT)
    fmt["sqr_laser_min_dist"] = float(F32((0.3 + 0.05 * (s % 3)) ** 2))
    fmt["sqr_laser_max_dist"] = float(F32((25.0 - s) ** 2))
    fmt["laser_z_min_value"] = -0.5 - 0.1 * (s % 4)
    fmt["laser_z_max_value"] = 0.5 + 0.1 * (s % 4)
    return fmt


def beam_angles64(p):
    return float(F32(p["angle_min"])) + np.arange(p["n_beams"]) * float(F32(p["angle_increment"]))


def session_data(seed, steps, p):
    """A trajectory through its own synthetic room: per step the ranges in `p`'s beam geometry with the projector's
    dropped edge values (NaN, +-inf, negative, 0, just below range_min, at the cutoff), the true pose and a noisy hint."""
    from hector_slam_b200 import synth

    rng = np.random.default_rng(seed)
    world = synth.World(1, seed=1000 + seed)
    angles = beam_angles64(p).astype(F32)
    x, y, a = rng.uniform(-2, 2), rng.uniform(-1.5, 1.5), rng.uniform(-3, 3)
    truth, ranges = [], []
    for k in range(steps):
        pose = np.array([x, y, a], F32)
        truth.append(pose)
        r = (world.cast(pose, angles) + rng.normal(0.0, 0.01, angles.shape[0])).astype(F32)
        ranges.append(np.ascontiguousarray(edge_ranges(r.size, p, 7 * k + seed, base=r, dropped_only=True)))
        a += rng.uniform(-0.08, 0.08)
        step = rng.uniform(0.03, 0.12)
        x = float(np.clip(x + step * np.cos(a), -6.0, 6.0))
        y = float(np.clip(y + step * np.sin(a), -4.0, 4.0))
    truth = np.asarray(truth, F32)
    hints = truth + rng.uniform(-1, 1, truth.shape).astype(F32) * np.array([0.04, 0.04, 0.02], F32)
    return dict(truth=truth, ranges=ranges, hints=hints.astype(F32))


def make_rep(s, proj=None, cloud=None, with_proj=True, with_cloud=True, **kw):
    from hector_slam_b200 import capi

    rep = capi.MapRepB200(RES, SIZE, levels=LEVELS, update_factor_free=0.4 + 0.02 * (s % 3),
                          update_factor_occupied=0.6 + 0.1 * (s % 4), **kw)
    dist, ang = ((0.0, 0.0), (0.15, 0.1), (0.3, 0.5))[s % 3]
    rep.setMapUpdateMinDistDiff(dist)
    rep.setMapUpdateMinAngleDiff(ang)
    if with_proj:
        rep.set_laser_projection(**(proj or member_proj(s)))
    if with_cloud:
        rep.set_cloud_format(member_transform(s), **(cloud or member_cloud(s)))
    return rep


def same(a, b):
    return np.array_equal(np.asarray(a, F32).view(np.uint32), np.asarray(b, F32).view(np.uint32))


def assert_same_state(a, b, tag):
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


def close_all(*groups):
    for g in groups:
        for x in (g if isinstance(g, (list, tuple)) else [g]):
            x.close()


def test_projected_scan_to_points_equals_oracle_and_cloud_conversion(hsb_lib, pyoracle, oracle_kinds):
    """Edge scans of every member format (NaN, +-inf, negative, range_min and the float below it, cutoff and the float
    below it, rear-close returns, a tilted mount, an all-dropped scan), a 1-beam scan and a scan at the staging limit:
    endpoints, count and origo equal the oracle container and hsb_cloud_to_points on the projected cloud."""
    from hector_slam_b200 import capi

    kind = "reference" if "reference" in oracle_kinds else "port"
    cases = []
    for s in range(8):
        p = member_proj(s)
        for seed in range(3):
            cases.append((s, p, edge_ranges(p["n_beams"], p, 31 * s + seed)))
        cases.append((s, p, np.full(p["n_beams"], np.nan, F32)))
    one = dict(member_proj(0), n_beams=1)
    cases += [(0, one, np.array([2.5], F32)), (1, one, np.array([np.inf], F32))]
    big = dict(member_proj(0), n_beams=LIMIT, angle_increment=float(F32(2 * math.pi / LIMIT)))
    cases.append((2, big, edge_ranges(LIMIT, big, 5)))
    reps = {}
    for s, p, r in cases:
        key = (s, p["n_beams"], p["angle_min"])
        if key not in reps:
            reps[key] = make_rep(s, proj=p)
        rep = reps[key]
        T = member_transform(s)
        for transform in (None, member_transform(s + 1)):
            Tu = T if transform is None else transform
            got, og = rep.projected_scan_to_points(r, transform)
            cloud = project(r, p)
            want, wog = pyoracle.cloud_to_points(cloud, Tu, *(member_cloud(s)[k] for k in (
                "sqr_laser_min_dist", "sqr_laser_max_dist", "laser_z_min_value", "laser_z_max_value")), SCALE, kind=kind)
            assert same(got, want) and same(og, wog), (s, p["n_beams"])
            if transform is None:
                alt, aog = rep.cloud_to_points(cloud)
                assert same(got, alt) and same(og, aog), (s, p["n_beams"])
    over = make_rep(0, proj=dict(big, n_beams=LIMIT + 1))
    with pytest.raises(capi.HsbError) as e:
        over.projected_scan_to_points(np.full(LIMIT + 1, 3.0, F32))
    assert e.value.status == -5 and "scan too long" in str(e.value)
    close_all(list(reps.values()), over)


@pytest.mark.parametrize("gather", ["ldg", "tex"])
def test_single_projected_step_bitwise_equals_cloud_step(hsb_lib, pyoracle, oracle_kinds, gather):
    """40 steps on four members: sync and nowait steps, map_without_matching steps (also straight after a matched one),
    empty scans, a per-call transform and the format's.  Pose, covariance, gate, kept count of every step and the end
    state equal hsb_slam_update_cloud on the numpy-projected cloud, and every kept count equals the oracle container's.
    (The poses against the node's compiled update: test_poses_against_the_reference_update_on_the_same_map.)"""
    from hector_slam_b200 import capi

    mode = capi.GATHER_LDG if gather == "ldg" else capi.GATHER_TEX
    kind = "reference" if "reference" in oracle_kinds else "port"
    M, steps = 4, 40
    data = [session_data(s, steps, member_proj(s)) for s in range(M)]
    fused = [make_rep(s, gather_mode=mode) for s in range(M)]
    twins = [make_rep(s, gather_mode=mode) for s in range(M)]
    covs = {s: np.full((3, 3), 5.0, F32) for s in range(M)}
    covs_two = {s: c.copy() for s, c in covs.items()}
    fired = np.zeros(2, int)
    seen = set()
    prev_without = [False] * M
    for k in range(steps):
        for s in range(M):
            p = member_proj(s)
            without = (k % 7 == 3) or (k % 11 == 5 and s % 2 == 0)
            r = data[s]["ranges"][k]
            if k % 13 == 9:
                r = np.full(p["n_beams"], np.nan, F32)   # empty scan: pose = hint, covariance untouched
                seen.add("empty")
            T = member_transform(s + 7) if k % 4 == 2 else None
            hint = data[s]["truth" if without else "hints"][k]
            nowait = k % 3 == 1
            a = fused[s].slam_update_projected(hint, r, transform=T, map_without_matching=without, nowait=nowait,
                                               cov_inout=covs[s])
            b = twins[s].slam_update_cloud(hint, project(r, p), transform=T, map_without_matching=without, nowait=nowait,
                                           cov_inout=covs_two[s])
            assert all(same(x, y) for x, y in zip(a[:2], b[:2])) and a[2:] == b[2:], (k, s, a, b)
            if without and k > 0 and not prev_without[s]:
                seen.add("without-after-match")
            prev_without[s] = without
            if not without:
                shape = fused[s].last_launch_shape()
                assert (shape["warps_per_scan"], shape["scans_per_block"], shape["unroll"]) == (8, 1, 4), shape
            covs[s], covs_two[s] = a[1], b[1]
            fired[int(a[2])] += 1
            pts, _ = oracle_container(pyoracle, kind, s, r, T)
            assert pts.shape[0] == a[3], (k, s)
        if k % 10 == 9:
            for s in range(M):
                assert_same_state(fused[s], twins[s], (k, s))
    assert fired[0] > 0 and fired[1] > 0, fired
    assert {"empty", "without-after-match"} <= seen
    close_all(fused, twins)


def oracle_container(pyoracle, kind, s, r, T=None):
    """Member s's DataContainer of ranges r as the node builds it: the restated projection, then the cloud converter."""
    cf = member_cloud(s)
    return pyoracle.cloud_to_points(project(r, member_proj(s)), member_transform(s) if T is None else T,
                                    cf["sqr_laser_min_dist"], cf["sqr_laser_max_dist"], cf["laser_z_min_value"],
                                    cf["laser_z_max_value"], SCALE, kind=kind)


def test_poses_against_the_reference_update_on_the_same_map(hsb_lib, pyoracle, oracle_kinds):
    """The 40-step runs of four members against the node's compiled HectorSlamProcessor::update on the oracle
    containers, one step at a time on the same map: before every step the reference's log-odds planes are uploaded into
    the handle, so each step's pose difference is that step's own, not an accumulation of earlier map differences.

    Where the reference is reproducible — its pose does not move past 1e-4 when the same scan is summed in reversed or
    rotated order or the hint moves by 3e-5 (m, m, rad), measured on a probe holding the same planes — the device is
    within 1e-4 m / 1e-4 rad.  On these runs many steps are not reproducible in the reference itself (the hints are up to
    4 cm / 0.02 rad off and the maps hold a few scans: Gauss-Newton stops before its fixed point, cf.
    test_oracle_golden.py::test_reference_sensitivity_on_a_sparse_map); there the device, whose summation order is
    another such change, must stay within twice the largest of those moves."""
    kind = "reference" if "reference" in oracle_kinds else "port"
    M, steps = 4, 40
    pert = [np.array(v, F32) for v in ([3e-5, -3e-5, 3e-5], [-3e-5, 3e-5, -3e-5])]
    stable = unstable = 0
    worst_stable, worst_ratio = 0.0, 0.0
    for s in range(M):
        data = session_data(s, steps, member_proj(s))
        rep = make_rep(s)
        orcs = []
        for _ in range(2):   # the reference, and a probe that receives its planes
            o = pyoracle.Oracle(kind, RES, SIZE, LEVELS)
            o.set_update_factors(0.4 + 0.02 * (s % 3), 0.6 + 0.1 * (s % 4))
            o.set_map_update_thresholds(*((0.0, 0.0), (0.15, 0.1), (0.3, 0.5))[s % 3])
            orcs.append(o)
        orc, probe = orcs
        for k in range(steps):
            without = (k % 7 == 3) or (k % 11 == 5 and s % 2 == 0)
            hint = data["truth" if without else "hints"][k]
            r = data["ranges"][k]
            T = member_transform(s + 7) if k % 4 == 2 else None
            pts, og = oracle_container(pyoracle, kind, s, r, T)
            planes = [orc.get_logodds(l) for l in range(LEVELS)]
            for l in range(LEVELS):
                rep.upload_level(l, planes[l])
            got, _, _, kept = rep.slam_update_projected(hint, r, transform=T, map_without_matching=without)
            want, _ = orc.update(pts, hint, map_without_matching=without, origo=og)
            assert kept == pts.shape[0], (s, k)
            if without:
                assert same(got, want), (s, k)
                continue
            for l in range(LEVELS):
                probe.set_logodds(l, planes[l])
            base, _ = probe.match(hint, pts, og)
            assert same(base, want), (s, k)   # the probe is the reference at this step
            moves = [probe.match(hint, np.ascontiguousarray(alt), og)[0] for alt in (pts[::-1], np.roll(pts, 137, axis=0))]
            moves += [probe.match((hint + d).astype(F32), pts, og)[0] for d in pert]
            spread = max(max(pose_err(m, base)) for m in moves)
            err = max(pose_err(got, want))
            if spread <= 1e-4:
                stable += 1
                worst_stable = max(worst_stable, err)
                assert err <= 1e-4, (s, k, err, spread)
            else:
                unstable += 1
                worst_ratio = max(worst_ratio, err / spread)
                assert err <= 2.0 * spread, (s, k, err, spread)
        rep.close()
        close_all(orcs)
    report(f"projected step vs {kind} update, same map every step: {stable} reproducible steps, worst {worst_stable:.2e}; "
           f"{unstable} steps where the reference itself moves past 1e-4, worst device / reference-spread {worst_ratio:.2f}")
    assert stable >= 60, (stable, unstable)


def test_group_projected_step_bitwise_equals_single_steps(hsb_lib):
    """12 members (four beam counts, differing angles, cutoffs, range windows, mounts, thresholds, update factors and
    gate thresholds), 40 steps with per-scan transforms on odd steps: every result and the final member state equal
    twin handles stepped with hsb_slam_update_projected."""
    from hector_slam_b200 import capi

    M, steps = 12, 40
    data = [session_data(s, steps, member_proj(s)) for s in range(M)]
    grp_reps = [make_rep(s) for s in range(M)]
    one_reps = [make_rep(s) for s in range(M)]
    group = capi.SlamGroup(grp_reps)
    fired = np.zeros(2, int)
    for k in range(steps):
        hints = np.stack([d["hints"][k] for d in data])
        T = np.stack([member_transform(s + k) for s in range(M)]) if k % 2 else None
        mwm = [k % 9 == 4 and s % 3 == 0 for s in range(M)]
        out = group.slam_update_projected(hints, [d["ranges"][k] for d in data], transforms=T, map_without_matching=mwm,
                                          nowait=(k % 3 == 1))
        single = [one_reps[s].slam_update_projected(hints[s], data[s]["ranges"][k], transform=None if T is None else T[s],
                                                    map_without_matching=mwm[s]) for s in range(M)]
        assert_same_step(out, single, k)
        for s in range(M):
            fired[int(out[2][s])] += 1
    assert fired[0] > 0 and fired[1] > 0, fired
    for s in range(M):
        assert_same_state(grp_reps[s], one_reps[s], s)
    group.close()
    close_all(grp_reps, one_reps)


def test_edge_sessions_in_permuted_groups(hsb_lib):
    """All-dropped scans (kept 0: pose = hint, covariance untouched), a one-beam member and map_without_matching
    sessions (also straight after a match) over three groups of the same handles in different session orders."""
    from hector_slam_b200 import capi

    M, steps = 6, 18
    projs = [member_proj(s) for s in range(M - 1)] + [dict(member_proj(0), n_beams=1, angle_min=0.3)]
    data = [session_data(20 + s, steps, projs[s]) for s in range(M)]
    grp_reps = [make_rep(s, projs[s]) for s in range(M)]
    one_reps = [make_rep(s, projs[s]) for s in range(M)]
    rng = np.random.default_rng(4)
    orders = [list(range(M)), list(range(M))[::-1], [int(x) for x in rng.permutation(M)]]
    groups = [capi.SlamGroup([grp_reps[s] for s in o]) for o in orders]
    covs = {s: np.full((3, 3), 7.0, F32) for s in range(M)}
    covs_one = {s: c.copy() for s, c in covs.items()}
    kinds_seen, prev_matched = set(), np.zeros(M, bool)
    for k in range(steps):
        kind = rng.choice(["match", "match", "dropped", "without"], M)
        if k == 0:
            kind[:] = "match"
        if k == 1:
            kind[0] = "without"
        order = orders[k % 3]
        hints, ranges, mwm, cin = [], [], [], []
        for s in order:
            r = data[s]["ranges"][k].copy()
            if kind[s] == "dropped":
                r[:] = F32(projs[s]["range_min"]) * F32(0.5)
            hints.append(data[s]["truth"][k] if kind[s] == "without" else data[s]["hints"][k])
            ranges.append(r)
            mwm.append(kind[s] == "without")
            cin.append(covs[s])
            if kind[s] == "without" and prev_matched[s]:
                kinds_seen.add("without-after-match")
            kinds_seen.add(str(kind[s]))
        P, Cv, U, K = groups[k % 3].slam_update_projected(np.stack(hints), ranges, map_without_matching=mwm,
                                                          cov_inout=np.stack(cin))
        single = []
        for i, s in enumerate(order):
            single.append(one_reps[s].slam_update_projected(hints[i], ranges[i], map_without_matching=mwm[i],
                                                            cov_inout=covs_one[s]))
            if kind[s] == "dropped":
                assert K[i] == 0 and same(P[i], hints[i]) and same(Cv[i], covs[s]), (k, s)
        assert_same_step((P, Cv, U, K), single, k)
        for i, s in enumerate(order):
            covs[s], covs_one[s] = Cv[i], single[i][1]
            prev_matched[s] = kind[s] == "match"
    assert {"match", "dropped", "without", "without-after-match"} <= kinds_seen, kinds_seen
    for s in range(M):
        assert_same_state(grp_reps[s], one_reps[s], s)
    close_all(groups, grp_reps, one_reps)


def test_mixing_with_other_calls_without_synchronisation(hsb_lib):
    """Between nowait group projected steps the same members take group cloud steps, single steps of the other kinds, a
    projection change between two nowait steps, torch-stream batch cloud matches and downloads, with no caller
    synchronisation.  Everything equals the same sequence driven by single calls."""
    import torch

    from hector_slam_b200 import capi

    M, steps = 4, 14
    data = [session_data(60 + s, steps, member_proj(s)) for s in range(M)]
    grp_reps = [make_rep(s) for s in range(M)]
    one_reps = [make_rep(s) for s in range(M)]
    projs = [member_proj(s) for s in range(M)]
    group = capi.SlamGroup(grp_reps)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)

    def batch(rep, hint, cloud):
        d_h = torch.from_numpy(np.repeat(hint[None], 4, axis=0)).to(dev)
        d_p = torch.from_numpy(np.tile(cloud, (4, 1))).to(dev)
        d_o = torch.from_numpy((np.arange(5) * cloud.shape[0]).astype(np.int32)).to(dev)
        poses = torch.zeros((4, 3), dtype=torch.float32, device=dev)
        torch.cuda.current_stream(dev).synchronize()
        rep.match_batch_cloud_device(4, d_h.data_ptr(), d_p.data_ptr(), d_o.data_ptr(), cloud.shape[0], None,
                                     poses.data_ptr(), None, None, stream.cuda_stream)
        with torch.cuda.stream(stream):
            return poses.cpu().numpy()

    for k in range(steps):
        hints = np.stack([d["hints"][k] for d in data])
        rs = [d["ranges"][k] for d in data]
        if k % 4 == 1:
            out = group.slam_update_cloud(hints, [project(rs[s], projs[s]) for s in range(M)], nowait=True)
            assert_same_step(out, [one_reps[s].slam_update_cloud(hints[s], project(rs[s], projs[s])) for s in range(M)], k)
        else:
            out = group.slam_update_projected(hints, rs, nowait=True)
            assert_same_step(out, [one_reps[s].slam_update_projected(hints[s], rs[s]) for s in range(M)], k)
        if k % 4 == 2:
            x = grp_reps[0].slam_update_projected(data[0]["truth"][k], rs[0], nowait=True)
            y = one_reps[0].slam_update_projected(data[0]["truth"][k], rs[0])
            assert all(same(u, v) for u, v in zip(x[:2], y[:2])) and x[2:] == y[2:], k
            x = grp_reps[1].slam_update_cloud(data[1]["truth"][k], project(rs[1], projs[1]), nowait=True)
            y = one_reps[1].slam_update_cloud(data[1]["truth"][k], project(rs[1], projs[1]))
            assert all(same(u, v) for u, v in zip(x[:2], y[:2])) and x[2:] == y[2:], k
        if k == 8:   # between two nowait group steps: read at the next step's conversion
            projs[3] = dict(projs[3], angle_min=projs[3]["angle_min"] + 0.01, range_cutoff=5.0)
            for r in (grp_reps[3], one_reps[3]):
                r.set_laser_projection(**projs[3])
        if k % 3 == 2:
            c = project(rs[2], projs[2])
            assert np.array_equal(batch(grp_reps[2], data[2]["hints"][k], c), batch(one_reps[2], data[2]["hints"][k], c)), k
        if k % 4 == 3:
            assert np.array_equal(grp_reps[3].download_occupancy(0), one_reps[3].download_occupancy(0)), k
    for s in range(M):
        assert_same_state(grp_reps[s], one_reps[s], s)
    group.close()
    close_all(grp_reps, one_reps)


def test_validation_leaves_every_member_unchanged(hsb_lib):
    """No projection, no cloud format, offsets that disagree with n_beams and a scan past the staging limit are each
    rejected before any member changes; the next step (map_without_matching everywhere, so the coarse levels write
    the containers the members hold) still equals the single-call twins.  A tuning without a projected kernel fails."""
    from hector_slam_b200 import capi

    M, steps = 3, 12
    data = [session_data(150 + s, steps, member_proj(s)) for s in range(M)]
    grp_reps = [make_rep(s, with_proj=(s != 1), with_cloud=(s != 2)) for s in range(M)]
    one_reps = [make_rep(s) for s in range(M)]
    group = capi.SlamGroup(grp_reps)
    step_no = [0]

    def valid_step(without):
        k = step_no[0]
        step_no[0] += 1
        hints = np.stack([d["truth" if without else "hints"][k] for d in data])
        out = group.slam_update_projected(hints, [d["ranges"][k] for d in data], map_without_matching=[without] * M,
                                          nowait=(k % 2 == 1))
        single = [one_reps[s].slam_update_projected(hints[s], data[s]["ranges"][k], map_without_matching=without)
                  for s in range(M)]
        assert_same_step(out, single, k)

    def rejected(status, texts, ranges):
        hints = np.stack([d["hints"][step_no[0]] for d in data])
        with pytest.raises(capi.HsbError) as e:
            group.slam_update_projected(hints, ranges)
        assert e.value.status == status and all(t in str(e.value) for t in texts), str(e.value)
        return str(e.value)

    ranges = [d["ranges"][0] for d in data]
    rejected(-1, ["session 1", "hsb_set_laser_projection"], ranges)
    grp_reps[1].set_laser_projection(**member_proj(1))
    rejected(-1, ["session 2", "hsb_set_cloud_format"], ranges)
    grp_reps[2].set_cloud_format(member_transform(2), **member_cloud(2))
    with pytest.raises(capi.HsbError) as e:
        make_rep(0, with_cloud=False).slam_update_projected(data[0]["hints"][0], ranges[0])
    assert e.value.status == -1 and "hsb_set_cloud_format" in str(e.value)
    valid_step(False)
    valid_step(False)

    n = [r.shape[0] for r in ranges]
    flat = np.concatenate(ranges)
    for offs in ([0, n[0], n[0] - 1, flat.shape[0]], [0, n[0] + 1, n[0] + n[1], flat.shape[0]],
                 [0, n[0], n[0] + n[1], flat.shape[0] - 1]):
        rejected(-1, ["offsets" if offs[2] < offs[1] else "beams"], (flat, np.array(offs, np.int32)))
    valid_step(True)
    valid_step(False)

    for bad in (ranges[0][:-1], np.concatenate([ranges[0], ranges[0][:1]])):
        with pytest.raises(capi.HsbError) as e:
            grp_reps[0].slam_update_projected(data[0]["hints"][0], bad)
        assert e.value.status == -1 and "beams" in str(e.value), str(e.value)
    valid_step(True)

    big = dict(member_proj(0), n_beams=LIMIT + 1, angle_increment=float(F32(1e-4)))
    grp_reps[0].set_laser_projection(**big)
    msg = rejected(-5, ["scan too long for the fused conversion (%d points)" % (LIMIT + 1)],
                   [np.full(LIMIT + 1, 3.0, F32), ranges[1], ranges[2]])
    probe = make_rep(0, big)
    with pytest.raises(capi.HsbError) as e:
        probe.slam_update_projected(data[0]["hints"][0], np.full(LIMIT + 1, 3.0, F32))
    assert e.value.status == -5 and str(e.value) == msg
    probe.set_laser_projection(**member_proj(0))
    nan, inf = float("nan"), float("inf")
    for bad in (dict(angle_min=nan), dict(angle_increment=inf), dict(range_min=-inf), dict(range_cutoff=nan),
                dict(range_cutoff=-1.0, range_max=nan), dict(n_beams=0)):
        with pytest.raises(capi.HsbError) as e:
            probe.set_laser_projection(**dict(member_proj(0), **bad))
        assert e.value.status == -1, bad
    # a rejected projection leaves the previous one: the step still runs with it
    assert probe.slam_update_projected(data[0]["hints"][0], ranges[0])[3] > 0
    probe.set_tuning(warps_per_scan=4)
    with pytest.raises(capi.HsbError) as e:
        probe.slam_update_projected(data[0]["hints"][0], ranges[0])
    assert e.value.status == -5 and "tuning" in str(e.value)
    probe.close()
    grp_reps[0].set_laser_projection(**member_proj(0))
    valid_step(True)
    valid_step(False)
    for s in range(M):
        assert_same_state(grp_reps[s], one_reps[s], s)
    group.close()
    close_all(grp_reps, one_reps)


@pytest.mark.parametrize("M", [1, 16])
def test_launch_count(hsb_lib, M):
    """A single projected step is three launches (also without matching); a group step is three launches counted on
    handles[0], and the other members' counts do not move."""
    from hector_slam_b200 import capi

    reps = [make_rep(s) for s in range(M)]
    data = [session_data(90 + s, 4, member_proj(s)) for s in range(M)]
    before = reps[0].launch_count
    reps[0].slam_update_projected(data[0]["hints"][0], data[0]["ranges"][0])
    reps[0].slam_update_projected(data[0]["hints"][0], data[0]["ranges"][0], nowait=True)
    reps[0].slam_update_projected(data[0]["truth"][0], data[0]["ranges"][0], map_without_matching=True)
    assert reps[0].launch_count - before == 3 + 3 + 5   # without matching: conversion, gate, publish + the map write
    group = capi.SlamGroup(reps)
    for k in range(1, 4):
        before = [r.launch_count for r in reps]
        group.slam_update_projected(np.stack([d["hints"][k] for d in data]), [d["ranges"][k] for d in data],
                                    map_without_matching=[k == 3 and s % 2 == 0 for s in range(M)], nowait=(k == 2))
        after = [r.launch_count for r in reps]
        assert after[0] - before[0] == 3, (k, before[0], after[0])
        assert after[1:] == before[1:], k
    group.close()
    close_all(reps)


def test_facade_update_projected_and_update_many_projected(hsb_lib):
    """hsb200::SlamProcessor::updateManyProjected and updateProjected (C++ façade, through its shim) equal each other
    and hsb_slam_update_projected on a third processor's handle: poses, covariances, kept counts and maps."""
    L = C.CDLL(os.path.join(ROOT, "hector_slam_b200", "lib", "libhsb200_host.so"))
    lib = hsb_lib
    vp, i, f, d = C.c_void_p, C.c_int, C.c_float, C.c_double
    L.hsbp_create.restype = vp
    L.hsbp_create.argtypes = [f, i, i, f, f, i, i]
    L.hsbp_destroy.argtypes = [vp]
    L.hsbp_handle.restype = vp
    L.hsbp_handle.argtypes = [vp]
    L.hsbp_set_laser_projection.argtypes = [vp, i, f, f, f, f, d]
    L.hsbp_set_cloud_format.argtypes = [vp, vp, f, f, f, f]
    L.hsbp_set_map_update_thresholds.argtypes = [vp, f, f]
    L.hsbp_update_projected.argtypes = [vp, vp, i, vp, vp, i, vp]
    L.hsbp_update_many_projected.argtypes = [vp, i, vp, vp, vp, vp, vp, vp]
    L.hsbp_get_pose_and_cov.argtypes = [vp, vp, vp]
    L.hsbp_get_grid_map.argtypes = [vp, i, vp]
    M, steps = 3, 8
    data = [session_data(110 + s, steps, member_proj(s)) for s in range(M)]
    sets = [[L.hsbp_create(RES, SIZE, SIZE, 0.5, 0.5, LEVELS, 0) for _ in range(M)] for _ in range(3)]
    many, one, capi_ps = sets
    assert all(all(x) for x in sets)
    for s in range(M):
        pj, cf, T = member_proj(s), member_cloud(s), np.ascontiguousarray(member_transform(s), np.float64)
        for p in (many[s], one[s], capi_ps[s]):
            assert L.hsbp_set_laser_projection(p, pj["n_beams"], pj["angle_min"], pj["angle_increment"], pj["range_min"],
                                               pj["range_max"], pj["range_cutoff"]) == 0
            assert L.hsbp_set_cloud_format(p, T.ctypes.data, cf["sqr_laser_min_dist"], cf["sqr_laser_max_dist"],
                                           cf["laser_z_min_value"], cf["laser_z_max_value"]) == 0
            L.hsbp_set_map_update_thresholds(p, (0.0, 0.15, 0.3)[s], (0.0, 0.1, 0.5)[s])
    arr = (C.c_void_p * M)(*many)
    cov3 = {s: np.zeros(9, F32) for s in range(M)}
    for k in range(steps):
        rs = [dd["ranges"][k] for dd in data]
        flat = np.ascontiguousarray(np.concatenate(rs), F32)
        offs = np.zeros(M + 1, np.int32)
        offs[1:] = np.cumsum([x.shape[0] for x in rs])
        hints = np.ascontiguousarray(np.stack([dd["hints"][k] for dd in data]), F32)
        Ts = np.ascontiguousarray(np.stack([member_transform(s + k) for s in range(M)]), np.float64)
        use_T = k % 2 == 1
        mwm = np.array([0, int(k % 3 == 2), 0], np.int32)
        kept = np.zeros(M, np.int32)
        assert L.hsbp_update_many_projected(C.cast(arr, C.c_void_p), M, flat.ctypes.data, offs.ctypes.data,
                                            Ts.ctypes.data if use_T else None, hints.ctypes.data, mwm.ctypes.data,
                                            kept.ctypes.data) == 0
        for s in range(M):
            p1, c1, p2, c2 = np.zeros(3, F32), np.zeros(9, F32), np.zeros(3, F32), np.zeros(9, F32)
            Tp = Ts[s].ctypes.data if use_T else None
            k1 = C.c_int(-1)
            assert L.hsbp_update_projected(one[s], rs[s].ctypes.data, rs[s].shape[0], Tp, hints[s].ctypes.data,
                                           int(mwm[s]), C.byref(k1)) == 0
            p3, upd, k3 = np.zeros(3, F32), C.c_int(0), C.c_int(-1)
            assert lib.hsb_slam_update_projected(L.hsbp_handle(capi_ps[s]), hints[s].ctypes.data, rs[s].ctypes.data,
                                                 rs[s].shape[0], Tp, int(mwm[s]), 0, p3.ctypes.data, cov3[s].ctypes.data,
                                                 C.addressof(upd), C.addressof(k3)) == 0
            L.hsbp_get_pose_and_cov(many[s], p1.ctypes.data, c1.ctypes.data)
            L.hsbp_get_pose_and_cov(one[s], p2.ctypes.data, c2.ctypes.data)
            assert same(p1, p2) and same(c1, c2) and kept[s] == k1.value, (k, s)
            assert same(p1, p3) and same(c1, cov3[s]) and k3.value == k1.value, (k, s)
    for s in range(M):
        for l in range(LEVELS):
            sz = SIZE >> l
            x, y, z = (np.zeros((sz, sz), F32) for _ in range(3))
            assert L.hsbp_get_grid_map(many[s], l, x.ctypes.data) == 0
            assert L.hsbp_get_grid_map(one[s], l, y.ctypes.data) == 0
            assert L.hsbp_get_grid_map(capi_ps[s], l, z.ctypes.data) == 0
            assert np.array_equal(x, y) and np.array_equal(x, z), (s, l)
    for p in many + one + capi_ps:
        L.hsbp_destroy(p)
