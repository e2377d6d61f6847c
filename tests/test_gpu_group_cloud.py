"""hsb_group_slam_update_cloud — the group SLAM step from the node's default input (projected point clouds, converted in
the group's match kernel) — against the same sessions stepped one by one with hsb_slam_update_cloud on twin handles:
bit-identical poses, covariances, gate decisions, kept counts, planes and handle state.  Every member has its own cloud
format (laser transform, distance window, z window), update factors and gate thresholds, so a session that read another
member's settings would differ.  Also: edge sessions in permuted groups, the oracle's converter and the two-call path,
mixing with other calls without synchronisation, M = 1 and nowait, validation, launch accounting and the C++ façade."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import ROOT

pytestmark = pytest.mark.gpu

RES, SIZE, LEVELS = 0.05, 512, 3
SCALE = 1.0 / RES


def member_transform(s, k=None):
    """Laser transform of member s (its cloud format's), or the per-scan one of step k."""
    from hector_slam_b200 import synth

    j = s if k is None else s + 7 * k + 3
    return synth.laser_transform(xyz=(0.04 * (j % 4), -0.03 * (j % 3), 0.2 + 0.05 * (j % 2)),
                                 rpy=(0.01 * (j % 3), -0.012 * (j % 2), 0.02 * (j % 5)))


def member_format(s):
    """Member s's distance and z windows (floats as the node stores them)."""
    d_min, d_max = (0.3, 0.45, 0.6)[s % 3], (9.0, 12.0, 30.0, 6.0)[s % 4]
    z = (1.0, 0.09, 0.15)[s % 3]   # the tilted lasers see far points leave a narrow z window
    return dict(sqr_laser_min_dist=float(np.float32(d_min * d_min)), sqr_laser_max_dist=float(np.float32(d_max * d_max)),
                laser_z_min_value=-z, laser_z_max_value=z)


def session_data(seed, steps):
    """A trajectory through its own synthetic room: per step the projected cloud (laser frame), the level-0 endpoints
    of the same ranges, the true pose and a noisy hint."""
    from hector_slam_b200 import synth

    rng = np.random.default_rng(seed)
    world = synth.World(1, seed=1000 + seed)
    x, y, a = rng.uniform(-2, 2), rng.uniform(-1.5, 1.5), rng.uniform(-3, 3)
    truth, clouds, scans = [], [], []
    for _ in range(steps):
        p = np.array([x, y, a], np.float32)
        truth.append(p)
        r = world.cast(p) + rng.normal(0.0, 0.01, 1081)
        clouds.append(np.ascontiguousarray(synth.ranges_to_cloud(r), np.float32))
        scans.append(np.ascontiguousarray(synth.ranges_to_points(r, SCALE), np.float32))
        a += rng.uniform(-0.08, 0.08)
        step = rng.uniform(0.03, 0.12)
        x = float(np.clip(x + step * np.cos(a), -6.0, 6.0))
        y = float(np.clip(y + step * np.sin(a), -4.0, 4.0))
    truth = np.asarray(truth, np.float32)
    hints = truth + rng.uniform(-1, 1, truth.shape).astype(np.float32) * np.array([0.04, 0.04, 0.02], np.float32)
    return dict(truth=truth, clouds=clouds, scans=scans, hints=hints.astype(np.float32))


def make_rep(s, cloud_format=True, **kw):
    """Handle of member s: update factors, gate thresholds and cloud format differ between members."""
    from hector_slam_b200 import capi

    rep = capi.MapRepB200(RES, SIZE, levels=LEVELS, update_factor_free=0.4 + 0.02 * (s % 3),
                          update_factor_occupied=0.6 + 0.1 * (s % 4), **kw)
    dist, ang = ((0.0, 0.0), (0.15, 0.1), (0.3, 0.5))[s % 3]
    rep.setMapUpdateMinDistDiff(dist)
    rep.setMapUpdateMinAngleDiff(ang)
    if cloud_format:
        rep.set_cloud_format(member_transform(s), **member_format(s))
    return rep


def assert_same_state(a, b, tag):
    """Planes, probability planes, gate pose and both dirty rectangles of every level."""
    for l in range(LEVELS):
        assert np.array_equal(a.download_level(l), b.download_level(l)), (tag, l)
        assert np.array_equal(a.download_prob(l), b.download_prob(l)), (tag, l)
        assert a.get_mirror_dirty_rect(l) == b.get_mirror_dirty_rect(l), (tag, l)
    assert a.get_dirty_rects() == b.get_dirty_rects(), tag
    assert np.array_equal(a.last_map_update_pose(), b.last_map_update_pose()), tag


def assert_same_step(group_out, single_outs, tag):
    P, Cv, U, K = group_out
    for i, (p, c, u, kept) in enumerate(single_outs):
        assert np.array_equal(P[i], p), (tag, i, P[i], p)
        assert np.array_equal(Cv[i], c), (tag, i)
        assert U[i] == u, (tag, i)
        assert K[i] == kept, (tag, i, K[i], kept)


def close_all(*groups):
    for g in groups:
        for x in (g if isinstance(g, (list, tuple)) else [g]):
            x.close()


def test_group_cloud_step_equals_single_cloud_steps(hsb_lib):
    """12 members, 40 steps, per-scan transforms on every other step: every pose, covariance, gate decision and kept
    count and the final handle state equal twin handles stepped with hsb_slam_update_cloud in the (8, 1, 4) shape."""
    from hector_slam_b200 import capi

    M, steps = 12, 40
    data = [session_data(s, steps) for s in range(M)]
    grp_reps = [make_rep(s) for s in range(M)]
    one_reps = [make_rep(s) for s in range(M)]
    group = capi.SlamGroup(grp_reps)
    fired = np.zeros(2, int)
    for k in range(steps):
        hints = np.stack([d["hints"][k] for d in data])
        Ts = np.stack([member_transform(s, k) for s in range(M)]) if k % 2 else None
        out = group.slam_update_cloud(hints, [d["clouds"][k] for d in data], transforms=Ts)
        single = []
        for s in range(M):
            single.append(one_reps[s].slam_update_cloud(hints[s], data[s]["clouds"][k],
                                                        transform=None if Ts is None else Ts[s]))
            shape = one_reps[s].last_launch_shape()
            assert (shape["warps_per_scan"], shape["scans_per_block"], shape["unroll"]) == (8, 1, 4), shape
        assert_same_step(out, single, k)
        for s in range(M):
            fired[int(out[2][s])] += 1
    assert fired[0] > 0 and fired[1] > 0, fired   # the gate both fires and holds back
    for s in range(M):
        assert_same_state(grp_reps[s], one_reps[s], s)
    group.close()
    close_all(grp_reps, one_reps)


def test_edge_sessions_in_permuted_groups(hsb_lib):
    """Empty clouds, clouds whose every point is filtered out (kept 0: pose = hint, covariance untouched), clouds
    thinned by the z window, map_without_matching (also straight after a matched step: the coarse levels then write the
    last MATCHED scan), over three groups of the same handles in different session orders."""
    from hector_slam_b200 import capi

    M, steps = 6, 18
    data = [session_data(20 + s, steps) for s in range(M)]
    grp_reps = [make_rep(s) for s in range(M)]
    one_reps = [make_rep(s) for s in range(M)]
    rng = np.random.default_rng(4)
    orders = [list(range(M)), list(range(M))[::-1], [int(x) for x in rng.permutation(M)]]
    groups = [capi.SlamGroup([grp_reps[s] for s in o]) for o in orders]
    covs = {s: np.full((3, 3), 7.0, np.float32) for s in range(M)}
    covs_one = {s: c.copy() for s, c in covs.items()}
    kinds_seen = set()
    prev_matched = np.zeros(M, bool)
    for k in range(steps):
        kind = rng.choice(["match", "match", "empty", "filtered", "zthin", "without"], M)
        if k == 0:
            kind[:] = "match"
        if k == 1:
            kind[0] = "without"   # straight after a matched step
        order = orders[k % 3]
        hints, clouds, mwm, cin = [], [], [], []
        for s in order:
            cloud = data[s]["clouds"][k].copy()
            if kind[s] == "empty":
                cloud = np.zeros((0, 3), np.float32)
            elif kind[s] == "filtered":
                cloud[:, :2] *= np.float32(0.001)   # every point inside the minimum distance
            elif kind[s] == "zthin":
                cloud[::3, 2] = 5.0                 # a third leaves the z window
            hints.append(data[s]["truth"][k] if kind[s] == "without" else data[s]["hints"][k])
            clouds.append(cloud)
            mwm.append(kind[s] == "without")
            cin.append(covs[s])
            if kind[s] == "without" and prev_matched[s]:
                kinds_seen.add("without-after-match")
            kinds_seen.add(str(kind[s]))
        P, Cv, U, K = groups[k % 3].slam_update_cloud(np.stack(hints), clouds, map_without_matching=mwm,
                                                       cov_inout=np.stack(cin))
        single = []
        for i, s in enumerate(order):
            single.append(one_reps[s].slam_update_cloud(hints[i], clouds[i], map_without_matching=mwm[i],
                                                        cov_inout=covs_one[s]))
            if kind[s] == "filtered":
                assert K[i] == 0 and clouds[i].shape[0] > 0, (k, s)
                assert np.array_equal(P[i], hints[i]) and np.array_equal(Cv[i], covs[s]), (k, s)
            if kind[s] == "zthin":
                assert 0 < K[i] < clouds[i].shape[0], (k, s)
        assert_same_step((P, Cv, U, K), single, k)
        for i, s in enumerate(order):
            covs[s], covs_one[s] = Cv[i], single[i][1]
            prev_matched[s] = kind[s] in ("match", "zthin")
    assert {"match", "empty", "filtered", "zthin", "without", "without-after-match"} <= kinds_seen, kinds_seen
    for s in range(M):
        assert_same_state(grp_reps[s], one_reps[s], s)
    close_all(groups, grp_reps, one_reps)


def test_against_oracle_converter_and_two_call_path(hsb_lib, pyoracle, oracle_kinds):
    """Every kept count equals the node's compiled converter's (pyoracle.cloud_to_points); twins driven by that
    conversion + hsb_slam_update with its origo give the same poses and end with identical planes."""
    from hector_slam_b200 import capi

    kind = "reference" if "reference" in oracle_kinds else "port"
    M, steps = 5, 12
    data = [session_data(130 + s, steps) for s in range(M)]
    grp_reps = [make_rep(s) for s in range(M)]
    two_reps = [make_rep(s) for s in range(M)]
    group = capi.SlamGroup(grp_reps)
    scale = grp_reps[0].getScaleToMap()
    foreign = 0   # sessions whose count under member 0's format differs from their own
    for k in range(steps):
        hints = np.stack([d["hints"][k] for d in data])
        Ts = np.stack([member_transform(s, k) for s in range(M)]) if k % 3 == 1 else None
        mwm = [k % 5 == 4 and s % 2 == 0 for s in range(M)]
        P, _, U, K = group.slam_update_cloud(hints, [d["clouds"][k] for d in data], transforms=Ts,
                                             map_without_matching=mwm)
        for s in range(M):
            T = member_transform(s) if Ts is None else Ts[s]
            f = member_format(s)
            pts, origo = pyoracle.cloud_to_points(data[s]["clouds"][k], T, f["sqr_laser_min_dist"], f["sqr_laser_max_dist"],
                                                  f["laser_z_min_value"], f["laser_z_max_value"], scale, kind=kind)
            assert K[s] == pts.shape[0], (k, s, K[s], pts.shape[0])
            f0 = member_format(0)
            other, _ = pyoracle.cloud_to_points(data[s]["clouds"][k], member_transform(0), f0["sqr_laser_min_dist"],
                                                f0["sqr_laser_max_dist"], f0["laser_z_min_value"], f0["laser_z_max_value"],
                                                scale, kind=kind)
            foreign += other.shape[0] != pts.shape[0]
            p, _, u = two_reps[s].slam_update(hints[s], pts, map_without_matching=mwm[s], origo=origo)
            assert np.array_equal(P[s], p) and U[s] == u, (k, s)
    assert foreign >= steps, foreign   # the members' formats differ in effect
    for s in range(M):
        for l in range(LEVELS):
            assert np.array_equal(grp_reps[s].download_level(l), two_reps[s].download_level(l)), (s, l)
    group.close()
    close_all(grp_reps, two_reps)


def test_mixing_with_other_calls_without_synchronisation(hsb_lib):
    """Between nowait group cloud steps the same members take group endpoint steps, single hsb_slam_update and
    hsb_slam_update_cloud steps, a reset, a change of cloud format, torch-stream batch matches and occupancy downloads,
    with no synchronisation by the caller.  Everything equals the same sequence driven only by single calls."""
    import torch

    from hector_slam_b200 import capi

    M, steps = 4, 16
    data = [session_data(60 + s, steps) for s in range(M)]
    grp_reps = [make_rep(s) for s in range(M)]
    one_reps = [make_rep(s) for s in range(M)]
    group = capi.SlamGroup(grp_reps)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)

    def batch(rep, hint, scan):
        d_h = torch.from_numpy(np.repeat(hint[None], 8, axis=0)).to(dev)
        d_p = torch.from_numpy(scan).to(dev)
        poses = torch.zeros((8, 3), dtype=torch.float32, device=dev)
        torch.cuda.current_stream(dev).synchronize()   # the inputs are on the device
        rep.match_batch_device(8, d_h.data_ptr(), d_p.data_ptr(), None, scan.shape[0], scan.shape[0], poses.data_ptr(),
                               None, stream.cuda_stream)
        with torch.cuda.stream(stream):
            return poses.cpu().numpy()   # reads the results: waits for this stream only

    for k in range(steps):
        hints = np.stack([d["hints"][k] for d in data])
        if k % 4 == 1:   # a group endpoint step on the same members
            P, Cv, U = group.slam_update(hints, [d["scans"][k] for d in data], nowait=True)
            for s in range(M):
                p, c, u = one_reps[s].slam_update(hints[s], data[s]["scans"][k])
                assert np.array_equal(P[s], p) and np.array_equal(Cv[s], c) and U[s] == u, (k, s)
        else:
            out = group.slam_update_cloud(hints, [d["clouds"][k] for d in data], nowait=True)
            assert_same_step(out, [one_reps[s].slam_update_cloud(hints[s], data[s]["clouds"][k]) for s in range(M)], k)
        if k % 4 == 2:   # single steps of both kinds on members right after the group step
            h = data[0]["truth"][k]
            x = grp_reps[0].slam_update(h, data[0]["scans"][k], nowait=True)
            y = one_reps[0].slam_update(h, data[0]["scans"][k])
            assert all(np.array_equal(u, v) for u, v in zip(x, y)), k
            x = grp_reps[1].slam_update_cloud(data[1]["truth"][k], data[1]["clouds"][k], nowait=True)
            y = one_reps[1].slam_update_cloud(data[1]["truth"][k], data[1]["clouds"][k])
            assert all(np.array_equal(u, v) for u, v in zip(x, y)), k
        if k == 6:
            grp_reps[2].reset()
            one_reps[2].reset()
        if k == 8:   # read at the next step's conversion
            for r in (grp_reps[3], one_reps[3]):
                r.set_cloud_format(member_transform(3, 99), **member_format(4))
        if k % 3 == 2:
            assert np.array_equal(batch(grp_reps[2], data[2]["hints"][k], data[2]["scans"][k]),
                                  batch(one_reps[2], data[2]["hints"][k], data[2]["scans"][k])), k
        if k % 4 == 3:
            assert np.array_equal(grp_reps[3].download_occupancy(0), one_reps[3].download_occupancy(0)), k
    for s in range(M):
        assert_same_state(grp_reps[s], one_reps[s], s)
    group.close()
    close_all(grp_reps, one_reps)


def test_single_member_group_and_nowait(hsb_lib):
    """M = 1 equals hsb_slam_update_cloud bit for bit; nowait = 1 equals nowait = 0 for a 5-member group, with
    hsb_on_map_updated of each member as the completion point before the planes are read."""
    from hector_slam_b200 import capi

    steps = 14
    d = session_data(77, steps)
    a, b = make_rep(1), make_rep(1)
    ga = capi.SlamGroup([a])
    for k in range(steps):
        out = ga.slam_update_cloud(d["hints"][k][None], [d["clouds"][k]], map_without_matching=[k == 5])
        assert_same_step(out, [b.slam_update_cloud(d["hints"][k], d["clouds"][k], map_without_matching=(k == 5))], k)
    assert_same_state(a, b, "M=1")
    ga.close()
    close_all([a, b])

    M = 5
    data = [session_data(40 + s, steps) for s in range(M)]

    def run(nowait):
        reps = [make_rep(s) for s in range(M)]
        grp = capi.SlamGroup(reps)
        out = []
        for k in range(steps):
            out.append(grp.slam_update_cloud(np.stack([x["hints"][k] for x in data]), [x["clouds"][k] for x in data],
                                             map_without_matching=[k % 6 == 5] * M, nowait=nowait))
        for r in reps:
            r.onMapUpdated()
        planes = [[r.download_level(l) for l in range(LEVELS)] for r in reps]
        grp.close()
        return out, planes, reps

    (oa, pa, ra), (ob, pb, rb) = run(False), run(True)
    for k in range(steps):
        for x, y in zip(oa[k], ob[k]):
            assert np.array_equal(x, y), k
    for s in range(M):
        for l in range(LEVELS):
            assert np.array_equal(pa[s][l], pb[s][l]), (s, l)
        assert_same_state(ra[s], rb[s], s)
    close_all(ra, rb)




def test_validation_leaves_every_member_unchanged(hsb_lib):
    """A member without a cloud format, bad offsets and an oversize cloud are rejected before any member changes.  The
    step after each rejection is map_without_matching everywhere, so its coarse levels write the last-match container
    the members hold: it still equals the single-call twins, and the group keeps working."""
    from hector_slam_b200 import capi

    M, steps = 3, 8
    data = [session_data(150 + s, steps) for s in range(M)]
    grp_reps = [make_rep(s, cloud_format=(s != 1)) for s in range(M)]
    one_reps = [make_rep(s) for s in range(M)]
    group = capi.SlamGroup(grp_reps)
    step_no = [0]

    def valid_step(without):
        k = step_no[0]
        step_no[0] += 1
        hints = np.stack([d["truth" if without else "hints"][k] for d in data])
        out = group.slam_update_cloud(hints, [d["clouds"][k] for d in data], map_without_matching=[without] * M,
                                      nowait=(k % 2 == 1))
        single = [one_reps[s].slam_update_cloud(hints[s], data[s]["clouds"][k], map_without_matching=without)
                  for s in range(M)]
        assert_same_step(out, single, k)

    def rejected(status, text, clouds):
        hints = np.stack([d["hints"][step_no[0]] for d in data])
        with pytest.raises(capi.HsbError) as e:
            group.slam_update_cloud(hints, clouds)
        assert e.value.status == status and text in str(e.value), str(e.value)
        return str(e.value)

    clouds = [d["clouds"][0] for d in data]
    rejected(-1, "session 1", clouds)   # member 1 has no cloud format
    grp_reps[1].set_cloud_format(member_transform(1), **member_format(1))
    valid_step(False)
    valid_step(False)

    n = [c.shape[0] for c in clouds]
    pts = np.concatenate(clouds)
    for offs in ([1, n[0], n[0] + n[1], pts.shape[0]], [0, n[0], n[0] - 1, pts.shape[0]],
                 [0, n[0] + n[1], n[0], pts.shape[0]]):
        rejected(-1, "offsets", (pts, np.array(offs, np.int32)))
    valid_step(True)
    valid_step(False)

    big = np.ascontiguousarray(np.tile(clouds[0], (40, 1))[:30000])
    msg = rejected(-5, "scan too long for the fused conversion (30000 points)", [big, clouds[1], clouds[2]])
    probe = make_rep(0)   # the single call's limit and wording (on a handle of its own: its state is not compared)
    with pytest.raises(capi.HsbError) as e:
        probe.slam_update_cloud(data[0]["hints"][0], big)
    assert e.value.status == -5 and str(e.value) == msg
    probe.close()
    valid_step(True)
    valid_step(False)
    for s in range(M):
        assert_same_state(grp_reps[s], one_reps[s], s)
    group.close()
    close_all(grp_reps, one_reps)


@pytest.mark.parametrize("M", [1, 16])
def test_launch_count(hsb_lib, M):
    """A group cloud step is three launches, counted on handles[0], also with map_without_matching sessions; the other
    members' counts do not move."""
    from hector_slam_b200 import capi

    reps = [make_rep(s) for s in range(M)]
    group = capi.SlamGroup(reps)
    data = [session_data(90 + s, 3) for s in range(M)]
    for k in range(3):
        before = [r.launch_count for r in reps]
        group.slam_update_cloud(np.stack([d["hints"][k] for d in data]), [d["clouds"][k] for d in data],
                                map_without_matching=[k == 2 and s % 2 == 0 for s in range(M)], nowait=(k == 1))
        after = [r.launch_count for r in reps]
        assert after[0] - before[0] == 3, (k, before[0], after[0])
        assert after[1:] == before[1:], k
    group.close()
    close_all(reps)


def test_facade_update_many_cloud(hsb_lib):
    """hsb200::SlamProcessor::updateManyCloud and updateCloud (C++ façade, through its shim) equal each other per
    processor — poses, covariances, kept counts and maps — with per-processor cloud formats and gate thresholds."""
    L = C.CDLL(os.path.join(ROOT, "hector_slam_b200", "lib", "libhsb200_host.so"))
    vp, i, f = C.c_void_p, C.c_int, C.c_float
    L.hsbp_create.restype = vp
    L.hsbp_create.argtypes = [f, i, i, f, f, i, i]
    L.hsbp_destroy.argtypes = [vp]
    L.hsbp_set_cloud_format.argtypes = [vp, vp, f, f, f, f]
    L.hsbp_set_map_update_thresholds.argtypes = [vp, f, f]
    L.hsbp_update_cloud.argtypes = [vp, vp, i, vp, vp, i, vp]
    L.hsbp_update_many_cloud.argtypes = [vp, i, vp, vp, vp, vp, vp, vp]
    L.hsbp_get_pose_and_cov.argtypes = [vp, vp, vp]
    L.hsbp_get_grid_map.argtypes = [vp, i, vp]
    M, steps = 3, 8
    data = [session_data(110 + s, steps) for s in range(M)]
    many = [L.hsbp_create(RES, SIZE, SIZE, 0.5, 0.5, LEVELS, 0) for _ in range(M)]
    one = [L.hsbp_create(RES, SIZE, SIZE, 0.5, 0.5, LEVELS, 0) for _ in range(M)]
    assert all(many) and all(one)
    for s in range(M):
        T, fm = member_transform(s), member_format(s)
        for p in (many[s], one[s]):
            assert L.hsbp_set_cloud_format(p, T.ctypes.data, fm["sqr_laser_min_dist"], fm["sqr_laser_max_dist"],
                                           fm["laser_z_min_value"], fm["laser_z_max_value"]) == 0
            L.hsbp_set_map_update_thresholds(p, (0.0, 0.15, 0.3)[s], (0.0, 0.1, 0.5)[s])
    arr = (C.c_void_p * M)(*many)
    for k in range(steps):
        clouds = [d["clouds"][k] for d in data]
        pts = np.ascontiguousarray(np.concatenate(clouds), np.float32)
        offs = np.zeros(M + 1, np.int32)
        offs[1:] = np.cumsum([x.shape[0] for x in clouds])
        hints = np.ascontiguousarray(np.stack([d["hints"][k] for d in data]), np.float32)
        Ts = np.ascontiguousarray(np.stack([member_transform(s, k) for s in range(M)])) if k % 2 else None
        mwm = np.array([0, int(k % 3 == 2), 0], np.int32)
        kept = np.zeros(M, np.int32)
        assert L.hsbp_update_many_cloud(C.cast(arr, C.c_void_p), M, pts.ctypes.data, offs.ctypes.data,
                                        None if Ts is None else Ts.ctypes.data, hints.ctypes.data, mwm.ctypes.data,
                                        kept.ctypes.data) == 0
        for s in range(M):
            p1, c1, p2, c2 = (np.zeros(3, np.float32), np.zeros(9, np.float32), np.zeros(3, np.float32),
                              np.zeros(9, np.float32))
            k1 = C.c_int(-1)
            assert L.hsbp_update_cloud(one[s], clouds[s].ctypes.data, clouds[s].shape[0],
                                       None if Ts is None else Ts[s].ctypes.data, hints[s].ctypes.data, int(mwm[s]),
                                       C.byref(k1)) == 0
            L.hsbp_get_pose_and_cov(many[s], p1.ctypes.data, c1.ctypes.data)
            L.hsbp_get_pose_and_cov(one[s], p2.ctypes.data, c2.ctypes.data)
            assert np.array_equal(p1, p2) and np.array_equal(c1, c2) and kept[s] == k1.value, (k, s)
    for s in range(M):
        for l in range(LEVELS):
            sz = SIZE >> l
            x, y = np.zeros((sz, sz), np.float32), np.zeros((sz, sz), np.float32)
            assert L.hsbp_get_grid_map(many[s], l, x.ctypes.data) == 0
            assert L.hsbp_get_grid_map(one[s], l, y.ctypes.data) == 0
            assert np.array_equal(x, y), (s, l)
    for p in many + one:   # any member first: its cached group goes with it
        L.hsbp_destroy(p)
