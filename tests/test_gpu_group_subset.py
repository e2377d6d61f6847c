"""The group SLAM steps over a subset of the group's members (hsb_group_slam_update_subset and its _cloud, _ranges and
_projected forms): session k steps members[k], in any order, and members left out are neither read nor changed.

Against twin handles stepped with the single-handle call only when their member was selected: bit-identical poses,
covariances, gate decisions and kept counts, and bit-identical member state (every level's log-odds and probability,
the texture twin, gate pose, both dirty rectangles, the last match's container through a following updateByScan).
Also: the identity subset against the full step, unselected members untouched, ordering against nowait steps and
caller-stream batch matches, launch accounting, rejections and the C++ façade.  Every case runs on a TEX and an LDG
group.  Members differ in beam geometry, laser mount, cloud thresholds, update factors and gate thresholds."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from conftest import ROOT
from twin_probe import probe_twin

pytestmark = pytest.mark.gpu

RES, SIZE, LEVELS = 0.05, 512, 3
SCALE = 1.0 / RES
F32 = np.float32
KINDS = ("endpoints", "cloud", "ranges", "projected")
MODES = pytest.mark.parametrize("mode", [2, 1], ids=["tex", "ldg"])   # capi.GATHER_TEX, capi.GATHER_LDG

# n_beams, angle_min (deg), angle_increment (deg), range_min, range_max of the members' lasers
GEOM = [(1081, -135.0, 0.25, 0.1, 30.0), (720, -180.0, 0.5, 0.2, 12.0), (360, -120.0, 0.75, 0.3, 20.0)]


def geometry(s):
    n, a0, da, rmin, rmax = GEOM[s % 3]
    return dict(n_beams=n, angle_min=float(F32(math.radians(a0))), angle_increment=float(F32(math.radians(da))),
                range_min=float(F32(rmin)), range_max=float(F32(rmax)))


def beam_angles(g):
    """fp32 beam angles accumulated as the node accumulates them"""
    out = np.empty(g["n_beams"], F32)
    a = F32(g["angle_min"])
    for i in range(out.size):
        out[i] = a
        a = F32(a + F32(g["angle_increment"]))
    return out


def member_transform(s):
    from hector_slam_b200 import synth

    return synth.laser_transform(xyz=(0.04 * (s % 4), -0.03 * (s % 3), 0.2 + 0.05 * (s % 2)),
                                 rpy=(0.01 * (s % 3), -0.012 * (s % 2), 0.02 * (s % 5)))


def member_cloud(s):
    d_min, d_max, z = (0.3, 0.45, 0.6)[s % 3], (9.0, 12.0, 30.0, 6.0)[s % 4], (1.0, 0.5, 0.3)[s % 3]
    return dict(sqr_laser_min_dist=float(F32(d_min * d_min)), sqr_laser_max_dist=float(F32(d_max * d_max)),
                laser_z_min_value=-z, laser_z_max_value=z)


def make_rep(s, mode, cloud_format=True):
    """Member s's handle: every input kind's format set (the cloud format unless cloud_format is False)."""
    from hector_slam_b200 import capi

    rep = capi.MapRepB200(RES, SIZE, levels=LEVELS, update_factor_free=0.4 + 0.02 * (s % 3),
                          update_factor_occupied=0.6 + 0.1 * (s % 4), gather_mode=mode)
    dist, ang = ((0.0, 0.0), (0.15, 0.1), (0.3, 0.5))[s % 3]
    rep.setMapUpdateMinDistDiff(dist)
    rep.setMapUpdateMinAngleDiff(ang)
    g = geometry(s)
    rep.set_scan_format(**g)
    rep.set_laser_projection(**g, range_cutoff=30.0)
    if cloud_format:
        rep.set_cloud_format(member_transform(s), **member_cloud(s))
    return rep


def session_data(seed, steps, g):
    """A trajectory through its own synthetic room: per step the ranges in geometry g, the same scan as level-0
    endpoints and as a Point32 cloud in the laser frame, the true pose and a noisy hint."""
    from hector_slam_b200 import synth

    rng = np.random.default_rng(seed)
    world = synth.World(1, seed=1000 + seed)
    ang = beam_angles(g)
    x, y, a = rng.uniform(-2, 2), rng.uniform(-1.5, 1.5), rng.uniform(-3, 3)
    truth, ranges, scans, clouds = [], [], [], []
    for _ in range(steps):
        p = np.array([x, y, a], F32)
        truth.append(p)
        r = (world.cast(p, ang) + rng.normal(0.0, 0.01, ang.size)).astype(F32)
        ranges.append(np.ascontiguousarray(r))
        scans.append(np.ascontiguousarray(synth.ranges_to_points(r, SCALE, ang), F32))
        clouds.append(np.ascontiguousarray(synth.ranges_to_cloud(r, ang), F32))
        a += rng.uniform(-0.08, 0.08)
        step = rng.uniform(0.03, 0.12)
        x = float(np.clip(x + step * np.cos(a), -6.0, 6.0))
        y = float(np.clip(y + step * np.sin(a), -4.0, 4.0))
    truth = np.asarray(truth, F32)
    hints = truth + rng.uniform(-1, 1, truth.shape).astype(F32) * np.array([0.04, 0.04, 0.02], F32)
    return dict(truth=truth, ranges=ranges, scans=scans, clouds=clouds, hints=hints.astype(F32))


def scan_of(kind, d, k):
    return {"endpoints": d["scans"], "cloud": d["clouds"], "ranges": d["ranges"], "projected": d["ranges"]}[kind][k]


def group_step(group, kind, hints, scans, mwm, members=None, nowait=False, cov=None):
    """One group step of `kind` -> (poses, covs, updated, kept or None)"""
    kw = dict(map_without_matching=mwm, nowait=nowait, cov_inout=cov, members=members)
    if kind == "endpoints":
        return group.slam_update(hints, scans, **kw) + (None,)
    return {"cloud": group.slam_update_cloud, "ranges": group.slam_update_ranges,
            "projected": group.slam_update_projected}[kind](hints, scans, **kw)


def single_step(rep, kind, hint, scan, without, cov=None):
    """The single-handle call of `kind` -> (pose, cov, updated, kept or None)"""
    if kind == "endpoints":
        return rep.slam_update(hint, scan, map_without_matching=without, cov_inout=cov) + (None,)
    return {"cloud": rep.slam_update_cloud, "ranges": rep.slam_update_ranges,
            "projected": rep.slam_update_projected}[kind](hint, scan, map_without_matching=without, cov_inout=cov)


def bits(a):
    return np.ascontiguousarray(a, F32).view(np.uint32)


def assert_same_session(out, i, ref, tag):
    P, Cv, U, K = out
    p, c, u, kept = ref
    assert np.array_equal(bits(P[i]), bits(p)), (tag, i, P[i], p)
    assert np.array_equal(bits(Cv[i]), bits(c)), (tag, i)
    assert bool(U[i]) == bool(u), (tag, i)
    if K is not None:
        assert K[i] == kept, (tag, i, K[i], kept)


def assert_same_state(a, b, tag, probe=True, levels=LEVELS):
    """Every level's log-odds and probability, the texture twin (probe over the written area), both dirty rectangles
    (read without reset) and the gate pose."""
    for l in range(levels):
        la = a.download_level(l)
        assert np.array_equal(bits(la), bits(b.download_level(l))), (tag, l)
        assert np.array_equal(bits(a.download_prob(l)), bits(b.download_prob(l))), (tag, l)
        assert a.get_mirror_dirty_rect(l) == b.get_mirror_dirty_rect(l), (tag, l)
        if probe:
            nz = np.nonzero(la)
            if nz[0].size:
                L = type("L", (), {})()
                L.sx, L.sy = la.shape[1], la.shape[0]
                rect = (int(nz[1].min()), int(nz[0].min()), int(nz[1].max()), int(nz[0].max()))
                probe_twin(a, l, L, la, rect, tag, max_cells=4000)
    assert a.get_dirty_rects() == b.get_dirty_rects(), tag
    assert np.array_equal(bits(a.last_map_update_pose()), bits(b.last_map_update_pose())), tag


def assert_same_container(a, b, d, k, tag):
    """The last match's container (points, count, origo) through a following updateByScan, whose coarse levels write
    it; both handles take the same write."""
    pose = d["truth"][k]
    a.updateByScan(d["scans"][k][::3], pose)
    b.updateByScan(d["scans"][k][::3], pose)
    for l in range(1, LEVELS):
        assert np.array_equal(bits(a.download_level(l)), bits(b.download_level(l))), (tag, l)


def snapshot(rep):
    return ([(bits(rep.download_level(l)).copy(), bits(rep.download_prob(l)).copy(), rep.get_mirror_dirty_rect(l))
             for l in range(LEVELS)], rep.get_dirty_rects(), bits(rep.last_map_update_pose()).copy(), rep.launch_count)


def assert_snapshot(rep, snap, tag):
    now = snapshot(rep)
    for l in range(LEVELS):
        assert np.array_equal(now[0][l][0], snap[0][l][0]) and np.array_equal(now[0][l][1], snap[0][l][1]), (tag, l)
        assert now[0][l][2] == snap[0][l][2], (tag, l)
    assert now[1] == snap[1] and np.array_equal(now[2], snap[2]) and now[3] == snap[3], tag


def close_all(*groups):
    for g in groups:
        for x in (g if isinstance(g, (list, tuple)) else [g]):
            x.close()


@MODES
@pytest.mark.parametrize("kind", KINDS)
def test_subset_run_equals_single_calls(hsb_lib, kind, mode):
    """M = 6, 30 seeded ticks: each tick steps a random subset in a random session order (K = M, K = 1 and K = 0
    included), some sessions map_without_matching.  Every session equals the single call on the member's twin; every
    member's full state equals its twin's every 10 ticks and at the end."""
    from hector_slam_b200 import capi

    M, ticks = 6, 30
    data = [session_data(300 + s, ticks, geometry(s)) for s in range(M)]
    grp = [make_rep(s, mode) for s in range(M)]
    one = [make_rep(s, mode) for s in range(M)]
    group = capi.SlamGroup(grp)
    rng = np.random.default_rng(17 + KINDS.index(kind))
    step = [0] * M   # each member's own position in its trajectory: it advances only when the member is stepped
    covs = [np.full((3, 3), 5.0, F32) for _ in range(M)]
    covs_one = [c.copy() for c in covs]
    seen_K, fired = set(), np.zeros(2, int)
    for t in range(ticks):
        K = {0: M, 1: 1, 2: 0}.get(t, int(rng.integers(0, M + 1)))
        members = [int(j) for j in rng.permutation(M)[:K]]
        seen_K.add(K)
        without = [bool(rng.random() < 0.2) and step[j] > 0 for j in members]
        hints, scans = [], []
        for j, w in zip(members, without):
            d, k = data[j], step[j]
            hints.append(d["truth" if w else "hints"][k])
            scans.append(scan_of(kind, d, k))
        hints = np.asarray(hints, F32).reshape(K, 3)
        out = group_step(group, kind, hints, scans, without, members=members, nowait=(t % 3 == 1),
                         cov=np.stack([covs[j] for j in members]) if K else None)
        for i, j in enumerate(members):
            ref = single_step(one[j], kind, hints[i], scans[i], without[i], cov=covs_one[j])
            assert_same_session(out, i, ref, (t, j))
            covs[j], covs_one[j] = out[1][i].copy(), ref[1]
            fired[int(ref[2])] += 1
            step[j] += 1
        if t % 10 == 9:
            for j in range(M):
                assert_same_state(grp[j], one[j], (t, j))
    assert {0, 1, M} <= seen_K, seen_K
    assert fired[0] > 0 and fired[1] > 0, fired
    for j in range(M):
        assert_same_state(grp[j], one[j], ("end", j))
        assert_same_container(grp[j], one[j], data[j], min(step[j], ticks - 1), ("container", j))
    group.close()
    close_all(grp, one)


@MODES
def test_identity_subset_equals_full_step(hsb_lib, mode):
    """members = 0..M-1 against the full call on twin groups, every input kind in turn: the same bits and end states,
    although the subset call sizes its map-write grids from its own member list."""
    from hector_slam_b200 import capi

    M, ticks = 5, 12
    data = [session_data(400 + s, ticks, geometry(s)) for s in range(M)]
    ra = [make_rep(s, mode) for s in range(M)]
    rb = [make_rep(s, mode) for s in range(M)]
    ga, gb = capi.SlamGroup(ra), capi.SlamGroup(rb)
    for t in range(ticks):
        kind = KINDS[t % 4]
        hints = np.stack([d["hints"][t] for d in data])
        scans = [scan_of(kind, d, t) for d in data]
        mwm = [t % 5 == 4 and s % 2 == 0 for s in range(M)]
        full = group_step(ga, kind, hints, scans, mwm, nowait=(t % 2 == 1))
        sub = group_step(gb, kind, hints, scans, mwm, members=list(range(M)), nowait=(t % 2 == 1))
        for x, y in zip(full, sub):
            if x is not None:
                assert np.array_equal(bits(x), bits(y)) if x.dtype == F32 else np.array_equal(x, y), (t, kind)
    for s in range(M):
        assert_same_state(ra[s], rb[s], s)
        assert_same_container(ra[s], rb[s], data[s], ticks - 1, s)
    close_all([ga, gb], ra, rb)


@MODES
def test_unselected_members_untouched(hsb_lib, mode):
    """Members left out of a subset step keep their planes, both dirty rectangles (read without reset), gate pose,
    launch count and last-match container; a member without a cloud format may be left out of a cloud step."""
    from hector_slam_b200 import capi

    M = 5
    data = [session_data(500 + s, 4, geometry(s)) for s in range(M)]
    grp = [make_rep(s, mode, cloud_format=(s != 3)) for s in range(M)]
    twin = [make_rep(s, mode) for s in range(M)]
    group = capi.SlamGroup(grp)
    # a first step of every member (endpoints: member 3 has no cloud format), mirrored on the twins
    hints = np.stack([d["hints"][0] for d in data])
    out = group.slam_update(hints, [d["scans"][0] for d in data])
    for s in range(M):
        assert_same_session(out + (None,), s, single_step(twin[s], "endpoints", hints[s], data[s]["scans"][0], False),
                            s)
    for kind, members in (("cloud", [4, 1]), ("endpoints", [2]), ("projected", [0, 2, 4]), ("ranges", [1])):
        left_out = [j for j in range(M) if j not in members]
        snaps = {j: snapshot(grp[j]) for j in left_out}
        k = 1 + KINDS.index(kind) % 3
        hints = np.stack([data[j]["hints"][k] for j in members])
        out = group_step(group, kind, hints, [scan_of(kind, data[j], k) for j in members], None, members=members,
                         nowait=(kind == "projected"))
        for i, j in enumerate(members):
            assert_same_session(out, i, single_step(twin[j], kind, hints[i], scan_of(kind, data[j], k), False),
                                (kind, j))
        for j in left_out:
            if j == 0 and snaps[j][3] != grp[0].launch_count:   # handles[0] carries the step's launches
                assert grp[0].launch_count - snaps[j][3] == 3, kind
                snaps[j] = snaps[j][:3] + (grp[0].launch_count,)
            assert_snapshot(grp[j], snaps[j], (kind, j))
    for s in range(M):
        assert_same_state(grp[s], twin[s], s)
        assert_same_container(grp[s], twin[s], data[s], 3, s)
    group.close()
    close_all(grp, twin)


@MODES
def test_ordering(hsb_lib, mode):
    """(1) A nowait full step, at once a nowait subset step without member j, then j's planes and a single step on j:
    equal to j's twin (j still waits for the map write of the full step), also when the pending write came from
    another group.  (2) A selected member's _device batch match still queued on a caller stream is ordered before the
    subset step, which rewrites the planes the match reads."""
    import torch

    from hector_slam_b200 import capi

    M, ticks = 4, 6
    data = [session_data(600 + s, ticks + 2, geometry(s)) for s in range(M)]
    grp = [make_rep(s, mode) for s in range(M)]
    one = [make_rep(s, mode) for s in range(M)]
    group = capi.SlamGroup(grp)
    solo = capi.SlamGroup([grp[3]])   # another group holding member 3
    t = 0
    for t in range(ticks):
        j = t % M
        hints = np.stack([d["hints"][t] for d in data])
        if j == 3:   # the pending write comes from the other group
            out = solo.slam_update(hints[3:4], [data[3]["scans"][t]], nowait=True)
            ref = single_step(one[3], "endpoints", hints[3], data[3]["scans"][t], False)
            assert_same_session(out + (None,), 0, ref, (t, "solo"))
            others = [0, 1, 2]
        else:
            out = group.slam_update(hints, [d["scans"][t] for d in data], nowait=True)
            for s in range(M):
                assert_same_session(out + (None,), s, single_step(one[s], "endpoints", hints[s], data[s]["scans"][t],
                                                                  False), (t, s))
            others = [s for s in range(M) if s != j]
        others = others[::-1]
        out = group.slam_update(hints[others], [data[s]["scans"][t + 1] for s in others], members=others, nowait=True)
        for i, s in enumerate(others):
            assert_same_session(out + (None,), i, single_step(one[s], "endpoints", hints[s], data[s]["scans"][t + 1],
                                                              False), (t, s, "subset"))
        for l in range(LEVELS):   # read at once: after the pending write of the step that included j
            assert np.array_equal(bits(grp[j].download_level(l)), bits(one[j].download_level(l))), (t, j, l)
        x = grp[j].slam_update(data[j]["hints"][t + 1], data[j]["scans"][t + 1], nowait=True)
        y = one[j].slam_update(data[j]["hints"][t + 1], data[j]["scans"][t + 1])
        assert all(np.array_equal(bits(u), bits(v)) for u, v in zip(x[:2], y[:2])) and x[2] == y[2], (t, j)
    for s in range(M):
        grp[s].onMapUpdated()
        assert_same_state(grp[s], one[s], s, probe=False)

    # (2) a batch match queued on a torch stream against member 1's map, then a subset step that writes that map
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    k = ticks + 1
    scan = data[1]["scans"][k]
    d_h = torch.from_numpy(np.repeat(data[1]["hints"][k][None], 64, axis=0)).to(dev)
    d_p = torch.from_numpy(scan).to(dev)
    torch.cuda.current_stream(dev).synchronize()

    def batch(rep):
        poses = torch.zeros((64, 3), dtype=torch.float32, device=dev)
        rep.match_batch_device(64, d_h.data_ptr(), d_p.data_ptr(), None, scan.shape[0], scan.shape[0],
                               poses.data_ptr(), None, stream.cuda_stream)
        return poses

    pg, po = batch(grp[1]), batch(one[1])
    hints = np.stack([data[s]["hints"][k] for s in (2, 1)])
    out = group.slam_update(hints, [data[s]["scans"][k] for s in (2, 1)], members=[2, 1], nowait=True)
    for i, s in enumerate((2, 1)):
        assert_same_session(out + (None,), i, single_step(one[s], "endpoints", hints[i], data[s]["scans"][k], False),
                            ("batch", s))
    with torch.cuda.stream(stream):
        assert np.array_equal(pg.cpu().numpy().view(np.uint32), po.cpu().numpy().view(np.uint32))
    for s in range(M):
        assert_same_state(grp[s], one[s], ("batch", s), probe=False)
    close_all([solo, group], grp, one)


@MODES
def test_launch_count(hsb_lib, mode):
    """Three launches per step of K >= 1, counted on handles[0] also when member 0 is not selected; none for K = 0;
    the other members' counts do not move."""
    from hector_slam_b200 import capi

    M = 6
    reps = [make_rep(s, mode) for s in range(M)]
    group = capi.SlamGroup(reps)
    data = [session_data(700 + s, 5, geometry(s)) for s in range(M)]
    for k, (kind, members) in enumerate((("endpoints", [3, 5]), ("projected", [0]), ("cloud", []), ("ranges", [2, 1, 4]),
                                         ("projected", []))):
        before = [r.launch_count for r in reps]
        hints = np.stack([data[j]["hints"][k] for j in members]) if members else np.zeros((0, 3), F32)
        group_step(group, kind, hints, [scan_of(kind, data[j], k) for j in members], None, members=members,
                   nowait=(k % 2 == 1))
        after = [r.launch_count for r in reps]
        assert after[0] - before[0] == (3 if members else 0), (k, before[0], after[0])
        assert after[1:] == before[1:], k
    group.close()
    close_all(reps)


@MODES
def test_rejections(hsb_lib, mode):
    """K < 0, K > M, members NULL with K > 0, an index outside [0, M), a member listed twice, and a selected member
    without the kind's format: HSB_ERR_INVALID_ARG naming the session where there is one; no member's state moved and
    nothing was launched.  K = 0 with every other argument NULL is a no-op."""
    from hector_slam_b200 import capi

    M = 4
    data = [session_data(800 + s, 3, geometry(s)) for s in range(M)]
    grp = [make_rep(s, mode, cloud_format=(s != 2)) for s in range(M)]
    twin = [make_rep(s, mode) for s in range(M)]
    group = capi.SlamGroup(grp)
    hints = np.stack([d["hints"][0] for d in data])
    out = group.slam_update(hints, [d["scans"][0] for d in data])
    for s in range(M):
        single_step(twin[s], "endpoints", hints[s], data[s]["scans"][0], False)
    snaps = [snapshot(r) for r in grp]
    lib = group.lib
    pts = np.ascontiguousarray(np.concatenate([d["scans"][1] for d in data]), F32)
    offs = np.zeros(M + 1, np.int32)
    offs[1:] = np.cumsum([d["scans"][1].shape[0] for d in data])
    poses, cov, upd = np.zeros((M, 3), F32), np.zeros((M, 9), F32), np.zeros(M, np.int32)

    def raw(K, members):
        m = None if members is None else np.ascontiguousarray(members, np.int32)
        return lib.hsb_group_slam_update_subset(group.g, K, None if m is None else m.ctypes.data, hints.ctypes.data,
                                                pts.ctypes.data, offs.ctypes.data, None, None, 0, poses.ctypes.data,
                                                cov.ctypes.data, upd.ctypes.data)

    def err():
        return (lib.hsb_last_error(grp[0].h) or b"").decode()

    for K, members, text in ((-1, [0], "K is -1"), (M + 1, [0, 1, 2, 3, 0], "K is 5"), (2, None, "members is NULL"),
                             (2, [0, M], "session 1: member 4"), (2, [-1, 0], "session 0: member -1"),
                             (3, [1, 3, 1], "session 2: member 1 is listed twice")):
        assert raw(K, members) == -1, (K, members)
        assert text in err(), (text, err())
    with pytest.raises(capi.HsbError) as e:   # member 2 has no cloud format: session 1 of this step
        group.slam_update_cloud(hints[[0, 2]], [data[0]["clouds"][1], data[2]["clouds"][1]], members=[0, 2])
    assert e.value.status == -1 and "session 1" in str(e.value) and "hsb_set_cloud_format" in str(e.value), str(e.value)
    with pytest.raises(capi.HsbError) as e:   # a ranges scan that is not its member's beam count
        group.slam_update_ranges(hints[[3]], [data[1]["ranges"][1]], members=[3])
    assert e.value.status == -1 and "session 0" in str(e.value), str(e.value)
    for name in ("hsb_group_slam_update_subset", "hsb_group_slam_update_cloud_subset",
                 "hsb_group_slam_update_ranges_subset", "hsb_group_slam_update_projected_subset"):
        nulls = [0 if t is C.c_int else None for t in getattr(lib, name).argtypes[3:]]   # nowait is the int
        assert getattr(lib, name)(group.g, 0, None, *nulls) == 0, name
    for s in range(M):
        assert_snapshot(grp[s], snaps[s], s)
    # the group still works, and every member still equals its twin
    members = [3, 0, 1]
    hints2 = np.stack([data[j]["hints"][2] for j in members])
    out = group.slam_update(hints2, [data[j]["scans"][2] for j in members], members=members,
                            map_without_matching=[False, True, False])
    for i, j in enumerate(members):
        assert_same_session(out + (None,), i, single_step(twin[j], "endpoints", hints2[i], data[j]["scans"][2], i == 1),
                            j)
    for s in range(M):
        assert_same_state(grp[s], twin[s], s, probe=False)
    group.close()
    close_all(grp, twin)


def test_facade_subset_overloads(hsb_lib):
    """hsb200::SlamProcessor's subset overloads of updateMany, updateManyCloud, updateManyRanges and
    updateManyProjected (through their shims) over changing subsets equal per-processor update* calls: poses,
    covariances and planes; the processors left out keep their poses.  (The façade's processors take the default
    gather mode.)"""
    L = C.CDLL(os.path.join(ROOT, "hector_slam_b200", "lib", "libhsb200_host.so"))
    vp, i, f, d = C.c_void_p, C.c_int, C.c_float, C.c_double
    L.hsbp_create.restype = vp
    L.hsbp_create.argtypes = [f, i, i, f, f, i, i]
    L.hsbp_destroy.argtypes = [vp]
    L.hsbp_set_cloud_format.argtypes = [vp, vp, f, f, f, f]
    L.hsbp_set_scan_format.argtypes = [vp, i, f, f, f, f]
    L.hsbp_set_laser_projection.argtypes = [vp, i, f, f, f, f, d]
    L.hsbp_set_map_update_thresholds.argtypes = [vp, f, f]
    L.hsbp_update.argtypes = [vp, vp, i, vp, vp, i, vp, vp]
    L.hsbp_update_cloud.argtypes = [vp, vp, i, vp, vp, i, vp]
    L.hsbp_update_ranges.argtypes = [vp, vp, i, vp, i, vp]
    L.hsbp_update_projected.argtypes = [vp, vp, i, vp, vp, i, vp]
    L.hsbp_update_many_subset.argtypes = [vp, i, vp, i, vp, vp, vp, vp, vp]
    L.hsbp_update_many_cloud_subset.argtypes = [vp, i, vp, i, vp, vp, vp, vp, vp, vp]
    L.hsbp_update_many_ranges_subset.argtypes = [vp, i, vp, i, vp, vp, vp, vp, vp]
    L.hsbp_update_many_projected_subset.argtypes = [vp, i, vp, i, vp, vp, vp, vp, vp, vp]
    L.hsbp_get_pose_and_cov.argtypes = [vp, vp, vp]
    L.hsbp_get_grid_map.argtypes = [vp, i, vp]

    M, ticks = 4, 12
    data = [session_data(900 + s, ticks, geometry(s)) for s in range(M)]
    many = [L.hsbp_create(RES, SIZE, SIZE, 0.5, 0.5, LEVELS, 0) for _ in range(M)]
    one = [L.hsbp_create(RES, SIZE, SIZE, 0.5, 0.5, LEVELS, 0) for _ in range(M)]
    assert all(many) and all(one)
    for s in range(M):
        T, fm, g = member_transform(s), member_cloud(s), geometry(s)
        for p in (many[s], one[s]):
            assert L.hsbp_set_cloud_format(p, T.ctypes.data, fm["sqr_laser_min_dist"], fm["sqr_laser_max_dist"],
                                           fm["laser_z_min_value"], fm["laser_z_max_value"]) == 0
            assert L.hsbp_set_scan_format(p, g["n_beams"], g["angle_min"], g["angle_increment"], g["range_min"],
                                          g["range_max"]) == 0
            assert L.hsbp_set_laser_projection(p, g["n_beams"], g["angle_min"], g["angle_increment"], g["range_min"],
                                               g["range_max"], 30.0) == 0
            L.hsbp_set_map_update_thresholds(p, (0.0, 0.15, 0.3, 0.0)[s], (0.0, 0.1, 0.5, 0.0)[s])
    arr = (C.c_void_p * M)(*many)
    rng = np.random.default_rng(5)
    step = [0] * M
    last = {s: (np.zeros(3, F32), np.zeros(9, F32)) for s in range(M)}
    for t in range(ticks):
        kind = KINDS[t % 4]
        K = (M, 2, 1, 3)[t % 4] if t < 8 else int(rng.integers(1, M + 1))
        members = np.ascontiguousarray(rng.permutation(M)[:K], np.int32)
        scans = [scan_of(kind, data[j], step[j]) for j in members]
        hints = np.ascontiguousarray(np.stack([data[j]["hints"][step[j]] for j in members]), F32)
        mwm = np.array([int(t % 5 == 4 and n == 0) for n in range(K)], np.int32)
        flat = np.ascontiguousarray(np.concatenate([x.reshape(-1) for x in scans]), F32)
        width = {"endpoints": 2, "cloud": 3}.get(kind, 1)
        offs = np.zeros(K + 1, np.int32)
        offs[1:] = np.cumsum([x.size // width for x in scans])
        kept = np.zeros(K, np.int32)
        base = (C.cast(arr, vp), M, members.ctypes.data, K, flat.ctypes.data, offs.ctypes.data)
        if kind == "endpoints":
            assert L.hsbp_update_many_subset(*base, None, hints.ctypes.data, mwm.ctypes.data) == 0
        elif kind == "cloud":
            assert L.hsbp_update_many_cloud_subset(*base, None, hints.ctypes.data, mwm.ctypes.data, kept.ctypes.data) == 0
        elif kind == "ranges":
            assert L.hsbp_update_many_ranges_subset(*base, hints.ctypes.data, mwm.ctypes.data, kept.ctypes.data) == 0
        else:
            assert L.hsbp_update_many_projected_subset(*base, None, hints.ctypes.data, mwm.ctypes.data,
                                                       kept.ctypes.data) == 0
        for n, j in enumerate(members):
            x = np.ascontiguousarray(scans[n])
            k1 = C.c_int(-1)
            if kind == "endpoints":
                p2, c2 = np.zeros(3, F32), np.zeros(9, F32)
                assert L.hsbp_update(one[j], x.ctypes.data, x.shape[0], None, hints[n].ctypes.data, int(mwm[n]),
                                     p2.ctypes.data, c2.ctypes.data) == 0
            elif kind == "cloud":
                assert L.hsbp_update_cloud(one[j], x.ctypes.data, x.shape[0], None, hints[n].ctypes.data, int(mwm[n]),
                                           C.byref(k1)) == 0
            elif kind == "ranges":
                assert L.hsbp_update_ranges(one[j], x.ctypes.data, x.size, hints[n].ctypes.data, int(mwm[n]),
                                            C.byref(k1)) == 0
            else:
                assert L.hsbp_update_projected(one[j], x.ctypes.data, x.size, None, hints[n].ctypes.data, int(mwm[n]),
                                               C.byref(k1)) == 0
            if kind != "endpoints":
                assert kept[n] == k1.value, (t, j)
            step[j] += 1
        for s in range(M):
            p1, c1, p2, c2 = np.zeros(3, F32), np.zeros(9, F32), np.zeros(3, F32), np.zeros(9, F32)
            L.hsbp_get_pose_and_cov(many[s], p1.ctypes.data, c1.ctypes.data)
            L.hsbp_get_pose_and_cov(one[s], p2.ctypes.data, c2.ctypes.data)
            assert np.array_equal(bits(p1), bits(p2)) and np.array_equal(bits(c1), bits(c2)), (t, s, kind)
            if s not in members:
                assert np.array_equal(bits(p1), bits(last[s][0])) and np.array_equal(bits(c1), bits(last[s][1])), (t, s)
            last[s] = (p1, c1)
    for s in range(M):
        for l in range(LEVELS):
            sz = SIZE >> l
            x, y = np.zeros((sz, sz), F32), np.zeros((sz, sz), F32)
            assert L.hsbp_get_grid_map(many[s], l, x.ctypes.data) == 0
            assert L.hsbp_get_grid_map(one[s], l, y.ctypes.data) == 0
            assert np.array_equal(bits(x), bits(y)), (s, l)
    for p in many + one:   # any member first: its cached group goes with it
        L.hsbp_destroy(p)
