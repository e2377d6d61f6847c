"""hsb_group_slam_update — HectorSlamProcessor::update for many handles (one SLAM session, one map each) in one device
pass — against the same sessions stepped one by one with hsb_slam_update: bit-identical poses, covariances, gate
decisions, planes and handle state, also with mixed session kinds, permuted groups, interleaved single calls and
nowait steps; against the oracle on the golden SLAM run; argument validation; launch accounting; the C++ façade's
updateMany."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import ROOT, load_golden, pose_err

pytestmark = pytest.mark.gpu

RES, SIZE, LEVELS = 0.05, 512, 3
SCALE = 1.0 / RES


def session_data(seed, steps):
    """A trajectory through its own synthetic room (World seed), its scans (level-0 cells) and noisy hints."""
    from hector_slam_b200 import synth

    rng = np.random.default_rng(seed)
    world = synth.World(1, seed=1000 + seed)
    x, y, a = rng.uniform(-2, 2), rng.uniform(-1.5, 1.5), rng.uniform(-3, 3)
    truth, scans = [], []
    for _ in range(steps):
        p = np.array([x, y, a], np.float32)
        truth.append(p)
        scans.append(synth.make_scan(world, p, rng, scale_to_map=SCALE))
        a += rng.uniform(-0.08, 0.08)
        step = rng.uniform(0.03, 0.12)
        x = float(np.clip(x + step * np.cos(a), -6.0, 6.0))
        y = float(np.clip(y + step * np.sin(a), -4.0, 4.0))
    truth = np.asarray(truth, np.float32)
    hints = truth + rng.uniform(-1, 1, truth.shape).astype(np.float32) * np.array([0.04, 0.04, 0.02], np.float32)
    return truth, scans, hints.astype(np.float32)


def make_rep(s, **kw):
    """Handle of session s: update factors and gate thresholds differ between sessions."""
    from hector_slam_b200 import capi

    rep = capi.MapRepB200(RES, SIZE, levels=LEVELS, update_factor_free=0.4 + 0.02 * (s % 3),
                          update_factor_occupied=0.6 + 0.1 * (s % 4), **kw)
    dist, ang = ((0.0, 0.0), (0.15, 0.1), (0.3, 0.5))[s % 3]
    rep.setMapUpdateMinDistDiff(dist)
    rep.setMapUpdateMinAngleDiff(ang)
    return rep


def assert_same_state(a, b, tag):
    """Planes, gate pose and both dirty rectangles of every level."""
    for l in range(LEVELS):
        assert np.array_equal(a.download_level(l), b.download_level(l)), (tag, l)
        assert np.array_equal(a.download_prob(l), b.download_prob(l)), (tag, l)
        assert a.get_mirror_dirty_rect(l) == b.get_mirror_dirty_rect(l), (tag, l)
    assert a.get_dirty_rects() == b.get_dirty_rects(), tag
    assert np.array_equal(a.last_map_update_pose(), b.last_map_update_pose()), tag


def close_all(*groups):
    for g in groups:
        for x in (g if isinstance(g, (list, tuple)) else [g]):
            x.close()


def test_group_step_equals_single_steps(hsb_lib):
    """12 sessions, 40 steps: every pose, covariance and gate decision and the final handle state equal 12 handles
    stepped with hsb_slam_update."""
    from hector_slam_b200 import capi

    M, steps = 12, 40
    data = [session_data(s, steps) for s in range(M)]
    grp_reps = [make_rep(s) for s in range(M)]
    one_reps = [make_rep(s) for s in range(M)]
    group = capi.SlamGroup(grp_reps)
    fired = np.zeros(2, int)
    for k in range(steps):
        hints = np.stack([d[2][k] for d in data])
        P, Cv, U = group.slam_update(hints, [d[1][k] for d in data])
        for s in range(M):
            p, c, u = one_reps[s].slam_update(hints[s], data[s][1][k])
            assert np.array_equal(P[s], p), (k, s, P[s], p)
            assert np.array_equal(Cv[s], c), (k, s)
            assert U[s] == u, (k, s)
            fired[int(u)] += 1
    assert fired[0] > 0 and fired[1] > 0, fired   # the gate both fires and holds back
    for s in range(M):
        assert_same_state(grp_reps[s], one_reps[s], s)
    group.close()
    close_all(grp_reps, one_reps)


def test_mixed_sessions_and_permuted_groups(hsb_lib):
    """Empty scans, map_without_matching (also right after a matched step: the coarse levels then write the last
    MATCHED scan), sessions whose gate holds the map write back, a non-zero origo, and the session order permuted
    between calls (three groups over the same handles)."""
    from hector_slam_b200 import capi

    M, steps = 6, 18
    data = [session_data(20 + s, steps) for s in range(M)]
    grp_reps = [make_rep(s) for s in range(M)]
    one_reps = [make_rep(s) for s in range(M)]
    for r in (grp_reps[5], one_reps[5]):   # writes only on its first step (FLT_MAX gate), then never
        r.setMapUpdateMinDistDiff(100.0)
        r.setMapUpdateMinAngleDiff(100.0)
    rng = np.random.default_rng(4)
    orders = [list(range(M)), list(range(M))[::-1], list(rng.permutation(M))]
    groups = [capi.SlamGroup([grp_reps[s] for s in o]) for o in orders]
    origo = np.array([[0.0, 0.0], [2.4, -0.6]] * 3, np.float32)
    covs = {s: np.full((3, 3), 7.0, np.float32) for s in range(M)}
    covs_one = {s: c.copy() for s, c in covs.items()}
    kinds_seen = set()
    prev_matched = np.zeros(M, bool)
    for k in range(steps):
        kind = rng.choice(["match", "match", "empty", "without"], M)
        if k == 0:
            kind[:] = "match"
        if k == 1:
            kind[0] = "without"   # straight after a matched step
        order = orders[k % 3]
        hints, scans, mwm, og, cin = [], [], [], [], []
        for s in order:
            scan = data[s][1][k] if kind[s] != "empty" else np.zeros((0, 2), np.float32)
            hints.append(data[s][0][k] if kind[s] == "without" else data[s][2][k])
            scans.append(scan)
            mwm.append(kind[s] == "without")
            og.append(origo[s])
            cin.append(covs[s])
            if kind[s] == "without" and prev_matched[s]:
                kinds_seen.add("without-after-match")
            kinds_seen.add(kind[s])
        P, Cv, U = groups[k % 3].slam_update(np.stack(hints), scans, origo=np.stack(og), map_without_matching=mwm,
                                             cov_inout=np.stack(cin))
        for i, s in enumerate(order):
            p, c, u = one_reps[s].slam_update(hints[i], scans[i], map_without_matching=mwm[i], cov_inout=covs_one[s],
                                              origo=og[i])
            assert np.array_equal(P[i], p), (k, s, kind[s])
            assert np.array_equal(Cv[i], c), (k, s, kind[s])
            assert U[i] == u, (k, s, kind[s])
            covs[s], covs_one[s] = Cv[i], c
            prev_matched[s] = kind[s] == "match"
            if s == 5 and k > 0 and kind[s] != "without":
                assert not u
    assert {"match", "empty", "without", "without-after-match"} <= kinds_seen, kinds_seen
    for s in range(M):
        assert_same_state(grp_reps[s], one_reps[s], s)
    close_all(groups, grp_reps, one_reps)


def test_group_against_oracle(hsb_lib, pyoracle):
    """8 sessions replay the golden SLAM run, map_without_matching on every fourth step at the golden estimate: every
    session within 1e-4 m / rad of the oracle's update(), planes within 1e-5."""
    from hector_slam_b200 import capi

    g = load_golden("slam3.npz")
    res, size = float(g["res"]), int(g["size"])
    M = 8
    reps = [capi.MapRepB200(res, size, levels=3, update_factor_free=0.4, update_factor_occupied=0.9) for _ in range(M)]
    for r in reps:
        r.setMapUpdateMinDistDiff(0.2)
        r.setMapUpdateMinAngleDiff(0.03)
    group = capi.SlamGroup(reps)
    orc = pyoracle.Oracle("port", res, size, 3)
    orc.set_update_factors(0.4, 0.9)
    orc.set_map_update_thresholds(0.2, 0.03)
    hint_g = np.repeat(g["first_hint"][None], M, axis=0).astype(np.float32)
    hint_o = g["first_hint"].copy()
    for k in range(g["scans"].shape[0]):
        scan = g["scans"][k]
        without = (k % 4 == 3)
        if without:
            hint_g[:] = g["est"][k]
            hint_o = g["est"][k].copy()
        P, _, U = group.slam_update(hint_g, [scan] * M, map_without_matching=[without] * M)
        want, _ = orc.update(scan, hint_o, map_without_matching=without)
        for s in range(M):
            ex, ey, ea = pose_err(P[s], want)
            assert max(ex, ey) <= 1e-4 and ea <= 1e-4, (k, s, ex, ey, ea)
            if without:
                assert U[s] and np.array_equal(P[s], hint_g[s])
        hint_g, hint_o = P.copy(), want
    for s in range(M):
        for l in range(3):
            got, ref = reps[s].download_level(l), orc.get_logodds(l)
            diff = np.abs(got - ref)
            assert (diff > 1e-5).sum() <= max(3, int(2e-3 * (got != 0).sum())), (s, l, int((diff > 1e-5).sum()))
    group.close()
    close_all(reps)
    orc.close()


def test_single_member_group_and_nowait(hsb_lib):
    """M = 1 equals hsb_slam_update bit for bit; nowait = 1 equals nowait = 0 for a 5-session group, with
    hsb_on_map_updated of each member as the completion point before the planes are read."""
    from hector_slam_b200 import capi

    steps = 14
    d = session_data(77, steps)
    a, b = make_rep(1), make_rep(1)
    ga = capi.SlamGroup([a])
    for k in range(steps):
        P, Cv, U = ga.slam_update(d[2][k][None], [d[1][k]])
        p, c, u = b.slam_update(d[2][k], d[1][k])
        assert np.array_equal(P[0], p) and np.array_equal(Cv[0], c) and U[0] == u, k
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
            out.append(grp.slam_update(np.stack([x[2][k] for x in data]), [x[1][k] for x in data], nowait=nowait))
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


def test_mixing_with_other_calls_without_synchronisation(hsb_lib):
    """Between nowait group steps, members take single SLAM steps, a reset, batch matches on a torch stream, occupancy
    downloads and plain map writes — with no synchronisation by the caller.  Everything equals the same sequence on
    handles driven only by single calls."""
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
        hints = np.stack([d[2][k] for d in data])
        P, Cv, U = group.slam_update(hints, [d[1][k] for d in data], nowait=True)
        for s in range(M):
            p, c, u = one_reps[s].slam_update(hints[s], data[s][1][k])
            assert np.array_equal(P[s], p) and np.array_equal(Cv[s], c) and U[s] == u, (k, s)
        if k % 4 == 1:   # a single step on a member right after the group step
            h = data[0][0][k]
            x = grp_reps[0].slam_update(h, data[0][1][k], nowait=True)
            y = one_reps[0].slam_update(h, data[0][1][k])
            assert all(np.array_equal(u, v) for u, v in zip(x, y)), k
        if k == 6:
            grp_reps[1].reset()
            one_reps[1].reset()
        if k % 3 == 2:
            assert np.array_equal(batch(grp_reps[2], data[2][0][k], data[2][1][k]),
                                  batch(one_reps[2], data[2][0][k], data[2][1][k])), k
        if k % 4 == 3:
            assert np.array_equal(grp_reps[3].download_occupancy(0), one_reps[3].download_occupancy(0)), k
        if k == 9:
            grp_reps[1].updateByScan(data[1][1][k], data[1][0][k])
            one_reps[1].updateByScan(data[1][1][k], data[1][0][k])
    for s in range(M):
        assert_same_state(grp_reps[s], one_reps[s], s)
    group.close()
    close_all(grp_reps, one_reps)


def test_validation(hsb_lib):
    import torch

    from hector_slam_b200 import capi

    a, b = make_rep(0), make_rep(1)
    bad = [capi.MapRepB200(RES, SIZE // 2, levels=LEVELS), capi.MapRepB200(RES, SIZE, levels=2),
           capi.MapRepB200(RES * 2, SIZE, levels=LEVELS), capi.MapRepB200(RES, SIZE, levels=LEVELS, start=(0.4, 0.5)),
           capi.MapRepB200(RES, SIZE, levels=LEVELS, max_iterations=[6, 0, 0]),
           capi.MapRepB200(RES, SIZE, levels=LEVELS, gather_mode=capi.GATHER_LDG)]
    assert a.gather_mode == capi.GATHER_TEX
    for r in bad:
        with pytest.raises(capi.HsbError) as e:
            capi.SlamGroup([a, r])
        assert e.value.status == -1 and "differs" in str(e.value)
    for reps in ([], [a, b, a], [a, None]):
        with pytest.raises(capi.HsbError) as e:
            capi.SlamGroup(reps)
        assert e.value.status == -1
    g = capi.SlamGroup([a, b])
    scan = session_data(3, 1)[1][0]
    n = scan.shape[0]
    for offs in ([1, n, 2 * n], [0, n, n - 1], [0, 2 * n, n]):
        with pytest.raises(capi.HsbError) as e:
            g.slam_update(np.zeros((2, 3), np.float32), (np.concatenate([scan, scan]), np.array(offs, np.int32)))
        assert e.value.status == -1
    P, _, _ = g.slam_update(np.zeros((2, 3), np.float32), [scan, scan])   # the group still works
    assert np.all(np.isfinite(P))
    g.close()
    if torch.cuda.device_count() >= 2:
        c = make_rep(0, device=1)
        with pytest.raises(capi.HsbError) as e:
            capi.SlamGroup([a, c])
        assert e.value.status == -1
        c.close()
    close_all(bad, [a, b])


@pytest.mark.parametrize("M", [1, 16])
def test_launch_count(hsb_lib, M):
    """A group step is three launches, counted on handles[0]; the other members' counts do not move."""
    from hector_slam_b200 import capi

    reps = [make_rep(s) for s in range(M)]
    group = capi.SlamGroup(reps)
    data = [session_data(90 + s, 2) for s in range(M)]
    for k in range(2):
        before = [r.launch_count for r in reps]
        group.slam_update(np.stack([d[2][k] for d in data]), [d[1][k] for d in data], nowait=(k == 1))
        after = [r.launch_count for r in reps]
        assert after[0] - before[0] == 3, (before[0], after[0])
        assert after[1:] == before[1:]
    group.close()
    close_all(reps)


def test_facade_update_many(hsb_lib):
    """hsb200::SlamProcessor::updateMany (C++ façade, through its shim) equals update() per processor: poses,
    covariances and maps."""
    L = C.CDLL(os.path.join(ROOT, "hector_slam_b200", "lib", "libhsb200_host.so"))
    L.hsbp_create.restype = C.c_void_p
    L.hsbp_create.argtypes = [C.c_float, C.c_int, C.c_int, C.c_float, C.c_float, C.c_int, C.c_int]
    L.hsbp_destroy.argtypes = [C.c_void_p]
    L.hsbp_update.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    L.hsbp_update_many.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.hsbp_get_pose_and_cov.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.hsbp_get_grid_map.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    M, steps = 3, 8
    data = [session_data(110 + s, steps) for s in range(M)]
    many = [L.hsbp_create(RES, SIZE, SIZE, 0.5, 0.5, LEVELS, 0) for _ in range(M)]
    one = [L.hsbp_create(RES, SIZE, SIZE, 0.5, 0.5, LEVELS, 0) for _ in range(M)]
    assert all(many) and all(one)
    arr = (C.c_void_p * M)(*many)
    for k in range(steps):
        scans = [d[1][k] for d in data]
        pts = np.ascontiguousarray(np.concatenate(scans), np.float32)
        offs = np.zeros(M + 1, np.int32)
        offs[1:] = np.cumsum([x.shape[0] for x in scans])
        hints = np.ascontiguousarray(np.stack([d[2][k] for d in data]), np.float32)
        mwm = np.array([0, int(k % 3 == 2), 0], np.int32)
        assert L.hsbp_update_many(C.cast(arr, C.c_void_p), M, pts.ctypes.data, offs.ctypes.data, None, hints.ctypes.data,
                                  mwm.ctypes.data) == 0
        for s in range(M):
            p1, c1, p2, c2 = (np.zeros(3, np.float32), np.zeros(9, np.float32), np.zeros(3, np.float32),
                              np.zeros(9, np.float32))
            scan = np.ascontiguousarray(scans[s])
            assert L.hsbp_update(one[s], scan.ctypes.data, scan.shape[0], None, hints[s].ctypes.data, int(mwm[s]),
                                 p2.ctypes.data, c2.ctypes.data) == 0
            L.hsbp_get_pose_and_cov(many[s], p1.ctypes.data, c1.ctypes.data)
            assert np.array_equal(p1, p2) and np.array_equal(c1, c2), (k, s)
    for s in range(M):
        for l in range(LEVELS):
            sz = SIZE >> l
            x, y = np.zeros((sz, sz), np.float32), np.zeros((sz, sz), np.float32)
            assert L.hsbp_get_grid_map(many[s], l, x.ctypes.data) == 0
            assert L.hsbp_get_grid_map(one[s], l, y.ctypes.data) == 0
            assert np.array_equal(x, y), (s, l)
    for p in many + one:   # any member first: its cached group goes with it
        L.hsbp_destroy(p)
