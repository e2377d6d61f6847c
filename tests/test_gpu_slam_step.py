"""hsb_slam_update — HectorSlamProcessor::update (slam_main/HectorSlamProcessor.h:71-113) as one stream-ordered
call — against (1) the same step driven from the host through hsb_match_data / hsb_update_by_scan (bit-identical
poses, flags and planes) and (2) the oracle's update(), with the gate active and with map_without_matching.
Also the map writer on maps whose coarse levels have rows that are not 16-byte multiples (scalar sweep)."""
import numpy as np
import pytest

from conftest import load_golden, pose_err
from oracle import pose32

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("thresholds", [(0.0, 0.0), (0.35, 0.05)])
def test_fused_equals_host_driven_step(hsb_lib, thresholds):
    from hector_slam_b200 import capi

    g = load_golden("slam3.npz")
    res, size = float(g["res"]), int(g["size"])
    dist, ang = thresholds
    fused = capi.MapRepB200(res, size, levels=3, update_factor_free=0.4, update_factor_occupied=0.9)
    plain = capi.MapRepB200(res, size, levels=3, update_factor_free=0.4, update_factor_occupied=0.9)
    fused.setMapUpdateMinDistDiff(dist)
    fused.setMapUpdateMinAngleDiff(ang)
    assert np.all(fused.last_map_update_pose() == np.finfo(np.float32).max)
    last = np.full(3, np.finfo(np.float32).max, np.float32)
    hint_f = g["first_hint"].copy()
    hint_p = g["first_hint"].copy()
    n_upd = 0
    for k in range(g["scans"].shape[0]):
        scan = g["scans"][k]
        pf, cf, uf = fused.slam_update(hint_f, scan)
        pp, cp = plain.matchData(hint_p, scan)
        up = pose32.pose_difference_larger_than(pp, last, dist, ang)
        if up:
            plain.updateByScan(scan, pp)
            plain.onMapUpdated()
            last = pp.copy()
        assert np.array_equal(pf, pp), (k, pf, pp)
        assert np.array_equal(cf, cp), k
        assert uf == up, (k, uf, up)
        n_upd += int(uf)
        hint_f, hint_p = pf, pp
    assert np.array_equal(fused.last_map_update_pose(), last)
    if dist > 0:
        assert 0 < n_upd < g["scans"].shape[0]   # the gate is really exercised
    for l in range(3):
        assert np.array_equal(fused.download_level(l), plain.download_level(l)), l
        assert np.array_equal(fused.download_prob(l), plain.download_prob(l)), l
    fused.reset()
    assert np.all(fused.last_map_update_pose() == np.finfo(np.float32).max)
    fused.close()
    plain.close()


def test_fused_against_oracle_with_map_without_matching(hsb_lib, pyoracle):
    """Scans alternate between matched steps and map_without_matching steps at the golden estimate: the latter
    write level 0 from the new scan and the coarse levels from the containers of the last MATCHED scan (Q11)."""
    from hector_slam_b200 import capi

    g = load_golden("slam3.npz")
    res, size = float(g["res"]), int(g["size"])
    rep = capi.MapRepB200(res, size, levels=3, update_factor_free=0.4, update_factor_occupied=0.9)
    orc = pyoracle.Oracle("port", res, size, 3)
    orc.set_update_factors(0.4, 0.9)
    for d, a in ((0.2, 0.03),):
        rep.setMapUpdateMinDistDiff(d)
        rep.setMapUpdateMinAngleDiff(a)
        orc.set_map_update_thresholds(d, a)
    hint_g = g["first_hint"].copy()
    hint_o = g["first_hint"].copy()
    for k in range(g["scans"].shape[0]):
        scan = g["scans"][k]
        without = (k % 4 == 3)
        if without:
            hint_g = g["est"][k].copy()
            hint_o = g["est"][k].copy()
        pose, _, upd = rep.slam_update(hint_g, scan, map_without_matching=without)
        want, _ = orc.update(scan, hint_o, map_without_matching=without)
        ex, ey, ea = pose_err(pose, want)
        assert max(ex, ey) <= 1e-4 and ea <= 1e-4, (k, ex, ey, ea)
        if without:
            assert upd and np.array_equal(pose, hint_g)
        hint_g, hint_o = pose, want
    for l in range(3):
        got, ref = rep.download_level(l), orc.get_logodds(l)
        diff = np.abs(got - ref)
        assert (diff > 1e-5).sum() <= max(3, int(2e-3 * (got != 0).sum())), (l, int((diff > 1e-5).sum()))
    rep.close()
    orc.close()


def test_empty_scan_step(hsb_lib):
    from hector_slam_b200 import capi

    rep = capi.MapRepB200(0.05, 256, levels=2)
    cov0 = np.arange(9, dtype=np.float32)
    pose, cov, upd = rep.slam_update([0.3, -0.2, 0.1], np.zeros((0, 2), np.float32), cov_inout=cov0)
    assert np.array_equal(pose, np.array([0.3, -0.2, 0.1], np.float32))   # ScanMatcher.h:68: the hint comes back
    assert np.array_equal(cov.reshape(9), cov0)                            # untouched
    assert upd                                                             # FLT_MAX gate fires, nothing to write
    assert np.all(rep.download_level(0) == 0)
    rep.close()


@pytest.mark.parametrize("size", [250, 1000])
def test_map_writer_on_unaligned_rows(hsb_lib, pyoracle, size):
    """size 250 -> coarse level 125 (scalar sweep); size 1000 -> 500 / 250 (vector, vector, scalar)."""
    from hector_slam_b200 import capi, synth

    levels = 3
    res = 50.0 / size   # the synthetic room (ROOM_W x ROOM_D metres) must fit the map
    rep = capi.MapRepB200(res, size, levels=levels, update_factor_free=0.4, update_factor_occupied=0.9)
    orc = pyoracle.Oracle("port", res, size, levels)
    orc.set_update_factors(0.4, 0.9)
    world = synth.World(1, seed=5)
    rng = np.random.default_rng(3)
    scale = 1.0 / res
    for k in range(6):
        pose = np.array([rng.uniform(-3, 3), rng.uniform(-3, 3), rng.uniform(-3, 3)], np.float32)
        scan = synth.make_scan(world, pose, rng, scale_to_map=scale)
        rep.matchData(pose, scan)      # fills the coarse containers on both sides
        orc.match(pose, scan)
        rep.updateByScan(scan, pose)
        orc.update_by_scan(scan, pose)
        rep.onMapUpdated()
        orc.on_map_updated()
    for l in range(levels):
        got, ref = rep.download_level(l), orc.get_logodds(l)
        assert (got != 0).sum() > 0
        diff = np.abs(got - ref)
        assert (diff > 1e-5).sum() <= max(3, int(2e-3 * (got != 0).sum())), (size, l, int((diff > 1e-5).sum()))
    rep.close()
    orc.close()


def test_nowait_step_equals_the_synchronous_step(hsb_lib):
    """hsb_slam_update_nowait returns when the pose has arrived and leaves the map write on the stream: the whole run —
    poses, gate decisions, final planes — must equal the synchronous call's, also when a batch match on other streams
    follows a step immediately (it has to wait for the pending map write)."""
    from hector_slam_b200 import capi

    g = load_golden("slam3.npz")

    def run(nowait):
        rep = capi.MapRepB200(float(g["res"]), int(g["size"]), levels=3, update_factor_free=0.4, update_factor_occupied=0.9)
        rep.setMapUpdateMinDistDiff(0.2)     # the trajectory advances 0.155 m per scan: the gate fires every other step
        rep.setMapUpdateMinAngleDiff(0.9)
        hint, traj, flags, probes = g["first_hint"], [], [], []
        for k in range(g["scans"].shape[0]):
            hint, cov, upd = rep.slam_update(hint, g["scans"][k], nowait=nowait)
            traj.append(hint)
            flags.append(upd)
            if k % 3 == 2:   # a batch call straight after the step: sees the map INCLUDING this step's write
                P, _ = rep.match_batch(np.repeat(hint[None], 4, axis=0), g["scans"][k], None)
                probes.append(P[0])
        rep.onMapUpdated()
        planes = [rep.download_level(l) for l in range(3)]
        rep.close()
        return np.asarray(traj), flags, np.asarray(probes), planes

    a, b = run(False), run(True)
    assert np.array_equal(a[0], b[0]) and a[1] == b[1] and np.array_equal(a[2], b[2])
    assert any(a[1]) and not all(a[1])
    for l in range(3):
        assert np.array_equal(a[3][l], b[3][l])


def test_scan_inside_the_launch_equals_the_copy_path(hsb_lib):
    """Single-scan calls send the scan inside the kernel parameters (tuning key inline_scan, default on, scans of up to
    1280 endpoints): poses, covariances, gate decisions and planes of a SLAM run must equal the host-to-device-copy
    path's bit for bit — through hsb_slam_update (sync and nowait), through hsb_match_data + hsb_update_by_scan (the
    kernel has to leave the endpoints on the device for the coarse levels), with an empty scan and with a scan too long
    to be inlined in between."""
    from hector_slam_b200 import capi

    g = load_golden("slam3.npz")
    long_scan = np.concatenate([g["scans"][0], g["scans"][1]]).astype(np.float32)   # 2162 endpoints: copy path in both

    def run(inline, mode):
        rep = capi.MapRepB200(float(g["res"]), int(g["size"]), levels=3, update_factor_free=0.4, update_factor_occupied=0.9)
        rep.set_tuning(inline_scan=inline)
        rep.setMapUpdateMinDistDiff(0.2)
        rep.setMapUpdateMinAngleDiff(0.9)
        hint, out = g["first_hint"], []
        for k in range(g["scans"].shape[0]):
            scan = g["scans"][k]
            if k == 5:
                scan = long_scan
            if k == 7:
                scan = np.zeros((0, 2), np.float32)
            if mode == "host":
                p, c = rep.matchData(hint, scan)
                rep.updateByScan(scan, p)
                rep.onMapUpdated()
                out.append((p, c, True))
            else:
                p, c, u = rep.slam_update(hint, scan, nowait=(mode == "nowait"))
                out.append((p, c, u))
            hint = p
        rep.onMapUpdated()
        planes = [rep.download_level(l) for l in range(3)]
        launches = rep.launch_count
        rep.close()
        return out, planes, launches

    for mode in ("sync", "nowait", "host"):
        a, pa, la = run(1, mode)
        b, pb, lb = run(0, mode)
        for k, (x, y) in enumerate(zip(a, b)):
            assert np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]) and x[2] == y[2], (mode, k, x, y)
        for l in range(3):
            assert np.array_equal(pa[l], pb[l]), (mode, l)
        assert la == lb   # same kernels either way: only the copy operation is gone
