"""CPU: the oracles against the golden vectors generated from the compiled reference
(oracle/gen_golden.py).  The plain-C port must reproduce them BIT FOR BIT; where the compiled
reference itself is present (oracle/_ref) it is re-run too, which also guards the fixtures."""
import numpy as np
import pytest

from conftest import apply_diff, golden_planes, load_golden


def make(pyoracle, kind, g):
    o = pyoracle.Oracle(kind, float(g["res"]), int(g["size"]), int(g["levels"]))
    if "factors" in g.files:
        o.set_update_factors(float(g["factors"][0]), float(g["factors"][1]))
    return o


def set_planes(o, planes):
    for l, p in enumerate(planes):
        o.set_logodds(l, p)


@pytest.mark.parametrize("name", ["match3.npz", "match1.npz"])
def test_match_goldens_bit_exact(pyoracle, oracle_kinds, name):
    g = load_golden(name)
    for kind in oracle_kinds:
        o = make(pyoracle, kind, g)
        set_planes(o, golden_planes(g))
        for k in range(g["scans"].shape[0]):
            p, c = o.match(g["hints"][k], g["scans"][k])
            assert np.array_equal(p, g["ref_poses"][k]), (kind, k)
            assert np.array_equal(c.reshape(9), g["ref_cov"][k]), (kind, k)
        # matches land within 1.5 cm / 2 mrad of the synthetic ground truth (noise sigma 1 cm)
        assert np.abs(g["ref_poses"][:, :2] - g["truth"][:, :2]).max() < 0.015
        o.close()


def test_three_evaluation_variant(pyoracle, oracle_kinds):
    """BASELINE.json config 1's "3 GN iters": ScanMatcher::matchData(maxIterations=2)."""
    g = load_golden("match1.npz")
    for kind in oracle_kinds:
        o = make(pyoracle, kind, g)
        set_planes(o, golden_planes(g))
        for k in range(g["scans"].shape[0]):
            p, c = o.match_level(0, g["hints"][k], g["scans"][k], 2)
            assert np.array_equal(p, g["ref_poses_3eval"][k])
            assert np.array_equal(c.reshape(9), g["ref_cov_3eval"][k])
        o.close()


def test_per_evaluation_hessians(pyoracle, oracle_kinds):
    g = load_golden("match3.npz")
    for kind in oracle_kinds:
        o = make(pyoracle, kind, g)
        set_planes(o, golden_planes(g))
        for i in range(len(g["ev_level"])):
            l, k = int(g["ev_level"][i]), int(g["ev_scan"][i])
            pts = (g["scans"][k] * np.float32(2.0 ** -l)).astype(np.float32)
            H, d = o.hessian_derivs(l, g["ev_pose"][i], pts)
            assert np.array_equal(H.reshape(9), g["ev_H"][i])
            assert np.array_equal(d, g["ev_dTr"][i])
        # pose conversions (GridMapBase.h:226-239) and log-odds increments (GridMapLogOdds.h:187-203)
        for k in range(4):
            for l in range(3):
                m = o.map_coords_pose(l, g["conv_world"][k])
                assert np.array_equal(m, g["conv_map"][k, l])
                assert np.array_equal(o.world_coords_pose(l, m), g["conv_back"][k, l])
        assert np.array_equal(o.logodds_increments(), g["increments"])
        assert np.allclose(g["increments"], [-0.405465156, 2.19722438], rtol=0, atol=1e-7)
        o.close()


def test_interpolation_bounds_and_single_steps(pyoracle, oracle_kinds):
    g = load_golden("interp.npz")
    for kind in oracle_kinds:
        o = pyoracle.Oracle(kind, float(g["res"]), int(g["size"]), int(g["levels"]))
        for l in range(int(g["levels"])):
            o.set_logodds(l, g[f"plane{l}"])
            assert np.array_equal(o.get_prob(l), g[f"prob{l}"])
        for i in range(len(g["ev_level"])):
            l = int(g["ev_level"][i])
            H, d = o.hessian_derivs(l, g["ev_pose"][i], g["ev_pts"][i])
            assert np.array_equal(H.reshape(9), g["ev_H"][i])
            assert np.array_equal(d, g["ev_dTr"][i])
            p, _ = o.match_level(l, g["step_hint"][i], g["ev_pts"][i], 0)
            assert np.array_equal(p, g["step_pose"][i])
        o.close()
    # the fixtures do exercise the rotation clamp (ScanMatcher.h:209-215)
    dpsi = g["step_pose"][:, 2] - g["step_hint"][:, 2]
    assert np.sum(g["step_clamped"]) >= 3
    assert np.all(np.abs(np.abs(dpsi[g["step_clamped"]]) - 0.2) < 1e-5)


def test_map_update_goldens(pyoracle, oracle_kinds):
    g = load_golden("match3.npz")
    for kind in oracle_kinds:
        o = make(pyoracle, kind, g)
        base = golden_planes(g)
        set_planes(o, base)
        o.match(g["hints"][0], g["scans"][0])
        o.update_by_scan(g["scans"][0], g["upd1_pose"])
        o.on_map_updated()
        want1 = apply_diff(base, g, "upd1")
        for l in range(3):
            assert np.array_equal(o.get_logodds(l), want1[l]), (kind, l)
        o.match(g["hints"][1], g["scans"][1])
        o.update_by_scan(g["scans"][2], g["upd2_pose"])
        o.on_map_updated()
        want2 = apply_diff(want1, g, "upd2")
        for l in range(3):
            assert np.array_equal(o.get_logodds(l), want2[l]), (kind, l)
        p, c = o.match(g["hints"][3], g["scans"][3])
        assert np.array_equal(p, g["after_upd_pose"])
        assert np.array_equal(c.reshape(9), g["after_upd_cov"])
        o.close()


def test_edge_cases(pyoracle, oracle_kinds):
    g = load_golden("match1.npz")
    for kind in oracle_kinds:
        o = make(pyoracle, kind, g)
        set_planes(o, golden_planes(g))
        cov_in = np.arange(9, dtype=np.float32)
        p, c = o.match(g["hints"][0], np.zeros((0, 2), np.float32), cov_in=cov_in)
        assert np.array_equal(p, g["hints"][0]) and np.array_equal(c.reshape(9), cov_in)  # ScanMatcher.h:68,189
        far = (g["scans"][0] + np.float32(1e5)).astype(np.float32)
        p, c = o.match(g["hints"][0], far)
        assert np.array_equal(p, g["edge_far_pose"]) and np.all(c == 0)
        assert np.abs(p - g["hints"][0]).max() < 1e-5  # only the world->map->world round trip
        o.close()


def test_slam_run_matches_golden(pyoracle, oracle_kinds):
    """HectorSlamProcessor::update over a short trajectory starting on an empty map (Q12)."""
    g = load_golden("slam3.npz")
    for kind in oracle_kinds:
        o = make(pyoracle, kind, g)
        o.set_map_update_thresholds(0.0, 0.0)
        hint = g["first_hint"]
        for k in range(g["scans"].shape[0]):
            pose, _ = o.update(g["scans"][k], hint)
            assert np.array_equal(pose, g["est"][k]), (kind, k)
            hint = pose
        final = golden_planes(g, "final")
        for l in range(3):
            assert np.array_equal(o.get_logodds(l), final[l])
        assert np.abs(g["est"][:, :2] - g["traj"][:, :2]).max() < 0.02
        o.close()


def test_port_equals_reference_on_fresh_inputs(pyoracle, oracle_kinds):
    """Beyond the fixtures: a fresh seeded world, both oracles, bit-for-bit (needs oracle/_ref)."""
    if "reference" not in oracle_kinds:
        pytest.skip("compiled reference (oracle/_ref/libhsref.so) not present")
    from hector_slam_b200 import synth

    world = synth.World(1, seed=77)
    rng = np.random.default_rng(3)
    poses = world.sample_free_poses(24, rng)
    pts, offs = synth.make_scan_batch(world, poses, noise_seed=9)
    hints = synth.perturb_hints(poses, seed=4)
    res = []
    for kind in ("reference", "port"):
        o = pyoracle.Oracle(kind, 0.05, 1024, 3)
        o.set_update_factors(0.4, 0.9)
        pyoracle.build_map_known_poses(o, world)
        P, Cv, _ = o.match_batch(hints, pts, offs, nthreads=1)
        P2, _, _ = o.match_batch(hints, pts, offs, nthreads=3)
        assert np.array_equal(P, P2)
        res.append((P, Cv, [o.get_logodds(l) for l in range(3)]))
        o.close()
    assert np.array_equal(res[0][0], res[1][0]) and np.array_equal(res[0][1], res[1][1])
    for l in range(3):
        assert np.array_equal(res[0][2][l], res[1][2][l])


def test_reference_sensitivity_on_a_sparse_map(pyoracle, oracle_kinds):
    """How much the REFERENCE's own answer moves under mathematically irrelevant changes on the first steps of a
    SLAM stream (map written once or twice, i.e. sparse): (a) the scan's points summed in reverse / rotated order,
    (b) the hint moved by 3e-5 (m, m, rad).  Measured with the compiled reference: on this 2048^2 stream most steps
    are bit-stable, but several move by 1e-4 .. 4e-4 — bilinear interpolation makes the objective piecewise, a
    last-bit difference can tip an endpoint into the neighbouring cell, and 14 evaluations do not always reach the
    fixed point on a one-scan map.  So the 1e-4 parity bar of the GPU tests is, on sparse maps, tighter than the
    reference's own reproducibility; that the GPU stream tests pass it is a property of the shipped reduction order
    (DESIGN.md, "A finding about parity on sparse maps").  This test pins the fact, with the oracle only."""
    from hector_slam_b200 import synth

    size = 2048
    world = synth.World.for_map_size(size)
    orc = pyoracle.Oracle(oracle_kinds[0], 0.05, size, 3)
    orc.set_update_factors(0.4, 0.9)
    orc.set_map_update_thresholds(0.4, 0.9)
    pose = np.array([3.0, 2.0, 0.1])
    rng = np.random.default_rng(5)
    hint = pose.astype(np.float32)
    order, hintsens = [], []
    for k in range(36):
        scan = np.ascontiguousarray(synth.make_scan(world, pose, rng))
        fwd, _ = orc.match(hint, scan)
        rev, _ = orc.match(hint, np.ascontiguousarray(scan[::-1]))
        rot, _ = orc.match(hint, np.ascontiguousarray(np.roll(scan, 137, axis=0)))
        per, _ = orc.match((hint + np.array([3e-5, -3e-5, 3e-5], np.float32)).astype(np.float32), scan)
        order.append(float(max(np.abs(fwd - rev).max(), np.abs(fwd - rot).max())))
        hintsens.append(float(np.abs(per - fwd).max()))
        hint, _ = orc.update(scan, hint)
        h = pose[2]
        pose = pose + np.array([0.0125 * np.cos(h), 0.0125 * np.sin(h), 0.0075])
    orc.close()
    order, hintsens = np.asarray(order), np.asarray(hintsens)
    assert np.median(order) <= 1e-6                         # most steps: order does not matter at all
    assert max(order.max(), hintsens.max()) >= 1e-4         # some steps: the reference itself moves past the bar
    assert max(order.max(), hintsens.max()) <= 2e-3         # ... but not arbitrarily far


def test_covariance_and_map_tools_port_equals_reference(pyoracle, oracle_kinds):
    """The "next" rows the port restates — sigma-point covariance (OccGridMapUtil.h:106-187) and hector_map_tools'
    ray cast / getDist (HectorMapTools.h:133-237) — against the reference headers compiled in oracle/_ref: bit-exact."""
    if "reference" not in oracle_kinds:
        pytest.skip("oracle/_ref not built here")
    g = load_golden("match3.npz")
    port, ref = make(pyoracle, "port", g), make(pyoracle, "reference", g)
    set_planes(port, golden_planes(g))
    set_planes(ref, golden_planes(g))
    for k in range(0, g["scans"].shape[0], 3):
        for l in range(int(g["levels"])):
            pm = port.map_coords_pose(l, g["ref_poses"][k])
            pts = (g["scans"][k] * np.float32(2.0 ** -l)).astype(np.float32)
            a, b = port.covariance_for_pose(l, pm, pts), ref.covariance_for_pose(l, pm, pts)
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
            assert a[0][0, 0] > 0 and np.array_equal(a[1], a[1].T)
    rng = np.random.default_rng(0)
    size = int(g["size"])
    for l in range(int(g["levels"])):
        lo = port.get_logodds(l)
        occ = np.where(lo < 0, 0, np.where(lo > 0, 100, -1)).astype(np.int8)   # publishMap, HectorMappingRos.cpp:448-468
        mt = pyoracle.RefMapTools(occ, port.cell_length(l), port.map_origin(l))
        s = size >> l
        hits = 0
        for _ in range(1500):
            b, e = rng.integers(-5, s + 5, 2), rng.integers(-5, s + 5, 2)
            assert port.raycast(l, b, e) == mt.raycast(b, e)
            bw, ew = rng.uniform(-14, 14, 2).astype(np.float32), rng.uniform(-14, 14, 2).astype(np.float32)
            a, r = port.get_dist(l, bw, ew), mt.get_dist(bw, ew)
            assert a[0] == r[0] and a[2] == r[2] and np.array_equal(a[1], r[1])
            hits += a[2]
        assert hits > 50
        mt.close()
    port.close()
    ref.close()


def test_next_rows_goldens_bit_exact(pyoracle):
    """tests/golden/next.npz (generated from the compiled reference: node converter source text, OccGridMapUtil.h,
    HectorMapTools.h): the C port reproduces every vector bit for bit on any machine."""
    from hector_slam_b200 import synth

    g, m = load_golden("next.npz"), load_golden("match3.npz")
    fmt = synth.CLOUD_FORMAT
    co, ko = g["cloud_offsets"], g["cloud_kept_offsets"]
    for k in range(len(co) - 1):
        pts, og = pyoracle.cloud_to_points(g["cloud_xyz"][co[k]:co[k + 1]], g["cloud_T"][k], fmt["sqr_laser_min_dist"],
                                           fmt["sqr_laser_max_dist"], fmt["laser_z_min_value"], fmt["laser_z_max_value"], 20.0)
        assert np.array_equal(pts, g["cloud_kept"][ko[k]:ko[k + 1]]) and np.array_equal(og, g["cloud_origo"][k])
    o = make(pyoracle, "port", m)
    set_planes(o, golden_planes(m))
    for l in range(3):
        for k in range(m["scans"].shape[0]):
            a, b = o.covariance_for_pose(l, o.map_coords_pose(l, m["ref_poses"][k]),
                                         (m["scans"][k] * np.float32(2.0 ** -l)).astype(np.float32))
            assert np.array_equal(a, g["cov_map"][l, k]) and np.array_equal(b, g["cov_world"][l, k])
    assert np.array_equal(o.map_origin(0), g["map_origin"])
    for i in range(len(g["ray_dist"])):
        d, h = o.raycast(0, g["ray_begin"][i], g["ray_end"][i])
        assert d == g["ray_dist"][i] and h == tuple(g["ray_hit"][i])
        d, hw, f = o.get_dist(0, g["gd_begin"][i], g["gd_end"][i])
        assert np.float32(d) == g["gd_dist"][i] and f == bool(g["gd_found"][i]) and np.array_equal(hw, g["gd_hit"][i])
    o.close()


def test_deep_golden_bit_exact(pyoracle):
    """tests/golden/deep.npz (oracle/gen_golden.py deep, from the compiled reference): a 14-step SLAM run with three
    map_without_matching steps on a 1000 x 640 x 8 and a 2048 x 2048 x 5 map, then matchData on the final maps under the
    default and the mixed iteration schedule with the matcher's hook reports.  The C port reproduces every array bit
    for bit on any machine: run poses and covariances, all 13 planes, match poses, covariances and hooks."""
    import subprocess

    from conftest import ROOT
    from oracle import gen_golden, record_oracle

    if not record_oracle.available("port"):
        subprocess.run(["make", "-C", f"{ROOT}/oracle", "-f", "record.mk", "port"], check=True, capture_output=True)
    want, got = load_golden("deep.npz"), gen_golden.deep_arrays("port")
    assert sorted(want.files) == sorted(got)
    for k in want.files:
        a, b = want[k], np.asarray(got[k])
        assert a.shape == b.shape and a.dtype == b.dtype, k
        if a.dtype == np.float32:
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), k
        else:
            assert np.array_equal(a, b), k
    for tag, g in gen_golden.DEEP_GEOMS.items():
        L = g[2]
        assert all(np.any(want[f"{tag}_final{l}"] != 0) for l in range(L)), tag       # every level was written
        assert not np.array_equal(want[f"{tag}_default_poses"], want[f"{tag}_mixed_poses"]), tag
    # the 5-level run tracks the path it was simulated on (noise sigma 1 cm).  (The 8-level one does not: its coarsest
    # levels, 7 x 5 cells of 6.4 m, throw the reference's matcher off: see oracle/gen_golden.py deep_run.)
    traj = gen_golden.deep_run(gen_golden.DEEP_GEOMS["g5"])[3]
    assert np.abs(want["g5_run_est"][:, :2] - traj[:, :2]).max() < 0.02
    assert np.abs(want["g5_default_poses"] - want["g5_match_hints"]).max() < 0.15
