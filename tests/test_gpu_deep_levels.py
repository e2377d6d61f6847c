"""GPU: handles of four to eight levels (tests/deep_cases.py) through the entry points whose per-level arrays only such
handles index beyond entry 2: the match kernel's level descriptors and record offsets, the map writer's level grid,
the group's members x levels tables, the tile header's eight rectangles, the dirty-rectangle block, pt_scale = 2^-l
for l >= 3 and the coarse last-match containers.  Both gather modes unless noted.

  * geometry: level sizes, origins and both pose conversions on every level equal the C port's bit for bit; the record
    size is the sum of 3 + 15 evaluations under every schedule; one cell below the minimum hsb_create refuses.
  * match: at W = 1, 2, 4, 8 and the auto shape, through the batch and the single-scan entry, every recorded H / dTr
    on every level lies within tests/test_gpu_match_record.py's float64 bound at the device's own pose, every estimate
    is pose32.step of the one before, every hand-off is the port's conversion bit for bit, the designed edge endpoints
    are classified as built on every level, TEX == LDG, and the record and `fixpoint` change no result bit; an empty
    scan fills every level's start pose; a 4096-scan batch in the launcher's own shape equals its scans matched alone.
  * golden: poses and covariances on deep.npz's final maps against the compiled reference's, 1e-4 m / rad and 1e-3
    relative, where the reference's own path is well conditioned (all of the 5-level map's matches).
  * input kinds: ranges, clouds and projected scans match as their converted endpoints do, bit for bit.
  * map writer: hsb_update_level_by_scan on each level, hsb_update_by_scan after a match and after a
    map_without_matching step (the stale container scaled by up to 2^-7), every cell against oracle/mapwrite.py, the
    probability plane against libm expf, the dirty rectangles of all levels, the texture twin by one-endpoint
    likelihoods, beams that collapse on the coarse levels, and two launches per write at any depth.
  * steps: a 20-step run through hsb_slam_update / _nowait equals matchData + updateByScan + onMapUpdated, poses,
    gate decisions and planes bit for bit; a group of five 8-level handles stepped whole and by subsets with mixed
    map_without_matching equals the single steps; a group refuses members that differ in levels or in
    max_iterations[5] only.
  * scoring, queries, export on levels 3..7: ray casts, getDist and occupancy equal the port's bit for bit; the group
    forms of likelihood, covariance, best hypothesis, getDist, ray cast, occupancy and batch match equal the single
    calls; level == levels and level == -1 are refused.
  * tile transport between two 8-level handles: header (level count, eight rectangles, cell total), the replica's
    planes and mirror rectangles, the overflow path one row short, and the two-step rectangle path on levels 3..7.
  * planes: upload / download / probability / refresh round trips on each level, hsb_reset clears all.
  * trace: refused on 5..8 levels, accepted on 4, where it changes no bit and its slots are ordered times.
"""
import math

import numpy as np
import pytest

import deep_cases as dc
import maptools_cases as mtc
import match_cases as mcs
from conftest import load_golden, report
from oracle import gen_golden, mapwrite as mw, pose32, record_oracle
from oracle.likelihood64 import same_bits_or_nan
from test_gpu_map_write import Pair, level_scans, scan_for, write_all
from test_gpu_match_geometry import RESET, batch_record, check_sums, scaled_cond
from test_gpu_match_record import port_record  # noqa: F401 (a fixture)

pytestmark = pytest.mark.gpu

f32 = np.float32
MODES = (1, 2)   # LDG, TEX
G8 = dc.GEOMS[0]
_SETUPS = {}
_WORST = {}


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def same(a, b):
    return np.array_equal(bits(a), bits(b))


def make_rep(g, mode=0, iters=None, **kw):
    from hector_slam_b200 import capi

    sx, sy, L, start, res = g
    return capi.MapRepB200(res, sx, sy, levels=L, start=start, gather_mode=mode, max_iterations=iters, **kw)


def make_port(g):
    sx, sy, L, start, res = g
    return record_oracle.RecordOracle("port", res, sx, L, start=start, size_y=sy)


class Setup:
    """match_cases.field planes on an LDG and a TEX handle under one schedule and under the edge scans' schedule, the C
    port with the same planes, and deep_cases.designed_scans built with the device as the matcher."""

    def __init__(self, gi, sched):
        g = dc.GEOMS[gi]
        self.g, self.levels, self.iters = g, g[2], dc.schedule(sched, g[2])
        self.family = f"deep {dc.IDS[gi]}-{sched}"
        self.reps = {m: make_rep(g, m, self.iters) for m in MODES}
        self.edge_reps = {m: make_rep(g, m, mcs.edge_iterations(g[2])) for m in MODES}
        self.port = make_port(g)
        dc.set_fields(g, self.port, *self.reps.values(), *self.edge_reps.values())
        self.prob = [self.reps[1].download_prob(l) for l in range(self.levels)]
        for l in range(self.levels):
            assert same(self.prob[l], self.reps[2].download_prob(l)) and same(self.prob[l], self.port.get_prob(l)), l
        self.cases = mcs.Cases(g, self.prob, self.port, seed=300 + gi)
        rep = self.edge_reps[1]

        def runner(hint, pts):
            rep.set_tuning(**RESET)
            return rep.matchData(hint, pts, record=True)[2]

        scans, self.designed, self.edge_index = dc.designed_scans(g, self.cases, runner)
        if not dc.has_edges(g):
            # on a 4-cell level a singular solve can make the pose NaN (the reference is undefined from there on, and the
            # float64 bound has nothing to say): such a scan is left out, as tests/test_deep_oracle.py leaves it out
            scans = [s for s in scans if np.all(np.isfinite(self.port.match_record(s[0], s[1], self.iters)[2]))]
            assert len(scans) >= 4
        self.scans = [(h, p, tag, True) for h, p, tag in scans]
        self.hints = np.stack([s[0] for s in scans]).astype(np.float32)
        self.pts = np.concatenate([s[1] for s in scans]).astype(np.float32)
        self.offs = np.concatenate([[0], np.cumsum([s[1].shape[0] for s in scans])]).astype(np.int32)

    def close(self):
        for r in list(self.reps.values()) + list(self.edge_reps.values()):
            r.close()
        self.port.close()


@pytest.fixture(scope="module")
def setups(hsb_lib, port_record):
    def get(gi, sched="default"):
        if (gi, sched) not in _SETUPS:
            _SETUPS[(gi, sched)] = Setup(gi, sched)
        return _SETUPS[(gi, sched)]

    yield get
    for s in _SETUPS.values():
        s.close()
    from test_gpu_match_geometry import _WORST as sums

    for fam in sorted(k for k in sums if k.startswith("deep ")):
        report(f"deep levels [{fam}]: sums max err / tol = {sums[fam]:.3f}")
    for k in sorted(_WORST):
        report(f"deep levels [{k}]: {_WORST[k]}")


# ---- geometry ------------------------------------------------------------------------------------------------------------
def test_create_rejects_one_cell_below_the_minimum(hsb_lib):
    from hector_slam_b200 import capi

    import torch

    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for sx, sy, L in dc.REJECTED:
        for _ in range(3):
            with pytest.raises(capi.HsbError, match="coarsest level"):
                capi.MapRepB200(0.05, sx, sy, levels=L)
    assert torch.cuda.mem_get_info()[0] >= free0 - (1 << 20), "a refused hsb_create leaked device memory"


@pytest.mark.parametrize("gi", range(len(dc.GEOMS)), ids=dc.IDS)
def test_geometry_and_getters(setups, gi):
    S = setups(gi)
    rep, port, g = S.reps[2], S.port, S.g
    assert rep.getMapLevels() == g[2]
    rng = np.random.default_rng(gi)
    poses = np.stack([rng.uniform(-0.2, 1.2, 64) * g[0] * g[4], rng.uniform(-0.2, 1.2, 64) * g[1] * g[4],
                      rng.uniform(-4, 4, 64)], axis=1).astype(np.float32)
    for l, (a, b) in enumerate(mcs.level_sizes(g)):
        sx, sy, cell = rep.level_info(l)
        assert (sx, sy) == (a, b) == port.level_size(l)
        assert f32(cell) == f32(port.cell_length(l))
        assert same(rep.map_origin(l), port.map_origin(l)), l
        for p in list(poses) + list(S.hints):
            assert same(rep.map_coords_pose(l, p), port.map_coords_pose(l, p)), (l, p)
            assert same(rep.world_coords_pose(l, p), port.world_coords_pose(l, p)), (l, p)
    for name in dc.SCHEDULES:
        r = make_rep(g, 1, dc.schedule(name, g[2]))
        assert r.record_floats == dc.record_floats(g[2], dc.schedule(name, g[2])), name
        r.close()


# ---- match ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gi,sched", dc.GS, ids=dc.GS_IDS)
def test_match_records_every_w(setups, gi, sched):
    S = setups(gi, sched)
    port = S.port
    for W in (1, 2, 4, 8, 0):
        tune = dict(warps_per_scan=W, scans_per_block=1) if W else {}
        P1, C1, recs, raw1, shape = batch_record(S.reps[1], S, **tune)
        P2, C2, _, raw2, _ = batch_record(S.reps[2], S, **tune)
        Wr = shape["warps_per_scan"]
        assert W == 0 or Wr == W
        assert same(raw1, raw2) and same(P1, P2) and same(C1, C2), W                # TEX == LDG
        check_sums(S, recs, Wr, shape["staged_points"], f"{S.family} W{W}", power=False)
        for b, (h, pts, tag, _) in enumerate(S.scans):
            nxt = h
            for l in range(S.levels - 1, -1, -1):
                r = recs[l]
                assert same_bits_or_nan(r["start"][b], nxt), (tag, l)                # hand-off
                if pts.shape[0] == 0:
                    continue                                                         # every level starts at the hint
                prev = port.map_coords_pose(l, r["start"][b])
                for e in range(r["H"].shape[1]):
                    want = pose32.step(prev, r["H"][b, e], r["dTr"][b, e])
                    assert same_bits_or_nan(r["est"][b, e], want), (tag, W, l, e)
                    prev = r["est"][b, e]
                nxt = port.world_coords_pose(l, f32([prev[0], prev[1], pose32.normalize_angle(prev[2])]))
            assert same_bits_or_nan(P1[b], nxt), (tag, W)
        # the record changes nothing, nor does ending a level at a fixed point
        for mode in MODES:
            rep = S.reps[mode]
            for fix in (0, 1):
                rep.set_tuning(**{**RESET, **tune, "fixpoint": fix})
                P0, C0 = rep.match_batch(S.hints, S.pts, S.offs)
                assert same(P0, P1) and same(C0, C1), (W, mode, fix)
            rep.set_tuning(**RESET, fixpoint=1)
    # the single-scan entry: the batch's auto-shape record is not its shape, so its sums are held to the bound afresh
    for mode in MODES:
        rep = S.reps[mode]
        rep.set_tuning(**RESET)
        for b, (h, pts, tag, _) in enumerate(S.scans):
            p, c, rec = rep.matchData(h, pts, record=True)
            p0, c0 = rep.matchData(h, pts)
            assert same(p, p0) and same(c, c0), (mode, tag)
            if mode == 1:
                one = [{k: np.asarray(v)[None] for k, v in r.items()} for r in rec]
                sh = rep.last_launch_shape()
                check_sums(S, one, sh["warps_per_scan"], sh["staged_points"], f"{S.family} single", scans=[S.scans[b]],
                           power=False)
            if tag == "empty":
                for l in range(S.levels):
                    assert same(rec[l]["start"], h) and not rec[l]["H"].any(), l


@pytest.mark.parametrize("gi", [i for i, g in enumerate(dc.GEOMS) if dc.has_edges(g)],
                         ids=[dc.IDS[i] for i, g in enumerate(dc.GEOMS) if dc.has_edges(g)])
def test_edges_on_every_level(setups, gi):
    S = setups(gi)
    h, pts, _, _ = S.scans[S.edge_index]
    assert {d[0] for d in S.designed} == set(range(S.levels))
    for mode in MODES:
        rep = S.edge_reps[mode]
        rep.set_tuning(**RESET)
        _, _, rec = rep.matchData(h, pts, record=True)
        mcs.check_edges(S.cases, rec, pts, S.designed)
        if mode == 1:
            sh = rep.last_launch_shape()
            Se = type("E", (), dict(scans=[S.scans[S.edge_index]], levels=S.levels, reps=S.edge_reps, prob=S.prob,
                                    family=S.family + " edges", zero=[]))
            check_sums(Se, [{k: np.asarray(v)[None] for k, v in r.items()} for r in rec], sh["warps_per_scan"],
                       sh["staged_points"], Se.family, power=False)


def test_one_wave_batch_equals_single_scans(setups):
    """4096 scans of 1081 endpoints on the 8-level map, in the shape the launcher picks for a large batch (reported):
    each scan's record equals the one it gets matched alone with the same warps per scan."""
    S = setups(0, "mixed")
    h, pts = S.scans[1][0], S.scans[1][1]
    B = 4096
    rng = np.random.default_rng(9)
    hints = (h + rng.uniform(-0.05, 0.05, (B, 3))).astype(np.float32)
    for mode in MODES:
        rep = S.reps[mode]
        rep.set_tuning(**RESET)
        P, C, recs, raw = rep.match_batch_record(hints, np.tile(pts, (B, 1)), (np.arange(B + 1) * len(pts)).astype(np.int32))
        shape = rep.last_launch_shape()
        _WORST[f"batch of {B} on 8 levels, mode{mode}"] = f"launch shape {shape}"
        rep.set_tuning(**{**RESET, "warps_per_scan": shape["warps_per_scan"], "scans_per_block": 1})
        for b in range(0, B, 293):
            p, c, r1, raw1 = rep.match_batch_record(hints[b:b + 1], pts, None)
            assert same(raw1[0], raw[b]) and same(p[0], P[b]) and same(c[0], C[b]), (mode, b)
        rep.set_tuning(**RESET)


@pytest.mark.parametrize("tag", list(dc.GOLDEN))
def test_golden_matches(hsb_lib, tag):
    d = load_golden("deep.npz")
    g = dc.golden_geometry(d, tag)
    L = g[2]
    scans, hints = d[f"{tag}_match_scans"], d[f"{tag}_match_hints"]
    K = scans.shape[0]
    offs = (np.arange(K + 1) * scans.shape[1]).astype(np.int32)
    compared = 0
    for name in ("default", "mixed"):
        iters = dc.schedule(name, L)
        mis = record_oracle.level_iterations(L, iters)
        hk = d[f"{tag}_{name}_hooks"]
        # the reference's own path: every reported Hessian well conditioned, or the last bits decide where it ends
        ok = np.abs(d[f"{tag}_{name}_poses"] - hints).max(axis=1) < 0.5      # (6.4 m cells move the 8-level matches by metres)
        off = 0
        for l in range(L - 1, -1, -1):
            for e in range(mis[l]):
                H = hk[:, off + 3 + 12 * e: off + 12 + 12 * e].reshape(K, 3, 3)
                ok &= np.array([scaled_cond(x) < 1e3 for x in H])
            off += 3 + 12 * mis[l]
        for mode in MODES:
            rep = make_rep(g, mode, iters)
            for l in range(L):
                rep.upload_level(l, d[f"{tag}_final{l}"])
            P, C = rep.match_batch(hints, scans.reshape(-1, 2), offs)
            rep.close()
            err = np.abs(P.astype(np.float64) - d[f"{tag}_{name}_poses"])[ok]
            if ok.any():
                assert err.max() <= 1e-4, (tag, name, mode, err.max(axis=0))
                want = d[f"{tag}_{name}_cov"][ok].astype(np.float64)
                got = C.reshape(K, 9)[ok].astype(np.float64)
                assert np.all(np.abs(got - want) <= 1e-3 * np.abs(want).max(axis=1, keepdims=True) + 1e-3), (tag, name, mode)
                _WORST[f"golden {tag}-{name} mode{mode}"] = f"{int(ok.sum())} of {K} matches compared, worst pose error {err.max():.2e}"
            compared += int(ok.sum())
    if tag == "g5":
        assert compared == 4 * K
    else:
        report(f"deep levels [golden {tag}]: {compared} of {4 * K} matches on a well-conditioned reference path")


# ---- input kinds -----------------------------------------------------------------------------------------------------------
def test_converted_inputs_equal_their_endpoints(hsb_lib):
    from hector_slam_b200 import synth

    world = synth.World(1, seed=1234)
    rng = np.random.default_rng(3)
    poses = world.sample_free_poses(6, rng)
    ranges = synth.make_range_batch(world, poses)
    hints = synth.perturb_hints(poses, seed=2).astype(np.float32)
    fmt, sf = synth.CLOUD_FORMAT, synth.SCAN_FORMAT
    T = synth.laser_transform()
    for mode in MODES:
        rep = make_rep(G8, mode, dc.schedule("mixed", 8))
        dc.set_fields(G8, rep)
        rep.set_scan_format(**sf)
        rep.set_cloud_format(T, fmt["sqr_laser_min_dist"], fmt["sqr_laser_max_dist"], fmt["laser_z_min_value"],
                             fmt["laser_z_max_value"])
        rep.set_laser_projection(sf["n_beams"], sf["angle_min"], sf["angle_increment"], sf["range_min"], sf["range_max"])

        def batch(pts_list):
            offs = np.concatenate([[0], np.cumsum([p.shape[0] for p in pts_list])]).astype(np.int32)
            return rep.match_batch(hints, np.concatenate(pts_list), offs)

        P, C = rep.match_batch_ranges(hints, ranges)
        P0, C0 = batch([rep.scan_to_points(r) for r in ranges])
        assert same(P, P0) and same(C, C0), ("ranges", mode)
        clouds = [synth.ranges_to_cloud(r) for r in ranges]
        offs = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int32)
        P, C, og = rep.match_batch_cloud(hints, np.concatenate(clouds), offs)
        conv = [rep.cloud_to_points(c) for c in clouds]
        P0, C0 = batch([c[0] for c in conv])
        assert same(P, P0) and same(C, C0) and same(og, np.stack([c[1] for c in conv])), ("cloud", mode)
        P, C, og = rep.match_batch_projected(hints, ranges)
        conv = [rep.projected_scan_to_points(r) for r in ranges]
        P0, C0 = batch([c[0] for c in conv])
        assert same(P, P0) and same(C, C0) and same(og, np.stack([c[1] for c in conv])), ("projected", mode)
        rep.close()


# ---- map writer ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gi", [0, 1, 3], ids=[dc.IDS[i] for i in (0, 1, 3)])
def test_update_level_by_scan_on_every_level(hsb_lib, gi):
    sx, sy, L, start, res = dc.GEOMS[gi]
    pair = Pair(res, sx, sy, L, start=start)
    rng = np.random.default_rng(sx + 3 * sy)
    pair.preload(rng, uniform=(gi != 0))
    for l, Lv in enumerate(pair.lv):
        for name, pose, pts, origo in level_scans(Lv, rng):
            if l < 3 and not name.startswith("family@(" + str(Lv.sx // 2)):
                continue          # levels 0..2 are tests/test_gpu_map_write.py's: one family each keeps them in the run
            counts = [r.launch_count for r in pair.reps]

            def fn(h, rep, m, l=l, pts=pts, pose=pose, origo=origo):
                rep.update_level_by_scan(l, pts, pose, origo)
                return [m.update_level(l, pts, pose, origo) if k == l else None for k in range(L)]
            before, writes = write_all(pair, fn)
            for r, c in zip(pair.reps, counts):
                assert r.launch_count - c <= 2, (l, name, r.launch_count - c)
            pair.check(before, writes, f"{dc.IDS[gi]} level {l} {name}", probe=name.startswith("family") or name == "4 beams")
        assert pair.reps[0].get_dirty_rects() == pair.models[0].dirty
        pair.reset_rects()
    pair.close()


@pytest.mark.parametrize("gi", [0, 1], ids=[dc.IDS[i] for i in (0, 1)])
def test_update_by_scan_all_levels(hsb_lib, gi):
    """updateByScan after a match, after a map_without_matching step (the coarse levels draw the stale container, scaled
    by 2^-l), with beams a few level-0 cells long that collapse to start == end on the coarse levels, two launches per
    write whatever the depth."""
    sx, sy, L, start, res = dc.GEOMS[gi]
    pair = Pair(res, sx, sy, L, 0.35, 0.8, start=start)
    rng = np.random.default_rng(17 + sx)
    pair.preload(rng, uniform=False)
    L0 = pair.lv[0]
    for rep in pair.reps:
        rep.setMapUpdateMinDistDiff(0.0)
        rep.setMapUpdateMinAngleDiff(0.0)
    collapsed = np.zeros(L, bool)
    short = np.zeros(L, bool)
    for k in range(4):
        c0 = (sx // 2 + 9 * k, sy // 2 - 7 * k)
        pose_a, scan_a = scan_for(L0, c0, 0.2 * k, rng)
        # beams of 1 .. 400 level-0 cells: on level l they span 2^-l of that, so some end in the start cell (dropped)
        # and some one to three cells away
        ring = np.float64([(c0[0] + r * math.cos(a), c0[1] + r * math.sin(a))
                           for r in (1, 3, 9, 30, 70, 130, 260, 400) for a in np.linspace(0.1, 6.2, 9)])
        scan_a = np.concatenate([scan_a, mw.points_for_targets(L0, pose_a, ring)])
        origo_a = f32([0.5 * k, -0.25 * k])
        pose_b, scan_b = scan_for(L0, (sx // 3, sy // 3 + k), -0.7, rng)
        origo_b = f32([-1.0, 0.5])

        def after_match(h, rep, m):
            rep.matchData(pose_a, scan_a, origo=origo_a)
            m.match(scan_a, origo_a)
            n0 = rep.launch_count
            rep.updateByScan(scan_b, pose_b, origo_b)
            assert rep.launch_count - n0 == 2, rep.launch_count - n0
            return m.update_by_scan(scan_b, pose_b, origo_b)

        def stale(h, rep, m):
            n0 = rep.launch_count
            pose, _, upd = rep.slam_update(pose_a, scan_b, map_without_matching=True, origo=origo_b)
            assert upd and same(pose, pose_a) and rep.launch_count - n0 <= 3, rep.launch_count - n0
            return m.update_by_scan(scan_b, pose_a, origo_b)

        for what, fn in (("after match", after_match), ("stale container", stale)):
            before, writes = write_all(pair, fn)
            pair.check(before, writes, f"{dc.IDS[gi]} updateByScan {what} {k}", probe=(k == 0))
            for l in range(1, L):
                assert writes[0][l] is not None and writes[0][l].box is not None, (what, l)
        for l in range(1, L):
            b = mw.beams(pair.lv[l], scan_a, pose_a, origo_a, float(f32(2.0 ** -l)))
            d = np.maximum(np.abs(b.x1 - b.x0), np.abs(b.y1 - b.y0))
            collapsed[l] |= bool(np.any(d == 0))
            short[l] |= bool(np.any(b.kept & (d >= 1) & (d <= 3)))
        for rep, m in zip(pair.reps, pair.models):
            assert rep.get_dirty_rects() == m.dirty
            assert [rep.get_dirty_rect(l) for l in range(L)] == m.dirty
            assert [rep.get_mirror_dirty_rect(l) for l in range(L)] == m.dirty
    assert collapsed[3:].all() and short[3:].all(), (collapsed, short)
    pair.close()


# ---- fused and group steps ---------------------------------------------------------------------------------------------------
def run_inputs(g, steps=20):
    scans, mwm, hints, _ = gen_golden.deep_run(g)
    k = np.arange(steps) % len(scans)
    return scans[k], mwm[k], hints[k]


@pytest.mark.parametrize("gi", [0, 2], ids=[dc.IDS[i] for i in (0, 2)])
def test_fused_steps_equal_the_host_sequence(hsb_lib, gi):
    g = dc.GEOMS[gi]
    L = g[2]
    scans, mwm, hints = run_inputs(g)

    def run(kind, mode):
        rep = make_rep(g, mode, update_factor_free=0.4, update_factor_occupied=0.9)
        rep.setMapUpdateMinDistDiff(0.2)
        rep.setMapUpdateMinAngleDiff(0.2)
        out, last = [], None
        for k in range(len(scans)):
            if kind == "host":
                if mwm[k]:
                    p, c = hints[k].copy(), np.zeros((3, 3), np.float32)
                else:
                    p, c = rep.matchData(hints[k], scans[k])
                u = bool(mwm[k]) or last is None or pose32.pose_difference_larger_than(p, last, f32(0.2), f32(0.2))
                if u:
                    rep.updateByScan(scans[k], p)
                    rep.onMapUpdated()
                    last = p
            else:
                p, c, u = rep.slam_update(hints[k], scans[k], map_without_matching=bool(mwm[k]), nowait=(kind == "nowait"))
                if mwm[k]:
                    c = np.zeros((3, 3), np.float32)
            out.append((p, c, u))
        rep.onMapUpdated()
        planes = [rep.download_level(l) for l in range(L)] + [rep.download_prob(l) for l in range(L)]
        end = rep.get_dirty_rects()
        rep.close()
        return out, planes, end

    for mode in MODES:
        want, wp, wend = run("host", mode)
        if gi == 2:   # (on the 8-level map the coarsest levels move every matched pose by metres: the gate always opens)
            assert any(u for _, _, u in want) and not all(u for _, _, u in want), "the gate opens and stays closed"
        for kind in ("sync", "nowait"):
            got, gp, gend = run(kind, mode)
            for k, (a, b) in enumerate(zip(got, want)):
                assert same(a[0], b[0]) and same(a[1], b[1]) and a[2] == b[2], (mode, kind, k, a, b)
            assert all(same(x, y) for x, y in zip(gp, wp)), (mode, kind)
            assert gend == wend, (mode, kind)


def test_group_of_deep_handles_equals_single_steps(hsb_lib):
    from hector_slam_b200 import capi, synth

    g, M, L = G8, 5, 8
    iters = dc.schedule("mixed", L)
    scans, _, hints = run_inputs(g, 12)
    world = synth.World(1, seed=1234)
    rng = np.random.default_rng(8)
    poses = world.sample_free_poses(12 * M, rng)
    ranges = synth.make_range_batch(world, poses).reshape(12, M, -1)
    fmt, sf = synth.CLOUD_FORMAT, synth.SCAN_FORMAT

    def make():
        rep = make_rep(g, 0, iters, update_factor_free=0.4, update_factor_occupied=0.9)
        rep.setMapUpdateMinDistDiff(0.0)
        rep.setMapUpdateMinAngleDiff(0.0)
        rep.set_scan_format(**sf)
        rep.set_cloud_format(synth.laser_transform(), fmt["sqr_laser_min_dist"], fmt["sqr_laser_max_dist"],
                             fmt["laser_z_min_value"], fmt["laser_z_max_value"])
        rep.set_laser_projection(sf["n_beams"], sf["angle_min"], sf["angle_increment"], sf["range_min"], sf["range_max"])
        return rep

    grp, one = [make() for _ in range(M)], [make() for _ in range(M)]
    group = capi.SlamGroup(grp)
    for k in range(12):
        members = None if k % 3 else [int(v) for v in rng.permutation(M)[:3]]
        mem = list(range(M)) if members is None else members
        h = np.stack([poses[k * M + s] for s in mem]).astype(np.float32)
        mwm = [(s + k) % 4 == 1 for s in mem]
        kind = ("endpoints", "cloud", "ranges", "projected")[k % 4]
        if kind == "endpoints":
            h = np.stack([hints[(k + s) % len(hints)] for s in mem])
            sc = [scans[(k + s) % len(scans)] for s in mem]
            P, Cv, U = group.slam_update(h, sc, map_without_matching=mwm, members=members)
            single = [one[s].slam_update(h[i], sc[i], map_without_matching=mwm[i]) for i, s in enumerate(mem)]
        elif kind == "cloud":
            cl = [synth.ranges_to_cloud(ranges[k, s]) for s in mem]
            P, Cv, U, kept = group.slam_update_cloud(h, cl, map_without_matching=mwm, members=members)
            single = [one[s].slam_update_cloud(h[i], cl[i], map_without_matching=mwm[i]) for i, s in enumerate(mem)]
        elif kind == "ranges":
            rr = [ranges[k, s] for s in mem]
            P, Cv, U, kept = group.slam_update_ranges(h, rr, map_without_matching=mwm, members=members)
            single = [one[s].slam_update_ranges(h[i], rr[i], map_without_matching=mwm[i]) for i, s in enumerate(mem)]
        else:
            rr = [ranges[k, s] for s in mem]
            P, Cv, U, kept = group.slam_update_projected(h, rr, map_without_matching=mwm, members=members)
            single = [one[s].slam_update_projected(h[i], rr[i], map_without_matching=mwm[i]) for i, s in enumerate(mem)]
        for i, s in enumerate(mem):
            assert same(P[i], single[i][0]) and same(Cv[i], single[i][1]) and U[i] == single[i][2], (k, kind, s)
            if kind != "endpoints":
                assert kept[i] == single[i][3], (k, kind, s)
    for s in range(M):
        for l in range(L):
            assert same(grp[s].download_level(l), one[s].download_level(l)), (s, l)
            assert same(grp[s].download_prob(l), one[s].download_prob(l)), (s, l)
            assert np.any(grp[s].download_level(l) != 0), (s, l)
        assert grp[s].get_dirty_rects() == one[s].get_dirty_rects()
        assert same(grp[s].last_map_update_pose(), one[s].last_map_update_pose())
    group.close()
    # members that differ in the depth only, or in one schedule entry beyond the third
    other = make_rep((g[0], g[1], 7, g[3], g[4]), 0, iters[:7])
    it5 = list(iters)
    it5[5] = 3
    other5 = make_rep(g, 0, it5)
    for bad in (other, other5):
        with pytest.raises(capi.HsbError, match="differs"):
            capi.SlamGroup([grp[0], bad])
        bad.close()
    for r in grp + one:
        r.close()


# ---- scoring, queries, export on the coarse levels -----------------------------------------------------------------------------
def test_queries_scores_and_export_on_levels_3_to_7(hsb_lib):
    from hector_slam_b200 import capi

    g, L, M = G8, 8, 3
    reps = [make_rep(g) for s in range(M)]
    port = make_port(g)
    planes = []
    for s, rep in enumerate(reps):
        planes.append([mtc.plane(a, b, seed=10 * s + l, occupied=0.1) for l, (a, b) in enumerate(mcs.level_sizes(g))])
        for l in range(L):
            rep.upload_level(l, planes[s][l])
    group = capi.SlamGroup(reps)
    rng = np.random.default_rng(12)
    scan = rng.uniform(-300, 300, (700, 2)).astype(np.float32)
    for l in range(3, L):
        sx, sy = mcs.level_sizes(g)[l]
        rays_b, rays_e, wb, we = [], [], [], []
        for s, rep in enumerate(reps):
            port.set_logodds(l, planes[s][l])
            occ = mtc.occupancy(planes[s][l])
            assert np.array_equal(rep.download_occupancy(l), occ), (s, l)
            rect = (1, 0, sx - 2, sy - 1)
            assert np.array_equal(rep.download_occupancy_rect(l, rect), occ[:, 1:sx - 1]), (s, l)
            assert same(rep.download_level_rect(l, rect), planes[s][l][:, 1:sx - 1]), (s, l)
            b, e = mtc.cell_rays(sx, sy, occ, seed=100 * s + l, n_random=300)
            dist, hit = rep.raycast_batch(l, b, e)
            for i in range(len(b)):
                d, hh = port.raycast(l, b[i], e[i])
                assert f32(d) == dist[i] and tuple(hit[i]) == hh, (s, l, i, b[i], e[i])
            bw, ew, nan = mtc.world_rays(sx, sy, port.map_origin(l), port.cell_length(l), seed=7 * s + l, n_random=200)
            dist, hw, found = rep.get_dist_batch(l, bw, ew)
            for i in np.flatnonzero(~nan):
                d, h1, f = port.get_dist(l, bw[i], ew[i])
                assert f32(d) == dist[i] and f == found[i] and same(h1, hw[i]), (s, l, i)
            rays_b.append(b), rays_e.append(e), wb.append(bw), we.append(ew)
        # the group forms equal the single calls
        dist, hit = group.raycast(l, rays_b, rays_e)
        one = [reps[s].raycast_batch(l, rays_b[s], rays_e[s]) for s in range(M)]
        assert same(dist, np.concatenate([o[0] for o in one])) and np.array_equal(hit, np.concatenate([o[1] for o in one])), l
        dist, hw, found = group.get_dist(l, wb, we)
        one = [reps[s].get_dist_batch(l, wb[s], we[s]) for s in range(M)]
        assert np.array_equal(bits(dist), bits(np.concatenate([o[0] for o in one]))), l
        assert np.array_equal(bits(hw), bits(np.concatenate([o[1] for o in one]))) and np.array_equal(found, np.concatenate([o[2] for o in one])), l
        grids = [np.full((sy, sx), 7, np.int8) for _ in range(M)]
        for s, rep in enumerate(reps):
            rep.get_mirror_dirty_rect(l, reset=True)
            rep.upload_level(l, planes[s][l])
        rects = group.sync_occupancy(l, grids)
        for s in range(M):
            assert rects[s] == (0, 0, sx - 1, sy - 1) and np.array_equal(grids[s], mtc.occupancy(planes[s][l])), (s, l)
        poses = [np.stack([rng.uniform(0.2, 0.8, 9) * g[0] * g[4] - 0.3 * g[0] * g[4],
                           rng.uniform(0.2, 0.8, 9) * g[1] * g[4] - 0.7 * g[1] * g[4], rng.uniform(-3, 3, 9)], axis=1).astype(np.float32)
                 for _ in range(M)]
        scans = [scan[: 300 + 100 * s] for s in range(M)]
        for s, r in enumerate(reps):       # finite planes for the scores: one NaN cell makes a whole sum NaN
            r.upload_level(l, mcs.field(sx, sy, l) + f32(0.2 * s))
        lh = group.likelihood(l, poses, scans)
        one = np.concatenate([reps[s].likelihood_batch(l, poses[s], scans[s]) for s in range(M)])
        assert same(lh, one), l
        assert np.all(np.isfinite(one)) and len(np.unique(one)) > M, "the poses see the level"
        cm, cw = group.covariance(l, poses, scans)
        onec = [reps[s].covariance_batch(l, poses[s], scans[s]) for s in range(M)]
        assert np.array_equal(bits(cm), bits(np.concatenate([o[0] for o in onec]))), l
        assert np.array_equal(bits(cw), bits(np.concatenate([o[1] for o in onec]))), l
        out, best4, index = group.best_hypothesis(l, poses, scans)
        assert same(out, one)
        for s in range(M):
            seg = one[9 * s: 9 * s + 9]
            assert index[s] == int(np.argmax(seg)) and best4[s, 0] == seg.max() and same(best4[s, 1:], poses[s][index[s]]), (l, s)
    # hypotheses matched over all eight levels
    hints = [np.stack([f32([0.0, 0.0, 0.1 * k]) for k in range(4)]) for _ in range(M)]
    scans = [scan[: 300 + 100 * s] for s in range(M)]
    P, Cv = group.match_batch(hints, scans)
    W = reps[0].last_launch_shape()["warps_per_scan"]
    for s, rep in enumerate(reps):
        rep.set_tuning(warps_per_scan=W, scans_per_block=1)
        p, c = rep.match_batch(hints[s], scans[s], None)
        rep.set_tuning(warps_per_scan=0, scans_per_block=0)
        assert same(P[4 * s: 4 * s + 4], p) and same(Cv[4 * s: 4 * s + 4], c), s
    # level == levels and level == -1
    rep = reps[0]
    for bad in (L, -1):
        for call in (lambda: rep.likelihood_batch(bad, poses[0], scans[0]), lambda: rep.covariance_batch(bad, poses[0], scans[0]),
                     lambda: rep.raycast_batch(bad, rays_b[0], rays_e[0]), lambda: rep.get_dist_batch(bad, wb[0], we[0]),
                     lambda: rep.download_occupancy_rect(bad, (0, 0, 1, 1)), lambda: rep.download_level_rect(bad, (0, 0, 1, 1)),
                     lambda: group.likelihood(bad, poses, scans), lambda: group.covariance(bad, poses, scans),
                     lambda: group.best_hypothesis(bad, poses, scans), lambda: group.raycast(bad, rays_b, rays_e),
                     lambda: group.get_dist(bad, wb, we), lambda: group.sync_occupancy(bad, grids)):
            with pytest.raises(capi.HsbError):
                call()
    group.close()
    port.close()
    for r in reps:
        r.close()


# ---- tile transport --------------------------------------------------------------------------------------------------------
def test_tiles_between_two_eight_level_handles(hsb_lib):
    import torch

    g, L = G8, 8
    sx, sy = g[0], g[1]
    a = make_rep(g, 0, update_factor_free=0.4, update_factor_occupied=0.9)
    b = make_rep(g, 0, update_factor_free=0.4, update_factor_occupied=0.9)
    c = make_rep(g, 0, update_factor_free=0.4, update_factor_occupied=0.9)
    lf, lo = a.logodds_increments()
    m = mw.MultiMap(g[4], sx, sy, L, lf, lo, start=g[3])
    rng = np.random.default_rng(71)
    for l, Lv in enumerate(m.lv):
        plane = mw.preload((Lv.sy, Lv.sx), rng)
        for r in (a, b, c):
            r.upload_level(l, plane)
            r.get_dirty_rect(l, reset=True)
            r.get_mirror_dirty_rect(l, reset=True)
        m.set_plane(l, plane)
    pose, scan = scan_for(m.lv[0], (sx // 2, sy // 2), 0.3, rng)
    a.matchData(pose, scan)
    m.match(scan)
    a.updateByScan(scan, pose)
    m.update_by_scan(scan, pose)
    rects = a.get_dirty_rects()
    assert rects == m.dirty and all(r is not None for r in rects), rects
    cells = [(r[2] - r[0] + 1) * (r[3] - r[1] + 1) for r in rects]
    st = torch.cuda.current_stream().cuda_stream
    # the two-step path on the coarse levels, to the third handle
    for l in range(3, L):
        buf = torch.empty(cells[l], dtype=torch.float32, device="cuda")
        a.pack_rect_device(l, rects[l], buf.data_ptr(), st)
        c.unpack_rect_device(l, rects[l], buf.data_ptr(), st)
        x0, y0, x1, y1 = rects[l]
        assert same(buf.cpu().numpy().reshape(y1 - y0 + 1, x1 - x0 + 1), m.planes[l][y0:y1 + 1, x0:x1 + 1]), l
        assert same(c.download_level(l), m.planes[l]) and same(c.download_prob(l), mw.prob(m.planes[l])), l
    # one row short: nothing shipped, the rectangles kept, the replica counts it
    total = sum(cells)
    cap = 4 << 20
    buf = torch.zeros(cap // 4, dtype=torch.float32, device="cuda")
    short = 4 * (64 + total - (rects[0][2] - rects[0][0] + 1))
    a.pack_dirty_device(buf.data_ptr(), short, True, st)
    b.unpack_dirty_device(buf.data_ptr(), short, st)
    hdr = buf[:64].view(torch.int32).cpu().numpy()
    assert hdr[1] == L and hdr[2] == 1 and hdr[3] == total
    assert a.get_dirty_rects() == rects and b.replication_overflows(reset=True) == 1
    assert all(b.get_mirror_dirty_rect(l) is None for l in range(L))
    # exactly enough
    exact = 4 * (64 + total)
    a.pack_dirty_device(buf.data_ptr(), exact, True, st)
    b.unpack_dirty_device(buf.data_ptr(), exact, st)
    hdr = buf[:64].view(torch.int32).cpu().numpy()
    assert hdr[1] == L and hdr[2] == 0 and hdr[3] == total
    assert [tuple(int(v) for v in hdr[4 + 4 * l: 8 + 4 * l]) for l in range(L)] == rects
    assert a.get_dirty_rects() == [None] * L and b.replication_overflows() == 0
    for l in range(L):
        assert same(b.download_level(l), m.planes[l]) and same(a.download_level(l), m.planes[l]), l
        assert same(b.download_prob(l), a.download_prob(l)) and same(b.download_prob(l), mw.prob(m.planes[l])), l
        assert b.get_mirror_dirty_rect(l) == rects[l], l
    pa, _ = a.matchData(pose, scan)
    pb, _ = b.matchData(pose, scan)
    assert same(pa, pb)
    for r in (a, b, c):
        r.close()


# ---- planes ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gi", [0, 3], ids=[dc.IDS[i] for i in (0, 3)])
def test_planes_round_trip_and_reset(hsb_lib, gi):
    import torch

    from hector_slam_b200 import parallel

    g = dc.GEOMS[gi]
    L = g[2]
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(5 + gi)
    for mode in MODES:
        rep = make_rep(g, mode)
        planes = [mw.preload((b, a), rng) for a, b in mcs.level_sizes(g)]
        for l in range(L):
            rep.upload_level(l, planes[l])
        for l in range(L):                       # (after every upload: a level's upload leaves the others alone)
            assert same(rep.download_level(l), planes[l]) and same(rep.download_prob(l), mw.prob(planes[l])), (mode, l)
        # refresh: log-odds changed behind the handle's back through the device pointer
        for l in range(L):
            sx, sy = mcs.level_sizes(g)[l]
            new = mw.preload((sy, sx), rng)
            rep.get_mirror_dirty_rect(l, reset=True)
            view = parallel.level_plane_tensor(rep, l, dev)
            view.copy_(torch.from_numpy(new).to(dev))
            rep.refresh_level(l, torch.cuda.current_stream().cuda_stream)
            torch.cuda.current_stream().synchronize()
            assert same(rep.download_level(l), new) and same(rep.download_prob(l), mw.prob(new)), (mode, l)
            assert rep.get_mirror_dirty_rect(l) == (0, 0, sx - 1, sy - 1), (mode, l)
        rep.reset()
        for l in range(L):
            assert not rep.download_level(l).any() and np.all(rep.download_prob(l) == f32(0.5)), (mode, l)
        rep.close()


# ---- trace -------------------------------------------------------------------------------------------------------------------
def test_trace_is_refused_above_four_levels_and_ordered_on_four(hsb_lib):
    import torch

    from hector_slam_b200 import capi

    for L in (5, 6, 7, 8):
        rep = make_rep((512, 512, L, (0.5, 0.5), 0.05), 1)
        with pytest.raises(capi.HsbError, match="trace records at most 4 levels") as e:
            rep.set_tuning(trace=1)
        assert e.value.status == -5                                    # HSB_ERR_UNSUPPORTED
        rep.set_tuning(trace=0)                                        # turning it off is always allowed
        p, _ = rep.match_batch(np.zeros((3, 3), np.float32), np.ones((50, 2), np.float32), None)
        assert rep.read_trace(3).shape[0] == 0                         # nothing was recorded
        rep.close()
    g = (512, 384, 4, (0.3, 0.7), 0.05)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for mode in MODES:
        rep = make_rep(g, mode)
        dc.set_fields(g, rep)
        port = make_port(g)
        cases = mcs.Cases(g, [rep.download_prob(l) for l in range(4)], port, seed=77)
        B = 40
        hints = np.stack([cases.hint(k) for k in range(B)]).astype(np.float32)
        pts = cases.scan(1081, hints[0], nonfinite=False)
        for tune in (dict(warps_per_scan=1, scans_per_block=1), dict(warps_per_scan=8, scans_per_block=1), {}):
            rep.set_tuning(**{**RESET, **tune, "trace": 0})
            P0, C0 = rep.match_batch(hints, pts, None)
            rep.set_tuning(trace=1)
            P1, C1 = rep.match_batch(hints, pts, None)
            assert same(P0, P1) and same(C0, C1), (mode, tune)
            tr = rep.read_trace(B + 5)
            assert tr.shape == (B, 8)
            t = tr[:, :6].astype(np.int64)
            assert np.all(np.diff(t, axis=1) >= 0) and np.all(t[:, 0] > 0), (mode, tune)     # start, 4 levels, end
            assert np.all(tr[:, 7] < sms) and np.all(tr[:, 6] < 64), (mode, tune)
        rep.set_tuning(**RESET, trace=0)
        rep.close()
        port.close()
