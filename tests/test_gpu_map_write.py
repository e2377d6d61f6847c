"""GPU: the map writer (K2: update_mark_kernel / update_apply_kernel and their group twins, update_kernel.cuh) held to
oracle/mapwrite.py's order-free plane with no cell excepted, bit for bit, on every entry point that writes the map.

The writer sums nothing: each cell is at most two fp32 additions, so it can be pinned exactly.  Per write:
  1. the log-odds plane equals mapwrite's `dev` plane on every cell;
  2. the probability plane equals mapwrite.prob (libm expf) of the device's own log-odds on every cell;
  3. no cell outside the write's box changed, and the replication and mirror dirty rectangles equal the union of the
     model's boxes since the last reset;
  4. the texture twin: handles in the TEX and the LDG gather mode fed the same sequence have the same planes, and a
     one-endpoint likelihood at every integer cell of the dirty box (x <= sx-2, y <= sy-2: the interpolation's bounds)
     returns 1 - (1 - P) of the model's P in both modes.  At an integer cell the bilinear weights are 1 and 0, so the
     likelihood reads exactly the one texel: any twin addressing error shows, and where P >= 0.5 the value is P itself;
  5. mapwrite's `ref` plane (the reference's beam-order result) differs from `dev` only on freed-then-hit cells where
     fl(fl(l + lf) - lf) != l (SURVEY.md Q10); the counts go to the parity report.

Maps: every width residue mod 4 is written (404 / 202 / 101, 150 / 75, 243 / 121, 257 / 128, 5, 7), square and
non-square, on the scalar apply path (width % 4 != 0) and the uint4 path, with boxes beyond one pass of either sweep.
"""
import numpy as np
import pytest

from conftest import report
from oracle import mapwrite as mw
from twin_probe import probe_twin

pytestmark = pytest.mark.gpu

LDG, TEX = 1, 2
STATS = {"writes": 0, "freed_then_hit": 0, "ref_ne_dev": 0, "max_ulp": 0, "max_abs": 0.0}   # LDG handles only


def sm_count():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def same(a, b):
    return np.array_equal(bits(a), bits(b))


class Pair:
    """The same map on an LDG-mode and a TEX-mode handle, each followed by its own order-free model."""

    def __init__(self, res, sx, sy, levels, ffree=0.4, focc=0.9, start=(0.5, 0.5)):
        from hector_slam_b200 import capi

        self.reps = [capi.MapRepB200(res, sx, sy, levels=levels, start=start, update_factor_free=ffree,
                                     update_factor_occupied=focc, gather_mode=m) for m in (LDG, TEX)]
        lf, lo = self.reps[0].logodds_increments()
        self.models = [mw.MultiMap(res, sx, sy, levels, lf, lo, start=start) for _ in self.reps]
        self.levels = levels
        self.lv = self.models[0].lv
        for l, L in enumerate(self.lv):
            assert self.reps[0].level_info(l)[:2] == (L.sx, L.sy)
            assert same(self.reps[0].map_coords_pose(l, [1.25, -0.5, 0.0])[:2],
                        np.float32(mw._affine(L.mtw, np.float32(1.25), np.float32(-0.5))))

    def preload(self, rng, uniform=True):
        for l, L in enumerate(self.lv):
            plane = mw.preload((L.sy, L.sx), rng, uniform)
            for rep, m in zip(self.reps, self.models):
                rep.upload_level(l, plane)
                m.set_plane(l, plane)
        self.reset_rects()

    def reset_rects(self):
        for rep, m in zip(self.reps, self.models):
            for l in range(self.levels):
                rep.get_dirty_rect(l, reset=True)
                rep.get_mirror_dirty_rect(l, reset=True)
                assert rep.get_dirty_rect(l) is None and rep.get_mirror_dirty_rect(l) is None
            m.dirty = [None] * self.levels

    def planes(self):
        return [[rep.download_level(l) for l in range(self.levels)] for rep in self.reps]

    def check(self, before, writes, what, probe=True, same_sequence=True):
        """writes[h][l]: the model's Write of handle h on level l (None: the level was not written).  same_sequence:
        both handles were given the same poses (a matched step may legitimately differ between the gather modes)."""
        after = self.planes()
        for h, (rep, m) in enumerate(zip(self.reps, self.models)):
            for l, L in enumerate(self.lv):
                got = after[h][l]
                w = writes[h][l] if writes is not None else None
                bad = bits(got) != bits(m.planes[l])
                assert not bad.any(), (what, h, l, int(bad.sum()), np.argwhere(bad)[:5].tolist())        # 1
                assert same(rep.download_prob(l), mw.prob(got)), (what, h, l)                             # 2
                changed = np.argwhere(bits(got) != bits(before[h][l]))                                    # 3
                if changed.size:
                    assert w is not None and w.box is not None, (what, h, l)
                    assert (changed[:, 1].min() >= w.box[0] and changed[:, 0].min() >= w.box[1]
                            and changed[:, 1].max() <= w.box[2] and changed[:, 0].max() <= w.box[3]), (what, h, l)
                assert rep.get_dirty_rect(l) == m.dirty[l], (what, h, l, rep.get_dirty_rect(l), m.dirty[l])
                assert rep.get_mirror_dirty_rect(l) == m.dirty[l], (what, h, l)
                if w is not None:
                    q10(w, count=(h == 0))                                                                  # 5
            if probe:
                for l in range(self.levels):
                    probe_twin(rep, l, self.lv[l], m.planes[l], m.dirty[l], what)                        # 4
        if same_sequence:
            assert all(same(a, b) for a, b in zip(*after)), f"{what}: LDG and TEX planes differ"

    def close(self):
        for r in self.reps:
            r.close()


def q10(w, count=True):
    """Assertion 5 on one write, and the figures for the report (ulp: distance of the fp32 bit patterns)."""
    if count:
        STATS["writes"] += 1
        STATS["freed_then_hit"] += int((w.cls == mw.FREED_THEN_HIT).sum())
    if not w.ref_defined:
        return
    diff = bits(w.ref) != bits(w.dev)
    assert not np.any(diff & ~w.deviation)
    assert np.all(w.cls[diff] == mw.FREED_THEN_HIT)
    if diff.any() and count:
        STATS["max_abs"] = max(STATS["max_abs"], float(np.abs(w.ref.astype(np.float64) - w.dev)[diff].max()))
        ulp = np.abs(w.ref.view(np.int32).astype(np.int64) - w.dev.view(np.int32).astype(np.int64))[diff]
        STATS["ref_ne_dev"] += int(diff.sum())
        STATS["max_ulp"] = max(STATS["max_ulp"], int(ulp.max()))


def write_all(pair, fn):
    """Run fn(h, rep, model) -> list of Writes per level on both handles; returns (before, writes)."""
    before = pair.planes()
    writes = [fn(h, rep, m) for h, (rep, m) in enumerate(zip(pair.reps, pair.models))]
    return before, writes


def scan_for(L, start, psi, rng, pt_scale=1.0, n_random=48):
    pose = mw.pose_for_cell(L, start[0], start[1], psi)
    return pose, mw.points_for_targets(L, pose, mw.family_targets(L, start, rng, n_random), pt_scale)


def level_scans(L, rng):
    """(name, pose, points, origo) for one level: the families at several starts, and the special cases"""
    out = []
    starts = [(L.sx // 2, L.sy // 2), (0, L.sy // 2), (L.sx - 1, L.sy - 1), (L.sx // 3, 0), (L.sx // 2, L.sy - 1)]
    for k, st in enumerate(starts):
        pose, pts = scan_for(L, st, (0.0, 0.3, -2.0, 1.5707964, 3.0)[k], rng)
        out.append((f"family@{st}", pose, pts, (0.0, 0.0) if k % 2 == 0 else (0.25, -0.5)))
    pose, pts = scan_for(L, (-3, L.sy // 2), 0.0, rng)
    out.append(("start outside", pose, pts, (0.0, 0.0)))
    c = (L.sx // 2, L.sy // 2)
    pose = mw.pose_for_cell(L, c[0], c[1], 0.1)
    out.append(("0 beams", pose, np.zeros((0, 2), np.float32), (0.0, 0.0)))
    out.append(("1 beam", pose, mw.points_for_targets(L, pose, [(L.sx - 1, 0)]), (0.0, 0.0)))
    out.append(("4 beams", pose, mw.points_for_targets(L, pose, [(0, 0), (L.sx - 1, 0), (0, L.sy - 1),
                                                                  (L.sx - 1, L.sy - 1)]), (0.0, 0.0)))
    wave = 4 * (sm_count() * 6) + 37    # beyond one wave of the mark grid (sm_count * 6 CTAs of 4 beams, one level)
    t = np.stack([rng.uniform(-2, L.sx + 2, wave), rng.uniform(-2, L.sy + 2, wave)], axis=1)
    out.append(("beyond one wave", pose, mw.points_for_targets(L, pose, t), (0.0, 0.0)))
    pts = mw.points_for_targets(L, pose, mw.family_targets(L, c, rng, 8))
    pts[::7, 0] = np.inf
    pts[3::11, 1] = np.nan
    pts[5::13] = np.float32([-3e9, 4e9])
    out.append(("non-finite endpoints", pose, pts, (0.0, 0.0)))
    out.append(("non-finite pose", np.float32([np.nan, 0.0, 0.0]), pts[:8], (0.0, 0.0)))
    return out


MAPS = [(256, 256, 3), (404, 300, 3), (150, 404, 2), (243, 200, 2), (257, 131, 1), (5, 7, 1), (7, 4, 1)]


@pytest.mark.parametrize("geom", MAPS, ids=lambda g: "x".join(map(str, g)))
def test_update_level_by_scan(hsb_lib, geom):
    """hsb_update_level_by_scan on every level: scan families at starts in the middle, on the edges and outside, 0 / 1
    / 4 beams, more beams than one wave of the mark grid, non-finite endpoints and a non-finite pose."""
    sx, sy, levels = geom
    pair = Pair(0.05, sx, sy, levels)
    rng = np.random.default_rng(sx * 7 + sy)
    pair.preload(rng)
    for l, L in enumerate(pair.lv):
        for name, pose, pts, origo in level_scans(L, rng):
            def fn(h, rep, m, l=l, pts=pts, pose=pose, origo=origo):
                rep.update_level_by_scan(l, pts, pose, origo)
                return [m.update_level(l, pts, pose, origo) if k == l else None for k in range(levels)]
            before, writes = write_all(pair, fn)
            pair.check(before, writes, f"{geom} level {l} {name}", probe=name.startswith("family") or name == "4 beams")
        pair.reset_rects()
    report(f"map_write Q10: {STATS}")
    pair.close()


@pytest.mark.parametrize("geom", [(404, 300, 3), (150, 404, 2)], ids=lambda g: "x".join(map(str, g)))
def test_update_by_scan_after_match(hsb_lib, geom):
    """updateByScan: level 0 from the given scan, the coarse levels from the last MATCHED scan with its origo, also
    when that is not the written one (SURVEY.md Q11)."""
    sx, sy, levels = geom
    pair = Pair(0.05, sx, sy, levels, 0.35, 0.8)
    rng = np.random.default_rng(11 + sx)
    pair.preload(rng)
    L0 = pair.lv[0]
    for k in range(4):
        pose_a, scan_a = scan_for(L0, (sx // 2 + 3 * k, sy // 2 - 2 * k), 0.2 * k, rng)
        origo_a = np.float32([0.5 * k, -0.25 * k])
        if k % 2:
            pose_b, scan_b, origo_b = pose_a, scan_a, origo_a
        else:
            pose_b, scan_b = scan_for(L0, (sx // 3, sy // 3 + k), -0.7, rng)
            origo_b = np.float32([-1.0, 0.5])

        def fn(h, rep, m):
            rep.matchData(pose_a, scan_a, origo=origo_a)
            m.match(scan_a, origo_a)
            rep.updateByScan(scan_b, pose_b, origo_b)
            return m.update_by_scan(scan_b, pose_b, origo_b)
        before, writes = write_all(pair, fn)
        pair.check(before, writes, f"{geom} updateByScan {k}")
    report(f"map_write Q10: {STATS}")
    pair.close()


def test_fused_slam_update(hsb_lib):
    """hsb_slam_update: map_without_matching (the coarse levels keep the last matched container, none at first), a
    matched write, and a step whose gate stays closed (planes and rectangles bitwise unchanged)."""
    sx, sy, levels = 404, 300, 3
    pair = Pair(0.05, sx, sy, levels)
    rng = np.random.default_rng(21)
    pair.preload(rng)
    L0 = pair.lv[0]
    og = np.float32([0.5, -0.25])
    steps = []
    for k in range(2):
        pose, scan = scan_for(L0, (sx // 2 + 5 * k, sy // 2), 0.4 * k, rng)
        steps.append(("mwm", pose, scan))
    pose, scan = scan_for(L0, (sx // 2, sy // 2 + 4), 0.1, rng)
    steps.insert(1, ("match", pose, scan))
    for h, rep in enumerate(pair.reps):
        rep.setMapUpdateMinDistDiff(0.0)
        rep.setMapUpdateMinAngleDiff(0.0)
    for name, hint, scan in steps:
        def fn(h, rep, m):
            pose, _, upd = rep.slam_update(hint, scan, map_without_matching=(name == "mwm"), origo=og)
            assert upd
            if name == "mwm":
                assert same(pose, hint)
            else:
                m.match(scan, og)
            return m.update_by_scan(scan, pose, og)
        before, writes = write_all(pair, fn)
        pair.check(before, writes, f"slam_update {name}", same_sequence=(name == "mwm"))
    # gate closed: the matched pose is within the thresholds of the last written one
    for rep in pair.reps:
        rep.setMapUpdateMinDistDiff(1e9)
        rep.setMapUpdateMinAngleDiff(1e9)
    pair.reset_rects()
    hint, scan = steps[-1][1], steps[-1][2]
    before = pair.planes()
    probs = [[rep.download_prob(l) for l in range(levels)] for rep in pair.reps]
    for rep, m in zip(pair.reps, pair.models):
        _, _, upd = rep.slam_update(hint, scan, origo=og)
        assert not upd
        m.match(scan, og)
    after = pair.planes()
    for h, rep in enumerate(pair.reps):
        for l in range(levels):
            assert same(after[h][l], before[h][l]) and same(rep.download_prob(l), probs[h][l])
            assert rep.get_dirty_rect(l) is None and rep.get_mirror_dirty_rect(l) is None
    # and the next forced write draws the coarse levels from the scan that step matched
    for rep in pair.reps:
        rep.setMapUpdateMinDistDiff(0.0)
    pose2, scan2 = scan_for(L0, (sx // 2 - 9, sy // 2 + 2), -0.3, rng)

    def fn(h, rep, m):
        rep.slam_update(pose2, scan2, map_without_matching=True, origo=og)
        return m.update_by_scan(scan2, pose2, og)
    before, writes = write_all(pair, fn)
    pair.check(before, writes, "slam_update mwm after a closed gate")
    report(f"map_write Q10: {STATS}")
    pair.close()


def test_fused_cloud_step_counts_on_device(hsb_lib):
    """hsb_slam_update_cloud: the kept-endpoint count is known only on the device (points outside the distance window
    and the height band are dropped), so every level's writer reads n_dev < n."""
    sx, sy, levels = 243, 200, 2
    res = 0.05
    pair = Pair(res, sx, sy, levels)
    rng = np.random.default_rng(31)
    pair.preload(rng)
    L0 = pair.lv[0]
    T = np.float64([1, 0, 0, 0.1, 0, 1, 0, -0.05, 0, 0, 1, 0.2])
    for rep in pair.reps:
        rep.setMapUpdateMinDistDiff(0.0)
        rep.setMapUpdateMinAngleDiff(0.0)
        rep.set_cloud_format(T, 0.3 ** 2, 8.0 ** 2, -0.5, 1.0)
    for k in range(2):
        pose, scan = scan_for(L0, (sx // 2 + 4 * k, sy // 2 - 3 * k), 0.25 * k, rng)
        xyz = np.zeros((scan.shape[0], 3), np.float32)
        xyz[:, :2] = scan * np.float32(res)
        xyz[::9, :2] *= np.float32(1e-3)            # inside the minimum distance
        xyz[1::9, 2] = np.float32(3.0)              # above the height band
        xyz = np.concatenate([xyz, np.float32([[20.0, 1.0, 0.0], [0.0, -30.0, 0.0]])])   # beyond the maximum

        def fn(h, rep, m):
            got_pose, _, upd, kept = rep.slam_update_cloud(pose, xyz)
            pts, origo = rep.cloud_to_points(xyz)
            assert upd and kept == pts.shape[0] < xyz.shape[0], (kept, pts.shape, xyz.shape)
            m.match(pts, origo)
            return m.update_by_scan(pts, got_pose, origo)
        before, writes = write_all(pair, fn)
        pair.check(before, writes, f"slam_update_cloud {k}", same_sequence=False)
    pair.close()


@pytest.mark.parametrize("pdl", [1, 0], ids=["pdl", "no_pdl"])
def test_single_write_launch_counts(hsb_lib, pdl):
    """Launches of the single-handle writes, with and without programmatic dependent launch: mark + apply for a write
    with endpoints on some level and none for a write without, behind one match launch for a matched step, the gate
    kernel for a map_without_matching step of endpoints, and conversion, gate and count publication for one of a
    cloud."""
    sx, sy, levels, res = 256, 256, 3, 0.05
    pair = Pair(res, sx, sy, levels)
    rng = np.random.default_rng(71)
    L0 = pair.lv[0]
    pose, scan = scan_for(L0, (sx // 2, sy // 2), 0.3, rng)
    xyz = np.zeros((scan.shape[0], 3), np.float32)
    xyz[:, :2] = scan * np.float32(res)
    none = np.zeros((0, 2), np.float32)
    steps = [
        ("update_by_scan, no endpoints, no container", 0, lambda r: r.updateByScan(none, pose)),
        ("update_level_by_scan, no endpoints", 0, lambda r: r.update_level_by_scan(1, none, pose)),
        ("update_level_by_scan", 2, lambda r: r.update_level_by_scan(1, scan * np.float32(0.5), pose)),
        ("update_by_scan", 2, lambda r: r.updateByScan(scan, pose)),
        ("slam_update map_without_matching", 3, lambda r: r.slam_update(pose, scan, map_without_matching=True)),
        ("slam_update", 3, lambda r: r.slam_update(pose, scan)),
        ("update_by_scan, no endpoints, matched container", 2, lambda r: r.updateByScan(none, pose)),
        ("slam_update, no endpoints", 1, lambda r: r.slam_update(pose, none)),
        ("update_by_scan, no endpoints, empty container", 0, lambda r: r.updateByScan(none, pose)),
        ("slam_update_cloud map_without_matching", 5,
         lambda r: r.slam_update_cloud(pose, xyz, map_without_matching=True)),
        ("slam_update_cloud", 3, lambda r: r.slam_update_cloud(pose, xyz)),
    ]
    for rep in pair.reps:
        rep.set_tuning(pdl=pdl)
        rep.setMapUpdateMinDistDiff(0.0)
        rep.setMapUpdateMinAngleDiff(0.0)
        rep.set_cloud_format(np.float64([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0]), 0.0, 1e6, -1.0, 1.0)
        for name, want, fn in steps:
            n0 = rep.launch_count
            fn(rep)
            assert rep.launch_count - n0 == want, (name, rep.gather_mode, rep.launch_count - n0)
    pair.close()


def test_group_step_odd_width(hsb_lib):
    """hsb_group_slam_update on a 243 x 200 geometry (level widths 243, 121: the scalar apply path), members with
    different update factors, one of them map_without_matching (its coarse levels keep the last matched container)."""
    from hector_slam_b200 import capi

    sx, sy, levels = 243, 200, 2
    factors = [(0.4, 0.9), (0.3, 0.7), (0.45, 0.6)]
    reps = [capi.MapRepB200(0.05, sx, sy, levels=levels, update_factor_free=f, update_factor_occupied=o)
            for f, o in factors]
    models = []
    rng = np.random.default_rng(41)
    for rep in reps:
        rep.setMapUpdateMinDistDiff(0.0)
        rep.setMapUpdateMinAngleDiff(0.0)
        lf, lo = rep.logodds_increments()
        m = mw.MultiMap(0.05, sx, sy, levels, lf, lo)
        for l, L in enumerate(m.lv):
            plane = mw.preload((L.sy, L.sx), rng)
            rep.upload_level(l, plane)
            m.set_plane(l, plane)
            rep.get_dirty_rect(l, reset=True)
            rep.get_mirror_dirty_rect(l, reset=True)
        models.append(m)
    assert len({tuple(r.logodds_increments()) for r in reps}) == 3
    L0 = models[0].lv[0]
    pose0, scan0 = scan_for(L0, (100, 90), 0.0, rng)
    reps[2].matchData(pose0, scan0)            # the mwm member's stale container
    models[2].match(scan0, (0.0, 0.0))
    group = capi.SlamGroup(reps)
    mwm = np.array([0, 0, 1], bool)
    for step in range(2):
        hints, scans, origos = [], [], []
        for k in range(3):
            pose, scan = scan_for(L0, (sx // 2 + 7 * k - 3 * step, sy // 2 + 5 * step), 0.3 * k - 0.2 * step, rng)
            hints.append(pose)
            scans.append(scan)
            origos.append(np.float32([0.25 * k, -0.5 * step]))
        poses, _, upd = group.slam_update(np.asarray(hints), scans, np.asarray(origos), mwm)
        for k, (rep, m) in enumerate(zip(reps, models)):
            assert upd[k]
            if mwm[k]:
                assert same(poses[k], hints[k])
            else:
                m.match(scans[k], origos[k])
            ws = m.update_by_scan(scans[k], poses[k], origos[k])
            for l in range(levels):
                got = rep.download_level(l)
                bad = bits(got) != bits(m.planes[l])
                assert not bad.any(), (step, k, l, int(bad.sum()))
                assert same(rep.download_prob(l), mw.prob(got))
                assert rep.get_dirty_rect(l) == m.dirty[l] and rep.get_mirror_dirty_rect(l) == m.dirty[l]
                if ws[l] is not None:
                    q10(ws[l])
                probe_twin(rep, l, m.lv[l], m.planes[l], m.dirty[l], f"group {step} member {k}")
    group.close()
    for r in reps:
        r.close()


@pytest.mark.parametrize("path", ["scalar", "uint4"])
def test_box_beyond_one_sweep_pass(hsb_lib, path):
    """One level whose box is larger than one pass of the apply grid: at most sm_count * 8 CTAs of 256 threads, one
    cell per thread on the scalar path, 16 on the uint4 path.  Four beams from the middle to the corners."""
    one_pass = sm_count() * 8 * 256 * (1 if path == "scalar" else 16)
    side = int(np.ceil(np.sqrt(one_pass * 1.05)))
    sx = side + (-side) % 4 + (1 if path == "scalar" else 0)
    sy = side
    assert sx * sy > one_pass and (sx % 4 != 0) == (path == "scalar")
    pair = Pair(0.05, sx, sy, 1)
    rng = np.random.default_rng(51)
    pair.preload(rng, uniform=False)   # PRELOAD values only: few distinct log-odds for mapwrite.prob
    L = pair.lv[0]
    pose = mw.pose_for_cell(L, sx // 2, sy // 2, 0.0)
    pts = mw.points_for_targets(L, pose, [(0, 0), (sx - 1, 0), (0, sy - 1), (sx - 1, sy - 1)])

    def fn(h, rep, m):
        rep.update_level_by_scan(0, pts, pose)
        return [m.update_level(0, pts, pose)]
    before, writes = write_all(pair, fn)
    assert writes[0][0].box == (0, 0, sx - 1, sy - 1)
    pair.check(before, writes, f"{path} box {sx} x {sy}")
    pair.close()


def test_replica_follows_owner_through_tiles(hsb_lib):
    """pack_dirty_device / unpack_dirty_device on one GPU between two handles of a 243 x 200 x 3 map (widths 243, 121,
    60): afterwards the replica's log-odds and probability planes equal the owner's bit for bit."""
    import torch

    from hector_slam_b200 import capi

    sx, sy, levels = 243, 200, 3
    owner = capi.MapRepB200(0.05, sx, sy, levels=levels, update_factor_free=0.4, update_factor_occupied=0.9)
    replica = capi.MapRepB200(0.05, sx, sy, levels=levels, update_factor_free=0.4, update_factor_occupied=0.9)
    lf, lo = owner.logodds_increments()
    m = mw.MultiMap(0.05, sx, sy, levels, lf, lo)
    rng = np.random.default_rng(61)
    for l, L in enumerate(m.lv):
        plane = mw.preload((L.sy, L.sx), rng)
        for r in (owner, replica):
            r.upload_level(l, plane)
            r.get_dirty_rect(l, reset=True)
            r.get_mirror_dirty_rect(l, reset=True)
        m.set_plane(l, plane)
    L0 = m.lv[0]
    for k in range(3):
        pose, scan = scan_for(L0, (60 + 50 * k, 70 + 20 * k), 0.5 * k, rng)
        owner.matchData(pose, scan)
        m.match(scan)
        owner.updateByScan(scan, pose)
        m.update_by_scan(scan, pose)
    cap = 4 << 20
    buf = torch.zeros(cap // 4, dtype=torch.float32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    assert owner.get_dirty_rects() == m.dirty
    owner.pack_dirty_device(buf.data_ptr(), cap, True, st)
    replica.unpack_dirty_device(buf.data_ptr(), cap, st)
    for l in range(levels):
        assert same(owner.download_level(l), m.planes[l])
        assert same(replica.download_level(l), owner.download_level(l))
        assert same(replica.download_prob(l), owner.download_prob(l))
    assert owner.get_dirty_rects() == [None] * levels and replica.replication_overflows() == 0
    owner.close()
    replica.close()
