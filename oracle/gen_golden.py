"""Generate tests/golden/*.npz from the COMPILED REFERENCE (oracle/_ref/libhsref.so).

TEST INFRASTRUCTURE.  Run in the build container, where /root/reference exists:

    make -C oracle && python oracle/gen_golden.py
    make -C oracle -f record.mk && python oracle/gen_golden.py deep      (deep.npz: 8- and 5-level maps)

The reference ships no golden vectors (SURVEY.md §4/§8c), so these fixtures are produced by the
unmodified reference headers themselves (compiled against oracle/shim).  They pin
  * the plain-C port (tests/test_oracle_golden.py, bit-exact), and
  * the CUDA path (tests/test_gpu_*.py, within the 1e-4 m / 1e-4 rad parity bar)
on machines where /root/reference is absent (the GPU box).

Everything is seeded; the world is one 20 m x 14 m room with 8 pillars (hector_slam_b200/synth.py)
on a 512 x 512 level-0 grid at 0.05 m so that the fixtures stay small.
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from hector_slam_b200 import synth  # noqa: E402
from oracle.pyoracle import Oracle, build_map_known_poses  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
SIZE = 512
RES = 0.05
K = 16


def sparse(plane):
    idx = np.flatnonzero(plane.reshape(-1) != 0).astype(np.int32)
    return idx, plane.reshape(-1)[idx].astype(np.float32)


def planes_sparse(orc, prefix, out, base=None):
    """Store the level planes sparsely; with `base` (list of planes) only the cells that changed."""
    planes = []
    for l in range(orc.levels):
        cur = orc.get_logodds(l)
        planes.append(cur)
        if base is None:
            idx, val = sparse(cur)
        else:
            idx = np.flatnonzero(cur.reshape(-1) != base[l].reshape(-1)).astype(np.int32)
            val = cur.reshape(-1)[idx].astype(np.float32)
        out[f"{prefix}_idx{l}"] = idx
        out[f"{prefix}_val{l}"] = val
    return planes


def main(kind="reference"):
    os.makedirs(OUT, exist_ok=True)
    world = synth.World(1, seed=1234)
    rng = np.random.default_rng(2024)
    truth = world.sample_free_poses(K, rng, margin=0.8)
    pts, offs = synth.make_scan_batch(world, truth, noise_seed=7)
    assert np.all(np.diff(offs) == synth.N_BEAMS)
    scans = pts.reshape(K, synth.N_BEAMS, 2)

    # ---------------- 3-level: fixed point of 14 evaluations ------------------------------------
    o3 = Oracle(kind, RES, SIZE, 3)
    o3.set_update_factors(0.4, 0.9)
    build_map_known_poses(o3, world)
    hints3 = synth.perturb_hints(truth, seed=1, dxy=0.1, dpsi=0.05)
    out = dict(res=np.float32(RES), size=np.int32(SIZE), levels=np.int32(3), factors=np.float32([0.4, 0.9]),
               scans=scans, hints=hints3, truth=truth.astype(np.float64))
    base = planes_sparse(o3, "map", out)
    poses, covs = [], []
    for k in range(K):
        p, c = o3.match(hints3[k], scans[k])
        poses.append(p)
        covs.append(c.reshape(9))
    out["ref_poses"] = np.asarray(poses, np.float32)
    out["ref_cov"] = np.asarray(covs, np.float32)
    # per-evaluation H / dTr on every level at the level's hint pose (scan 0..3)
    ev_level, ev_scan, ev_pose, ev_H, ev_d = [], [], [], [], []
    for k in range(4):
        for l in range(3):
            pm = o3.map_coords_pose(l, hints3[k])
            pl = (scans[k] * np.float32(2.0 ** -l)).astype(np.float32)
            H, d = o3.hessian_derivs(l, pm, pl)
            ev_level.append(l)
            ev_scan.append(k)
            ev_pose.append(pm)
            ev_H.append(H.reshape(9))
            ev_d.append(d)
    out.update(ev_level=np.int32(ev_level), ev_scan=np.int32(ev_scan), ev_pose=np.float32(ev_pose),
               ev_H=np.float32(ev_H), ev_dTr=np.float32(ev_d))
    # pose conversions
    out["conv_world"] = hints3[:4]
    out["conv_map"] = np.float32([[o3.map_coords_pose(l, hints3[k]) for l in range(3)] for k in range(4)])
    out["conv_back"] = np.float32([[o3.world_coords_pose(l, o3.map_coords_pose(l, hints3[k])) for l in range(3)]
                                   for k in range(4)])
    out["increments"] = o3.logodds_increments()

    # ---------------- map write: match (fills coarse containers) then updateByScan --------------
    upd_pose = poses[0]
    o3.match(hints3[0], scans[0])
    o3.update_by_scan(scans[0], upd_pose)
    o3.on_map_updated()
    base = planes_sparse(o3, "upd1", out, base)
    out["upd1_pose"] = upd_pose
    # a second write from another pose, after a match with ANOTHER scan (Q11: coarse levels then
    # use the matched scan, level 0 the given one)
    o3.match(hints3[1], scans[1])
    o3.update_by_scan(scans[2], poses[2])
    o3.on_map_updated()
    base = planes_sparse(o3, "upd2", out, base)
    out["upd2_pose"] = poses[2]
    # rotation clamp (ScanMatcher.h:209-215): hint rotated by 0.3 rad, first steps hit +-0.2 rad
    # match again on the modified map (probabilities must have been refreshed)
    p, c = o3.match(hints3[3], scans[3])
    out["after_upd_pose"] = p
    out["after_upd_cov"] = c.reshape(9)
    np.savez_compressed(os.path.join(OUT, "match3.npz"), **out)
    o3.close()

    # ---------------- 1-level: 6 evaluations, step-by-step fidelity ------------------------------
    o1 = Oracle(kind, RES, SIZE, 1)
    o1.set_update_factors(0.4, 0.9)
    build_map_known_poses(o1, world)
    hints1 = synth.perturb_hints(truth, seed=3, dxy=0.03, dpsi=0.015)
    out = dict(res=np.float32(RES), size=np.int32(SIZE), levels=np.int32(1), factors=np.float32([0.4, 0.9]),
               scans=scans, hints=hints1, truth=truth.astype(np.float64))
    planes_sparse(o1, "map", out)
    out["ref_poses"] = np.float32([o1.match(hints1[k], scans[k])[0] for k in range(K)])
    out["ref_cov"] = np.float32([o1.match(hints1[k], scans[k])[1].reshape(9) for k in range(K)])
    # "3 GN iters" of BASELINE.json config 1: ScanMatcher::matchData(maxIterations = 2) = 3 evaluations
    out["ref_poses_3eval"] = np.float32([o1.match_level(0, hints1[k], scans[k], 2)[0] for k in range(K)])
    out["ref_cov_3eval"] = np.float32([o1.match_level(0, hints1[k], scans[k], 2)[1].reshape(9) for k in range(K)])

    # ---------------- edge cases ------------------------------------------------------------------
    e = {}
    # empty scan: pose = hint, cov untouched
    cov_in = np.arange(9, dtype=np.float32)
    p, c = o1.match(hints1[0], np.zeros((0, 2), np.float32), cov_in=cov_in)
    e["empty_pose"], e["empty_cov"] = p, c.reshape(9)
    # every endpoint outside the map: H = 0 -> gate fails -> pose = hint after the round trip
    far = (scans[0] + np.float32(1e5)).astype(np.float32)
    p, c = o1.match(hints1[0], far)
    e["far_pose"], e["far_cov"] = p, c.reshape(9)
    out.update({"edge_" + k: v for k, v in e.items()})
    np.savez_compressed(os.path.join(OUT, "match1.npz"), **out)
    o1.close()

    # ---------------- random plane: interpolation incl. the [0, S-2] bounds (Q6) and the Q1 gradient
    RS = 64
    orr = Oracle(kind, 0.1, RS, 2)
    rng = np.random.default_rng(5)
    out = dict(res=np.float32(0.1), size=np.int32(RS), levels=np.int32(2))
    for l in range(2):
        s_ = RS >> l
        plane = rng.normal(0.0, 2.0, (s_, s_)).astype(np.float32)
        plane[rng.uniform(size=plane.shape) < 0.05] = np.float32(60.0)   # saturated cells (P = 1)
        orr.set_logodds(l, plane)
        out[f"plane{l}"] = plane
        out[f"prob{l}"] = orr.get_prob(l)
    ev_pose, ev_pts, ev_H, ev_d, ev_level = [], [], [], [], []
    st_hint, st_pose, st_clamped, st_cond = [], [], [], []
    for trial in range(28):
        l = trial % 2
        s_ = RS >> l
        pm = np.float32([rng.uniform(0, s_), rng.uniform(0, s_), rng.uniform(-3.2, 3.2)])
        pts = rng.uniform(-0.8 * s_, 0.8 * s_, (256, 2)).astype(np.float32)
        if trial >= 12:  # a handful of endpoints close to the sensor: rotation barely constrained,
            # so the raw Gauss-Newton step in psi is often beyond the +-0.2 rad clamp
            pm = np.float32([rng.uniform(8, s_ - 8), rng.uniform(8, s_ - 8), rng.uniform(-3.2, 3.2)])
            pts[:] = 0
            pts[:8] = rng.uniform(-2.0, 2.0, (8, 2)).astype(np.float32)
            pts[8:] = np.float32(1e6)  # the rest is out of the map and contributes nothing
        if trial < 2:  # pose at the origin, no rotation: endpoints exactly on / just beyond the bounds
            pm = np.float32([0.0, 0.0, 0.0])
            lim = np.float32(s_ - 2)
            pts[:8] = np.float32([[lim, 5.0], [np.nextafter(lim, np.float32(1e9)), 5.0], [5.0, lim],
                                  [5.0, np.nextafter(lim, np.float32(1e9))], [0.0, 0.0], [-0.0, 3.5],
                                  [np.nextafter(np.float32(0), np.float32(-1)), 3.0], [lim, lim]])
        H, d = orr.hessian_derivs(l, pm, pts)
        # one Gauss-Newton step from this pose (ScanMatcher::matchData with maxIterations = 0 runs
        # exactly the pre-loop evaluation, ScanMatcher.h:74): exercises the H^-1 dTr solve and the
        # +-0.2 rad clamp (:209-215), which well-converging scans in a real map hardly ever hit
        hint_w = orr.world_coords_pose(l, pm)
        step_pose, _ = orr.match_level(l, hint_w, pts, 0)
        with np.errstate(all="ignore"):
            try:
                dstep = np.linalg.solve(H.astype(np.float64), d.astype(np.float64))
            except np.linalg.LinAlgError:
                dstep = np.full(3, np.nan)
        st_hint.append(hint_w)
        st_pose.append(step_pose)
        st_clamped.append(bool(abs(dstep[2]) > 0.2))
        st_cond.append(np.linalg.cond(H.astype(np.float64)))
        ev_pose.append(pm)
        ev_pts.append(pts)
        ev_H.append(H.reshape(9))
        ev_d.append(d)
        ev_level.append(l)
    out.update(ev_level=np.int32(ev_level), ev_pose=np.float32(ev_pose), ev_pts=np.float32(ev_pts), ev_H=np.float32(ev_H),
               ev_dTr=np.float32(ev_d), step_hint=np.float32(st_hint), step_pose=np.float32(st_pose),
               step_clamped=np.array(st_clamped), step_cond=np.float64(st_cond))
    print("step clamped:", st_clamped)
    assert sum(st_clamped) >= 3
    np.savez_compressed(os.path.join(OUT, "interp.npz"), **out)
    orr.close()

    # ---------------- first scan on an empty map + a short SLAM run (HectorSlamProcessor::update) -
    os_ = Oracle(kind, RES, SIZE, 3)
    os_.set_update_factors(0.4, 0.9)
    os_.set_map_update_thresholds(0.0, 0.0)
    rng = np.random.default_rng(99)
    traj = [np.array([-3.0, -2.0, 0.2])]
    for i in range(11):
        traj.append(traj[-1] + np.array([0.15, 0.04, 0.02]))
    traj = np.asarray(traj)
    sl_scans = np.stack([synth.make_scan(world, p, rng) for p in traj])
    est = []
    hint = traj[0].astype(np.float32)
    for k in range(len(traj)):
        pose, cov = os_.update(sl_scans[k], hint)
        est.append(pose)
        hint = pose  # the node feeds the last estimate back (HectorMappingRos.cpp:314)
    out = dict(res=np.float32(RES), size=np.int32(SIZE), levels=np.int32(3), factors=np.float32([0.4, 0.9]),
               scans=sl_scans.astype(np.float32), traj=traj, est=np.float32(est), first_hint=traj[0].astype(np.float32))
    planes_sparse(os_, "final", out)
    np.savez_compressed(os.path.join(OUT, "slam3.npz"), **out)
    os_.close()
    gen_next(kind)
    for f in sorted(os.listdir(OUT)):
        print(f, os.path.getsize(os.path.join(OUT, f)))


def gen_next(kind="reference"):
    """next.npz — the "next" rows of SURVEY.md §8f, from the compiled reference: the node's point-cloud converter
    (HectorMappingRos.cpp:509-542, source text compiled by oracle/ros_conv_driver.cpp), the sigma-point covariance
    (OccGridMapUtil.h:106-187) and hector_map_tools' ray cast / getDist (HectorMapTools.h:133-237, header compiled by
    oracle/maptools_driver.cpp) on the match3 map."""
    from oracle import pyoracle

    g = np.load(os.path.join(OUT, "match3.npz"))
    out = {}
    # point clouds
    rng = np.random.default_rng(77)
    fmt = synth.CLOUD_FORMAT
    world = synth.World(1, seed=1234)
    clouds, Ts, kept, origos = [], [], [], []
    for k in range(6):
        T = synth.laser_transform(xyz=rng.uniform(-0.3, 0.3, 3), rpy=rng.uniform(-0.06, 0.06, 3))
        pose = world.sample_free_poses(1, rng)[0]
        cloud = synth.ranges_to_cloud(world.cast(pose) + rng.normal(0, 0.01, synth.N_BEAMS))
        cloud[::11, 2] = rng.uniform(-1.6, 1.6, cloud[::11].shape[0])         # some outside the z window
        cloud[5] = (-0.5, 0.3, 0.0)
        cloud[6] = (0.3, 0.2, 0.0)
        pts, og = pyoracle.cloud_to_points(cloud, T, fmt["sqr_laser_min_dist"], fmt["sqr_laser_max_dist"],
                                           fmt["laser_z_min_value"], fmt["laser_z_max_value"], 20.0, kind=kind)
        clouds.append(cloud)
        Ts.append(T)
        kept.append(pts)
        origos.append(og)
    out["cloud_offsets"] = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int32)
    out["cloud_xyz"] = np.concatenate(clouds).astype(np.float32)
    out["cloud_T"] = np.asarray(Ts, np.float64)
    out["cloud_kept_offsets"] = np.concatenate([[0], np.cumsum([c.shape[0] for c in kept])]).astype(np.int32)
    out["cloud_kept"] = np.concatenate(kept).astype(np.float32)
    out["cloud_origo"] = np.asarray(origos, np.float32)
    # covariance + map tools on the match3 map
    size = int(g["size"])
    orc = Oracle(kind, float(g["res"]), size, 3)
    for l in range(3):
        p = np.zeros((size >> l) ** 2, np.float32)
        p[g[f"map_idx{l}"]] = g[f"map_val{l}"]
        orc.set_logodds(l, p.reshape(size >> l, size >> l))
    cm, cw = [], []
    for l in range(3):
        for k in range(K):
            a, b = orc.covariance_for_pose(l, orc.map_coords_pose(l, g["ref_poses"][k]),
                                           (g["scans"][k] * np.float32(2.0 ** -l)).astype(np.float32))
            cm.append(a)
            cw.append(b)
    out["cov_map"] = np.asarray(cm, np.float32).reshape(3, K, 3, 3)
    out["cov_world"] = np.asarray(cw, np.float32).reshape(3, K, 3, 3)
    port = Oracle("port", float(g["res"]), size, 3)   # only for the level geometry (map origin)
    lo = orc.get_logodds(0)
    occ = np.where(lo < 0, 0, np.where(lo > 0, 100, -1)).astype(np.int8)
    origin = port.map_origin(0)
    mt = pyoracle.RefMapTools(occ, float(g["res"]), origin)
    B = 400
    begin = rng.integers(int(0.3 * size), int(0.7 * size), (B, 2)).astype(np.int32)
    end = rng.integers(-5, size + 5, (B, 2)).astype(np.int32)
    bw = rng.uniform(-7, 7, (B, 2)).astype(np.float32)
    ew = rng.uniform(-14, 14, (B, 2)).astype(np.float32)
    rc = [mt.raycast(begin[i], end[i]) for i in range(B)]
    gd = [mt.get_dist(bw[i], ew[i]) for i in range(B)]
    out.update(ray_begin=begin, ray_end=end, ray_dist=np.float32([r[0] for r in rc]), ray_hit=np.int32([r[1] for r in rc]),
               gd_begin=bw, gd_end=ew, gd_dist=np.float32([r[0] for r in gd]), gd_hit=np.float32([r[1] for r in gd]),
               gd_found=np.int8([r[2] for r in gd]), map_origin=origin)
    mt.close()
    orc.close()
    port.close()
    np.savez_compressed(os.path.join(OUT, "next.npz"), **out)


# ---------------- deep pyramids: 8 and 5 levels (tests/deep_cases.py) ------------------------------------------------
# (sx, sy, levels, start, resolution): the 8-level map whose coarse widths take every residue mod 4, and the node's
# default size with two more levels than its default 3
DEEP_GEOMS = {"g8": (1000, 640, 8, (0.3, 0.7), 0.05), "g5": (2048, 2048, 5, (0.5, 0.5), 0.025)}
# maxIterations per level, level 0 first, in every encoding of hsb_config::max_iterations (0: the reference's literal,
# -1: none, n: n), truncated to the depth
DEEP_SCHEDULES = {"default": None, "mixed": [0, -1, 2, 7, -1, 1, 0, 4], "single": [-1] * 8}
DEEP_STEPS, DEEP_MWM, DEEP_MATCHES = 14, (6, 7, 11), 12


def deep_run(g):
    """A short SLAM run for geometry g: 1081-beam scans along a path in the one-room world, and which steps are
    map_without_matching (two in a row and one later, none first: the coarse levels then write from the container of
    the last matched scan).  Every step's hint is the path's pose, as when odometry supplies the start estimate: on
    the 8-level map the coarsest levels (6.4 m cells, 7 x 5 of them) send the reference's own matcher tens of metres
    off on a map of one or two scans, and a run that fed its estimates back would leave the map at the second step.
    -> (scans (K, 1081, 2), mwm (K,) bool, hints (K, 3), the path (K, 3) float64)"""
    world = synth.World(1, seed=1234)
    rng = np.random.default_rng(4242)
    traj = np.array([-3.0, -2.0, 0.2]) + np.arange(DEEP_STEPS)[:, None] * np.array([0.12, 0.05, 0.025])
    scans = np.stack([synth.make_scan(world, p, rng, 1.0 / g[4]) for p in traj]).astype(np.float32)
    mwm = np.zeros(DEEP_STEPS, bool)
    mwm[list(DEEP_MWM)] = True
    return scans, mwm, traj.astype(np.float32), traj


def deep_matches(g, traj):
    """DEEP_MATCHES scans from poses around the path, with perturbed hints, an empty one last"""
    world = synth.World(1, seed=1234)
    rng = np.random.default_rng(777)
    poses = traj[rng.integers(0, len(traj), DEEP_MATCHES)] + rng.uniform(-0.3, 0.3, (DEEP_MATCHES, 3)) * [1, 1, 0.3]
    scans = np.stack([synth.make_scan(world, p, rng, 1.0 / g[4]) for p in poses]).astype(np.float32)
    return scans, synth.perturb_hints(poses, seed=5, dxy=0.08, dpsi=0.04).astype(np.float32)


def deep_arrays(kind="reference"):
    """The arrays of deep.npz from the compiled reference or (kind="port") the C port: per geometry the run's poses,
    covariances and final planes, then matchData on the final map under the default and the mixed schedule with what
    the matcher reports to its hooks (oracle/record_oracle.py)."""
    from oracle.record_oracle import RecordOracle, port_hooks

    out = {}
    for tag, g in DEEP_GEOMS.items():
        sx, sy, L, start, res = g
        orc = RecordOracle(kind, res, sx, L, start=start, size_y=sy)
        orc.set_update_factors(0.4, 0.9)
        orc.set_map_update_thresholds(0.0, 0.0)
        scans, mwm, hints, traj = deep_run(g)
        est, cov = [], []
        for k in range(DEEP_STEPS):
            p, c = orc.update(scans[k], hints[k], map_without_matching=bool(mwm[k]))
            est.append(p)
            cov.append(c.reshape(9))
        out.update({f"{tag}_geom": np.float64([sx, sy, L, start[0], start[1], res]), f"{tag}_run_scans": scans,
                    f"{tag}_run_mwm": mwm, f"{tag}_run_hints": hints,
                    f"{tag}_run_est": np.float32(est), f"{tag}_run_cov": np.float32(cov)})
        for l in range(L):
            out[f"{tag}_final{l}"] = orc.get_logodds(l)
        mscans, mhints = deep_matches(g, traj)
        out[f"{tag}_match_scans"], out[f"{tag}_match_hints"] = mscans, mhints
        for name in ("default", "mixed"):
            iters = None if DEEP_SCHEDULES[name] is None else DEEP_SCHEDULES[name][:L]
            P, Cv, Hk = [], [], []
            for k in range(DEEP_MATCHES):
                if kind == "reference":
                    p, c, hooks, _ = orc.match_record(mhints[k], mscans[k], iters)
                else:
                    p, c, rec = orc.match_record(mhints[k], mscans[k], iters)
                    hooks = port_hooks(orc, rec, mscans[k].shape[0], iters)
                P.append(p)
                Cv.append(c.reshape(9))
                Hk.append(hooks)
            out[f"{tag}_{name}_poses"], out[f"{tag}_{name}_cov"] = np.float32(P), np.float32(Cv)
            out[f"{tag}_{name}_hooks"] = np.float32(Hk)
        orc.close()
    return out


def gen_deep(kind="reference"):
    np.savez_compressed(os.path.join(OUT, "deep.npz"), **deep_arrays(kind))


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "next":
        gen_next()
    elif len(sys.argv) > 1 and sys.argv[1] == "deep":
        gen_deep()
    else:
        main()
