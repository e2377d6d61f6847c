"""GPU: ending a level's Gauss-Newton loop at a fixed point (tuning key `fixpoint`) changes no bit.

Once an evaluation leaves the pose bitwise unchanged, every later evaluation of the level would repeat it exactly, so
the match kernel stops there (match_kernel.cuh).  Here `fixpoint = 1` (the default) is compared with `fixpoint = 0`,
which runs every evaluation, in the same process:

  * batch matches with and without the per-evaluation record, in every launch shape the auto-launcher picks
    (1 x 32, 1 x 28, 1 x 1 and 2 / 4 / 8 / 16 warps per scan), the paired path and both gather modes: poses,
    covariances and full records bitwise equal;
  * hsb_match_data (with / without record, scan inside the launch or copied), hsb_slam_update (waiting and nowait) and
    the fused cloud, ranges and projected steps, single and group: poses, covariances, gate decisions and every level's
    map bitwise equal;
  * edge cases in every batch: a scan entirely outside the map (H = 0 from the first evaluation) and an empty scan;
    on a one-level map, hints that already are a fixed point (the match stops after its first evaluation);
  * the trace's evaluation count of each scan equals what the full record predicts (per level: up to and including
    the first evaluation that leaves the pose unchanged), and bench-like scans do skip.
"""
import numpy as np
import pytest

from conftest import report

pytestmark = pytest.mark.gpu

RES, SIZE, LEVELS = 0.05, 512, 3
SCALE = 1.0 / RES
F32 = np.float32
MODES = (1, 2)   # LDG, TEX
RESET = dict(warps_per_scan=0, scans_per_block=0, unroll=0, stage_smem=1, partial=1, packed=0, seq=0, inline_scan=0,
             host_out=1, auto_group=1, trace=0, fixpoint=1)
# (warps per scan, scans per block): every shape the auto-launcher picks
SHAPES = [(1, 32), (1, 28), (1, 1), (2, 1), (4, 1), (8, 1), (16, 1)]


def bits(a):
    return np.ascontiguousarray(a, F32).view(np.uint32)


def same(a, b):
    """bitwise for float32 results, exact otherwise (gate flags, kept counts)"""
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype == F32 and b.dtype == F32:
        return np.array_equal(bits(a), bits(b))
    return a.dtype == b.dtype and np.array_equal(a, b)


@pytest.fixture(scope="module")
def env(hsb_lib):
    """A 512^2 3-level map built with known poses (bench.py's recipe on a one-room world), loaded into one handle per
    gather mode, and a batch of bench-like scans (hints +-0.1 m / +-0.05 rad) with the edge cases appended."""
    from hector_slam_b200 import capi, synth

    world = synth.World.for_map_size(SIZE)
    builder = capi.MapRepB200(RES, SIZE, levels=LEVELS, update_factor_free=0.4, update_factor_occupied=0.9)
    rng = np.random.default_rng(11)
    for p in world.mapping_poses():
        scan = synth.make_scan(world, p, rng, SCALE)
        p32 = p.astype(F32)
        builder.matchData(p32, scan)
        builder.updateByScan(scan, p32)
        builder.onMapUpdated()
    logodds = [builder.download_level(l) for l in range(LEVELS)]
    builder.close()
    reps = {}
    for mode in MODES:
        rep = capi.MapRepB200(RES, SIZE, levels=LEVELS, gather_mode=mode, update_factor_free=0.4,
                              update_factor_occupied=0.9)
        for l in range(LEVELS):
            rep.upload_level(l, logodds[l])
        reps[mode] = rep
    B = 160
    poses = world.sample_free_poses(B, np.random.default_rng(5))
    pts, offs = synth.make_scan_batch(world, poses, noise_seed=9, scale_to_map=SCALE)
    hints = synth.perturb_hints(poses, seed=3, dxy=0.1, dpsi=0.05)
    scans = [pts[offs[b]:offs[b + 1]] for b in range(B)]
    # a hint at the pose this match returns when started from its own result (the coarse levels still move it)
    rep = reps[2]
    rep.set_tuning(**RESET)
    again = hints[0]
    for _ in range(4):
        again, _ = rep.matchData(again, scans[0])
    scans += [np.zeros((0, 2), F32), (scans[1] + F32(1e5)).astype(F32), scans[0]]
    hints = np.concatenate([hints, np.stack([hints[0], hints[1], again])]).astype(F32)
    pts = np.concatenate(scans).astype(F32)
    offs = np.concatenate([[0], np.cumsum([s.shape[0] for s in scans])]).astype(np.int32)
    yield dict(world=world, logodds=logodds, reps=reps, scans=scans, hints=hints, pts=pts, offs=offs)
    for r in reps.values():
        r.close()


def batch(rep, e, record, **tuning):
    rep.set_tuning(**{**RESET, **tuning})
    if record:
        P, C, _, raw = rep.match_batch_record(e["hints"], e["pts"], e["offs"])
        return P, C, raw
    P, C = rep.match_batch(e["hints"], e["pts"], e["offs"])
    return P, C, None


def predicted_counts(rep, e, recs):
    """Evaluations each scan runs with `fixpoint` on, from the record of a run with it off: per level, up to and
    including the first evaluation whose estimate equals the pose it started from."""
    B = e["hints"].shape[0]
    out = np.zeros(B, np.int64)
    for b in range(B):
        if e["scans"][b].shape[0] == 0:
            continue
        for l in range(rep.levels - 1, -1, -1):
            r = recs[l]
            E = r["est"].shape[1]
            prev = rep.map_coords_pose(l, r["start"][b])
            ran = E
            for k in range(E):
                if np.array_equal(bits(r["est"][b, k]), bits(prev)):
                    ran = k + 1
                    break
                prev = r["est"][b, k]
            out[b] += ran
    return out


@pytest.mark.parametrize("mode", MODES)
def test_batch_every_shape(env, mode):
    e = env
    rep = e["reps"][mode]
    variants = [dict(warps_per_scan=W, scans_per_block=G) for W, G in SHAPES]
    variants += [dict(warps_per_scan=1, scans_per_block=32, stage_smem=0), dict(warps_per_scan=1, scans_per_block=1,
                                                                                 stage_smem=2)]
    if mode == 2:
        variants += [dict(warps_per_scan=W, scans_per_block=G, packed=1) for W, G in SHAPES]
    variants += [dict()]   # the auto shape of this batch
    for tune in variants:
        for record in (False, True):
            P0, C0, R0 = batch(rep, e, record, fixpoint=0, **tune)
            P1, C1, R1 = batch(rep, e, record, fixpoint=1, **tune)
            case = (mode, tune, record)
            assert np.array_equal(bits(P0), bits(P1)), case
            assert np.array_equal(bits(C0), bits(C1)), case
            if record:
                assert np.array_equal(bits(R0), bits(R1)), case
    rep.set_tuning(**RESET)
    report(f"fixpoint: mode {mode}, {len(variants)} launch shapes: poses, covariances and records bit-identical on / off")


@pytest.mark.parametrize("mode", MODES)
def test_trace_counts_match_record(env, mode):
    e = env
    rep = e["reps"][mode]
    B = e["hints"].shape[0]
    full = rep.level_evals()
    for W, G in SHAPES:
        P0, _, raw0 = batch(rep, e, True, fixpoint=0, trace=1, warps_per_scan=W, scans_per_block=G)
        tr0 = rep.read_trace(B)
        assert (tr0[:, 5] == sum(full) * np.array([s.shape[0] > 0 for s in e["scans"]])).all(), (W, G)
        want = predicted_counts(rep, e, rep.split_record(raw0))
        P1, _, _ = batch(rep, e, True, fixpoint=1, trace=1, warps_per_scan=W, scans_per_block=G)
        tr1 = rep.read_trace(B).astype(np.int64)
        assert np.array_equal(bits(P0), bits(P1)), (W, G)
        assert np.array_equal(tr1[:, 5], want), (W, G, np.flatnonzero(tr1[:, 5] != want)[:8])
    rep.set_tuning(**RESET)
    ran = tr1[:-3, 5]   # the bench-like scans
    assert (ran < sum(full)).sum() > 0
    assert tr1[-3, 5] == 0                   # empty scan
    assert tr1[-2, 5] == LEVELS              # outside the map: H = 0 at the first evaluation of every level
    report(f"fixpoint: mode {mode}, {ran.size} bench-like scans: {int((ran < sum(full)).sum())} skip, evaluations run "
           f"{int(ran.sum())} of {ran.size * sum(full)} ({1 - ran.sum() / (ran.size * sum(full)):.1%} skipped); the "
           f"re-matched hint ran {int(tr1[-1, 5])}")


@pytest.mark.parametrize("mode", MODES)
def test_match_data_paths(env, mode):
    e = env
    rep = e["reps"][mode]
    for k in (0, 7, len(e["scans"]) - 3, len(e["scans"]) - 2, len(e["scans"]) - 1):
        hint, scan = e["hints"][k], e["scans"][k]
        cov_in = np.arange(9, dtype=F32).reshape(3, 3)
        for inl in (0, 1):
            out = []
            for fp in (0, 1):
                rep.set_tuning(**{**RESET, "inline_scan": inl, "fixpoint": fp})
                p, c = rep.matchData(hint, scan, cov_inout=cov_in)
                pr, cr, rec = rep.matchData(hint, scan, cov_inout=cov_in, record=True)
                flat = np.concatenate([np.concatenate([rec[l]["start"], np.concatenate(
                    [rec[l]["H"].reshape(-1, 9), rec[l]["dTr"], rec[l]["est"]], axis=1).reshape(-1)])
                    for l in range(LEVELS - 1, -1, -1)])
                out.append((p, c, pr, cr, flat))
            for a, b in zip(out[0], out[1]):
                assert np.array_equal(bits(a), bits(b)), (mode, k, inl)
    rep.set_tuning(**RESET)


def test_fixed_point_hints(env):
    """One level: hints the match returns unchanged (found by re-matching from the result, in the 8-warp shape that a
    single scan and a small batch share); such a hint is a fixed point of the first evaluation unless the pose moved
    within the rounding of the map -> world conversion."""
    from hector_slam_b200 import capi

    e = env
    rep = capi.MapRepB200(RES, SIZE, levels=1, update_factor_free=0.4, update_factor_occupied=0.9)
    rep.upload_level(0, e["logodds"][0])
    rep.set_tuning(**RESET)
    hints, scans = [], []
    for k in range(24):
        h = e["hints"][k]
        for _ in range(12):
            p, _ = rep.matchData(h, e["scans"][k])
            if np.array_equal(bits(p), bits(h)):
                hints.append(h)
                scans.append(e["scans"][k])
                break
            h = p
    assert len(hints) > 0
    f = dict(hints=np.stack(hints).astype(F32), scans=scans, pts=np.concatenate(scans).astype(F32),
             offs=np.concatenate([[0], np.cumsum([s.shape[0] for s in scans])]).astype(np.int32))
    B = len(hints)
    for tune in [dict(warps_per_scan=W, scans_per_block=G) for W, G in SHAPES]:
        P0, C0, R0 = batch(rep, f, True, fixpoint=0, trace=1, **tune)
        want = predicted_counts(rep, f, rep.split_record(R0))
        P1, C1, R1 = batch(rep, f, True, fixpoint=1, trace=1, **tune)
        ran = rep.read_trace(B)[:, 5].astype(np.int64)
        assert np.array_equal(bits(P0), bits(P1)) and np.array_equal(bits(C0), bits(C1)), tune
        assert np.array_equal(bits(R0), bits(R1)), tune
        assert np.array_equal(ran, want), tune
        if tune["warps_per_scan"] == 8:
            first = int((ran == 1).sum())
            assert first > 0, ran
    report(f"fixpoint: {B} of 24 one-level hints are returned unchanged by the match; {first} of them stop after the "
           f"first evaluation")
    rep.close()


# ---- SLAM steps: twin handles, one with fixpoint off ------------------------------------------------------------------
def twins(e, n, mode=2):
    from hector_slam_b200 import capi, synth

    sides = []
    for fp in (0, 1):
        side = []
        for s in range(n):
            rep = capi.MapRepB200(RES, SIZE, levels=LEVELS, gather_mode=mode, update_factor_free=0.4,
                                  update_factor_occupied=0.9)
            for l in range(LEVELS):
                rep.upload_level(l, e["logodds"][l])
            rep.set_tuning(fixpoint=fp)
            rep.setMapUpdateMinDistDiff(0.1 * s)
            rep.set_scan_format(**synth.SCAN_FORMAT)
            rep.set_cloud_format(synth.laser_transform(), **synth.CLOUD_FORMAT)
            rep.set_laser_projection(**synth.SCAN_FORMAT, range_cutoff=30.0)
            side.append(rep)
        sides.append(side)
    return sides


def trajectory(e, seed, steps):
    """ranges along a short drive from a free pose, with hints off the true pose"""
    rng = np.random.default_rng(seed)
    pose = e["world"].sample_free_poses(1, rng)[0].astype(np.float64)
    out = []
    for _ in range(steps):
        r = (e["world"].cast(pose) + rng.normal(0.0, 0.01, 1081)).astype(F32)
        hint = (pose + rng.uniform(-1, 1, 3) * np.array([0.04, 0.04, 0.02])).astype(F32)
        out.append((hint, r))
        pose = pose + np.array([0.06 * np.cos(pose[2]), 0.06 * np.sin(pose[2]), rng.uniform(-0.05, 0.05)])
    return out


def same_state(a, b, tag):
    for l in range(LEVELS):
        assert np.array_equal(a.download_level(l), b.download_level(l)), (tag, l)
        assert np.array_equal(a.download_prob(l), b.download_prob(l)), (tag, l)
    assert np.array_equal(bits(a.last_map_update_pose()), bits(b.last_map_update_pose())), tag


def test_single_slam_steps(env):
    from hector_slam_b200 import synth

    e = env
    off, on = (side[0] for side in twins(e, 1))
    T = synth.laser_transform()
    for k, (hint, r) in enumerate(trajectory(e, 21, 12)):
        kind = k % 5
        res = []
        for rep in (off, on):
            if kind in (0, 1):
                res.append(rep.slam_update(hint, synth.ranges_to_points(r, SCALE), nowait=kind == 1))
            elif kind == 2:
                res.append(rep.slam_update_cloud(hint, synth.ranges_to_cloud(r), transform=T))
            elif kind == 3:
                res.append(rep.slam_update_ranges(hint, r))
            else:
                res.append(rep.slam_update_projected(hint, r, transform=T))
        for a, b in zip(res[0], res[1]):
            assert same(a, b), (k, kind)
    same_state(off, on, "single steps")
    off.close()
    on.close()


def test_group_slam_steps(env):
    from hector_slam_b200 import capi, synth

    e = env
    M = 3
    sides = twins(e, M)
    groups = [capi.SlamGroup(side) for side in sides]
    trajs = [trajectory(e, 40 + s, 8) for s in range(M)]
    T = np.stack([synth.laser_transform()] * M)
    for k in range(8):
        hints = np.stack([trajs[s][k][0] for s in range(M)])
        ranges = [trajs[s][k][1] for s in range(M)]
        kind = k % 4
        res = []
        for grp in groups:
            if kind == 0:
                res.append(grp.slam_update(hints, [synth.ranges_to_points(r, SCALE) for r in ranges], nowait=k % 2 == 1))
            elif kind == 1:
                res.append(grp.slam_update_cloud(hints, [synth.ranges_to_cloud(r) for r in ranges], transforms=T))
            elif kind == 2:
                res.append(grp.slam_update_ranges(hints, ranges))
            else:
                res.append(grp.slam_update_projected(hints, ranges, transforms=T))
        for a, b in zip(res[0], res[1]):
            assert same(a, b), (k, kind)
    for s in range(M):
        same_state(sides[0][s], sides[1][s], f"group session {s}")
    for grp in groups:
        grp.close()
    for side in sides:
        for rep in side:
            rep.close()
