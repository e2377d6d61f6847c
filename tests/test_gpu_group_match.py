"""Matching a group's pose hints in one pass (hsb_group_match_batch and its _subset form): every hint of a session runs
the full coarse-to-fine matchData on its member's map with the session's one scan, by one launch of the match kernel,
with one copy each way; the scan either sent with the call or the member's last matched scan as it lies on the device.

Every pose and covariance is compared in bits with hsb_match_batch in shared-scan mode on the member, run with the
warps per scan the group call reports, on maps written by mixed full, subset, nowait and map_without_matching group
steps of every input kind, on three non-square geometries, with ragged and empty sessions and non-finite hints, over
permuted member lists; the number of hints selects each of 8, 4, 2 and 1 warps per scan, and each is also forced
through handles[0]'s tuning.  Also: the CPU oracle, last-match mode (conversions that drop beams, right after nowait
steps of this group, of a member alone and of a second group), no member state change, relocalisation (match, then the
best hypothesis), launch accounting, rejections and the C++ façade.  Every group case runs on a TEX and an LDG group."""
import ctypes as C
import os

import numpy as np
import pytest

import maptools_cases as mc
from conftest import ROOT
from test_gpu_group_score import (GEOM, GEOMS, KINDS, SENTINEL, Tracker, bits, close_all, fleet, hypotheses, single_best,
                                  state, step)
from test_gpu_group_subset import geometry, group_step, session_data

pytestmark = pytest.mark.gpu

F32 = np.float32
MODES = pytest.mark.parametrize("mode", [2, 1], ids=["tex", "ldg"])   # capi.GATHER_TEX, capi.GATHER_LDG
COUNTS = (0, 1, 7, 33, 700)


def sm_count():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def auto_w(Q):
    """the warps per scan hsb_match_batch takes for one batch of Q scans under the default tuning"""
    want, W = sm_count() * 24 // max(Q, 1), 1
    while W * 2 <= want and W < 8:
        W *= 2
    return W


def ragged(rng, K, target):
    """K hint counts drawn from COUNTS (permuted), the largest replaced so that they sum to `target`"""
    c = [int(x) for x in rng.permutation(np.resize(COUNTS, K))]
    big = int(np.argmax(c))
    c[big] = 0
    c[big] = max(target - sum(c), 0)
    return c


def single_match(rep, hints, scan, W, restore=0):
    """hsb_match_batch in shared-scan mode on one member with W warps per scan -> (poses, cov (B, 9))"""
    rep.set_tuning(warps_per_scan=W)
    try:
        poses, cov = rep.match_batch(np.ascontiguousarray(hints, F32), np.ascontiguousarray(scan, F32).reshape(-1, 2))
    finally:
        rep.set_tuning(warps_per_scan=restore)
    return poses, cov.reshape(-1, 9)


def assert_match(g, reps, members, hints, scans, points, tag, restore=0):
    """The group call over `members` (None: all) against hsb_match_batch on each member, in bits.  scans: each session's
    scan; points: what the group call is given (the scans, or None for the last matched scans).
    -> (poses, cov (Q, 9), W the call reported)"""
    sel = list(range(len(reps))) if members is None else members
    poses, cov = g.match_batch(hints, points, members=members)
    cov = cov.reshape(-1, 9)
    W = reps[0].last_launch_shape()["warps_per_scan"]
    q = 0
    for k, j in enumerate(sel):
        n = hints[k].shape[0]
        if n:
            wp, wc = single_match(reps[j], hints[k], scans[k], W, restore)
            assert np.array_equal(bits(poses[q:q + n]), bits(wp)), tag + (k, j, W)
            assert np.array_equal(bits(cov[q:q + n]), bits(wc)), tag + (k, j, W)
            if scans[k].shape[0] == 0:   # an empty scan: the hint and a zero matrix
                assert np.array_equal(bits(poses[q:q + n]), bits(hints[k])) and not cov[q:q + n].any(), tag
        q += n
    assert q == poses.shape[0]
    return poses, cov, W


# ---- 1: against the single call ----------------------------------------------------------------------------------

@MODES
@pytest.mark.parametrize("geom", GEOMS, ids=mc.geom_id)
def test_against_single_calls(hsb_lib, geom, mode):
    """Fleets of 3 to 6 members, 8 ticks of full and subset, sync and nowait group steps of every input kind (some
    sessions map_without_matching); after every tick a group match over a permuted subset with ragged sessions (0 to
    hundreds of hints, NaN and infinite hints, angles past 120 rad), the scans sent with the call.  The first four ticks
    size the call so that the default tuning takes 8, 4, 2 and 1 warps per scan; the last four force each through
    handles[0]'s tuning.  Then one call over every member whose scans hold more than 1 MB of endpoints in all (more than
    131 072 points: past what the call stages in pinned memory), one session without hints.  Everything equals
    hsb_match_batch on the members in bits."""
    M, ticks = 3 + GEOMS.index(geom) + (1 if mode == 1 else 0), 8
    reps, g = fleet(geom, M, mode)
    track = Tracker(geom, M, mode)
    data = [session_data(5100 + s, ticks, geometry(s)) for s in range(M)]
    rng = np.random.default_rng(141)
    at = [0] * M
    sm = sm_count()
    seen, moved = set(), 0
    for t in range(ticks):
        members = None if t % 4 == 0 else [int(j) for j in rng.permutation(M)[:int(rng.integers(1, M + 1))]]
        step([g], data, at, KINDS[t % 4], members, rng, nowait=(t % 3 != 0), track=track)
        sel = [int(j) for j in rng.permutation(M)[:int(rng.integers(1, M + 1))]]
        forced = (0, 0, 0, 0, 8, 4, 2, 1)[t]
        target = (2 * sm, 5 * sm, 10 * sm, 14 * sm)[t % 4] if not forced else int(rng.integers(40, 3 * sm))
        counts = ragged(rng, len(sel), target)
        hints = [hypotheses(rng, track.pose[j], c) for j, c in zip(sel, counts)]
        scans = [track.scan(j)[::1 + k % 3] for k, j in enumerate(sel)]
        reps[0].set_tuning(warps_per_scan=forced)
        poses, _, W = assert_match(g, reps, sel, hints, scans, scans, ("tick", t), restore=forced)
        reps[0].set_tuning(warps_per_scan=0)
        assert W == (forced or auto_w(sum(counts))), (t, W, sum(counts))
        seen.add(W)
        h = np.concatenate(hints)
        ok = np.all(np.isfinite(h), axis=1)
        moved += int((np.abs(poses[ok, :2] - h[ok, :2]).max(axis=1) > 1e-3).sum())
    sel = [int(j) for j in rng.permutation(M)]
    counts = [(7, 0, 33, 1)[k % 4] for k in range(M)]
    hints = [hypotheses(rng, track.pose[j], c) for j, c in zip(sel, counts)]
    lengths = [48000 + 2000 * k for k in range(M)]
    scans = [(np.resize(track.scan(j), (n, 2)) + rng.normal(0.0, 0.25, (n, 2))).astype(F32) for j, n in zip(sel, lengths)]
    assert sum(s.shape[0] for s in scans) > 131072
    assert_match(g, reps, sel, hints, scans, scans, ("past 1 MB",))
    assert seen == {1, 2, 4, 8}
    assert moved > 100    # the hints were matched, not passed through
    close_all(g, reps, track)


# ---- 2: against the CPU oracle -----------------------------------------------------------------------------------

@MODES
def test_against_oracle(hsb_lib, pyoracle, oracle_kinds, mode):
    """The 3-level 2048^2 map the CPU oracle builds from known poses (the batch parity test's), uploaded into three
    members; each member's session matches 24 hints around its own pose with its own scan, in one group call.  Every
    pose the oracle does not diverge on lies within the batch tests' 1e-4 m / 1e-4 rad of the oracle's."""
    from hector_slam_b200 import capi, synth

    kind = "reference" if "reference" in oracle_kinds else "port"
    world = synth.World.for_map_size(2048)
    orc = pyoracle.Oracle(kind, 0.05, 2048, 3)
    orc.set_update_factors(0.4, 0.9)
    pyoracle.build_map_known_poses(orc, world)
    M, H = 3, 24
    reps = [capi.MapRepB200(0.05, 2048, levels=3, update_factor_free=0.4, update_factor_occupied=0.9, gather_mode=mode)
            for _ in range(M)]
    for rep in reps:
        for l in range(3):
            rep.upload_level(l, orc.get_logodds(l))
    g = capi.SlamGroup(reps)
    rng = np.random.default_rng(143)
    truth = world.sample_free_poses(M, rng)
    pts, offs = synth.make_scan_batch(world, truth, noise_seed=9)
    members = [2, 0, 1]
    scans = [np.ascontiguousarray(pts[offs[j]:offs[j + 1]], F32) for j in members]
    hints = [np.ascontiguousarray(synth.perturb_hints(np.repeat(truth[j][None], H, axis=0), seed=20 + j, dxy=0.1,
                                                      dpsi=0.05), F32) for j in members]
    poses, _ = g.match_batch(hints, scans, members=members)
    checked = 0
    for k, j in enumerate(members):
        n = scans[k].shape[0]
        want, _, _ = orc.match_batch(hints[k], np.tile(scans[k], (H, 1)), np.arange(H + 1, dtype=np.int32) * n)
        ok = np.abs(want[:, :2] - hints[k][:, :2]).max(axis=1) < 0.5   # oracle divergences (SURVEY.md Q4) are left out
        assert ok.mean() > 0.9, (k, j)
        got = poses[k * H:(k + 1) * H][ok].astype(np.float64)
        d = np.abs(got - want[ok].astype(np.float64))
        d[:, 2] = np.abs((d[:, 2] + np.pi) % (2 * np.pi) - np.pi)
        assert d[:, :2].max() <= 1e-4 and d[:, 2].max() <= 1e-4, (k, j, d.max(axis=0))
        assert np.abs(got[:, :2] - truth[j][:2]).max() < 0.03, (k, j)   # and close to the ground truth
        checked += int(ok.sum())
    assert checked >= 0.9 * M * H
    orc.close()
    close_all(g, reps)


# ---- 3: the last matched scan ------------------------------------------------------------------------------------

@MODES
def test_last_match_mode(hsb_lib, mode):
    """M = 5, 12 ticks of group steps of every input kind (full and subset, sync and nowait, some sessions
    map_without_matching; every 7th beam of a converted scan is one its conversion drops), and on some ticks a nowait
    single step of one member and a nowait step of a second group holding one member.  Straight after each, the group
    call without points over a permuted subset equals the call with the converted scans sent and hsb_match_batch on each
    member.  Before its first step a member returns its hints and zero covariances."""
    from hector_slam_b200 import capi

    M, ticks = 5, 12
    reps, g = fleet(GEOM, M, mode)
    solo = capi.SlamGroup([reps[3]])
    track = Tracker(GEOM, M, mode)
    data = [session_data(5300 + s, 3 * ticks, geometry(s)) for s in range(M)]
    rng = np.random.default_rng(147)
    at = [0] * M

    def check(ask, tag):
        hints = [hypotheses(rng, track.pose[j], int(rng.choice((1, 7, 33)))) for j in ask]
        scans = [track.scan(j) for j in ask]
        p_last, c_last, _ = assert_match(g, reps, ask, hints, scans, None, tag)
        p_sent, c_sent = g.match_batch(hints, scans, members=ask)
        assert np.array_equal(bits(p_last), bits(p_sent)) and np.array_equal(bits(c_last), bits(c_sent.reshape(-1, 9))), tag

    hints = [hypotheses(rng, (0, 0, 0), 5) for _ in range(M)]
    poses, cov = g.match_batch(hints)
    assert np.array_equal(bits(poses), bits(np.concatenate(hints))) and not cov.any()
    kept_below = 0
    for t in range(ticks):
        members = ([0, 3], [3, 1])[t] if t < 2 else None if t % 4 == 0 else \
            [int(j) for j in rng.permutation(M)[:int(rng.integers(1, M + 1))]]
        kind = KINDS[(t + t // 4) % 4]
        res = step([g], data, at, kind, members, rng, nowait=(t % 2 == 0), track=track, p_without=0.3)[0]
        if res[3] is not None:
            sel = list(range(M)) if members is None else members
            kept_below += sum(int(res[3][k]) < data[j]["ranges"][0].size for k, j in enumerate(sel))
        check([int(j) for j in rng.permutation(M)[:int(rng.integers(1, M + 1))]], ("group", t))
        if t % 3 == 2:
            j = t % M
            pose = reps[j].slam_update(data[j]["hints"][at[j]], data[j]["scans"][at[j]], nowait=True)[0]
            track.note(j, "endpoints", data[j]["scans"][at[j]], False, pose)
            at[j] += 1
            check([j, (j + 1) % M], ("single", t))
            k = at[3]
            pose = solo.slam_update(data[3]["hints"][k][None], [data[3]["scans"][k]], nowait=True)[0][0]
            track.note(3, "endpoints", data[3]["scans"][k], False, pose)
            at[3] += 1
            check([3, 0], ("other group", t))
    assert kept_below > 5      # conversions dropped beams: a stale count would have shown
    close_all(solo, g, reps, track)


# ---- 4: no state change ------------------------------------------------------------------------------------------

@MODES
def test_no_state_change(hsb_lib, mode):
    """Twin fleets take the same 8 ticks of group steps; fleet A matches, in both scan modes, over a subset after most
    of them.  Every step's results are equal in bits, and at the end every member's planes, grids, both dirty
    rectangles, gate pose and last matched scan are byte-identical to its twin's; the next group step gives the same
    bits on both fleets."""
    M, ticks = 5, 8
    a, ga = fleet(GEOM, M, mode)
    b, gb = fleet(GEOM, M, mode)
    track = Tracker(GEOM, M, mode)
    data = [session_data(5400 + s, ticks + 1, geometry(s)) for s in range(M)]
    rng = np.random.default_rng(149)
    at = [0] * M
    for t in range(ticks):
        members = None if t % 3 == 0 else [int(j) for j in rng.permutation(M)[:int(rng.integers(1, M + 1))]]
        ra, rb = step([ga, gb], data, at, KINDS[t % 4], members, rng, nowait=(t % 2 == 0), track=track)
        for x, y in zip(ra[:3], rb[:3]):
            assert np.array_equal(bits(x) if x.dtype != bool else x, bits(y) if y.dtype != bool else y), t
        if t % 4 != 3:
            sel = [int(j) for j in rng.permutation(M)[:int(rng.integers(1, M))]]
            hints = [hypotheses(rng, track.pose[j], 40) for j in sel]
            for points in (None, [track.scan(j) for j in sel]):
                ga.match_batch(hints, points, members=sel)
    poses = [hypotheses(rng, track.pose[j], 6, specials=False) for j in range(M)]
    la, lb = ga.likelihood(0, poses), gb.likelihood(0, poses)     # the last matched scans: the same points, the same size
    assert np.array_equal(bits(la), bits(lb)) and not np.isnan(la).any()
    for j in range(M):
        sa, sb = state(a[j]), state(b[j])
        for l, (x, y) in enumerate(zip(sa[0], sb[0])):
            assert all(np.array_equal(u, v) for u, v in zip(x[:3], y[:3])) and x[3] == y[3], (j, l)
        assert sa[1] == sb[1] and np.array_equal(sa[2], sb[2]), j
    ra, rb = step([ga, gb], data, at, "ranges", None, rng, nowait=False, p_without=0.3)
    for x, y in zip(ra[:3], rb[:3]):
        assert np.array_equal(bits(x) if x.dtype != bool else x, bits(y) if y.dtype != bool else y)
    close_all(ga, gb, a, b, track)


# ---- 5: relocalisation -------------------------------------------------------------------------------------------

def device_reloc(rep, hints, scan, W):
    """per member on the device: hsb_match_batch_device in shared-scan mode, then hsb_best_hypothesis_device on the
    returned poses -> (poses, best4)"""
    import torch

    B, n = hints.shape[0], scan.shape[0]
    d_h = torch.from_numpy(np.ascontiguousarray(hints, F32).reshape(-1)).cuda()
    d_p = torch.from_numpy(np.ascontiguousarray(scan, F32).reshape(-1)).cuda()
    d_out = torch.zeros(B * 3, dtype=torch.float32, device="cuda")
    d_cov = torch.zeros(B * 9, dtype=torch.float32, device="cuda")
    d_best = torch.zeros(4, dtype=torch.float32, device="cuda")
    rep.set_tuning(warps_per_scan=W)
    try:
        rep.match_batch_device(B, d_h.data_ptr(), d_p.data_ptr(), None, n, n, d_out.data_ptr(), d_cov.data_ptr())
        rep.best_hypothesis_device(0, B, d_out.data_ptr(), d_p.data_ptr(), None, n, d_best.data_ptr(), None, 0)
        torch.cuda.synchronize()
    finally:
        rep.set_tuning(warps_per_scan=0)
    return d_out.cpu().numpy().reshape(B, 3), d_best.cpu().numpy()


@MODES
def test_relocalisation(hsb_lib, mode):
    """Four robots whose 3-level maps of one synthetic room are written at known poses (registered to the world), each
    then stepped once by a group step at its own pose.  64 hints each, spread 0.25 m / 0.15 rad around the true pose:
    match_batch on the last matched scans, then best_hypothesis on the returned poses, equals the per-member device
    path in bits, and every winner lies within 5 cm / 0.03 rad of the true pose."""
    from hector_slam_b200 import capi, synth

    M, H = 4, 64
    world = synth.World(1, seed=77)
    reps = [capi.MapRepB200(0.05, 1024, levels=3, update_factor_free=0.4, update_factor_occupied=0.9, gather_mode=mode)
            for _ in range(M)]
    noise = np.random.default_rng(11)
    for p in world.mapping_poses():
        scan = synth.make_scan(world, p, noise)
        for rep in reps:
            rep.updateByScan(scan, p.astype(F32))
    g = capi.SlamGroup(reps)
    rng = np.random.default_rng(151)
    truth = world.sample_free_poses(M, rng).astype(F32)
    pts, offs = synth.make_scan_batch(world, truth, noise_seed=13)
    scans = [np.ascontiguousarray(pts[offs[j]:offs[j + 1]], F32) for j in range(M)]
    g.slam_update(truth + rng.uniform(-1, 1, (M, 3)).astype(F32) * F32([0.03, 0.03, 0.02]), scans)
    members = [3, 1, 0, 2]
    hints = [(truth[j][None] + rng.uniform(-1, 1, (H, 3)) * np.array([0.25, 0.25, 0.15])).astype(F32) for j in members]
    poses, _ = g.match_batch(hints, members=members)
    W = reps[0].last_launch_shape()["warps_per_scan"]
    _, best4, index = g.best_hypothesis(0, (poses, np.arange(M + 1, dtype=np.int32) * H), members=members)
    for k, j in enumerate(members):
        wp, wb = device_reloc(reps[j], hints[k], scans[j], W)
        assert np.array_equal(bits(poses[k * H:(k + 1) * H]), bits(wp)), k
        assert np.array_equal(bits(best4[k]), bits(wb)), (k, best4[k], wb)
        assert np.array_equal(bits(best4[k]), bits(single_best(reps[j], 0, wp, scans[j])[0])), k
        d = np.abs(best4[k, 1:].astype(np.float64) - truth[j])
        d[2] = abs((d[2] + np.pi) % (2 * np.pi) - np.pi)
        assert d[0] < 0.05 and d[1] < 0.05 and d[2] < 0.03, (k, best4[k], truth[j])
    close_all(g, reps)


# ---- 6: accounting and rejections --------------------------------------------------------------------------------

@MODES
def test_launches_and_rejections(hsb_lib, mode):
    """A call is one launch on handles[0], whichever members it lists; the other members' counts do not move.  Every
    rejection returns its code with its message, launches nothing and writes no output byte; K = 0 and Q = 0 queue
    nothing; a tuning without a group match kernel gives HSB_ERR_UNSUPPORTED; the group answers as before afterwards."""
    M = 4
    reps, g = fleet(GEOM, M, mode)
    track = Tracker(GEOM, M, mode)
    data = [session_data(5600 + s, 1, geometry(s)) for s in range(M)]
    rng = np.random.default_rng(153)
    step([g], data, [0] * M, "endpoints", None, rng, nowait=True, track=track, p_without=0.0)
    lib = g.lib
    hyp = [hypotheses(rng, track.pose[j], 10) for j in range(M)]
    scans = [track.scan(j) for j in range(M)]
    for members in (None, [2], [3, 1], [1, 0, 3, 2]):
        sel = list(range(M)) if members is None else members
        for points in (None, [scans[j] for j in sel]):
            counts = [r.launch_count for r in reps]
            g.match_batch([hyp[j] for j in sel], points, members=members)
            assert [r.launch_count for r in reps] == [counts[0] + 1] + counts[1:], members
            g.match_batch([hyp[j] for j in sel], points, members=members, want_cov=False)
            assert [r.launch_count for r in reps] == [counts[0] + 2] + counts[1:], members
    valid_members = [3, 0, 2]
    valid = [hyp[j] for j in valid_members]
    before = assert_match(g, reps, valid_members, valid, [scans[j] for j in valid_members], None, ("before",))

    Q, N = 12, 30
    hints = np.tile(track.pose[0], (Q, 1)).astype(F32)
    pts = np.ones((N, 2), F32)
    poses, cov = np.full((Q, 3), SENTINEL, F32), np.full((Q, 9), SENTINEL, F32)

    def p(x):
        if x is None:
            return None, None
        a = np.ascontiguousarray(x, np.int32)
        return a, a.ctypes.data

    def call(K, members, ho=(0, 4, 4, 12), hw=hints, xy=pts, so=(0, 10, 10, 30), out=True):
        m, mp = p(members)
        o, op = p(ho)
        s, sp = p(so)
        return lib.hsb_group_match_batch_subset(g.g, K, mp, op, None if hw is None else hw.ctypes.data,
                                                None if xy is None else xy.ctypes.data, sp,
                                                poses.ctypes.data if out else None, cov.ctypes.data)

    def err():
        return (lib.hsb_last_error(reps[0].h) or b"").decode()

    def c(**kw):
        K = kw.pop("K", 3)
        members = kw.pop("members", [0, 1, 2])
        return lambda: call(K, members, **kw)

    cases = [(c(K=-1, members=[0]), "K is -1"), (c(K=M + 1, members=[0, 1, 2, 3, 0]), "K is 5"),
             (c(members=None), "members is NULL"), (c(members=[0, 1, M]), "session 2: member 4"),
             (c(members=[-1, 0, 1]), "session 0: member -1"), (c(members=[1, 3, 1]), "session 2: member 1 is listed twice"),
             (c(ho=None), "hint_offsets is NULL"), (c(ho=(1, 4, 4, 12)), "hint_offsets[0] is 1"),
             (c(ho=(0, 4, 3, 12)), "hint_offsets decrease at session 1"),
             (c(xy=None), "both be given or both be NULL"), (c(so=None), "both be given or both be NULL"),
             (c(so=(2, 10, 10, 30)), "scan_offsets[0] is 2"), (c(so=(0, 10, 30, 20)), "scan_offsets decrease at session 2"),
             (c(hw=None), "hints_world is NULL"), (c(out=False), "out_poses_world is NULL")]
    fo, fp = p((0, 3, 3, 3, 12))
    cases += [(lambda: lib.hsb_group_match_batch(g.g, None, hints.ctypes.data, None, None, poses.ctypes.data, None),
               "hint_offsets is NULL"),
              (lambda: lib.hsb_group_match_batch(g.g, fp, hints.ctypes.data, pts.ctypes.data, None, poses.ctypes.data,
                                                 None), "both be given or both be NULL")]
    counts = [r.launch_count for r in reps]
    for fn, text in cases:
        assert fn() == -1, text
        assert text in err(), (text, err())
    # K = 0 reads nothing else; Q = 0 (every session empty) needs no hints and no outputs
    assert call(0, None, ho=None, hw=None, xy=None, so=None, out=False) == 0
    assert call(3, [0, 1, 2], ho=(0, 0, 0, 0), hw=None, out=False) == 0
    assert call(3, [0, 1, 2], ho=(0, 0, 0, 0), hw=None, xy=None, so=None, out=False) == 0
    # tunings of handles[0] whose launch shape has no group match kernel
    unsupported = [dict(warps_per_scan=16), dict(scans_per_block=2), dict(unroll=8)]
    if mode == 2:
        unsupported.append(dict(packed=1))
    for kw in unsupported:
        reps[0].set_tuning(**kw)
        assert call(3, [0, 1, 2]) == -5, kw
        assert "no group match kernel" in err() and f"{list(kw)[0]}=" in err(), (kw, err())
        reps[0].set_tuning(**{k: 0 for k in kw})
    assert [r.launch_count for r in reps] == counts
    assert (poses == SENTINEL).all() and (cov == SENTINEL).all()
    after = assert_match(g, reps, valid_members, valid, [scans[j] for j in valid_members], None, ("after",))
    assert np.array_equal(bits(before[0]), bits(after[0])) and np.array_equal(bits(before[1]), bits(after[1]))
    close_all(g, reps, track)


# ---- 7: the C++ façade -------------------------------------------------------------------------------------------

def test_facade(hsb_lib):
    """hsb200::SlamProcessor::matchMany (both overloads), through their shims, against the C-ABI group call on a second
    set of processors stepped with the same scans: the same bits, with the scans given and with each processor's last
    matched scan."""
    L = C.CDLL(os.path.join(ROOT, "hector_slam_b200", "lib", "libhsb200_host.so"))
    vp, i, f = C.c_void_p, C.c_int, C.c_float
    L.hsbp_create.restype = vp
    L.hsbp_create.argtypes = [f, i, i, f, f, i, i]
    L.hsbp_destroy.argtypes = [vp]
    L.hsbp_handle.restype = vp
    L.hsbp_handle.argtypes = [vp]
    L.hsbp_update.argtypes = [vp, vp, i, vp, vp, i, vp, vp]
    L.hsbp_match_many.argtypes = [vp, i, vp, vp, vp, vp, vp, vp]
    L.hsbp_match_many_subset.argtypes = [vp, i, vp, i, vp, vp, vp, vp, vp, vp]
    lib = hsb_lib

    sx0, sy0, levels, start = GEOM
    M, ticks = 4, 6
    data = [session_data(5700 + s, ticks, geometry(s)) for s in range(M)]
    sets = [[L.hsbp_create(mc.RES, sx0, sy0, start[0], start[1], levels, 0) for _ in range(M)] for _ in range(2)]
    assert all(q for s in sets for q in s)
    many, capi_set = sets
    hs = (C.c_void_p * M)(*[L.hsbp_handle(q) for q in capi_set])
    g = C.c_void_p()
    assert lib.hsb_group_create(C.cast(hs, vp), M, C.byref(g)) == 0
    arr = C.cast((C.c_void_p * M)(*many), vp)
    rng = np.random.default_rng(157)
    moved = 0
    for t in range(ticks):
        last = np.zeros((M, 3), F32)
        for s in range(M):
            x = data[s]["scans"][t]
            for st in sets:
                pose, cov = np.zeros(3, F32), np.zeros(9, F32)
                assert L.hsbp_update(st[s], x.ctypes.data, x.shape[0], None, data[s]["hints"][t].ctypes.data, 0,
                                     pose.ctypes.data, cov.ctypes.data) == 0
            last[s] = pose
        members = None if t % 2 == 0 else np.ascontiguousarray(rng.permutation(M)[:int(rng.integers(1, M + 1))], np.int32)
        sel = list(range(M)) if members is None else [int(j) for j in members]
        K = len(sel)
        ho = np.zeros(K + 1, np.int32)
        ho[1:] = np.cumsum(rng.integers(0, 12, K))
        Q = int(ho[-1])
        hints = np.concatenate([hypotheses(rng, last[j], int(ho[k + 1] - ho[k]), specials=False) for k, j in enumerate(sel)]
                               + [np.zeros((1, 3), F32)]).astype(F32)
        given = t % 3 != 2     # otherwise: the last matched scans
        scans = [data[j]["scans"][t][::2] for j in sel]
        so = np.zeros(K + 1, np.int32)
        so[1:] = np.cumsum([s.shape[0] for s in scans])
        pts = np.ascontiguousarray(np.concatenate(scans), F32)
        pp, sp = (pts.ctypes.data, so.ctypes.data) if given else (None, None)
        outs = [[np.zeros((Q + 1, 3), F32), np.zeros((Q + 1, 9), F32)] for _ in range(2)]
        (p1, c1), (p2, c2) = [[o.ctypes.data for o in out] for out in outs]
        common = (ho.ctypes.data, hints.ctypes.data, pp, sp)
        if members is None:
            assert L.hsbp_match_many(arr, M, *common, p1, c1) == 0
            assert lib.hsb_group_match_batch(g, *common, p2, c2) == 0
        else:
            mp = members.ctypes.data
            assert L.hsbp_match_many_subset(arr, M, mp, K, *common, p1, c1) == 0
            assert lib.hsb_group_match_batch_subset(g, K, mp, *common, p2, c2) == 0
        for x, y in zip(*outs):
            assert np.array_equal(bits(x), bits(y)), t
        moved += int((np.abs(outs[0][0][:Q, :2] - hints[:Q, :2]).max(axis=1) > 1e-4).sum())
    assert moved > 10
    lib.hsb_group_destroy(g)
    for q in many + capi_set:
        L.hsbp_destroy(q)
