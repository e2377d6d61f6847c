"""Groups of robots whose map pyramids differ in level count, iteration schedule and gather path
(hsb_group_create_heterogeneous): every group call runs each member's own levels, and every session and member state
stays bit-identical to the single-handle call on that member.

GPU.  One heterogeneous group of six members, each with a twin handle of the same configuration driven by single calls:
  (a) 1 level, TEX, 512 x 512 at 0.05 m        (b) 2 levels, TEX, 768 x 640 at 0.05 m started at (0.25, 0.6)
  (c) 3 levels, LDG, 1030 x 514 at 0.025 m     (d) 3 levels, TEX, 512 x 512 at 0.1 m, max_iterations [6, 0, -1]
  (e) 5 levels, LDG, 512 x 512 at 0.05 m       (f) 8 levels, TEX, 1024 x 1024 at 0.05 m
  - steps: all four input kinds, full and permuted subset forms, nowait, map_without_matching, three launches each;
  - end states on every level of every member, the last-match containers through likelihood with points=None;
  - occupancy sync, getDist, ray casts, likelihood, covariance and best hypothesis at level 0 over every member and at
    higher levels over the members that have them, and the level rule's rejection of a listed member without the level;
  - match_batch at W = 1, 2, 4 and 8;
  - a subset reset followed by steps, and queries straight after a nowait step;
  - tile replication: same-order replica bit-equal with every block the member's single pack, another order counted
    once and not applied, a reset 1-level member shipping its clear record alone;
  - the constructor's rejections."""
import numpy as np
import pytest

from test_gpu_group_match import assert_match
from test_gpu_group_mixed import grids_of, twin_sync
from test_gpu_group_score import assert_sessions, hypotheses, thinned
from test_gpu_group_subset import (KINDS, assert_same_session, assert_same_state, beam_angles, bits, close_all,
                                   geometry, group_step, member_cloud, member_transform, scan_of, session_data,
                                   single_step)

pytestmark = pytest.mark.gpu

F32 = np.float32
TEX, LDG = 2, 1   # capi.GATHER_TEX, capi.GATHER_LDG
# map_size_x, map_size_y, map_resolution, start, levels, gather mode, max_iterations
SPECS = [(512, 512, 0.05, (0.5, 0.5), 1, TEX, None),
         (768, 640, 0.05, (0.25, 0.6), 2, TEX, None),
         (1030, 514, 0.025, (0.5, 0.5), 3, LDG, None),
         (512, 512, 0.1, (0.1, 0.9), 3, TEX, [6, 0, -1]),
         (512, 512, 0.05, (0.5, 0.5), 5, LDG, None),
         (1024, 1024, 0.05, (0.5, 0.5), 8, TEX, None)]
A, B, C, D, E, F = range(6)
M = len(SPECS)
LEVELS = [s[4] for s in SPECS]
TICKS = 12
HSB_ERR_INVALID_ARG = -1
CLEARED_WORD = 4 + 4 * 8   # HSB_TILE_CLEARED_WORD (hsb_internal.h)


def make_rep(s):
    """Member s's handle: SPECS[s]'s map and pyramid, its own update factors, gate thresholds and formats"""
    from hector_slam_b200 import capi

    sx, sy, res, start, levels, mode, iters = SPECS[s]
    rep = capi.MapRepB200(res, sx, sy, levels=levels, start=start, max_iterations=iters,
                          update_factor_free=0.4 + 0.02 * (s % 3), update_factor_occupied=0.6 + 0.1 * (s % 4),
                          gather_mode=mode)
    dist, ang = ((0.0, 0.0), (0.15, 0.1), (0.3, 0.5))[s % 3]
    rep.setMapUpdateMinDistDiff(dist)
    rep.setMapUpdateMinAngleDiff(ang)
    g = geometry(s)
    rep.set_scan_format(**g)
    rep.set_laser_projection(**g, range_cutoff=30.0)
    rep.set_cloud_format(member_transform(s), **member_cloud(s))
    assert rep.gather_mode == mode
    return rep


def member_data(s):
    """session_data's trajectory with the endpoints in member s's own level-0 cell units"""
    from hector_slam_b200 import synth

    g = geometry(s)
    d = session_data(900 + s, TICKS + 8, g)   # (spare steps for the tests that step again)
    ang = beam_angles(g)
    d["scans"] = [np.ascontiguousarray(synth.ranges_to_points(r, 1.0 / SPECS[s][2], ang), F32) for r in d["ranges"]]
    return d


def having(level):
    """the members that have `level`"""
    return [j for j in range(M) if LEVELS[j] > level]


class Fleet:
    """The heterogeneous group, its members' twins, never-stepped converters (the last-match containers' endpoints), and
    every member's trajectory position."""

    def __init__(self):
        from hector_slam_b200 import capi

        self.grp = [make_rep(s) for s in range(M)]
        self.one = [make_rep(s) for s in range(M)]
        self.conv = [make_rep(s) for s in range(M)]
        self.g = capi.SlamGroup(self.grp, heterogeneous=True)
        self.data = [member_data(s) for s in range(M)]
        self.at = [0] * M
        self.last = [None] * M
        self.covs = [np.full((3, 3), 5.0, F32) for _ in range(M)]

    def tick(self, t, rng, members=None, nowait=None):
        kind = KINDS[t % 4]
        if members is None and t % 2 == 1:
            members = [int(j) for j in rng.permutation(M)[:int(rng.integers(1, M + 1))]]
        sel = list(range(M)) if members is None else members
        without = [bool(rng.random() < 0.2) and self.at[j] > 0 for j in sel]
        hints = np.asarray([self.data[j]["truth" if w else "hints"][self.at[j]] for j, w in zip(sel, without)],
                           F32).reshape(len(sel), 3)
        scans = [thinned(kind, scan_of(kind, self.data[j], self.at[j])) for j in sel]
        cov = np.stack([self.covs[j] for j in sel])
        launches = self.grp[0].launch_count
        out = group_step(self.g, kind, hints, scans, without, members=members,
                         nowait=(t % 3 == 1) if nowait is None else nowait, cov=cov)
        assert self.grp[0].launch_count - launches == 3, (t, kind)
        for i, j in enumerate(sel):
            ref = single_step(self.one[j], kind, hints[i], scans[i], without[i], cov=self.covs[j].copy())
            assert_same_session(out, i, ref, (t, kind, i, j))
            self.covs[j] = out[1][i].copy()
            if not without[i]:
                self.last[j] = (kind, scans[i])
            self.at[j] += 1
        return out

    def container(self, j):
        """the endpoints of member j's last matched input, as the matching *_to_points call returns them"""
        if self.last[j] is None:
            return np.zeros((0, 2), F32)
        kind, x = self.last[j]
        c = self.conv[j]
        if kind == "endpoints":
            return np.ascontiguousarray(x, F32)
        if kind == "ranges":
            return c.scan_to_points(x)
        return (c.cloud_to_points(x) if kind == "cloud" else c.projected_scan_to_points(x))[0]

    def close(self):
        self.g.close()
        close_all(self.grp, self.one, self.conv)


@pytest.fixture(scope="module")
def fleet(hsb_lib):
    """One stepped fleet shared by the tests below, in file order (the ones that change state run last)."""
    f = Fleet()
    rng = np.random.default_rng(77)
    for t in range(TICKS):
        f.tick(t, rng)
    yield f
    f.close()


def assert_states(f, tag, probe=True):
    for j in range(M):
        assert_same_state(f.grp[j], f.one[j], (tag, j), probe=probe, levels=LEVELS[j])


# ---- steps --------------------------------------------------------------------------------------------------------

def test_steps_and_end_state(fleet):
    """The fleet's steps (checked session by session in Fleet.tick) leave every member, on every one of its own levels,
    in its twin's state; every member has matched."""
    f = fleet
    for j in range(M):
        assert f.last[j] is not None, j
    assert_states(f, "end")


def test_last_match_containers(fleet):
    """likelihood with points=None reads each member's last-match container: at level 0 over every member, and at each
    higher level over the members that have it."""
    f = fleet
    rng = np.random.default_rng(5)
    for level in range(max(LEVELS)):
        sel = having(level)
        poses = [hypotheses(rng, f.data[j]["truth"][f.at[j] - 1], 7, specials=False) for j in sel]
        scans = [f.container(j) for j in sel]
        assert_sessions(f.g, f.one, level, None if len(sel) == M else sel, poses, scans, None, ("container", level))


# ---- queries ------------------------------------------------------------------------------------------------------

def test_scoring(fleet):
    """likelihood, covariance (map and world) and best hypothesis with scans given: level 0 over every member, each
    higher level over the members that have it in a permuted order."""
    f = fleet
    rng = np.random.default_rng(11)
    for level in range(max(LEVELS)):
        sel = having(level)
        if level > 0:
            sel = [sel[i] for i in rng.permutation(len(sel))]
        poses = [hypotheses(rng, f.data[j]["truth"][f.at[j] - 1], 6 + j) for j in sel]
        scans = [f.data[j]["scans"][f.at[j] - 1] for j in sel]
        assert_sessions(f.g, f.one, level, None if level == 0 else sel, poses, scans, scans, ("scans", level))


def test_ray_queries(fleet):
    """getDist and ray casts at level 0 over every member and at level 2 over (e), (c), (f), (d)."""
    f = fleet
    rng = np.random.default_rng(21)
    for level, members in ((0, None), (2, [E, C, F, D])):
        sel = list(range(M)) if members is None else members
        wb = rng.uniform(-15.0, 25.0, (400, 2)).astype(F32)
        we = rng.uniform(-15.0, 25.0, (400, 2)).astype(F32)
        cb = rng.integers(0, 520, (400, 2)).astype(np.int32)
        ce = rng.integers(-20, 1100, (400, 2)).astype(np.int32)
        d, h, fnd = f.g.get_dist(level, [wb] * len(sel), [we] * len(sel), members=members)
        cd, ch = f.g.raycast(level, [cb] * len(sel), [ce] * len(sel), members=members)
        for k, j in enumerate(sel):
            sd, sh, sf = f.one[j].get_dist_batch(level, wb, we)
            rd, rh = f.one[j].raycast_batch(level, cb, ce)
            tag = (level, k, j)
            assert np.array_equal(bits(d[k * 400:(k + 1) * 400]), bits(sd)), tag
            assert np.array_equal(bits(h[k * 400:(k + 1) * 400]), bits(sh)), tag
            assert np.array_equal(fnd[k * 400:(k + 1) * 400], sf), tag
            assert np.array_equal(bits(cd[k * 400:(k + 1) * 400]), bits(rd)), tag
            assert np.array_equal(ch[k * 400:(k + 1) * 400], rh), tag


def test_level_rule(fleet):
    """A level-taking call that lists a member without the level is rejected with HSB_ERR_INVALID_ARG naming the
    session and the member's level count, before anything is cleared: the following sync still returns the rectangle.
    Members that are not listed are not checked."""
    from hector_slam_b200 import capi

    f = fleet
    level = 1
    sel = [B, C, A]   # (a) has one level: session 2
    pose = [f.data[j]["truth"][f.at[j] - 1][None, :] for j in sel]
    scans = [f.data[j]["scans"][f.at[j] - 1] for j in sel]
    rays = [np.zeros((2, 2), F32)] * 3
    cells = [np.zeros((2, 2), np.int32)] * 3
    grids = grids_of([f.grp[B], f.grp[C]], level) + [np.zeros((1, 1), np.int8)]
    calls = [lambda: f.g.sync_occupancy(level, grids, members=sel),
             lambda: f.g.get_dist(level, rays, rays, members=sel),
             lambda: f.g.raycast(level, cells, cells, members=sel),
             lambda: f.g.likelihood(level, pose, scans, members=sel),
             lambda: f.g.covariance(level, pose, scans, members=sel),
             lambda: f.g.best_hypothesis(level, pose, scans, members=sel)]
    launches = f.grp[0].launch_count
    for i, call in enumerate(calls):
        with pytest.raises(capi.HsbError) as e:
            call()
        msg = str(e.value)
        assert e.value.status == HSB_ERR_INVALID_ARG and "session 2" in msg and "has 1 levels" in msg, (i, msg)
    assert f.grp[0].launch_count == launches
    # nothing was cleared: the members with the level still return their rectangles, equal to their twins'
    ok = [B, C]
    gg, tg = grids_of([f.grp[j] for j in ok], level), grids_of([f.one[j] for j in ok], level)
    rects = f.g.sync_occupancy(level, gg, members=ok)
    for k, j in enumerate(ok):
        assert rects[k] is not None, j
        assert rects[k] == twin_sync(f.one[j], level, tg[k]), j
        assert np.array_equal(gg[k], tg[k]), j


def test_occupancy(fleet):
    """Grids of each member's own shape: level 0 over every member, level 1 over (f), (b), (e), each of its members'
    higher levels over the members that have them."""
    f = fleet
    for level in range(max(LEVELS)):
        sel = having(level)
        if level == 1:
            sel = [F, B, E, C, D]
        gg, tg = grids_of([f.grp[j] for j in sel], level), grids_of([f.one[j] for j in sel], level)
        rects = f.g.sync_occupancy(level, gg, members=None if len(sel) == M else sel)
        for k, j in enumerate(sel):
            assert rects[k] == twin_sync(f.one[j], level, tg[k]), (level, k, j)
            assert np.array_equal(gg[k], tg[k]), (level, k, j)


def test_match_batch(fleet):
    """match_batch with scans and with the last-match containers, full and subset, against hsb_match_batch per member
    with W = 1, 2, 4 and 8 set through handles[0]'s tuning (a match changes no state)."""
    f = fleet
    rng = np.random.default_rng(13)
    hints = [hypotheses(rng, f.data[j]["truth"][f.at[j] - 1], (3, 0, 5, 2, 4, 3)[j], specials=False) for j in range(M)]
    scans = [f.data[j]["scans"][f.at[j] - 1] for j in range(M)]
    conts = [f.container(j) for j in range(M)]
    sub = [F, A, D]
    try:
        for W in (1, 2, 4, 8):
            f.grp[0].set_tuning(warps_per_scan=W)
            assert assert_match(f.g, f.grp, None, hints, scans, scans, ("scans",))[2] == W
            assert_match(f.g, f.grp, None, hints, conts, None, ("containers",))
            assert_match(f.g, f.grp, sub, [hints[j] for j in sub], [scans[j] for j in sub], [scans[j] for j in sub],
                         ("subset",))
    finally:
        f.grp[0].set_tuning(warps_per_scan=0)


# ---- tiles --------------------------------------------------------------------------------------------------------

def pack_buffers(reps):
    import torch

    from test_gpu_group_tiles import HEADER_WORDS, group_header_words

    cells = sum(r.level_info(l)[0] * r.level_info(l)[1] for r in reps for l in range(r.levels))
    words = group_header_words(len(reps)) + len(reps) * HEADER_WORDS + cells
    return (torch.zeros(words, dtype=torch.float32, device="cuda"),
            torch.zeros(HEADER_WORDS + cells, dtype=torch.float32, device="cuda"), words)


def test_tiles(fleet, hsb_lib):
    """Pack on the heterogeneous group, unpack on a heterogeneous replica group in the same order: every block equals the
    member's single pack (its own level count in word 1), group-header word 2 is the largest level count, the replica
    equals the owner in bits.  A replica group listing the handles in another order (blocks landing on members of
    another level count): counted once on its handles[0], nothing applied."""
    import torch

    from hector_slam_b200 import capi
    from test_gpu_group_tiles import HEADER_WORDS, group_header_words

    f = fleet
    assert [f.grp[j].get_dirty_rects() for j in range(M)] == [f.one[j].get_dirty_rects() for j in range(M)]
    buf, single, words = pack_buffers(f.grp)
    st = torch.cuda.current_stream().cuda_stream
    replica = [make_rep(s) for s in range(M)]
    rg = capi.SlamGroup(replica, heterogeneous=True)
    order = [A, C, B, D, F, E]
    rg2 = capi.SlamGroup([replica[j] for j in order], heterogeneous=True)
    try:
        f.g.pack_dirty_device(buf.data_ptr(), 4 * words, False, st)
        torch.cuda.synchronize()
        hdr = buf[:group_header_words(M)].view(torch.int32).cpu().numpy()
        assert hdr[1] == M and hdr[2] == max(LEVELS) and hdr[3] == 0, hdr[:5]
        for j in range(M):
            f.one[j].pack_dirty_device(single.data_ptr(), 4 * single.numel(), False, st)
            torch.cuda.synchronize()
            start = int(hdr[6 + 2 * j])
            assert int(hdr[5 + 2 * j]) == j
            head = single[:HEADER_WORDS].view(torch.int32)
            assert int(head[1]) == LEVELS[j]
            n = HEADER_WORDS + int(head[3])
            assert torch.equal(buf[start:start + n].view(torch.int32), single[:n].view(torch.int32)), j
        rg.unpack_dirty_device(buf.data_ptr(), 4 * words, st)
        torch.cuda.synchronize()
        for j in range(M):
            for l in range(LEVELS[j]):
                assert np.array_equal(bits(replica[j].download_level(l)), bits(f.grp[j].download_level(l))), (j, l)
        snap = [([bits(r.download_level(l)).copy() for l in range(r.levels)],
                 [r.get_mirror_dirty_rect(l) for l in range(r.levels)]) for r in replica]
        assert all(r.replication_overflows() == 0 for r in replica)
        rg2.unpack_dirty_device(buf.data_ptr(), 4 * words, st)
        torch.cuda.synchronize()
        assert replica[order[0]].replication_overflows(reset=True) == 1
        assert all(replica[j].replication_overflows() == 0 for j in range(M))
        for j, r in enumerate(replica):
            for l in range(r.levels):
                assert np.array_equal(bits(r.download_level(l)), snap[j][0][l]), ("wrong order", j, l)
                assert r.get_mirror_dirty_rect(l) == snap[j][1][l], ("wrong order", j, l)
    finally:
        rg2.close()
        rg.close()
        close_all(replica)


# ---- reset (changes state: runs last) -----------------------------------------------------------------------------

def test_reset_then_steps(fleet, hsb_lib):
    """A subset reset of (a), (e) and (c) against hsb_reset on their twins: every own level cleared, the others
    untouched; a pack then ships (a)'s clear record and no rows; steps after it, and queries straight after a nowait
    step, stay bit-equal to the twins."""
    import torch

    from test_gpu_group_tiles import HEADER_WORDS, group_header_words

    f = fleet
    sel = [A, E, C]
    f.g.reset(members=sel)
    for j in sel:
        f.one[j].reset()
    assert_states(f, "after reset", probe=False)
    for j in sel:
        for l in range(LEVELS[j]):
            assert not f.grp[j].download_level(l).any(), (j, l)
    # (a)'s block: its clear record and no rows (pack only (a): the others' rectangles stay as they are)
    buf, _, words = pack_buffers(f.grp)
    st = torch.cuda.current_stream().cuda_stream
    f.g.pack_dirty_device(buf.data_ptr(), 4 * words, True, st, members=[A])
    torch.cuda.synchronize()
    hdr = buf[:group_header_words(1) + HEADER_WORDS].view(torch.int32).cpu().numpy()
    blk = hdr[int(hdr[6]):int(hdr[6]) + HEADER_WORDS]
    assert hdr[2] == max(LEVELS) and blk[1] == 1 and blk[2] == 0 and blk[3] == 0, blk[:8]
    assert blk[CLEARED_WORD] == 1 and blk[4] > blk[6], blk[:8]
    f.one[A].pack_dirty_device(buf.data_ptr(), 4 * words, True, st)   # the twin's replication state follows
    torch.cuda.synchronize()
    rng = np.random.default_rng(9)
    for t in range(4):
        f.tick(TICKS + t, rng, members=None if t % 2 == 0 else [C, A, F], nowait=True)
        # straight after the nowait step: a query that waits for the step's map writes
        sel2 = having(0)
        poses = [f.data[j]["truth"][f.at[j] - 1][None, :] for j in sel2]
        scans = [f.data[j]["scans"][f.at[j] - 1] for j in sel2]
        assert_sessions(f.g, f.one, 0, None, poses, scans, scans, ("after nowait", t))
    assert_states(f, "after reset and steps")


# ---- rejections ---------------------------------------------------------------------------------------------------

def test_rejections(hsb_lib):
    """hsb_group_create_heterogeneous takes members of any level count, iteration schedule and gather mode, and refuses
    NULL and duplicate handles (and another device, with two GPUs) as hsb_group_create_mixed does; the mixed constructor
    still refuses these members."""
    import torch

    from hector_slam_b200 import capi

    reps = [make_rep(s) for s in (A, C, D)]
    capi.SlamGroup(reps, heterogeneous=True).close()
    with pytest.raises(capi.HsbError) as e:
        capi.SlamGroup(reps, mixed=True)
    assert e.value.status == HSB_ERR_INVALID_ARG and "levels" in str(e.value)
    for rs, what in (([], "M >= 1"), ([reps[0], reps[1], reps[0]], "listed twice"), ([reps[0], None], "is NULL")):
        with pytest.raises(capi.HsbError) as e:
            capi.SlamGroup(rs, heterogeneous=True)
        assert e.value.status == HSB_ERR_INVALID_ARG and "hsb_group_create_heterogeneous" in str(e.value), str(e.value)
        assert what in str(e.value), str(e.value)
    if torch.cuda.device_count() >= 2:
        far = capi.MapRepB200(0.05, 256, levels=2, device=1)
        with pytest.raises(capi.HsbError) as e:
            capi.SlamGroup([reps[0], far], heterogeneous=True)
        assert e.value.status == HSB_ERR_INVALID_ARG and "device" in str(e.value)
        far.close()
    close_all(reps)


# ---- C++ façade ---------------------------------------------------------------------------------------------------

def test_facade(hsb_lib):
    """hsb200::SlamProcessor::updateMany over a 1-level, a 2-level and a 3-level processor of different map sizes:
    without the opt-in it throws (hsb_group_create refuses them); with setHeterogeneousGroups(true) on ps[0] it equals
    update() per processor on a twin set — poses, covariances and every level of every map."""
    import ctypes as C
    import os

    from conftest import ROOT

    L = C.CDLL(os.path.join(ROOT, "hector_slam_b200", "lib", "libhsb200_host.so"))
    vp, i, fl = C.c_void_p, C.c_int, C.c_float
    L.hsbp_create.restype = vp
    L.hsbp_create.argtypes = [fl, i, i, fl, fl, i, i]
    L.hsbp_destroy.argtypes = [vp]
    L.hsbp_update.argtypes = [vp, vp, i, vp, vp, i, vp, vp]
    L.hsbp_update_many.argtypes = [vp, i, vp, vp, vp, vp, vp]
    L.hsbp_set_heterogeneous_groups.argtypes = [vp, i]
    L.hsbp_get_grid_map.argtypes = [vp, i, vp]
    L.hsbp_get_pose_and_cov.argtypes = [vp, vp, vp]
    procs = [(512, 512, 1), (640, 512, 2), (512, 768, 3)]   # hector_ugv, mapping_default, the node's default
    M, ticks = len(procs), 8
    data = [session_data(8300 + s, ticks, geometry(s)) for s in range(M)]
    sets = [[L.hsbp_create(0.05, sx, sy, 0.5, 0.5, lv, 0) for sx, sy, lv in procs] for _ in range(2)]
    assert all(q for s in sets for q in s)
    many, single = sets
    arr = C.cast((C.c_void_p * M)(*many), vp)
    for t in range(ticks):
        pts = np.ascontiguousarray(np.concatenate([data[s]["scans"][t] for s in range(M)]), F32)
        offsets = np.zeros(M + 1, np.int32)
        offsets[1:] = np.cumsum([data[s]["scans"][t].shape[0] for s in range(M)])
        hints = np.ascontiguousarray(np.stack([data[s]["hints"][t] for s in range(M)]), F32)
        if t == 0:
            assert L.hsbp_update_many(arr, M, pts.ctypes.data, offsets.ctypes.data, None, hints.ctypes.data, None) == -1
            L.hsbp_set_heterogeneous_groups(many[0], 1)
        assert L.hsbp_update_many(arr, M, pts.ctypes.data, offsets.ctypes.data, None, hints.ctypes.data, None) == 0
        for s in range(M):
            x = data[s]["scans"][t]
            pose, cov = np.zeros(3, F32), np.zeros(9, F32)
            assert L.hsbp_update(single[s], x.ctypes.data, x.shape[0], None, hints[s].ctypes.data, 0,
                                 pose.ctypes.data, cov.ctypes.data) == 0
            gp, gc = np.zeros(3, F32), np.zeros(9, F32)
            assert L.hsbp_get_pose_and_cov(many[s], gp.ctypes.data, gc.ctypes.data) == 0
            assert np.array_equal(bits(gp), bits(pose)) and np.array_equal(bits(gc), bits(cov)), (t, s)
    for s, (sx, sy, lv) in enumerate(procs):
        for l in range(lv):
            n = (sx >> l) * (sy >> l)
            a, b = np.zeros(n, F32), np.zeros(n, F32)
            assert L.hsbp_get_grid_map(many[s], l, a.ctypes.data) == 0
            assert L.hsbp_get_grid_map(single[s], l, b.ctypes.data) == 0
            assert np.array_equal(bits(a), bits(b)), (s, l)
    for st in sets:
        for q in st:
            L.hsbp_destroy(q)
