"""Groups of robots whose maps differ in size, resolution and start (hsb_group_create_mixed): every group call takes each
member's own geometry, and every session and member state stays bit-identical to the single-handle call on that member.

GPU, in both gather modes, every member created with that mode.  One mixed group of five 3-level members:
  (a) 1024 x 1024 at 0.05 m, (b) 768 x 1280 at 0.05 m started at (0.25, 0.6), (c) 1030 x 514 at 0.025 m (a width that
  is not a multiple of 4 on any level), (d) 512 x 512 at 0.1 m started at (0.1, 0.9), (e) a second (a).
Each member has a twin handle with the same configuration driven by single calls; members differ in update factors,
gate thresholds, scan formats, laser mounts and cloud thresholds.  The synthetic room (20 x 14 m) reaches past (c)'s map
in y and past (b)'s in x, so endpoints and beams land outside those maps.
  - steps: all four input kinds, full and subset forms (permuted), nowait, map_without_matching; the last-match
    container through likelihood with points=None; three launches per step on handles[0];
  - occupancy sync with grids of each member's own shape, once with occupancy_chunk = 1 byte while (c)'s whole level 0
    is dirty (its rows are wider than handles[0]'s);
  - getDist and ray casts with the same rays sent to every member;
  - likelihood, covariance (map and world) and best hypothesis, with scans and with the last-match containers;
  - match_batch at the group's warps per scan;
  - tile replication: pack on the mixed group, unpack on a mixed replica group in the same order (bit-equal, every block
    the member's single pack) and on one in another order (counted once on its handles[0], nothing applied);
  - the rejections of hsb_group_create_mixed, and hsb_group_create still refusing the mixed handles."""
import numpy as np
import pytest

import maptools_cases as mc
from test_gpu_group_match import assert_match
from test_gpu_group_occupancy import SENTINEL, n_chunks
from test_gpu_group_score import assert_sessions, hypotheses, thinned
from test_gpu_group_subset import (KINDS, assert_same_session, assert_same_state, beam_angles, bits, close_all,
                                   geometry, group_step, member_cloud, member_transform, scan_of, session_data,
                                   single_step)

pytestmark = pytest.mark.gpu

F32 = np.float32
LEVELS = 3
MODES = pytest.mark.parametrize("mode", [2, 1], ids=["tex", "ldg"])   # capi.GATHER_TEX, capi.GATHER_LDG
# map_size_x, map_size_y, map_resolution, start
SPECS = [(1024, 1024, 0.05, (0.5, 0.5)), (768, 1280, 0.05, (0.25, 0.6)), (1030, 514, 0.025, (0.5, 0.5)),
         (512, 512, 0.1, (0.1, 0.9)), (1024, 1024, 0.05, (0.5, 0.5))]
A, B, C, D, E = range(5)
M = len(SPECS)
TICKS = 16


def make_rep(s, mode):
    """Member s's handle: SPECS[s]'s map, its own update factors, gate thresholds and formats"""
    from hector_slam_b200 import capi

    sx, sy, res, start = SPECS[s]
    rep = capi.MapRepB200(res, sx, sy, levels=LEVELS, start=start, update_factor_free=0.4 + 0.02 * (s % 3),
                          update_factor_occupied=0.6 + 0.1 * (s % 4), gather_mode=mode)
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
    d = session_data(700 + s, TICKS + 2, g)   # (two spare steps for the tests that step again)
    ang = beam_angles(g)
    d["scans"] = [np.ascontiguousarray(synth.ranges_to_points(r, 1.0 / SPECS[s][2], ang), F32) for r in d["ranges"]]
    return d


def outside_share(rep, d):
    """the share of member d's endpoints (from the true poses) that fall outside the handle's level-0 map"""
    sx, sy, cell = rep.level_info(0)
    org = rep.map_origin(0)
    out = tot = 0
    for p, pts in zip(d["truth"], d["scans"]):
        c, s_ = np.cos(p[2]), np.sin(p[2])
        wx = p[0] + (c * pts[:, 0] - s_ * pts[:, 1]) * cell
        wy = p[1] + (s_ * pts[:, 0] + c * pts[:, 1]) * cell
        cx, cy = (wx - org[0]) / cell, (wy - org[1]) / cell
        out += int(np.sum((cx < 0) | (cy < 0) | (cx >= sx) | (cy >= sy)))
        tot += pts.shape[0]
    return out / max(tot, 1)


class Fleet:
    """The mixed group, its members' twins, never-stepped converters (the last-match containers' endpoints), and every
    member's trajectory position."""

    def __init__(self, mode):
        from hector_slam_b200 import capi

        self.grp = [make_rep(s, mode) for s in range(M)]
        self.one = [make_rep(s, mode) for s in range(M)]
        self.conv = [make_rep(s, mode) for s in range(M)]
        self.g = capi.SlamGroup(self.grp, mixed=True)
        self.data = [member_data(s) for s in range(M)]
        self.at = [0] * M
        self.last = [None] * M          # (kind, input) of each member's last matched step
        self.covs = [np.full((3, 3), 5.0, F32) for _ in range(M)]

    def tick(self, t, rng):
        kind = KINDS[t % 4]
        members = None if t % 2 == 0 else [int(j) for j in rng.permutation(M)[:int(rng.integers(1, M + 1))]]
        sel = list(range(M)) if members is None else members
        without = [bool(rng.random() < 0.2) and self.at[j] > 0 for j in sel]
        hints = np.asarray([self.data[j]["truth" if w else "hints"][self.at[j]] for j, w in zip(sel, without)],
                           F32).reshape(len(sel), 3)
        scans = [thinned(kind, scan_of(kind, self.data[j], self.at[j])) for j in sel]
        cov = np.stack([self.covs[j] for j in sel])
        launches = self.grp[0].launch_count
        out = group_step(self.g, kind, hints, scans, without, members=members, nowait=(t % 3 == 1), cov=cov)
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

    def run(self, seed):
        rng = np.random.default_rng(seed)
        for t in range(TICKS):
            self.tick(t, rng)

    def close(self):
        self.g.close()
        close_all(self.grp, self.one, self.conv)


@pytest.fixture(scope="module", params=[2, 1], ids=["tex", "ldg"])
def fleet(request, hsb_lib):
    """One stepped fleet per gather mode, shared by the query tests below (none of them changes a member's state
    except where a test says so, and those run last)."""
    f = Fleet(request.param)
    f.run(31 + request.param)
    yield f
    f.close()


# ---- steps --------------------------------------------------------------------------------------------------------

def test_steps_and_end_state(fleet):
    """The fleet's TICKS steps (checked session by session in Fleet.tick) leave every member in its twin's state;
    every member has matched; the trajectories reach past (b)'s and (c)'s maps."""
    f = fleet
    for j in range(M):
        assert f.last[j] is not None, j
        assert_same_state(f.grp[j], f.one[j], ("end", j))
    assert outside_share(f.grp[B], f.data[B]) > 0.0 and outside_share(f.grp[C], f.data[C]) > 0.0


def test_last_match_containers(fleet):
    """likelihood with points=None reads each member's last-match container: equal to the single call on the twin
    with the endpoints the matching conversion returns, on every level."""
    f = fleet
    rng = np.random.default_rng(5)
    for level in range(LEVELS):
        poses = [hypotheses(rng, f.data[j]["truth"][f.at[j] - 1], 9, specials=False) for j in range(M)]
        scans = [f.container(j) for j in range(M)]
        assert_sessions(f.g, f.one, level, None, poses, scans, None, ("container",))


# ---- scoring and matching -----------------------------------------------------------------------------------------

def test_scoring(fleet):
    """likelihood, covariance (map and world) and best hypothesis with scans given, full and subset, against the twins;
    the world covariances at each member's last pose at 0.025, 0.05 and 0.1 m differ and each equals its twin's."""
    f = fleet
    rng = np.random.default_rng(11)
    for level in range(LEVELS):
        poses = [hypotheses(rng, f.data[j]["truth"][f.at[j] - 1], 8 + j) for j in range(M)]
        scans = [f.data[j]["scans"][f.at[j] - 1] for j in range(M)]
        assert_sessions(f.g, f.one, level, None, poses, scans, scans, ("scans",))
        sub = [D, A, C]
        assert_sessions(f.g, f.one, level, sub, [poses[j] for j in sub], [scans[j] for j in sub],
                        [scans[j] for j in sub], ("subset",))
    poses = [f.data[j]["truth"][f.at[j] - 1][None, :] for j in range(M)]
    scans = [f.data[j]["scans"][f.at[j] - 1] for j in range(M)]
    _, cw = f.g.covariance(0, poses, scans)
    for j in range(M):
        assert np.array_equal(bits(cw[j]), bits(f.one[j].covariance_batch(0, poses[j], scans[j])[1][0])), j
    assert not np.array_equal(bits(cw[A]), bits(cw[C])) and not np.array_equal(bits(cw[A]), bits(cw[D]))
    assert not np.array_equal(bits(cw[C]), bits(cw[D]))


def test_match_batch(fleet):
    """match_batch with scans and with the last-match containers, full and subset, against hsb_match_batch per member
    at the warps per scan the group call reports (on the members themselves: a match changes no state)."""
    f = fleet
    rng = np.random.default_rng(13)
    hints = [hypotheses(rng, f.data[j]["truth"][f.at[j] - 1], (3, 0, 5, 2, 4)[j], specials=False) for j in range(M)]
    scans = [f.data[j]["scans"][f.at[j] - 1] for j in range(M)]
    assert_match(f.g, f.grp, None, hints, scans, scans, ("scans",))
    conts = [f.container(j) for j in range(M)]
    assert_match(f.g, f.grp, None, hints, conts, None, ("containers",))
    sub = [C, E, B]
    assert_match(f.g, f.grp, sub, [hints[j] for j in sub], [scans[j] for j in sub], [scans[j] for j in sub], ("subset",))


# ---- ray queries --------------------------------------------------------------------------------------------------

def shared_rays(f, level, seed, n=300):
    """the same world and cell rays for every member: (a)'s maptools cases, plus rays that lie inside (a) and outside
    (d) or the reverse"""
    rep = f.grp[A]
    sx, sy, cell = rep.level_info(level)
    cb, ce = mc.cell_rays(sx, sy, rep.download_occupancy(level), seed)
    wb, we, _ = mc.world_rays(sx, sy, rep.map_origin(level), cell, seed)
    rng = np.random.default_rng(seed)
    ic, iw = rng.choice(cb.shape[0], n), rng.choice(wb.shape[0], n)
    cb, ce, wb, we = cb[ic], ce[ic], wb[iw].copy(), we[iw].copy()
    dx, dy, _ = f.grp[D].level_info(level)
    lo, hi = min(dx, sx), max(dx, sx)
    span = rng.integers(lo, hi + 40, (n, 4)).astype(np.int32)   # in the larger map, past the smaller one
    inner = rng.integers(0, lo, (n, 4)).astype(np.int32)
    cb = np.concatenate([cb, inner[:, :2], span[:, :2]]).astype(np.int32)
    ce = np.concatenate([ce, span[:, 2:], inner[:, 2:]]).astype(np.int32)
    wxy = rng.uniform(-30.0, 50.0, (2 * n, 4)).astype(F32)   # spans (a), (d) and past both
    wb = np.concatenate([wb, wxy[:, :2]]).astype(F32)
    we = np.concatenate([we, wxy[:, 2:]]).astype(F32)
    return cb, ce, wb, we


def test_ray_queries(fleet):
    """getDist and ray casts: the same rays to every member, full and subset, against each twin's single calls."""
    f = fleet
    for level in range(LEVELS):
        cb, ce, wb, we = shared_rays(f, level, 40 + level)
        for members in (None, [D, B, A]):
            sel = list(range(M)) if members is None else members
            d, h, fnd = f.g.get_dist(level, [wb] * len(sel), [we] * len(sel), members=members)
            cd, ch = f.g.raycast(level, [cb] * len(sel), [ce] * len(sel), members=members)
            nw, nc = wb.shape[0], cb.shape[0]
            for k, j in enumerate(sel):
                sd, sh, sf = f.one[j].get_dist_batch(level, wb, we)
                rd, rh = f.one[j].raycast_batch(level, cb, ce)
                tag = (level, k, j)
                assert np.array_equal(bits(d[k * nw:(k + 1) * nw]), bits(sd)), tag
                assert np.array_equal(bits(h[k * nw:(k + 1) * nw]), bits(sh)), tag
                assert np.array_equal(fnd[k * nw:(k + 1) * nw], sf), tag
                assert np.array_equal(bits(cd[k * nc:(k + 1) * nc]), bits(rd)), tag
                assert np.array_equal(ch[k * nc:(k + 1) * nc], rh), tag
        # the same world rays measure in each member's own cell length (a miss is -cell length)
        dist_a = f.one[A].get_dist_batch(level, wb, we)[0]
        dist_d = f.one[D].get_dist_batch(level, wb, we)[0]
        assert not np.array_equal(bits(dist_a), bits(dist_d)), level


# ---- occupancy ----------------------------------------------------------------------------------------------------

def grids_of(reps, level, fill=SENTINEL):
    out = []
    for r in reps:
        sx, sy, _ = r.level_info(level)
        out.append(np.full((sy, sx), fill, np.int8))
    return out


def twin_sync(rep, level, grid):
    """hsb_get_mirror_dirty_rect(reset) + hsb_download_occupancy_rect + a row-by-row copy"""
    r = rep.get_mirror_dirty_rect(level, reset=True)
    if r is not None:
        grid[r[1]:r[3] + 1, r[0]:r[2] + 1] = rep.download_occupancy_rect(level, r)
    return r


def test_occupancy(fleet):
    """Grids of each member's own shape, every level, full and subset; then occupancy_chunk = 1 byte on handles[0]
    (a) with (c)'s whole level 0 dirty: one row per chunk at most, (c)'s rows wider than (a)'s."""
    f = fleet
    for level in range(LEVELS):
        for members in ([C, D], None):
            sel = list(range(M)) if members is None else members
            gg, tg = grids_of([f.grp[j] for j in sel], level), grids_of([f.one[j] for j in sel], level)
            rects = f.g.sync_occupancy(level, gg, members=members)
            for k, j in enumerate(sel):
                assert rects[k] == twin_sync(f.one[j], level, tg[k]), (level, k, j)
                assert np.array_equal(gg[k], tg[k]), (level, k, j)
    # (c)'s whole level 0 dirty on both sides, (a)'s and the others' a step's worth
    for rep in (f.grp[C], f.one[C]):
        rep.upload_level(0, f.grp[C].download_level(0))
    f.tick(TICKS, np.random.default_rng(3))   # a full endpoints step: every member writes
    gg, tg = grids_of(f.grp, 0), grids_of(f.one, 0)
    f.grp[A].set_tuning(occupancy_chunk=1)
    try:
        launches = f.grp[A].launch_count
        rects = f.g.sync_occupancy(0, gg)
        widths = [f.grp[j].level_info(0)[0] for j in range(M) if rects[j] is not None]
        assert rects[C] == (0, 0, SPECS[C][0] - 1, SPECS[C][1] - 1), rects[C]
        assert max(widths) == SPECS[C][0] > SPECS[A][0]
        assert f.grp[A].launch_count - launches == 1 + n_chunks(rects, 1, max(widths))
    finally:
        f.grp[A].set_tuning(occupancy_chunk=0)
    for j in range(M):
        assert rects[j] == twin_sync(f.one[j], 0, tg[j]), j
        assert np.array_equal(gg[j], tg[j]), j
        assert_same_state(f.grp[j], f.one[j], ("after occupancy", j), probe=False)


# ---- tiles --------------------------------------------------------------------------------------------------------

def test_tiles(fleet, hsb_lib):
    """Pack on the mixed group, unpack on a mixed replica group listing the same handles in the same order: the replica
    equals the owner in bits and each block equals the member's single pack.  Then a replica group listing them in
    another order, so that (c)'s block lands on (d) past (d)'s size: counted once on its handles[0], nothing applied."""
    import torch

    from hector_slam_b200 import capi
    from test_gpu_group_tiles import HEADER_WORDS, group_header_words

    f = fleet
    mode = f.grp[0].gather_mode
    rects = [f.grp[j].get_dirty_rects() for j in range(M)]
    assert rects == [f.one[j].get_dirty_rects() for j in range(M)]
    dx, dy, _ = f.grp[D].level_info(0)
    assert rects[C][0] is not None and (rects[C][0][2] >= dx or rects[C][0][3] >= dy), rects[C][0]
    cells = sum(r.level_info(l)[0] * r.level_info(l)[1] for r in f.grp for l in range(LEVELS))
    words = group_header_words(M) + M * HEADER_WORDS + cells
    buf = torch.zeros(words, dtype=torch.float32, device="cuda")
    single = torch.zeros(HEADER_WORDS + cells, dtype=torch.float32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    replica = [make_rep(s, mode) for s in range(M)]
    rg = capi.SlamGroup(replica, mixed=True)
    order = [A, B, D, C, E]   # (c)'s block (member 2) lands on (d)
    rg2 = capi.SlamGroup([replica[j] for j in order], mixed=True)
    try:
        f.g.pack_dirty_device(buf.data_ptr(), 4 * words, False, st)
        torch.cuda.synchronize()
        hdr = buf[:group_header_words(M)].view(torch.int32).cpu().numpy()
        assert hdr[3] == 0, "a block was deferred"
        for j in range(M):
            f.one[j].pack_dirty_device(single.data_ptr(), 4 * single.numel(), False, st)
            torch.cuda.synchronize()
            start = int(hdr[6 + 2 * j])
            assert int(hdr[5 + 2 * j]) == j
            n = HEADER_WORDS + int(single[:HEADER_WORDS].view(torch.int32)[3])
            assert torch.equal(buf[start:start + n].view(torch.int32), single[:n].view(torch.int32)), j
        rg.unpack_dirty_device(buf.data_ptr(), 4 * words, st)
        torch.cuda.synchronize()
        for j in range(M):
            for l in range(LEVELS):
                assert np.array_equal(bits(replica[j].download_level(l)), bits(f.grp[j].download_level(l))), (j, l)
        snap = [([bits(r.download_level(l)).copy() for l in range(LEVELS)],
                 [r.get_mirror_dirty_rect(l) for l in range(LEVELS)]) for r in replica]
        assert all(r.replication_overflows() == 0 for r in replica)
        rg2.unpack_dirty_device(buf.data_ptr(), 4 * words, st)
        torch.cuda.synchronize()
        assert replica[order[0]].replication_overflows(reset=True) == 1
        assert all(replica[j].replication_overflows() == 0 for j in range(M))
        for j, r in enumerate(replica):
            for l in range(LEVELS):
                assert np.array_equal(bits(r.download_level(l)), snap[j][0][l]), ("wrong order", j, l)
                assert r.get_mirror_dirty_rect(l) == snap[j][1][l], ("wrong order", j, l)
    finally:
        rg2.close()
        rg.close()
        close_all(replica)


# ---- rejections and accounting ------------------------------------------------------------------------------------

@MODES
def test_rejections(hsb_lib, mode):
    """hsb_group_create_mixed refuses another level count, resolved max_iterations, resolved gather mode and device
    (with two GPUs), NULL and duplicate handles, each naming the member and the field; hsb_group_create still refuses
    the mixed members with "differs"."""
    import torch

    from hector_slam_b200 import capi

    reps = [make_rep(s, mode) for s in range(M)]
    g = capi.SlamGroup(reps, mixed=True)
    g.close()
    with pytest.raises(capi.HsbError) as e:
        capi.SlamGroup(reps)
    assert e.value.status == -1 and "differs" in str(e.value)
    other = 1 if mode == 2 else 2
    bad = [(capi.MapRepB200(0.05, 256, levels=2, gather_mode=mode), "levels"),
           (capi.MapRepB200(0.05, 256, levels=LEVELS, max_iterations=[6, 0, 0], gather_mode=mode), "max_iterations"),
           (capi.MapRepB200(0.05, 256, levels=LEVELS, gather_mode=other), "resolved gather mode")]
    for r, field in bad:
        with pytest.raises(capi.HsbError) as e:
            capi.SlamGroup([reps[A], reps[C], r], mixed=True)
        assert e.value.status == -1 and field in str(e.value) and "handle 2" in str(e.value), str(e.value)
    for rs in ([], [reps[A], reps[C], reps[A]], [reps[A], None]):
        with pytest.raises(capi.HsbError) as e:
            capi.SlamGroup(rs, mixed=True)
        assert e.value.status == -1
    if torch.cuda.device_count() >= 2:
        from hector_slam_b200 import capi as cp

        far = cp.MapRepB200(0.05, 256, levels=LEVELS, device=1, gather_mode=mode)
        with pytest.raises(capi.HsbError) as e:
            capi.SlamGroup([reps[A], far], mixed=True)
        assert e.value.status == -1 and "device" in str(e.value)
        far.close()
    close_all([r for r, _ in bad], reps)
