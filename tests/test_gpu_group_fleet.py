"""A fleet server's group: every group call on one mixed group of about 300 members, past the 32- and 128-session
boundaries of the tile layout, the subset member list, the map writer's grid and the finish kernels.

GPU, in both gather modes.  M = max(300, ceil((8 SMs + 1) / levels)) members of 4 levels, three small geometries
assigned round-robin: (a) 128 x 128 at 0.1 m, (b) 136 x 104 at 0.1 m started at (0.3, 0.6) (levels 68 x 52, 34 x 26
and 17 x 13: widths that are not multiples of 4, odd ones), (c) 96 x 160 at 0.05 m.  A full step has K x levels
(session, level) slots, more than 8 x SMs: the map writer's mark and apply kernels run one CTA per slot.  Members
differ in update factors, gate thresholds, scan formats, laser mounts and cloud thresholds.  Each member has a twin
handle driven by single calls and a replica handle (the receiver of tile replication, and the converter the map
replay takes its endpoints from).
  - steps: full steps and permuted subsets of K = 129 and K = 33, all four input kinds, nowait, map_without_matching;
    every session equal to its twin's single step, three launches per step, unselected members untouched, every end
    state equal to the twin's, and members 0, 31, 32, 127, 128, 129, 255, 256 and M - 1 equal to a mapwrite replay of
    their own writes at the device's poses;
  - occupancy sync, full and K = 129, on two levels, and once in chunks of 4 KB that split inside and across rectangles;
  - getDist and ray casts over K = M with uneven ray counts and empty sessions at 0, 127, 128 and M - 1;
  - likelihood, covariance and best hypothesis over K = M with empty sessions at 128, 255 and M - 1, then again with
    other poses and other empty sessions (the accumulators of sessions past the first finish CTA are re-armed), and the
    likelihoods of sampled sessions within likelihood64's bound;
  - match_batch over K = M at the automatic warps per scan (1) and at 8;
  - tile replication: a full pack and unpack (the group header, block starts, ship flags, blocks byte-equal to the
    twins' single packs, replica planes and mirror rectangles), first deferrals at sessions 31, 32, 127, 128, 129 and
    256 (a smaller block still shipped after each), a member dirtier than the whole buffer, and subset packs of
    K = 128, 129 and M in permuted order.  These run last: they rewrite the owners' planes."""
import time

import numpy as np
import pytest

from conftest import report
from oracle import likelihood64
from oracle import mapwrite as mw
from test_gpu_group_dist import level_rays
from test_gpu_group_match import assert_match, auto_w, sm_count
from test_gpu_group_mixed import grids_of, twin_sync
from test_gpu_group_occupancy import n_chunks
from test_gpu_group_score import assert_sessions, hypotheses, thinned
from test_gpu_group_subset import (KINDS, assert_same_session, assert_same_state, beam_angles, bits, close_all,
                                   geometry, group_step, member_cloud, member_transform, scan_of, session_data,
                                   single_step)
from test_gpu_group_tiles import HEADER_WORDS, MAGIC, cells_of, group_header_words, layout

pytestmark = pytest.mark.gpu

F32 = np.float32
LEVELS = 4
# map_size_x, map_size_y, map_resolution, start
SPECS = [(128, 128, 0.1, (0.5, 0.5)), (136, 104, 0.1, (0.3, 0.6)), (96, 160, 0.05, (0.5, 0.5))]
TICKS = 10
CLEAN = [None] * LEVELS


def fleet_size(sms):
    return max(300, -(-(8 * sms + 1) // LEVELS))


def samples(M):
    """the sessions on either side of the 32-lane and 128-session boundaries, and the last"""
    return [0, 31, 32, 127, 128, 129, 255, 256, M - 1]


def make_rep(s, mode):
    """Member s's handle: SPECS[s % 3]'s map; scan format, gate thresholds and laser mount drawn from s // 3, so that
    they do not follow the geometry"""
    from hector_slam_b200 import capi

    sx, sy, res, start = SPECS[s % 3]
    t = s // 3
    rep = capi.MapRepB200(res, sx, sy, levels=LEVELS, start=start, update_factor_free=0.4 + 0.02 * (s % 5),
                          update_factor_occupied=0.6 + 0.1 * (s % 4), gather_mode=mode)
    dist, ang = ((0.0, 0.0), (0.15, 0.1), (0.3, 0.5))[t % 3]
    rep.setMapUpdateMinDistDiff(dist)
    rep.setMapUpdateMinAngleDiff(ang)
    g = geometry(t)
    rep.set_scan_format(**g)
    rep.set_laser_projection(**g, range_cutoff=30.0)
    rep.set_cloud_format(member_transform(s), **member_cloud(s))
    return rep


def member_data(s):
    """session_data's trajectory with the endpoints in member s's own level-0 cell units"""
    from hector_slam_b200 import synth

    g = geometry(s // 3)
    d = session_data(900 + s, TICKS + 2, g)   # (a spare step for the occupancy test)
    ang = beam_angles(g)
    d["scans"] = [np.ascontiguousarray(synth.ranges_to_points(r, 1.0 / SPECS[s % 3][2], ang), F32) for r in d["ranges"]]
    return d


def state_of(rep):
    return ([bits(rep.download_level(l)).copy() for l in range(LEVELS)], [rep.get_mirror_dirty_rect(l) for l in range(LEVELS)],
            rep.get_dirty_rects(), bits(rep.last_map_update_pose()).copy())


def same_state(a, b):
    return (all(np.array_equal(x, y) for x, y in zip(a[0], b[0])) and a[1] == b[1] and a[2] == b[2]
            and np.array_equal(a[3], b[3]))


def device_memory_used():
    import torch

    free, total = torch.cuda.mem_get_info()
    return total - free


class Fleet:
    """The mixed group of M members, their twins, their replicas (in a mixed replica group listing them in the same
    order), every member's trajectory position, and the writes of the sampled members."""

    def __init__(self, mode):
        from hector_slam_b200 import capi

        self.sms = sm_count()
        self.M = M = fleet_size(self.sms)
        self.mem0 = self.mem_peak = device_memory_used()
        t0 = time.perf_counter()
        self.grp = [make_rep(s, mode) for s in range(M)]
        self.one = [make_rep(s, mode) for s in range(M)]
        self.replica = [make_rep(s, mode) for s in range(M)]
        self.g = capi.SlamGroup(self.grp, mixed=True)
        self.rg = capi.SlamGroup(self.replica, mixed=True)
        self.create_s = time.perf_counter() - t0
        self.note_memory()
        self.data = [member_data(s) for s in range(M)]
        self.at = [0] * M
        self.covs = [np.full((3, 3), 5.0, F32) for _ in range(M)]
        self.writes = {j: [] for j in samples(M)}   # (kind, input, matched, pose, updated) per step of the member
        self.untouched = 0                          # unselected sampled members compared across a subset step
        self.buf = None

    def note_memory(self):
        self.mem_peak = max(self.mem_peak, device_memory_used())

    def tick(self, t, kind, members, nowait, rng):
        M = self.M
        sel = list(range(M)) if members is None else members
        left_out = [j for j in self.writes if j not in sel and j != 0]   # (handles[0] counts the group's launches)
        before = {j: state_of(self.grp[j]) for j in left_out}
        without = [bool(rng.random() < 0.2) and self.at[j] > 0 for j in sel]
        hints = np.asarray([self.data[j]["truth" if w else "hints"][self.at[j]] for j, w in zip(sel, without)],
                           F32).reshape(len(sel), 3)
        scans = [thinned(kind, scan_of(kind, self.data[j], self.at[j])) for j in sel]
        cov = np.stack([self.covs[j] for j in sel])
        launches = self.grp[0].launch_count
        out = group_step(self.g, kind, hints, scans, without, members=members, nowait=nowait, cov=cov)
        assert self.grp[0].launch_count - launches == 3, (t, kind)
        for i, j in enumerate(sel):
            ref = single_step(self.one[j], kind, hints[i], scans[i], without[i], cov=self.covs[j].copy())
            assert_same_session(out, i, ref, (t, kind, i, j))
            self.covs[j] = out[1][i].copy()
            if j in self.writes:
                self.writes[j].append((kind, scans[i], not without[i], out[0][i].copy(), bool(out[2][i])))
            self.at[j] += 1
        for j in left_out:
            assert same_state(state_of(self.grp[j]), before[j]), ("left out", t, j)
            self.untouched += 1
        self.note_memory()

    def run(self, seed):
        rng = np.random.default_rng(seed)
        for t in range(TICKS):
            K = (self.M, 129, 33)[t % 3]
            members = None if K == self.M else [int(j) for j in rng.permutation(self.M)[:K]]
            self.tick(t, KINDS[t % 4], members, t % 2 == 1, rng)

    def converted(self, j, kind, x):
        """the endpoints and origo the member's step drew from input x, through the replica's conversion calls"""
        c = self.replica[j]
        if kind == "endpoints":
            return x, (0.0, 0.0)
        if kind == "ranges":
            return c.scan_to_points(x), (0.0, 0.0)
        return c.cloud_to_points(x) if kind == "cloud" else c.projected_scan_to_points(x)

    def tile_buffer(self):
        """one device buffer large enough for every member's whole planes -> (buffer, capacity bytes)"""
        import torch

        if self.buf is None:
            cells = sum(r.level_info(l)[0] * r.level_info(l)[1] for r in self.grp for l in range(LEVELS))
            words = group_header_words(self.M) + self.M * HEADER_WORDS + cells
            self.buf = torch.zeros(words, dtype=torch.float32, device="cuda")
            self.note_memory()
        return self.buf, 4 * self.buf.numel()

    def close(self):
        self.g.close()
        self.rg.close()
        close_all(self.grp, self.one, self.replica)


@pytest.fixture(scope="module", params=[2, 1], ids=["tex", "ldg"])
def fleet(request, hsb_lib):
    """One stepped fleet per gather mode, shared by the tests below in file order."""
    t0 = time.perf_counter()
    f = Fleet(request.param)
    assert f.M * LEVELS > 8 * f.sms, (f.M, f.sms)
    mode = {2: "tex", 1: "ldg"}[request.param]
    report(f"group fleet [{mode}]: M = {f.M}, K x levels = {f.M * LEVELS} > 8 x SMs = {8 * f.sms} ({f.sms} SMs); "
           f"{3 * f.M} handles and two groups created in {f.create_s:.1f} s")
    f.run(51 + request.param)
    f.steps_s = time.perf_counter() - t0
    yield f
    report(f"group fleet [{mode}]: {time.perf_counter() - t0:.1f} s from creation to the last test (steps "
           f"{f.steps_s:.1f} s); device memory in use at most {(f.mem_peak - f.mem0) / 2 ** 20:.0f} MiB above the "
           f"{f.mem0 / 2 ** 20:.0f} MiB before the fleet")
    f.close()
    f.buf = None
    import torch

    torch.cuda.empty_cache()


# ---- steps --------------------------------------------------------------------------------------------------------

def test_steps_and_end_state(fleet):
    """The TICKS steps (each session checked against its twin in Fleet.tick) leave every member in its twin's state;
    sampled members left out of a subset step were untouched by it; the sampled members' planes and replication
    rectangles equal a mapwrite replay of their writes at the device's poses, cell for cell."""
    f = fleet
    M = f.M
    assert f.untouched > 0
    for j in range(M):
        assert f.at[j] > 0, j
        assert_same_state(f.grp[j], f.one[j], ("end", j), probe=j in f.writes, levels=LEVELS)
    written = 0
    for j, steps in f.writes.items():
        sx, sy, res, start = SPECS[j % 3]
        lf, lo = f.grp[j].logodds_increments()
        m = mw.MultiMap(res, sx, sy, LEVELS, lf, lo, start=start, follow="dev")
        for kind, x, matched, pose, updated in steps:
            pts, og = f.converted(j, kind, x)
            if matched:
                m.match(pts, og)
            if updated:
                m.update_by_scan(pts, pose, og)
                written += 1
        for l in range(LEVELS):
            got = f.grp[j].download_level(l)
            bad = bits(got) != bits(m.planes[l])
            assert not bad.any(), ("replay", j, l, int(bad.sum()), np.argwhere(bad)[:5].tolist())
            assert np.any(got != 0), ("replay: nothing written", j, l)
        assert f.grp[j].get_dirty_rects() == m.dirty, ("replay rectangles", j)
    report(f"group fleet: members {sorted(f.writes)} equal their mapwrite replay on every level ({written} writes); "
           f"{f.untouched} left-out member states unchanged across subset steps")


# ---- occupancy ----------------------------------------------------------------------------------------------------

def test_occupancy(fleet):
    """sync_occupancy with K = 129 (permuted) then with every member, on levels 0 and 2, against twin_sync on the
    twins; the reset clears every member's rectangle, sessions >= 128 included.  Then a full step and one sync in
    4 KB chunks: 1 + n_chunks launches, chunks split inside and across many members' rectangles."""
    f = fleet
    M = f.M
    rng = np.random.default_rng(9)
    sub = [int(j) for j in rng.permutation(M)[:129]]
    for level in (0, 2):
        for members in (sub, None):
            sel = list(range(M)) if members is None else members
            gg, tg = grids_of([f.grp[j] for j in sel], level), grids_of([f.one[j] for j in sel], level)
            rects = f.g.sync_occupancy(level, gg, members=members)
            for k, j in enumerate(sel):
                assert rects[k] == twin_sync(f.one[j], level, tg[k]), (level, k, j)
                assert np.array_equal(gg[k], tg[k]), (level, k, j)
            if members is None:
                assert any(rects[k] is not None for k in range(128, M)), level
        assert all(f.grp[j].get_mirror_dirty_rect(level) is None for j in range(M)), level
        assert f.g.sync_occupancy(level, grids_of(f.grp, level)) == [None] * M, level
    f.tick(TICKS, "endpoints", None, False, rng)   # every member writes again
    gg, tg = grids_of(f.grp, 0), grids_of(f.one, 0)
    chunk = 4096
    f.grp[0].set_tuning(occupancy_chunk=chunk)
    try:
        launches = f.grp[0].launch_count
        rects = f.g.sync_occupancy(0, gg)
        widths = [f.grp[j].level_info(0)[0] for j in range(M) if rects[j] is not None]
        chunks = n_chunks(rects, chunk, max(widths))
        assert f.grp[0].launch_count - launches == 1 + chunks
    finally:
        f.grp[0].set_tuning(occupancy_chunk=0)
    bytes_ = sum(0 if r is None else (r[2] - r[0] + 1) * (r[3] - r[1] + 1) for r in rects)
    assert len(widths) > 64 and chunks > len(widths), (len(widths), chunks)
    for j in range(M):
        assert rects[j] == twin_sync(f.one[j], 0, tg[j]), j
        assert np.array_equal(gg[j], tg[j]), j
    report(f"group fleet: occupancy in {chunks} chunks of {chunk} bytes over {len(widths)} rectangles ({bytes_} bytes)")


# ---- ray queries --------------------------------------------------------------------------------------------------

def test_ray_queries(fleet):
    """getDist and ray casts over K = M on levels 0 and 3: 1 to 40 rays per session, none at sessions 0, 127, 128
    and M - 1; each ray equal to the twin's single call."""
    f = fleet
    M = f.M
    rng = np.random.default_rng(17)
    for level in (0, LEVELS - 1):
        counts = [int(c) for c in rng.integers(1, 41, M)]
        for j in (0, 127, 128, M - 1):
            counts[j] = 0
        cells, worlds = [], []
        for j in range(M):
            occ = f.one[j].download_occupancy(level)
            if not (occ == 100).any():   # (level_rays starts some rays on occupied cells)
                occ[occ.shape[0] // 2, occ.shape[1] // 2] = 100
            cb, ce, wb, we = level_rays(f.one[j], level, 700 + 3 * j + level, max(counts[j], 1), occ)
            cells.append((cb[:counts[j]], ce[:counts[j]]))
            worlds.append((wb[:counts[j]], we[:counts[j]]))
        d, h, fnd = f.g.get_dist(level, [w[0] for w in worlds], [w[1] for w in worlds])
        cd, ch = f.g.raycast(level, [c[0] for c in cells], [c[1] for c in cells])
        q = 0
        for j in range(M):
            n = counts[j]
            if n:
                sd, sh, sf = f.one[j].get_dist_batch(level, *worlds[j])
                rd, rh = f.one[j].raycast_batch(level, *cells[j])
                tag = (level, j)
                assert np.array_equal(bits(d[q:q + n]), bits(sd)), tag
                assert np.array_equal(bits(h[q:q + n]), bits(sh)), tag
                assert np.array_equal(fnd[q:q + n], sf), tag
                assert np.array_equal(bits(cd[q:q + n]), bits(rd)), tag
                assert np.array_equal(ch[q:q + n], rh), tag
            q += n
        assert q == d.shape[0] == cd.shape[0] == sum(counts)
        assert level > 0 or (fnd.any() and (cd >= 0).any())


# ---- scoring and matching -----------------------------------------------------------------------------------------

def test_scoring(fleet):
    """likelihood, covariance (map and world) and best hypothesis over K = M on levels 0 and 2, against the twins in
    bits.  First round: poses around each member's last pose, sessions 128, 255 and M - 1 empty ({-1, 0, 0, 0}, index
    -1).  Second round right after: poses half a metre off (lower likelihoods) and sessions 129 and 256 empty, so that
    an accumulator left armed from the first round would show.  best_hypothesis makes two launches; the likelihoods of
    the sampled sessions lie within likelihood64's float64 bound."""
    f = fleet
    M = f.M
    rng = np.random.default_rng(23)
    scans = [f.data[j]["scans"][f.at[j] - 1][::3] for j in range(M)]
    worst = 0.0
    for level in (0, 2):
        for r, (empty, off) in enumerate((({128, 255, M - 1}, (0.0, 0.0, 0.0)), ({129, 256}, (0.5, -0.4, 0.3)))):
            poses = [np.zeros((0, 3), F32) if j in empty else
                     hypotheses(rng, f.data[j]["truth"][f.at[j] - 1] + F32(off), 6, specials=False) for j in range(M)]
            lh = assert_sessions(f.g, f.one, level, None, poses, scans, scans, ("round", r))
            launches = f.grp[0].launch_count
            _, best4, index = f.g.best_hypothesis(level, poses, scans)
            assert f.grp[0].launch_count - launches == 2
            for j in range(M):
                assert (index[j] == -1) == (j in empty), (level, r, j, index[j])
                if j in empty:
                    assert np.array_equal(best4[j], F32([-1, 0, 0, 0])), (level, r, j, best4[j])
            q = np.concatenate([[0], np.cumsum([p.shape[0] for p in poses])])
            for j in samples(M):
                if j in empty:
                    continue
                prob = f.one[j].download_prob(level)
                n = scans[j].shape[0]
                for b, p in enumerate(poses[j]):
                    ev = likelihood64.evaluate(prob, scans[j], f.one[j].map_coords_pose(level, p), 2.0 ** -level)
                    tol = ev.tol(-(-n // 32) + 5)
                    err = abs(float(lh[q[j] + b]) - ev.lh64)
                    assert err <= tol, (level, r, j, b, float(lh[q[j] + b]), ev.lh64, err, tol)
                    worst = max(worst, err / tol if tol else 0.0)
    assert worst > 0.0
    report(f"group fleet: sampled likelihoods within {worst:.3f} of likelihood64's bound")


def test_match_batch(fleet):
    """match_batch with 8 hints per session over K = M at the automatic warps per scan (1 at this size) and with 8
    forced on handles[0]: each pose and covariance equal to the member's hsb_match_batch at the same W."""
    f = fleet
    M = f.M
    rng = np.random.default_rng(29)
    hints = [hypotheses(rng, f.data[j]["truth"][f.at[j] - 1], 8, specials=False) for j in range(M)]
    scans = [f.data[j]["scans"][f.at[j] - 1][::2] for j in range(M)]
    _, _, W = assert_match(f.g, f.grp, None, hints, scans, scans, ("auto",))
    assert W == auto_w(8 * M) == 1, W
    f.grp[0].set_tuning(warps_per_scan=8)
    try:
        _, _, W = assert_match(f.g, f.grp, None, hints, scans, scans, ("W = 8",), restore=8)
        assert W == 8
    finally:
        f.grp[0].set_tuning(warps_per_scan=0)


# ---- tile replication (last: it rewrites the owners' planes) -------------------------------------------------------

def stream():
    import torch

    return torch.cuda.current_stream().cuda_stream


def words_of(buf):
    import torch

    torch.cuda.synchronize()
    return buf.view(torch.int32).cpu().numpy()


def round_trip(f, cap, reset=True, members=None):
    buf, _ = f.tile_buffer()
    st = stream()
    f.g.pack_dirty_device(buf.data_ptr(), cap, reset, st, members=members)
    f.rg.unpack_dirty_device(buf.data_ptr(), cap, st)
    return words_of(buf)


def assert_layout(w, rects, members, cap):
    """the group header and every block's ship flag are the host's layout -> blocks"""
    hdr, blocks = layout(rects, members, cap, LEVELS)
    got = [int(v) for v in w[:len(hdr)]]
    assert got == hdr, [(i, a, b) for i, (a, b) in enumerate(zip(got, hdr)) if a != b][:8]
    for k, (start, ship) in enumerate(blocks):
        assert w[start] == MAGIC and w[start + 2] == (0 if ship else 1), (k, members[k], start, ship)
    return blocks


def upload(f, which, rng):
    """a fresh plane on each listed owner level {member: levels}"""
    for j, levels in which.items():
        for l in levels:
            sx, sy, _ = f.grp[j].level_info(l)
            f.grp[j].upload_level(l, rng.uniform(-60.0, 50.0, (sy, sx)).astype(F32))


def assert_replica(f, j, levels, tag, prob=False):
    for l in levels:
        got = f.replica[j].download_level(l)
        assert np.array_equal(bits(got), bits(f.grp[j].download_level(l))), (tag, j, l)
        if prob:
            assert np.array_equal(bits(f.replica[j].download_prob(l)), bits(mw.prob(got))), (tag, j, l)


def ship_the_rest(f, which, tag):
    """the next pack with room for everything ships what is left: every owner clean, every replica equal"""
    _, cap = f.tile_buffer()
    w = round_trip(f, cap)
    assert w[3] == 0, tag
    for j, levels in which.items():
        assert_replica(f, j, levels, (tag, "next pack"))
    assert all(f.grp[j].get_dirty_rects() == CLEAN for j in range(f.M)), tag
    assert all(r.replication_overflows() == 0 for r in f.replica), tag


def test_tiles_full_round_trip(fleet):
    """After the steps: one full pack (no reset) and an unpack on the replica group.  The group header, every block
    start and ship flag are layout()'s; the sampled blocks are byte-equal to the twins' single packs; every replica
    plane equals its owner's (P equals mapwrite.prob on the sampled members) and its mirror rectangles are what it
    received.  A second pack with reset leaves every owner clean."""
    import torch

    f = fleet
    M = f.M
    rects = [f.grp[j].get_dirty_rects() for j in range(M)]
    assert rects == [f.one[j].get_dirty_rects() for j in range(M)]
    clean = [j for j in range(M) if cells_of(rects[j]) == 0]
    assert len(clean) < M // 10 and not set(clean) & set(samples(M)), clean
    buf, cap = f.tile_buffer()
    buf.zero_()
    w = round_trip(f, cap, reset=False)
    blocks = assert_layout(w, rects, list(range(M)), cap)
    assert all(ship for _, ship in blocks)
    single = torch.zeros(HEADER_WORDS + max(cells_of(r) for r in rects), dtype=torch.float32, device="cuda")
    for k in samples(M):
        single.zero_()
        f.one[k].pack_dirty_device(single.data_ptr(), 4 * single.numel(), False, stream())
        n = HEADER_WORDS + cells_of(rects[k])
        want = words_of(single)[:n]
        start = blocks[k][0]
        assert np.array_equal(w[start:start + n], want), (k, np.argwhere(w[start:start + n] != want)[:5].tolist())
    for j in range(M):
        assert_replica(f, j, range(LEVELS), "full", prob=j in samples(M))
        assert [f.replica[j].get_mirror_dirty_rect(l) for l in range(LEVELS)] == rects[j], j
        assert f.replica[j].replication_overflows() == 0, j
    assert [f.grp[j].get_dirty_rects() for j in range(M)] == rects
    ship_the_rest(f, {}, "full with reset")
    report(f"group fleet: full pack of {M} blocks ({len(clean)} clean: {clean}), {int(w[4])} words, replica equal; "
           f"blocks {samples(M)} byte-equal to the single packs")


def test_tiles_deferrals_at_the_boundaries(fleet):
    """Every member uploads one level; capacities chosen from layout() so that the first deferred block is session 31,
    32, 127, 128, 129 or 256 and the next, smaller block still ships; then a member dirtier than the whole buffer.  Each
    with reset: the deferred count, each replica member's overflow counter, only shipped owners cleared, shipped
    replicas equal and deferred ones unchanged; the next pack ships what was deferred."""
    f = fleet
    M = f.M
    G = group_header_words(M)
    base = G + HEADER_WORDS * M
    rng = np.random.default_rng(37)
    seen = []
    for case, d in enumerate((31, 32, 127, 128, 129, 256)):
        which = {j: [(j + case) % LEVELS] for j in range(M)}
        which[d], which[d + 1] = [0], [LEVELS - 1]
        upload(f, which, rng)
        rects = [f.grp[j].get_dirty_rects() for j in range(M)]
        cells = [cells_of(r) for r in rects]
        cap = 4 * (base + sum(cells[:d]) + cells[d + 1])
        hdr, blocks = layout(rects, list(range(M)), cap, LEVELS)
        ships = [s for _, s in blocks]
        first = ships.index(False)
        used = [start - G - HEADER_WORDS * k for k, (start, _) in enumerate(blocks)]
        assert first == d and ships[d + 1] and cells[d + 1] > 0 and all(cells), (d, first)
        if d >= 128:   # a deferral in a later chunk, after chunk 1 shipped rows: the layout carries `used` into it
            assert used[128] > 0
        if d >= 256:
            assert used[256] > used[128]
        before = {j: [bits(f.replica[j].download_level(l)).copy() for l in which[j]] for j in range(M) if not ships[j]}
        w = round_trip(f, cap)
        assert_layout(w, rects, list(range(M)), cap)
        assert w[3] == ships.count(False) == hdr[3]
        assert [f.replica[j].replication_overflows(reset=True) for j in range(M)] == [int(not s) for s in ships], d
        for j in range(M):
            if ships[j]:
                assert f.grp[j].get_dirty_rects() == CLEAN, (d, j)
                assert_replica(f, j, which[j], ("shipped", d))
            else:
                assert f.grp[j].get_dirty_rects() == rects[j], (d, j)
                for l, b in zip(which[j], before[j]):
                    got = bits(f.replica[j].download_level(l))
                    assert np.array_equal(got, b) and not np.array_equal(got, bits(f.grp[j].download_level(l))), (d, j, l)
        ship_the_rest(f, which, ("after", d))
        seen.append((d, ships.count(False), sum(ships[d + 1:])))
    # a member dirtier than the whole buffer: all four levels of a 128 x 128 member; small blocks on either side ship
    big = 255
    assert SPECS[big % 3][:2] == (128, 128)
    small = [big - 1, big + 1, big + 2, M - 1]
    which = {big: list(range(LEVELS)), **{j: [LEVELS - 1] for j in small}}
    upload(f, which, rng)
    rects = [f.grp[j].get_dirty_rects() for j in range(M)]
    cells = [cells_of(r) for r in rects]
    cap = 4 * (base + sum(cells[j] for j in small))
    assert cells[big] > cap // 4, (cells[big], cap)
    w = round_trip(f, cap)
    blocks = assert_layout(w, rects, list(range(M)), cap)
    assert [k for k, (_, s) in enumerate(blocks) if not s] == [big] and w[3] == 1
    assert [f.replica[j].replication_overflows(reset=True) for j in range(M)] == [int(j == big) for j in range(M)]
    assert f.grp[big].get_dirty_rects() == rects[big]
    for j in small:
        assert f.grp[j].get_dirty_rects() == CLEAN
        assert_replica(f, j, which[j], "beside the dirtiest")
    ship_the_rest(f, which, "dirtier than the buffer")
    report(f"group fleet: first deferrals (session, deferred, shipped after it) {seen}; a {cells[big]}-cell block "
           f"deferred from a {cap // 4}-word buffer")


def test_tiles_subset_packs(fleet):
    """Subset packs of K = 128 (the small member list), 129 and M (the large one), in permuted order, every member
    dirty: the header is layout()'s for that order, the selected members' blocks land on their replicas, the others
    keep their rectangles and their replicas; two launches per pack with reset, one per unpack."""
    f = fleet
    M = f.M
    rng = np.random.default_rng(41)
    _, cap = f.tile_buffer()
    for K in (128, 129, M):
        members = [int(j) for j in rng.permutation(M)[:K]]
        which = {j: [int(rng.integers(0, LEVELS))] for j in range(M)}
        upload(f, which, rng)
        rects = [f.grp[j].get_dirty_rects() for j in range(M)]
        left_out = [j for j in range(M) if j not in set(members)]
        before = {j: bits(f.replica[j].download_level(which[j][0])).copy() for j in left_out}
        la, lb = f.grp[0].launch_count, f.replica[0].launch_count
        w = round_trip(f, cap, members=members)
        assert (f.grp[0].launch_count - la, f.replica[0].launch_count - lb) == (2, 1), K
        blocks = assert_layout(w, [rects[j] for j in members], members, cap)
        assert all(s for _, s in blocks) and w[3] == 0
        for j in members:
            assert f.grp[j].get_dirty_rects() == CLEAN, (K, j)
            assert_replica(f, j, which[j], ("subset", K))
        for j in left_out:
            assert f.grp[j].get_dirty_rects() == rects[j], (K, j)
            assert np.array_equal(bits(f.replica[j].download_level(which[j][0])), before[j]), (K, j)
        ship_the_rest(f, which, ("after subset", K))
