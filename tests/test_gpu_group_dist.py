"""hector_map_server's obstacle-distance queries for a group's members in one pass (hsb_group_get_dist,
hsb_group_raycast and their _subset forms): every session's rays cast on its member's plane of a level by one launch,
with one copy each way.

Every ray's distance, hit and found flag are compared in bits: with the single calls (hsb_get_dist_batch,
hsb_raycast_batch) on maps written by mixed full, subset, nowait and map_without_matching group steps, every level,
ragged and empty sessions, permuted member lists; with HectorMapTools.h compiled unmodified (oracle/_ref; the C port
where it is absent) on per-member planes, the constructed long rays included (5000-step cap, end cell, offsets next to
a perfect square); across the grid-stride loop; right after nowait steps of this group, of a member alone and of a
second group.  Also: no member state changes (a twin fleet stepped without queries ends byte-identical), launch
accounting, rejections and the C++ façade.  Every group case runs on a TEX and an LDG group."""
import ctypes as C
import os

import numpy as np
import pytest

import maptools_cases as mc
from conftest import ROOT
from test_gpu_group_subset import geometry, session_data

pytestmark = pytest.mark.gpu

MODES = pytest.mark.parametrize("mode", [2, 1], ids=["tex", "ldg"])   # capi.GATHER_TEX, capi.GATHER_LDG
SLAM_GEOMS = [g for g in mc.GEOMS if g[2] > 1]   # the multi-level ones: a scan writes every level
GEOM = SLAM_GEOMS[0]
SENTINEL = 77


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def make_rep(geom, s, mode):
    from hector_slam_b200 import capi

    sx, sy, levels, start = geom
    rep = capi.MapRepB200(mc.RES, sx, sy, levels=levels, start=start, update_factor_free=0.4 + 0.02 * (s % 3),
                          update_factor_occupied=0.6 + 0.1 * (s % 4), gather_mode=mode)
    dist, ang = ((0.0, 0.0), (0.15, 0.1), (0.3, 0.5))[s % 3]
    rep.setMapUpdateMinDistDiff(dist)
    rep.setMapUpdateMinAngleDiff(ang)
    rep.set_scan_format(**geometry(s))
    assert rep.gather_mode == mode
    return rep


def fleet(geom, M, mode):
    from hector_slam_b200 import capi

    reps = [make_rep(geom, s, mode) for s in range(M)]
    return reps, capi.SlamGroup(reps)


def step(groups, data, at, t, members, rng, nowait):
    """one endpoints or ranges group step of `members` (None: all) on every group of `groups`, the same inputs
    -> the results of each group"""
    M = len(data)
    sel = list(range(M)) if members is None else members
    kind = ("endpoints", "ranges")[t % 2]
    without = [bool(rng.random() < 0.2) and at[j] > 0 for j in sel]
    hints = np.asarray([data[j]["truth" if w else "hints"][at[j]] for j, w in zip(sel, without)],
                       np.float32).reshape(len(sel), 3)
    scans = [data[j]["scans" if kind == "endpoints" else "ranges"][at[j]] for j in sel]
    out = []
    for g in groups:
        fn = g.slam_update if kind == "endpoints" else g.slam_update_ranges
        out.append(fn(hints, scans, map_without_matching=without, nowait=nowait, members=members)[:3])
    for j in sel:
        at[j] += 1
    return out


def level_rays(rep, level, seed, n, occ=None):
    """n cell rays and n world rays in and around the level (maptools_cases), NaN and absurd world points included.
    occ: the occupancy the cell rays take their begins on occupied cells from (None: the level's, downloaded; a given
    one keeps the handle's streams untouched)"""
    sx, sy, cell = rep.level_info(level)
    if occ is None:
        occ = rep.download_occupancy(level)
    cb, ce = mc.cell_rays(sx, sy, occ, seed)
    wb, we, _ = mc.world_rays(sx, sy, rep.map_origin(level), cell, seed)
    rng = np.random.default_rng(seed)
    ic, iw = rng.choice(cb.shape[0], n), rng.choice(wb.shape[0], n)
    wb, we = wb[iw].copy(), we[iw].copy()
    wb[rng.random(n) < 0.02] = np.float32(3e30)
    we[rng.random(n) < 0.02] = np.float32(-1e12)
    return cb[ic], ce[ic], wb, we


def ragged(rng, K, hi):
    """K ray counts in [0, hi], at least one session empty when K > 1"""
    n = [int(v) for v in rng.integers(0, hi + 1, K)]
    if K > 1:
        n[int(rng.integers(0, K))] = 0
    return n


def query_round(g, reps, level, members, counts, seed):
    """One getDist and one ray-cast round of the group against the single calls on each member, in bits."""
    cells, worlds = [], []
    for k, j in enumerate(members):
        cb, ce, wb, we = level_rays(reps[j], level, seed + 13 * j + k, max(counts[k], 1))
        cells.append((cb[:counts[k]], ce[:counts[k]]))
        worlds.append((wb[:counts[k]], we[:counts[k]]))
    d, h, f = g.get_dist(level, [w[0] for w in worlds], [w[1] for w in worlds], members=members)
    cd, ch = g.raycast(level, [c[0] for c in cells], [c[1] for c in cells], members=members)
    q = 0
    for k, j in enumerate(members):
        n = counts[k]
        sd, sh, sf = reps[j].get_dist_batch(level, *worlds[k])
        rd, rh = reps[j].raycast_batch(level, *cells[k])
        tag = (level, k, j)
        assert np.array_equal(bits(d[q:q + n]), bits(sd)), tag
        assert np.array_equal(bits(h[q:q + n]), bits(sh)), tag
        assert np.array_equal(f[q:q + n], sf), tag
        assert np.array_equal(bits(cd[q:q + n]), bits(rd)), tag
        assert np.array_equal(ch[q:q + n], rh), tag
        q += n
    assert q == d.shape[0] == cd.shape[0]
    return f


def close_all(*xs):
    for x in xs:
        for y in (x if isinstance(x, (list, tuple)) else [x]):
            y.close()


# ---- 1: against the single calls ----------------------------------------------------------------------------------

@MODES
@pytest.mark.parametrize("geom", SLAM_GEOMS, ids=mc.geom_id)
def test_against_single_calls(hsb_lib, geom, mode):
    """M = 5, 12 ticks of full and subset, sync and nowait, endpoint and range group steps (some sessions
    map_without_matching); after every tick a query round at one level, full or over a permuted subset, with ragged ray
    counts (an empty session every time); at the end a full round at every level.  Every ray equals the single call on
    its member in bits."""
    M, ticks = 5, 12
    reps, g = fleet(geom, M, mode)
    data = [session_data(2100 + s, ticks, geometry(s)) for s in range(M)]
    rng = np.random.default_rng(31)
    at = [0] * M
    levels = geom[2]
    hits = 0
    for t in range(ticks):
        members = None if t % 4 == 0 else [int(j) for j in rng.permutation(M)[:int(rng.integers(1, M + 1))]]
        step([g], data, at, t, members, rng, nowait=(t % 3 != 0))
        sel = [int(j) for j in rng.permutation(M)[:int(rng.integers(1, M + 1))]] if t % 2 else list(range(M))
        f = query_round(g, reps, t % levels, sel, ragged(rng, len(sel), 60), 500 * t)
        hits += int(f.sum())
    for l in range(levels):
        query_round(g, reps, l, [int(j) for j in rng.permutation(M)], ragged(rng, M, 200), 9000 + l)
    assert hits > 20
    close_all(g, reps)


# ---- 2: against the compiled header -------------------------------------------------------------------------------

def oracle_rays(geom, l, plane, cb, ce, wb, we):
    """(dist, hit) of the cell rays and (dist, hit_world, found) of the world rays from HectorMapTools.h over the
    thresholded plane (the C port without oracle/_ref), as test_gpu_map_io.expected_rays computes them"""
    from oracle import pyoracle

    sx, sy, levels, start = geom
    port = pyoracle.Oracle("port", mc.RES, sx, levels, start=start, size_y=sy)
    cell, origin = port.cell_length(l), port.map_origin(l)
    mt = pyoracle.RefMapTools(mc.occupancy(plane), cell, origin) if pyoracle.available("reference") else None
    if mt is None:
        port.set_logodds(l, plane)
    cast = [mt.raycast(b, e) if mt else port.raycast(l, b, e) for b, e in zip(cb, ce)]
    is_nan = np.isnan(wb).any(axis=1) | np.isnan(we).any(axis=1)
    gd = [(-1.0, np.zeros(2, np.float32), False) if nan else (mt.get_dist(b, e) if mt else port.get_dist(l, b, e))
          for b, e, nan in zip(wb, we, is_nan)]
    if mt:
        mt.close()
    port.close()
    gdist = np.float32([x[0] for x in gd])
    gdist[is_nan] = np.float32(-cell)
    return (np.float32([c[0] for c in cast]), np.int32([c[1] for c in cast]), gdist, np.float32([x[1] for x in gd]),
            np.array([x[2] for x in gd]))


@MODES
@pytest.mark.parametrize("geom", mc.GEOMS, ids=mc.geom_id)
def test_against_compiled_header(hsb_lib, geom, mode):
    """Three members with their own planes (mc.plane) on every level; the cell and world rays of maptools_cases split
    raggedly between them, members listed in reverse order: every ray equals the compiled header on its member's
    plane."""
    from hector_slam_b200 import capi

    sx, sy, levels, start = geom
    M = 3
    reps = [capi.MapRepB200(mc.RES, sx, sy, levels=levels, start=start, gather_mode=mode) for _ in range(M)]
    g = capi.SlamGroup(reps)
    members = [2, 1, 0]
    for l, (lx, ly) in enumerate(mc.level_sizes(geom)):
        planes = [mc.plane(lx, ly, seed=lx * 31 + ly + l + 1000 * j) for j in range(M)]
        for rep, p in zip(reps, planes):
            rep.upload_level(l, p)
        sess = []
        for k, j in enumerate(members):
            cb, ce = mc.cell_rays(lx, ly, mc.occupancy(planes[j]), seed=lx + 7 * ly + j)
            wb, we, _ = mc.world_rays(lx, ly, reps[j].map_origin(l), reps[j].level_info(l)[2], seed=lx + 3 * ly + j)
            cut_c, cut_w = (cb.shape[0] * (k + 1)) // (M + 1), (wb.shape[0] * (k + 1)) // (M + 1)
            sess.append((cb[:cut_c], ce[:cut_c], wb[:cut_w], we[:cut_w]))
        cd, ch = g.raycast(l, [s[0] for s in sess], [s[1] for s in sess], members=members)
        d, h, f = g.get_dist(l, [s[2] for s in sess], [s[3] for s in sess], members=members)
        qc = qw = 0
        for k, j in enumerate(members):
            cb, ce, wb, we = sess[k]
            dist, hit, gdist, ghit, gfound = oracle_rays(geom, l, planes[j], cb, ce, wb, we)
            nc, nw = cb.shape[0], wb.shape[0]
            assert np.array_equal(bits(cd[qc:qc + nc]), bits(dist)) and np.array_equal(ch[qc:qc + nc], hit), (l, j)
            gf = f[qw:qw + nw]
            assert np.array_equal(bits(d[qw:qw + nw]), bits(gdist)) and np.array_equal(gf, gfound), (l, j)
            assert np.array_equal(bits(h[qw:qw + nw][gf]), bits(ghit[gfound])) and not h[qw:qw + nw][~gf].any(), (l, j)
            qc, qw = qc + nc, qw + nw
    close_all(g, reps)


@MODES
@pytest.mark.parametrize("geom", mc.LONG, ids=mc.geom_id)
def test_constructed_long_rays(hsb_lib, geom, mode):
    """One member per constructed case of maptools_cases.lone_cases (the 5000-step cap, the end cell, hit offsets next
    to a perfect square in all four mirrors), its lone-cell plane uploaded: one ray-cast call covers every case and
    equals the compiled header; one getDist call over the same rays given as world points at the cell centres equals
    hsb_get_dist_batch on each member."""
    from hector_slam_b200 import capi
    from oracle import pyoracle

    sx, sy, _, start = geom
    cases = mc.lone_cases(sx, sy)
    M = len(cases)
    reps = [capi.MapRepB200(mc.RES, sx, sy, levels=1, start=start, gather_mode=mode) for _ in range(M)]
    g = capi.SlamGroup(reps)
    port = pyoracle.Oracle("port", mc.RES, sx, 1, start=start, size_y=sy)
    have_ref = pyoracle.available("reference")
    want = []
    for k, c in enumerate(cases):
        p = mc.lone_plane(sx, sy, c.cell, seed=k)
        reps[k].upload_level(0, p)
        if have_ref:
            mt = pyoracle.RefMapTools(mc.occupancy(p), port.cell_length(0), port.map_origin(0))
            want.append(mt.raycast(c.begin, c.end))
            mt.close()
        else:
            port.set_logodds(0, p)
            want.append(port.raycast(0, c.begin, c.end))
        assert want[-1] == ((float(c.dist), c.cell) if c.hit else (-1.0, (-1, -1))), (c, want[-1])
    members = [int(j) for j in np.random.default_rng(7).permutation(M)]
    d, h = g.raycast(0, [np.int32([cases[j].begin]) for j in members], [np.int32([cases[j].end]) for j in members],
                     members=members)
    for q, j in enumerate(members):
        assert (float(d[q]), tuple(int(v) for v in h[q])) == want[j], (cases[j], d[q], h[q])
    origin, cell = reps[0].map_origin(0), np.float32(reps[0].level_info(0)[2])

    def world(c):
        return (origin + (np.float32(c) + np.float32(0.5)) * cell).astype(np.float32)[None]

    wd, wh, wf = g.get_dist(0, [world(cases[j].begin) for j in members], [world(cases[j].end) for j in members],
                            members=members)
    for q, j in enumerate(members):
        sd, sh, sf = reps[j].get_dist_batch(0, world(cases[j].begin), world(cases[j].end))
        assert bits(wd[q]) == bits(sd[0]) and np.array_equal(bits(wh[q]), bits(sh[0])) and wf[q] == sf[0], cases[j]
    assert wf.sum() == sum(c.hit for c in cases)
    port.close()
    close_all(g, reps)


# ---- 3: grid-stride -----------------------------------------------------------------------------------------------

@MODES
def test_grid_stride(hsb_lib, mode):
    """16 members x 700 rays in one call: more rays than the launch has warps (at most 8 CTAs of 8 warps per SM).
    Equal to the same rays issued in calls of one member and at most 50 rays each."""
    import torch

    M, n = 16, 700
    reps, g = fleet(GEOM, M, mode)
    data = [session_data(2200 + s, 2, geometry(s)) for s in range(M)]
    at = [0] * M
    step([g], data, at, 0, None, np.random.default_rng(1), nowait=False)
    assert M * n > torch.cuda.get_device_properties(0).multi_processor_count * 8 * 8
    rays = [level_rays(reps[j], 0, 300 + j, n) for j in range(M)]
    d, h, f = g.get_dist(0, [r[2] for r in rays], [r[3] for r in rays])
    cd, ch = g.raycast(0, [r[0] for r in rays], [r[1] for r in rays])
    for j in range(M):
        for a in range(0, n, 50):
            q = slice(j * n + a, j * n + min(n, a + 50))
            r = [x[a:a + 50] for x in rays[j]]
            sd, sh, sf = g.get_dist(0, [r[2]], [r[3]], members=[j])
            rd, rh = g.raycast(0, [r[0]], [r[1]], members=[j])
            assert np.array_equal(bits(d[q]), bits(sd)) and np.array_equal(bits(h[q]), bits(sh)), (j, a)
            assert np.array_equal(f[q], sf) and np.array_equal(bits(cd[q]), bits(rd)) and np.array_equal(ch[q], rh)
    assert f.sum() > 20 and (cd >= 0).sum() > 20
    close_all(g, reps)


# ---- 4: ordering --------------------------------------------------------------------------------------------------

def settled(reps, g, level, members, worlds, cells):
    """the single calls on each member after hsb_on_map_updated, concatenated in ray order"""
    out = [[], [], [], [], []]
    for k, j in enumerate(members):
        reps[j].onMapUpdated()
        for i, x in enumerate(reps[j].get_dist_batch(level, *worlds[k]) + reps[j].raycast_batch(level, *cells[k])):
            out[i].append(x)
    return [np.concatenate(x) for x in out]


def any_occ(rep, level, seed):
    """an occupancy of the level's shape with occupied cells, for level_rays without touching the handle"""
    sx, sy, _ = rep.level_info(level)
    return mc.occupancy(mc.plane(sx, sy, seed))


def assert_round_settled(g, reps, level, members, seed, tag):
    cells, worlds = [], []
    for k, j in enumerate(members):
        cb, ce, wb, we = level_rays(reps[j], level, seed + k, 40, occ=any_occ(reps[j], level, seed + k))
        cells.append((cb, ce))
        worlds.append((wb, we))
    # the group call first, right after the step it must see
    got = g.get_dist(level, [w[0] for w in worlds], [w[1] for w in worlds], members=members)
    got += g.raycast(level, [c[0] for c in cells], [c[1] for c in cells], members=members)
    want = settled(reps, g, level, members, worlds, cells)
    for i, (x, y) in enumerate(zip(got, want)):
        assert np.array_equal(bits(x) if x.dtype == np.float32 else x, bits(y) if y.dtype == np.float32 else y), (tag, i)


@MODES
def test_ordering(hsb_lib, mode):
    """A query round right after (1) a nowait step of this group, (2) a member's own nowait single step, (3) a nowait
    step of a second group that shares a member sees the written maps: it equals the single calls issued after
    hsb_on_map_updated.  The rays run through the area the step wrote (the robot's surroundings)."""
    from hector_slam_b200 import capi

    M, ticks = 4, 6
    reps, g = fleet(GEOM, M, mode)
    solo = capi.SlamGroup([reps[3]])
    data = [session_data(2300 + s, 3 * ticks, geometry(s)) for s in range(M)]
    rng = np.random.default_rng(3)
    at = [0] * M
    for t in range(ticks):
        step([g], data, at, t, None, rng, nowait=True)                                            # (1)
        assert_round_settled(g, reps, t % GEOM[2], [int(j) for j in rng.permutation(M)], 40 * t, ("group", t))
        j = t % M                                                                                 # (2)
        reps[j].slam_update(data[j]["hints"][at[j]], data[j]["scans"][at[j]], nowait=True)
        at[j] += 1
        assert_round_settled(g, reps, 0, [j, (j + 1) % M], 40 * t + 7, ("single", t))
        k = at[3]                                                                                 # (3)
        solo.slam_update(data[3]["hints"][k][None], [data[3]["scans"][k]], nowait=True)
        at[3] += 1
        assert_round_settled(g, reps, 0, [3, 0], 40 * t + 11, ("other group", t))
    close_all(solo, g, reps)


# ---- 5: no state change -------------------------------------------------------------------------------------------

def state(rep):
    """every level's log-odds, probability and occupancy grid, both dirty rectangles (read without reset), gate pose"""
    lv = [(bits(rep.download_level(l)).copy(), bits(rep.download_prob(l)).copy(), rep.download_occupancy(l),
           rep.get_mirror_dirty_rect(l)) for l in range(rep.levels)]
    return lv, rep.get_dirty_rects(), bits(rep.last_map_update_pose()).copy()


def assert_same_state(a, b, tag):
    sa, sb = state(a), state(b)
    for l, (x, y) in enumerate(zip(sa[0], sb[0])):
        assert all(np.array_equal(u, v) for u, v in zip(x[:3], y[:3])) and x[3] == y[3], (tag, l)
    assert sa[1] == sb[1] and np.array_equal(sa[2], sb[2]), tag


@MODES
def test_no_state_change(hsb_lib, mode):
    """Twin fleets take the same 10 ticks of group steps; fleet A answers a query round over a subset after most of
    them.  Poses, covariances and gate decisions of every step are equal in bits, and at the end every member's planes,
    grids, both dirty rectangles and gate pose are byte-identical to its twin.  The rectangles of members left out of a
    round do not move during it."""
    M, ticks = 5, 10
    a, ga = fleet(GEOM, M, mode)
    b, gb = fleet(GEOM, M, mode)
    data = [session_data(2400 + s, ticks, geometry(s)) for s in range(M)]
    rng = np.random.default_rng(5)
    at = [0] * M
    occs = [any_occ(a[0], l, l) for l in range(GEOM[2])]
    for t in range(ticks):
        members = None if t % 3 == 0 else [int(j) for j in rng.permutation(M)[:int(rng.integers(1, M + 1))]]
        ra, rb = step([ga, gb], data, at, t, members, rng, nowait=(t % 2 == 0))
        for x, y in zip(ra, rb):
            assert np.array_equal(bits(x) if x.dtype != bool else x, bits(y) if y.dtype != bool else y), t
        if t % 4 != 3:
            sel = [int(j) for j in rng.permutation(M)[:int(rng.integers(1, M))]]
            left = [j for j in range(M) if j not in sel]
            before = {j: ([a[j].get_mirror_dirty_rect(l) for l in range(GEOM[2])], a[j].get_dirty_rects()) for j in left}
            for l in range(GEOM[2]):
                cells, worlds = zip(*[((r[0], r[1]), (r[2], r[3]))
                                      for r in (level_rays(a[j], l, 60 * t + j, 30, occ=occs[l]) for j in sel)])
                ga.get_dist(l, [w[0] for w in worlds], [w[1] for w in worlds], members=sel)
                ga.raycast(l, [c[0] for c in cells], [c[1] for c in cells], members=sel)
            for j in left:
                assert ([a[j].get_mirror_dirty_rect(l) for l in range(GEOM[2])], a[j].get_dirty_rects()) == before[j]
    for j in range(M):
        assert_same_state(a[j], b[j], j)
    close_all(ga, gb, a, b)


# ---- 6: accounting and rejections ---------------------------------------------------------------------------------

@MODES
def test_launches_and_rejections(hsb_lib, mode):
    """Each call with rays is one launch on handles[0], whichever members it lists; the other members' counts do not
    move.  Every rejection returns -1 with its message, launches nothing and writes no output byte; K = 0 and Q = 0
    queue nothing; the group still answers afterwards."""
    M = 4
    reps, g = fleet(GEOM, M, mode)
    data = [session_data(2500 + s, 1, geometry(s)) for s in range(M)]
    step([g], data, [0] * M, 0, None, np.random.default_rng(6), nowait=True)
    lib = g.lib
    rays = [level_rays(reps[j], 0, 70 + j, 10) for j in range(M)]
    for members in (None, [2], [3, 1], [1, 0, 3, 2]):
        counts = [r.launch_count for r in reps]
        sel = list(range(M)) if members is None else members
        g.get_dist(0, [rays[j][2] for j in sel], [rays[j][3] for j in sel], members=members)
        assert [r.launch_count for r in reps] == [counts[0] + 1] + counts[1:], members
        g.raycast(0, [rays[j][0] for j in sel], [rays[j][1] for j in sel], members=members)
        assert [r.launch_count for r in reps] == [counts[0] + 2] + counts[1:], members

    Q = 12
    wb, we = np.ones((Q, 2), np.float32), np.full((Q, 2), 2.0, np.float32)
    cb, ce = np.ones((Q, 2), np.int32), np.full((Q, 2), 40, np.int32)
    dist, hit, found = np.full(Q, SENTINEL, np.float32), np.full((Q, 2), SENTINEL, np.float32), np.full(Q, SENTINEL, np.int32)
    chit = np.full((Q, 2), SENTINEL, np.int32)

    def arr(x, dt=np.int32):
        return None if x is None else np.ascontiguousarray(x, dt)

    def gd(K, members, level=0, offsets=(0, 4, 4, 12), b=wb, e=we, out=dist):
        m, o = arr(members), arr(offsets)
        return lib.hsb_group_get_dist_subset(g.g, K, None if m is None else m.ctypes.data, level,
                                             None if o is None else o.ctypes.data, None if b is None else b.ctypes.data,
                                             None if e is None else e.ctypes.data, None if out is None else out.ctypes.data,
                                             hit.ctypes.data, found.ctypes.data)

    def rc(K, members, level=0, offsets=(0, 4, 4, 12), b=cb, e=ce, out=dist):
        m, o = arr(members), arr(offsets)
        return lib.hsb_group_raycast_subset(g.g, K, None if m is None else m.ctypes.data, level,
                                            None if o is None else o.ctypes.data, None if b is None else b.ctypes.data,
                                            None if e is None else e.ctypes.data, None if out is None else out.ctypes.data,
                                            chit.ctypes.data)

    def err():
        return (lib.hsb_last_error(reps[0].h) or b"").decode()

    full_off = arr((0, 3, 3, 3, 12))
    cases = []
    for fn in (gd, rc):
        cases += [(lambda fn=fn: fn(-1, [0]), "K is -1"), (lambda fn=fn: fn(M + 1, [0, 1, 2, 3, 0]), "K is 5"),
                  (lambda fn=fn: fn(3, None), "members is NULL"), (lambda fn=fn: fn(3, [0, 1, M]), "session 2: member 4"),
                  (lambda fn=fn: fn(3, [-1, 0, 1]), "session 0: member -1"), (lambda fn=fn: fn(3, [1, 3, 1]), "listed twice"),
                  (lambda fn=fn: fn(3, [0, 1, 2], level=-1), "level -1"),
                  (lambda fn=fn: fn(3, [0, 1, 2], level=GEOM[2]), "level 3"),
                  (lambda fn=fn: fn(3, [0, 1, 2], offsets=None), "offsets is NULL"),
                  (lambda fn=fn: fn(3, [0, 1, 2], offsets=(1, 4, 4, 12)), "offsets[0] is 1"),
                  (lambda fn=fn: fn(3, [0, 1, 2], offsets=(0, 4, 3, 12)), "offsets decrease at session 1"),
                  (lambda fn=fn: fn(3, [0, 1, 2], b=None), "must not be NULL"),
                  (lambda fn=fn: fn(3, [0, 1, 2], e=None), "must not be NULL"),
                  (lambda fn=fn: fn(3, [0, 1, 2], out=None), "out_dist must not be NULL")]
    cases += [(lambda: lib.hsb_group_get_dist(g.g, GEOM[2], full_off.ctypes.data, wb.ctypes.data, we.ctypes.data,
                                              dist.ctypes.data, None, None), "level 3"),
              (lambda: lib.hsb_group_raycast(g.g, 0, None, cb.ctypes.data, ce.ctypes.data, dist.ctypes.data, None),
               "offsets is NULL")]
    counts = [r.launch_count for r in reps]
    for call, text in cases:
        assert call() == -1, text
        assert text in err(), (text, err())
    # K = 0 reads nothing else; Q = 0 (every session empty) needs no rays and no outputs
    assert gd(0, None, level=-5, offsets=None, b=None, e=None, out=None) == 0
    assert rc(0, None, level=-5, offsets=None, b=None, e=None, out=None) == 0
    assert gd(3, [0, 1, 2], offsets=(0, 0, 0, 0), b=None, e=None, out=None) == 0
    assert rc(3, [0, 1, 2], offsets=(0, 0, 0, 0), b=None, e=None, out=None) == 0
    assert [r.launch_count for r in reps] == counts
    assert (dist == SENTINEL).all() and (hit == SENTINEL).all() and (found == SENTINEL).all() and (chit == SENTINEL).all()
    query_round(g, reps, 0, [3, 0, 2], [5, 0, 9], 11)   # still works
    close_all(g, reps)


# ---- 7: the C++ façade --------------------------------------------------------------------------------------------

def test_facade(hsb_lib):
    """hsb200::SlamProcessor::getDistMany (both overloads) and getDist, through their shims, against the C-ABI group
    call on a third set of processors stepped with the same scans: the same bits."""
    L = C.CDLL(os.path.join(ROOT, "hector_slam_b200", "lib", "libhsb200_host.so"))
    vp, i, f = C.c_void_p, C.c_int, C.c_float
    L.hsbp_create.restype = vp
    L.hsbp_create.argtypes = [f, i, i, f, f, i, i]
    L.hsbp_destroy.argtypes = [vp]
    L.hsbp_handle.restype = vp
    L.hsbp_handle.argtypes = [vp]
    L.hsbp_update.argtypes = [vp, vp, i, vp, vp, i, vp, vp]
    L.hsbp_get_dist.argtypes = [vp, i, i, vp, vp, vp, vp, vp]
    L.hsbp_get_dist_many.argtypes = [vp, i, i, vp, vp, vp, vp, vp, vp]
    L.hsbp_get_dist_many_subset.argtypes = [vp, i, vp, i, i, vp, vp, vp, vp, vp, vp]
    lib = hsb_lib

    sx0, sy0, levels, start = GEOM
    M, ticks = 4, 6
    data = [session_data(2600 + s, ticks, geometry(s)) for s in range(M)]
    sets = [[L.hsbp_create(mc.RES, sx0, sy0, start[0], start[1], levels, 0) for _ in range(M)] for _ in range(3)]
    assert all(p for s in sets for p in s)
    many, one, capi_set = sets
    hs = (C.c_void_p * M)(*[L.hsbp_handle(p) for p in capi_set])
    g = C.c_void_p()
    assert lib.hsb_group_create(C.cast(hs, vp), M, C.byref(g)) == 0
    arr = (C.c_void_p * M)(*many)
    rng = np.random.default_rng(8)
    found_any = 0
    for t in range(ticks):
        for s in range(M):
            x = data[s]["scans"][t]
            for st in sets:
                pose, cov = np.zeros(3, np.float32), np.zeros(9, np.float32)
                assert L.hsbp_update(st[s], x.ctypes.data, x.shape[0], None, data[s]["hints"][t].ctypes.data, 0,
                                     pose.ctypes.data, cov.ctypes.data) == 0
        level = t % levels
        members = None if t % 2 == 0 else np.ascontiguousarray(rng.permutation(M)[:int(rng.integers(1, M + 1))], np.int32)
        sel = list(range(M)) if members is None else [int(j) for j in members]
        K = len(sel)
        n = [int(v) for v in rng.integers(0, 30, K)]
        offsets = np.zeros(K + 1, np.int32)
        offsets[1:] = np.cumsum(n)
        Q = int(offsets[-1])
        # robots' surroundings: the rooms of session_data lie within a few metres of the origin
        wb = rng.uniform(-3, 3, (max(Q, 1), 2)).astype(np.float32)
        we = (wb + rng.uniform(-6, 6, wb.shape)).astype(np.float32)
        outs = [[np.zeros(max(Q, 1), np.float32), np.zeros((max(Q, 1), 2), np.float32), np.zeros(max(Q, 1), np.int32)]
                for _ in range(3)]
        ptrs = [[o.ctypes.data for o in out] for out in outs]
        if members is None:
            assert L.hsbp_get_dist_many(C.cast(arr, vp), M, level, offsets.ctypes.data, wb.ctypes.data, we.ctypes.data,
                                        *ptrs[0]) == 0
            assert lib.hsb_group_get_dist(g, level, offsets.ctypes.data, wb.ctypes.data, we.ctypes.data, *ptrs[2]) == 0
        else:
            assert L.hsbp_get_dist_many_subset(C.cast(arr, vp), M, members.ctypes.data, K, level, offsets.ctypes.data,
                                               wb.ctypes.data, we.ctypes.data, *ptrs[0]) == 0
            assert lib.hsb_group_get_dist_subset(g, K, members.ctypes.data, level, offsets.ctypes.data, wb.ctypes.data,
                                                 we.ctypes.data, *ptrs[2]) == 0
        for k, j in enumerate(sel):
            a, b = int(offsets[k]), int(offsets[k + 1])
            assert L.hsbp_get_dist(one[j], level, b - a, wb[a:].ctypes.data, we[a:].ctypes.data,
                                   outs[1][0][a:].ctypes.data, outs[1][1][a:].ctypes.data, outs[1][2][a:].ctypes.data) == 0
        for x, y, z in zip(*outs):
            assert np.array_equal(bits(x[:Q]) if x.dtype != np.int32 else x[:Q],
                                  bits(z[:Q]) if z.dtype != np.int32 else z[:Q]), t
            assert np.array_equal(bits(y[:Q]) if y.dtype != np.int32 else y[:Q],
                                  bits(z[:Q]) if z.dtype != np.int32 else z[:Q]), t
        found_any += int(outs[2][2][:Q].sum())
    assert found_any > 10
    lib.hsb_group_destroy(g)
    for p in many + one + capi_set:
        L.hsbp_destroy(p)
