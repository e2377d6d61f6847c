"""publishMap for a group's members in one pass (hsb_group_sync_occupancy and its _subset form): each listed member's
mirror rectangle of a level gathered (and cleared) with one launch, thresholded with one launch per chunk, copied once
per chunk and scattered into the caller's whole-level grids.

Against a twin fleet that gets the same inputs and publishes with the per-member single calls
(hsb_get_mirror_dirty_rect + hsb_download_occupancy_rect + a row-by-row copy): byte-identical rectangles and grids after
runs of mixed full, subset, nowait and map_without_matching group steps; grids equal to hsb_download_occupancy and to a
numpy threshold of the log-odds; bytes outside the rectangle untouched; the threshold's edge values; reset, upload and
refresh; ordering against nowait steps of this and other groups; unlisted members untouched; chunk boundaries at and
inside rectangles and rectangles larger than a chunk; launch and byte accounting; rejections; the C++ façade.  Maps are
non-square geometries of tests/maptools_cases.GEOMS, every level; every group case runs on a TEX and an LDG group."""
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


def make_rep(geom, s, mode):
    from hector_slam_b200 import capi

    sx, sy, levels, start = geom
    rep = capi.MapRepB200(mc.RES, sx, sy, levels=levels, start=start, update_factor_free=0.4 + 0.02 * (s % 3),
                          update_factor_occupied=0.6 + 0.1 * (s % 4), gather_mode=mode)
    dist, ang = ((0.0, 0.0), (0.15, 0.1), (0.3, 0.5))[s % 3]
    rep.setMapUpdateMinDistDiff(dist)
    rep.setMapUpdateMinAngleDiff(ang)
    rep.set_scan_format(**geometry(s))
    return rep


def twin_fleets(geom, M, mode):
    """(fleet A, group A, fleet B, group B): same configuration member for member"""
    from hector_slam_b200 import capi

    a = [make_rep(geom, s, mode) for s in range(M)]
    b = [make_rep(geom, s, mode) for s in range(M)]
    return a, capi.SlamGroup(a), b, capi.SlamGroup(b)


def new_grids(reps, fill=-1):
    """per level, one whole-level grid per member (-1 everywhere is a fresh map's grid)"""
    out = []
    for l in range(reps[0].levels):
        sx, sy, _ = reps[0].level_info(l)
        out.append([np.full((sy, sx), fill, np.int8) for _ in reps])
    return out


def single_sync(rep, level, grid, reset=True):
    """The per-member path the group call replaces."""
    r = rep.get_mirror_dirty_rect(level, reset=reset)
    if r is not None:
        grid[r[1]:r[3] + 1, r[0]:r[2] + 1] = rep.download_occupancy_rect(level, r)
    return r


def area(r):
    return 0 if r is None else (r[2] - r[0] + 1) * (r[3] - r[1] + 1)


def n_chunks(rects, cap, sx):
    """chunks of whole rows of at most max(cap, sx) bytes, rectangles in session order"""
    cap, used, n = max(cap, sx), 0, 0
    for r in rects:
        if r is None:
            continue
        w = r[2] - r[0] + 1
        for _ in range(r[3] - r[1] + 1):
            if n == 0 or used + w > cap:
                n, used = n + 1, 0
            used += w
    return n


def step_both(ga, gb, data, step, t, members, rng, nowait):
    """one endpoints or ranges group step of `members` (None: all) on both fleets, the same inputs"""
    M = len(data)
    sel = list(range(M)) if members is None else members
    kind = ("endpoints", "ranges")[t % 2]
    without = [bool(rng.random() < 0.2) and step[j] > 0 for j in sel]
    hints = np.asarray([data[j]["truth" if w else "hints"][step[j]] for j, w in zip(sel, without)],
                       np.float32).reshape(len(sel), 3)
    scans = [data[j]["scans" if kind == "endpoints" else "ranges"][step[j]] for j in sel]
    for g in (ga, gb):
        fn = g.slam_update if kind == "endpoints" else g.slam_update_ranges
        fn(hints, scans, map_without_matching=without, nowait=nowait, members=members)
    for j in sel:
        step[j] += 1


def publish_and_compare(ga, a, b, ga_grids, gb_grids, level, members, reset, tag):
    """the group call on fleet A, the single calls on fleet B; rectangles, every grid of the level, the accounting"""
    M = len(a)
    sel = list(range(M)) if members is None else members
    left_out = [j for j in range(M) if j not in sel]
    before_rects = {j: b[j].get_mirror_dirty_rect(level) for j in left_out}
    d2h = [r.d2h_bytes for r in a]
    launches = a[0].launch_count
    got = ga.sync_occupancy(level, [ga_grids[level][j] for j in sel], members=members, reset=reset)
    want = [single_sync(b[j], level, gb_grids[level][j], reset=reset) for j in sel]
    assert got == want, (tag, got, want)
    for j in range(M):
        assert np.array_equal(ga_grids[level][j], gb_grids[level][j]), (tag, j)
    for i, j in enumerate(sel):
        assert a[j].d2h_bytes - d2h[j] == area(got[i]), (tag, j)
    for j in left_out:
        assert a[j].d2h_bytes == d2h[j], (tag, j)
        assert a[j].get_mirror_dirty_rect(level) == before_rects[j] == b[j].get_mirror_dirty_rect(level), (tag, j)
    sx = a[0].level_info(level)[0]
    assert a[0].launch_count - launches == 1 + n_chunks(got, 32 << 20, sx), tag
    return got


@MODES
@pytest.mark.parametrize("geom", SLAM_GEOMS, ids=mc.geom_id)
def test_twin_fleets(hsb_lib, geom, mode):
    """M = 5, 16 ticks of full and subset, sync and nowait, endpoint and range group steps (some sessions
    map_without_matching) on both fleets; a publish after every other tick, full or subset, level by level, reset
    mostly set.  Rectangles and grids equal the twin's byte for byte every time.  At the end a full publish of every
    level: every kept grid equals hsb_download_occupancy and a numpy threshold of download_level."""
    M, ticks = 5, 16
    a, ga, b, gb = twin_fleets(geom, M, mode)
    data = [session_data(1100 + s, ticks, geometry(s)) for s in range(M)]
    rng = np.random.default_rng(23)
    ga_grids, gb_grids = new_grids(a), new_grids(b)
    step = [0] * M
    levels = geom[2]
    for t in range(ticks):
        members = None if t % 4 == 0 else [int(j) for j in rng.permutation(M)[:int(rng.integers(0, M + 1))]]
        step_both(ga, gb, data, step, t, members, rng, nowait=(t % 3 != 0))
        if t % 2 == 1:
            pub = None if t % 8 == 1 else [int(j) for j in rng.permutation(M)[:int(rng.integers(1, M + 1))]]
            publish_and_compare(ga, a, b, ga_grids, gb_grids, (t // 2) % levels, pub, reset=(t % 7 != 5), tag=t)
    for l in range(levels):
        publish_and_compare(ga, a, b, ga_grids, gb_grids, l, None, True, ("end", l))
        for j in range(M):
            assert np.array_equal(ga_grids[l][j], a[j].download_occupancy(l)), (l, j)
            assert np.array_equal(ga_grids[l][j], mc.occupancy(a[j].download_level(l))), (l, j)
    for x in (ga, gb, *a, *b):
        x.close()


@MODES
def test_untouched_bytes_and_clean_members(hsb_lib, mode):
    """Sentinel grids: only the cells of each rectangle are written; a member whose map did not change gets no
    rectangle and its grid is not touched; a second call finds nothing."""
    M = 4
    a, ga, b, gb = twin_fleets(GEOM, M, mode)
    data = [session_data(1200 + s, 2, geometry(s)) for s in range(M)]
    step = [0] * M
    step_both(ga, gb, data, step, 0, [1, 3], np.random.default_rng(1), nowait=True)
    for l in range(GEOM[2]):
        grids = new_grids(a, SENTINEL)[l]
        rects = ga.sync_occupancy(l, grids)
        assert rects[0] is None and rects[2] is None and rects[1] is not None and rects[3] is not None, rects
        for j in range(M):
            r = rects[j]
            outside = np.ones(grids[j].shape, bool)
            if r is not None:
                outside[r[1]:r[3] + 1, r[0]:r[2] + 1] = False
                assert np.array_equal(grids[j][~outside].reshape(r[3] - r[1] + 1, -1),
                                      b[j].download_occupancy_rect(l, r)), (l, j)
            assert (grids[j][outside] == SENTINEL).all(), (l, j)
        again = [g.copy() for g in grids]
        assert ga.sync_occupancy(l, again) == [None] * M
        assert all(np.array_equal(x, y) for x, y in zip(again, grids)), l
    for x in (ga, gb, *a, *b):
        x.close()


@MODES
@pytest.mark.parametrize("geom", mc.GEOMS, ids=mc.geom_id)
def test_threshold_edge_values(hsb_lib, geom, mode):
    """Planes carrying -0, +0, the smallest denormals, +-inf, NaN and 50 at the corners, along the last row and column
    and at random cells, planted by hsb_upload_level on every level: the synced grid equals the whole-level export
    (hsb_download_occupancy) and the numpy threshold."""
    from hector_slam_b200 import capi

    reps = [make_rep(geom, s, mode) for s in range(2)]
    g = capi.SlamGroup(reps)
    for l in range(geom[2]):
        sx, sy, _ = reps[0].level_info(l)
        planes = [mc.plane(sx, sy, 31 * l + s) for s in range(2)]
        for rep, p in zip(reps, planes):
            rep.upload_level(l, p)
        grids = [np.full((sy, sx), SENTINEL, np.int8) for _ in reps]
        assert g.sync_occupancy(l, grids, members=[1, 0])[::-1] == [(0, 0, sx - 1, sy - 1)] * 2
        for rep, p, grid in zip(reps, planes, grids[::-1]):
            assert np.array_equal(grid, rep.download_occupancy(l)), l
            assert np.array_equal(grid, mc.occupancy(p)), l
    g.close()
    for r in reps:
        r.close()


@MODES
def test_reset_upload_refresh(hsb_lib, mode):
    """reset = 0 returns the same rectangle again and clears nothing; reset = 1 clears it.  hsb_reset, hsb_upload_level
    and hsb_refresh_level each make the level's rectangle the whole level."""
    import torch

    M = 3
    a, ga, b, gb = twin_fleets(GEOM, M, mode)
    data = [session_data(1300 + s, 2, geometry(s)) for s in range(M)]
    ga_grids, gb_grids = new_grids(a), new_grids(b)
    step_both(ga, gb, data, [0] * M, 0, None, np.random.default_rng(2), nowait=False)
    for l in range(GEOM[2]):
        first = publish_and_compare(ga, a, b, ga_grids, gb_grids, l, None, False, ("keep", l))
        assert all(r is not None for r in first)
        assert publish_and_compare(ga, a, b, ga_grids, gb_grids, l, None, True, ("reset", l)) == first
        assert publish_and_compare(ga, a, b, ga_grids, gb_grids, l, None, True, ("clean", l)) == [None] * M
    sizes = [a[0].level_info(l)[:2] for l in range(GEOM[2])]
    a[0].reset()
    b[0].reset()
    plane = mc.plane(*sizes[1], 7)
    a[1].upload_level(1, plane)
    b[1].upload_level(1, plane)
    a[2].refresh_level(0)
    b[2].refresh_level(0)
    torch.cuda.synchronize()   # the refresh ran on the legacy default stream
    for l in range(GEOM[2]):
        whole = (0, 0, sizes[l][0] - 1, sizes[l][1] - 1)
        got = publish_and_compare(ga, a, b, ga_grids, gb_grids, l, None, True, ("whole", l))
        assert got[0] == whole and (got[1] == whole) == (l == 1) and (got[2] == whole) == (l == 0), (l, got)
        for j in range(M):
            assert np.array_equal(ga_grids[l][j], a[j].download_occupancy(l)), (l, j)
    for x in (ga, gb, *a, *b):
        x.close()


@MODES
def test_ordering(hsb_lib, mode):
    """(1) A publish right after a nowait group step sees that step's write.  (2) publish(reset) -> a single nowait step
    on member j -> a subset group step including j -> publish: equal to the twin, no write lost.  (3) A member that
    also belongs to a second group, stepped nowait through that group and published through this one."""
    from hector_slam_b200 import capi

    M = 4
    a, ga, b, gb = twin_fleets(GEOM, M, mode)
    solo_a, solo_b = capi.SlamGroup([a[3]]), capi.SlamGroup([b[3]])
    ticks = 8
    data = [session_data(1400 + s, 2 * ticks, geometry(s)) for s in range(M)]
    ga_grids, gb_grids = new_grids(a), new_grids(b)
    rng = np.random.default_rng(3)
    step = [0] * M
    for t in range(0, ticks, 2):
        step_both(ga, gb, data, step, t, None, rng, nowait=True)   # (1)
        publish_and_compare(ga, a, b, ga_grids, gb_grids, 0, None, True, ("after nowait", t))
        j = t % M
        for rep in (a[j], b[j]):   # (2)
            rep.slam_update(data[j]["hints"][step[j]], data[j]["scans"][step[j]], nowait=True)
        step[j] += 1
        others = [j] + [s for s in range(M) if s != j][:2]
        step_both(ga, gb, data, step, t + 1, others, rng, nowait=True)
        publish_and_compare(ga, a, b, ga_grids, gb_grids, 0, [j, (j + 1) % M], True, ("single then subset", t))
        publish_and_compare(ga, a, b, ga_grids, gb_grids, 0, None, True, ("rest", t))
        k = step[3]   # (3)
        for g in (solo_a, solo_b):
            g.slam_update(data[3]["hints"][k][None], [data[3]["scans"][k]], nowait=True)
        step[3] += 1
        publish_and_compare(ga, a, b, ga_grids, gb_grids, 0, [3, 1], True, ("other group", t))
    for l in range(GEOM[2]):
        publish_and_compare(ga, a, b, ga_grids, gb_grids, l, None, True, ("end", l))
        for j in range(M):
            assert np.array_equal(ga_grids[l][j], a[j].download_occupancy(l)), (l, j)
    for x in (solo_a, solo_b, ga, gb, *a, *b):
        x.close()


@MODES
def test_chunking(hsb_lib, mode):
    """The same rectangles (reset = 0) through staging capacities that end a chunk exactly at the end of a rectangle,
    inside one, and below one rectangle's size (the level's width, the least a chunk holds): the same bytes as the twin
    every time, one launch per chunk plus the gather."""
    M = 4
    a, ga, b, gb = twin_fleets(GEOM, M, mode)
    data = [session_data(1500 + s, 3, geometry(s)) for s in range(M)]
    step = [0] * M
    rng = np.random.default_rng(4)
    for t in range(3):
        step_both(ga, gb, data, step, t, None, rng, nowait=(t == 2))
    for l in range(GEOM[2]):
        sx = a[0].level_info(l)[0]
        rects = [b[j].get_mirror_dirty_rect(l) for j in range(M)]
        assert all(r is not None for r in rects), rects
        w1 = rects[1][2] - rects[1][0] + 1
        caps = {"end of a rectangle": area(rects[0]), "inside a rectangle": area(rects[0]) + 3 * w1,
                "below one rectangle": 1}
        assert caps["end of a rectangle"] >= sx and 3 < rects[1][3] - rects[1][1] + 1
        for name, cap in caps.items():
            a[0].set_tuning(occupancy_chunk=cap)
            ga_grids, gb_grids = new_grids(a, SENTINEL), new_grids(b, SENTINEL)
            launches = a[0].launch_count
            got = ga.sync_occupancy(l, ga_grids[l], reset=False)
            want = [single_sync(b[j], l, gb_grids[l][j], reset=False) for j in range(M)]
            assert got == want == rects, (l, name)
            assert all(np.array_equal(x, y) for x, y in zip(ga_grids[l], gb_grids[l])), (l, name)
            chunks = n_chunks(got, cap, sx)
            assert chunks > 1 and a[0].launch_count - launches == 1 + chunks, (l, name, chunks)
        a[0].set_tuning(occupancy_chunk=0)
    for x in (ga, gb, *a, *b):
        x.close()


def test_level_larger_than_one_chunk(hsb_lib):
    """An 8192^2 level is 64 MiB of cells: after an upload its whole-level rectangle goes in two chunks of the default
    32 MiB staging."""
    from hector_slam_b200 import capi

    n = 8192
    rep = capi.MapRepB200(mc.RES, n, n, levels=1)
    g = capi.SlamGroup([rep])
    rng = np.random.default_rng(5)
    p = rng.standard_normal((n, n), dtype=np.float32)
    p[0, 0], p[-1, -1], p[n // 2, 7], p[-1, 0] = 0.0, np.nan, -0.0, mc.MIN_DENORMAL
    rep.upload_level(0, p)
    grid = np.full((n, n), SENTINEL, np.int8)
    launches = rep.launch_count
    assert g.sync_occupancy(0, [grid]) == [(0, 0, n - 1, n - 1)]
    assert rep.launch_count - launches == 3
    assert np.array_equal(grid, rep.download_occupancy(0))
    assert np.array_equal(grid, mc.occupancy(p))
    g.close()
    rep.close()


@MODES
def test_rejections(hsb_lib, mode):
    """Every rejection: HSB_ERR_INVALID_ARG with a message, nothing launched, no rectangle cleared, no grid written.
    K = 0 queues nothing."""
    M = 4
    a, ga, b, gb = twin_fleets(GEOM, M, mode)
    data = [session_data(1600 + s, 1, geometry(s)) for s in range(M)]
    step_both(ga, gb, data, [0] * M, 0, None, np.random.default_rng(6), nowait=True)
    lib = ga.lib
    sx, sy, _ = a[0].level_info(0)
    grids = [np.full((sy, sx), SENTINEL, np.int8) for _ in range(M)]
    rects_before = [[r.get_mirror_dirty_rect(l) for l in range(GEOM[2])] for r in a]
    launches = a[0].launch_count
    ptrs = (C.c_void_p * M)(*[g.ctypes.data for g in grids])
    out = np.zeros((M, 4), np.int32)

    def raw(K, members, level=0, grid_ptrs=ptrs):
        m = None if members is None else np.ascontiguousarray(members, np.int32)
        return lib.hsb_group_sync_occupancy_subset(ga.g, K, None if m is None else m.ctypes.data, level,
                                                   None if grid_ptrs is None else C.cast(grid_ptrs, C.c_void_p),
                                                   out.ctypes.data, 1)

    def err():
        return (lib.hsb_last_error(a[0].h) or b"").decode()

    with_null = (C.c_void_p * M)(*[g.ctypes.data for g in grids])
    with_null[2] = None
    cases = ((lambda: raw(-1, [0]), "K is -1"), (lambda: raw(M + 1, [0, 1, 2, 3, 0]), "K is 5"),
             (lambda: raw(2, None), "members is NULL"), (lambda: raw(2, [0, M]), "session 1: member 4"),
             (lambda: raw(2, [-1, 0]), "session 0: member -1"), (lambda: raw(3, [1, 3, 1]), "listed twice"),
             (lambda: raw(2, [0, 1], level=-1), "level -1"), (lambda: raw(2, [0, 1], level=GEOM[2]), "level 3"),
             (lambda: raw(2, [0, 1], grid_ptrs=None), "grids is NULL"),
             (lambda: raw(M, [0, 1, 2, 3], grid_ptrs=with_null), "session 2: grid is NULL"),
             (lambda: lib.hsb_group_sync_occupancy(ga.g, GEOM[2], C.cast(ptrs, C.c_void_p), None, 1), "level 3"),
             (lambda: lib.hsb_group_sync_occupancy(ga.g, 0, None, None, 1), "grids is NULL"))
    for call, text in cases:
        assert call() == -1, text
        assert text in err(), (text, err())
    assert raw(0, None, grid_ptrs=None) == 0
    assert a[0].launch_count == launches
    assert all((g == SENTINEL).all() for g in grids)
    assert [[r.get_mirror_dirty_rect(l) for l in range(GEOM[2])] for r in a] == rects_before
    ga_grids, gb_grids = new_grids(a), new_grids(b)   # still works, still equal to the twin
    for l in range(GEOM[2]):
        publish_and_compare(ga, a, b, ga_grids, gb_grids, l, None, True, ("after", l))
    for x in (ga, gb, *a, *b):
        x.close()


def test_facade(hsb_lib):
    """hsb200::SlamProcessor::syncOccupancyMany (both overloads) and syncOccupancy, through their shims, against the
    C-ABI group call on a third set of processors stepped with the same scans: the same rectangles and grids."""
    L = C.CDLL(os.path.join(ROOT, "hector_slam_b200", "lib", "libhsb200_host.so"))
    vp, i, f = C.c_void_p, C.c_int, C.c_float
    L.hsbp_create.restype = vp
    L.hsbp_create.argtypes = [f, i, i, f, f, i, i]
    L.hsbp_destroy.argtypes = [vp]
    L.hsbp_handle.restype = vp
    L.hsbp_handle.argtypes = [vp]
    L.hsbp_update.argtypes = [vp, vp, i, vp, vp, i, vp, vp]
    L.hsbp_sync_occupancy.argtypes = [vp, i, vp, vp]
    L.hsbp_sync_occupancy_many.argtypes = [vp, i, i, vp, vp]
    L.hsbp_sync_occupancy_many_subset.argtypes = [vp, i, vp, i, i, vp, vp]
    lib = hsb_lib

    sx0, sy0, levels, start = GEOM
    M, ticks = 4, 6
    data = [session_data(1700 + s, ticks, geometry(s)) for s in range(M)]
    sets = [[L.hsbp_create(mc.RES, sx0, sy0, start[0], start[1], levels, 0) for _ in range(M)] for _ in range(3)]
    assert all(p for s in sets for p in s)
    many, one, capi_set = sets
    hs = (C.c_void_p * M)(*[L.hsbp_handle(p) for p in capi_set])
    g = C.c_void_p()
    assert lib.hsb_group_create(C.cast(hs, vp), M, C.byref(g)) == 0
    grids = [[[np.full(((sy0 >> l), (sx0 >> l)), -1, np.int8) for _ in range(M)] for l in range(levels)] for _ in sets]
    arr = (C.c_void_p * M)(*many)
    rng = np.random.default_rng(8)
    for t in range(ticks):
        for s in range(M):
            if t % 3 == 2 and s % 2:
                continue
            x = data[s]["scans"][t]
            for st in sets:
                pose, cov = np.zeros(3, np.float32), np.zeros(9, np.float32)
                assert L.hsbp_update(st[s], x.ctypes.data, x.shape[0], None, data[s]["hints"][t].ctypes.data, 0,
                                     pose.ctypes.data, cov.ctypes.data) == 0
        level = t % levels
        members = None if t % 2 == 0 else np.ascontiguousarray(rng.permutation(M)[:int(rng.integers(1, M + 1))], np.int32)
        sel = list(range(M)) if members is None else [int(j) for j in members]
        K = len(sel)
        r_many, r_capi = np.zeros((K, 4), np.int32), np.zeros((K, 4), np.int32)
        p_many = (C.c_void_p * K)(*[grids[0][level][j].ctypes.data for j in sel])
        p_capi = (C.c_void_p * K)(*[grids[2][level][j].ctypes.data for j in sel])
        if members is None:
            assert L.hsbp_sync_occupancy_many(C.cast(arr, vp), M, level, C.cast(p_many, vp), r_many.ctypes.data) == 0
            assert lib.hsb_group_sync_occupancy(g, level, C.cast(p_capi, vp), r_capi.ctypes.data, 1) == 0
        else:
            assert L.hsbp_sync_occupancy_many_subset(C.cast(arr, vp), M, members.ctypes.data, K, level,
                                                     C.cast(p_many, vp), r_many.ctypes.data) == 0
            assert lib.hsb_group_sync_occupancy_subset(g, K, members.ctypes.data, level, C.cast(p_capi, vp),
                                                       r_capi.ctypes.data, 1) == 0
        r_one = np.zeros((K, 4), np.int32)
        for n, j in enumerate(sel):
            assert L.hsbp_sync_occupancy(one[j], level, grids[1][level][j].ctypes.data, r_one[n].ctypes.data) == 0
        assert np.array_equal(r_many, r_capi) and np.array_equal(r_one, r_capi), t
        for j in range(M):
            assert np.array_equal(grids[0][level][j], grids[2][level][j]), (t, j)
            assert np.array_equal(grids[1][level][j], grids[2][level][j]), (t, j)
    lib.hsb_group_destroy(g)
    for p in many + one + capi_set:
        L.hsbp_destroy(p)
