"""GPU: the kernels that read whole cells out of a level plane or move cells between planes, held bit for bit on
non-square levels, long rays and plane edges, in both gather modes (LDG and TEX handles).

  N1  occupancy export and rectangle downloads (occupancy_rect_kernel, hsb_download_level_rect) against a numpy
      publishMap threshold of the uploaded plane, with -0, +0, +-min denormal, +-inf, NaN and 50 planted;
  N4  ray cast and getDist (warp_raycast, ray_kernel) against HectorMapTools.h compiled unmodified (oracle/_ref; the C
      port where it is absent) on the rays of tests/maptools_cases.py, and right after a nowait SLAM step;
  N3  hsb_likelihood_batch and hsb_covariance_batch right after a nowait SLAM step, their launch count, and a negative
      shared scan length;
  §6  tile replication between an owner and a replica on one device, both protocols (pack_rect / unpack_rect and
      pack_dirty / reset_dirty / unpack_dirty): log-odds, probabilities, texture twin, mirror and replication
      rectangles, the buffer header and the overflow boundary;
      hsb_refresh_level after a plane written from a caller's stream.
Every comparison is of bit patterns."""
import functools

import numpy as np
import pytest

import maptools_cases as mc
from oracle import mapwrite as mw
from twin_probe import probe_twin

pytestmark = pytest.mark.gpu

LDG, TEX = 1, 2
MODES = pytest.mark.parametrize("mode", [LDG, TEX], ids=["ldg", "tex"])
HEADER_WORDS, MAGIC = 64, 0x48534254   # HSB_TILE_HEADER_WORDS, HSB_TILE_MAGIC (hsb_internal.h)
INT_MAX = 2 ** 31 - 1
HSB_ERR_INVALID_ARG = -1


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def same(a, b):
    return np.array_equal(bits(a), bits(b))


def handle(geom, mode, **kw):
    from hector_slam_b200 import capi

    sx, sy, levels, start = geom
    rep = capi.MapRepB200(mc.RES, sx, sy, levels=levels, start=start, gather_mode=mode, **kw)
    assert rep.gather_mode == mode
    return rep


# ---- N1 ------------------------------------------------------------------------------------------------------------

def rects_for(sx, sy):
    """The four corners as single cells, the last row, the last column, the whole level, a 1 x n and an n x 1 strip."""
    n = max(1, min(sx, sy) // 2)
    return [(0, 0, 0, 0), (sx - 1, 0, sx - 1, 0), (0, sy - 1, 0, sy - 1), (sx - 1, sy - 1, sx - 1, sy - 1),
            (0, sy - 1, sx - 1, sy - 1), (sx - 1, 0, sx - 1, sy - 1), (0, 0, sx - 1, sy - 1),
            (sx // 3, sy // 2, sx // 3 + n - 1, sy // 2), (sx // 2, sy // 3, sx // 2, sy // 3 + n - 1)]


@MODES
@pytest.mark.parametrize("geom", mc.GEOMS, ids=mc.geom_id)
def test_occupancy_export_and_rect_downloads(hsb_lib, geom, mode):
    from hector_slam_b200 import capi

    rep = handle(geom, mode)
    planes = [mc.plane(lx, ly, seed=17 * lx + ly + l) for l, (lx, ly) in enumerate(mc.level_sizes(geom))]
    for l, p in enumerate(planes):
        rep.upload_level(l, p)
    for l, p in enumerate(planes):
        sx, sy = p.shape[1], p.shape[0]
        occ = rep.download_occupancy(l)
        assert occ.dtype == np.int8 and np.array_equal(occ, mc.occupancy(p)), (geom, l)
        full = rep.download_level(l)
        assert same(full, p)
        for r in rects_for(sx, sy):
            x0, y0, x1, y1 = r
            n = (x1 - x0 + 1) * (y1 - y0 + 1)
            b0 = rep.d2h_bytes
            win = rep.download_level_rect(l, r)
            b1 = rep.d2h_bytes
            owin = rep.download_occupancy_rect(l, r)
            b2 = rep.d2h_bytes
            assert same(win, full[y0:y1 + 1, x0:x1 + 1]), (geom, l, r)
            assert np.array_equal(owin, occ[y0:y1 + 1, x0:x1 + 1]), (geom, l, r)
            assert (b1 - b0, b2 - b1) == (4 * n, n), (geom, l, r)
        if sx != sy:   # valid only for the transposed geometry: rejected before any copy
            for r in [(sy - 1, sx - 1, sy - 1, sx - 1), (0, 0, sy - 1, sx - 1)]:
                b0 = rep.d2h_bytes
                for fn in (rep.download_level_rect, rep.download_occupancy_rect):
                    with pytest.raises(capi.HsbError) as e:
                        fn(l, r)
                    assert e.value.status == HSB_ERR_INVALID_ARG
                assert rep.d2h_bytes == b0
    rep.close()


# ---- N4 ------------------------------------------------------------------------------------------------------------

@functools.lru_cache(maxsize=None)
def expected_rays(geom):
    """Per level: (plane, cell rays, their expected (dist, hit), world rays, their expected (dist, hit_world, found),
    NaN mask, origin) from the compiled header over the numpy-thresholded plane, or the C port without oracle/_ref."""
    from oracle import pyoracle

    sx, sy, levels, start = geom
    port = pyoracle.Oracle("port", mc.RES, sx, levels, start=start, size_y=sy)
    have_ref = pyoracle.available("reference")
    out = []
    for l, (lx, ly) in enumerate(mc.level_sizes(geom)):
        cell = port.cell_length(l)
        origin = port.map_origin(l)
        p = mc.plane(lx, ly, seed=lx * 31 + ly + l)
        port.set_logodds(l, p)
        mt = pyoracle.RefMapTools(mc.occupancy(p), cell, origin) if have_ref else None
        begin, end = mc.cell_rays(lx, ly, mc.occupancy(p), seed=lx + 7 * ly)
        cast = [mt.raycast(b, e) if mt else port.raycast(l, b, e) for b, e in zip(begin, end)]
        dist = np.float32([c[0] for c in cast])
        hit = np.int32([c[1] for c in cast])
        bw, ew, is_nan = mc.world_rays(lx, ly, origin, cell, seed=lx + 3 * ly)
        gd = [(-1.0, np.zeros(2, np.float32), False) if nan else (mt.get_dist(b, e) if mt else port.get_dist(l, b, e))
              for b, e, nan in zip(bw, ew, is_nan)]
        gdist = np.float32([g[0] for g in gd])
        gdist[is_nan] = np.float32(-cell)
        ghit = np.float32([g[1] for g in gd])
        gfound = np.array([g[2] for g in gd])
        out.append((p, begin, end, dist, hit, bw, ew, gdist, ghit, gfound, origin))
        if mt:
            mt.close()
    port.close()
    return out


@MODES
@pytest.mark.parametrize("geom", mc.GEOMS, ids=mc.geom_id)
def test_raycast_and_get_dist(hsb_lib, geom, mode):
    rep = handle(geom, mode)
    exp = expected_rays(geom)
    for l, (p, begin, end, dist, hit, bw, ew, gdist, ghit, gfound, origin) in enumerate(exp):
        rep.upload_level(l, p)
        assert same(rep.map_origin(l), origin), (geom, l)
        d, h = rep.raycast_batch(l, begin, end)
        bad = (bits(d) != bits(dist)) | np.any(h != hit, axis=1)
        assert not bad.any(), (geom, l, int(bad.sum()), begin[bad][:3], end[bad][:3], d[bad][:3], dist[bad][:3])
        assert (dist >= 0).sum() > 200 and (dist == 0).sum() >= 8
        gd, gh, gf = rep.get_dist_batch(l, bw, ew)
        assert same(gd, gdist) and np.array_equal(gf, gfound), (geom, l, np.argwhere(bits(gd) != bits(gdist))[:5])
        assert same(gh[gf], ghit[gf]) and not gh[~gf].any()
        assert gf.sum() > 100
    rep.close()


@MODES
@pytest.mark.parametrize("geom", mc.LONG, ids=mc.geom_id)
def test_constructed_long_rays(hsb_lib, geom, mode):
    """The rays of tests/test_oracle_maptools.py's constructed cases, one occupied cell per ray: the 5000-step cap,
    the end cell, and hit offsets next to a perfect square in all four mirrors."""
    from oracle import pyoracle

    sx, sy, _, start = geom
    rep = handle(geom, mode)
    port = pyoracle.Oracle("port", mc.RES, sx, 1, start=start, size_y=sy)
    have_ref = pyoracle.available("reference")
    for k, c in enumerate(mc.lone_cases(sx, sy)):
        p = mc.lone_plane(sx, sy, c.cell, seed=k)
        rep.upload_level(0, p)
        d, h = rep.raycast_batch(0, np.int32([c.begin]), np.int32([c.end]))
        if have_ref:
            mt = pyoracle.RefMapTools(mc.occupancy(p), port.cell_length(0), port.map_origin(0))
            want = mt.raycast(c.begin, c.end)
            mt.close()
        else:
            port.set_logodds(0, p)
            want = port.raycast(0, c.begin, c.end)
        assert want == ((float(c.dist), c.cell) if c.hit else (-1.0, (-1, -1))), (c, want)   # the construction holds
        assert (float(d[0]), tuple(int(v) for v in h[0])) == want, (c, d[0], h[0])
    port.close()
    rep.close()


@MODES
@pytest.mark.parametrize("kind", ["endpoints", "ranges"])
def test_rays_right_after_a_nowait_step(hsb_lib, mode, kind):
    """hsb_get_dist_batch and hsb_raycast_batch issued right after a nowait SLAM step see the step's map write and leave
    the step's input alone (the scan and the rays go through the handle's one pinned staging): the rays, the poses and
    every level's plane equal those of a twin stepped synchronously.  The rays start around the robot."""
    from hector_slam_b200 import capi
    from test_gpu_group_subset import geometry, session_data

    fmt = geometry(0)
    ticks = 8
    data = session_data(40 + mode, ticks, fmt)
    twins = [capi.MapRepB200(0.05, 512, 512, levels=3, update_factor_free=0.4, update_factor_occupied=0.9,
                             gather_mode=mode) for _ in range(2)]
    for rep in twins:
        rep.set_scan_format(**fmt)
    rng = np.random.default_rng(7 + mode)
    ang = np.linspace(-np.pi, np.pi, 48, endpoint=False, dtype=np.float32)
    for t in range(ticks):
        level = t % 3
        sx, sy, _ = twins[0].level_info(level)
        p = data["truth"][t]
        wb = np.repeat(p[None, :2], ang.size, axis=0).astype(np.float32)
        we = (wb + np.float32(5.0) * np.stack([np.cos(ang), np.sin(ang)], axis=1)).astype(np.float32)
        cb = np.int32([sx // 2, sy // 2]) + rng.integers(-(sx // 5), sx // 5 + 1, (64, 2)).astype(np.int32)
        ce = np.stack([rng.integers(0, sx, 64), rng.integers(0, sy, 64)], axis=1).astype(np.int32)
        out = []
        for rep, nowait in zip(twins, (True, False)):
            if kind == "endpoints":
                pose = rep.slam_update(data["hints"][t], data["scans"][t], nowait=nowait)[0]
            else:
                pose = rep.slam_update_ranges(data["hints"][t], data["ranges"][t], nowait=nowait)[0]
            out.append((pose,) + rep.get_dist_batch(level, wb, we) + rep.raycast_batch(level, cb, ce))
        for i, (x, y) in enumerate(zip(*out)):
            assert np.array_equal(bits(x) if x.dtype == np.float32 else x, bits(y) if y.dtype == np.float32 else y), (t, i)
        assert out[0][3].sum() > 0, t   # some world ray hits a wall
    for l in range(3):
        assert same(twins[0].download_level(l), twins[1].download_level(l)), l
    for rep in twins:
        rep.close()


# ---- N3 ------------------------------------------------------------------------------------------------------------

@MODES
@pytest.mark.parametrize("kind", ["endpoints", "ranges"])
def test_scores_right_after_a_nowait_step(hsb_lib, mode, kind):
    """hsb_likelihood_batch and hsb_covariance_batch issued right after a nowait SLAM step see the step's map write and
    leave the step's input alone (the scan and the poses go through the handle's one pinned staging), with one shared
    scan and with per-pose offsets: the likelihoods, both covariance matrices, the poses and every level's plane equal
    those of a twin stepped synchronously.  The poses lie around the robot and are scored against the step's scan."""
    from hector_slam_b200 import capi
    from test_gpu_group_subset import geometry, session_data

    fmt = geometry(1)
    ticks = 8
    data = session_data(50 + mode, ticks, fmt)
    twins = [capi.MapRepB200(0.05, 512, 512, levels=3, update_factor_free=0.4, update_factor_occupied=0.9,
                             gather_mode=mode) for _ in range(2)]
    for rep in twins:
        rep.set_scan_format(**fmt)
    rng = np.random.default_rng(11 + mode)
    for t in range(ticks):
        level = t % 3
        scan = data["scans"][t]
        poses = (data["truth"][t] + rng.uniform(-1, 1, (6, 3)) * np.float32([0.1, 0.1, 0.05])).astype(np.float32)
        offsets = np.int32([0] + sorted(rng.integers(0, scan.shape[0] + 1, 5)) + [scan.shape[0]])
        out = []
        for rep, nowait in zip(twins, (True, False)):
            if kind == "endpoints":
                pose = rep.slam_update(data["hints"][t], scan, nowait=nowait)[0]
            else:
                pose = rep.slam_update_ranges(data["hints"][t], data["ranges"][t], nowait=nowait)[0]
            out.append((pose, rep.likelihood_batch(level, poses, scan), rep.likelihood_batch(level, poses, scan, offsets))
                       + rep.covariance_batch(level, poses, scan) + rep.covariance_batch(level, poses, scan, offsets))
        for i, (x, y) in enumerate(zip(*out)):
            assert same(x, y), (t, i)
        assert np.isfinite(out[0][1]).all(), t
    for l in range(3):
        assert same(twins[0].download_level(l), twins[1].download_level(l)), l
    for rep in twins:
        rep.close()


def score_handle(mode):
    """A 1-level 256^2 handle at resolution 0.25 from (0, 0), so that world = map cells x 0.25 exactly, and B = 5 map
    poses with their world twins."""
    from hector_slam_b200 import capi

    rep = capi.MapRepB200(0.25, 256, 256, levels=1, start=(0.0, 0.0), gather_mode=mode)
    rep.upload_level(0, mc.plane(256, 256, seed=3))
    rng = np.random.default_rng(5 + mode)
    pm = np.stack([rng.uniform(60, 200, 5), rng.uniform(60, 200, 5), rng.uniform(-3.1, 3.1, 5)], axis=1).astype(np.float32)
    return rep, pm, (pm * np.float32([0.25, 0.25, 1.0])).astype(np.float32)


@MODES
def test_score_launch_count(hsb_lib, mode):
    """Each hsb_likelihood_batch and hsb_covariance_batch call is one launch, in either scan layout."""
    rep, _, world = score_handle(mode)
    pts = np.random.default_rng(1).uniform(-40, 40, (300, 2)).astype(np.float32)
    offsets = np.int32([0, 0, 1, 100, 299, 300])
    calls = [lambda: rep.likelihood_batch(0, world, pts), lambda: rep.likelihood_batch(0, world, pts, offsets),
             lambda: rep.covariance_batch(0, world, pts), lambda: rep.covariance_batch(0, world, pts, offsets)]
    for i, call in enumerate(calls):
        n = rep.launch_count
        call()
        assert rep.launch_count == n + 1, i
    rep.close()


@MODES
def test_negative_shared_scan_length(hsb_lib, mode):
    """A negative n_shared with offsets NULL, through the C-ABI: no points are read, the likelihood's scan length is 0
    (1 - 0/0: NaN for every pose) and the covariance's is n_shared itself (each sigma point 1 - 0/n_shared = 1), so the
    covariance is oracle/likelihood64.py's fp32 formula on seven likelihoods of 1.0."""
    from oracle import likelihood64

    rep, pm, world = score_handle(mode)
    B = world.shape[0]
    lh = np.zeros(B, np.float32)
    assert hsb_lib.hsb_likelihood_batch(rep.h, 0, B, world.ctypes.data, None, None, -1, lh.ctypes.data) == 0
    assert np.isnan(lh).all(), lh
    cm, cw = np.zeros((B, 9), np.float32), np.zeros((B, 9), np.float32)
    assert hsb_lib.hsb_covariance_batch(rep.h, 0, B, world.ctypes.data, None, None, -1, cm.ctypes.data,
                                        cw.ctypes.data) == 0
    assert np.isfinite(cm).all() and np.isfinite(cw).all()
    for b in range(B):
        wm, ww = likelihood64.covariance_fp32(np.ones(7, np.float32), pm[b], 0.25)
        assert same(cm[b], wm.reshape(9)) and same(cw[b], ww.reshape(9)), (b, cm[b], wm, cw[b], ww)
    rep.close()


# ---- §6 -----------------------------------------------------------------------------------------------------------

REPL_MAPS = [(404, 300, 3, (0.5, 0.5)), (257, 131, 2, (0.3, 0.7))]


def union(rects):
    out = None
    for r in rects:
        out = mw.union(out, r)
    return out


class Replication:
    """An owner and a replica of one geometry in one gather mode, the replica's shipped rectangles since its last
    mirror reset, and the planes the replica must hold."""

    def __init__(self, geom, mode, seed):
        import torch

        self.geom = geom
        self.owner = handle(geom, mode, update_factor_free=0.4, update_factor_occupied=0.9)
        self.replica = handle(geom, mode, update_factor_free=0.4, update_factor_occupied=0.9)
        self.levels = geom[2]
        self.lv = mw.geometry(mc.RES, geom[0], geom[1], geom[2], geom[3])
        self.rng = np.random.default_rng(seed)
        for l, L in enumerate(self.lv):
            p = mw.preload((L.sy, L.sx), self.rng)
            self.owner.upload_level(l, p)
            self.replica.upload_level(l, p)
        for rep in (self.owner, self.replica):
            rep.get_dirty_rects(reset=True)
            for l in range(self.levels):
                rep.get_mirror_dirty_rect(l, reset=True)
        self.shipped = [[] for _ in range(self.levels)]
        self.want = [self.replica.download_level(l) for l in range(self.levels)]
        self.cap_max = 4 * (HEADER_WORDS + sum(L.sx * L.sy for L in self.lv)) + 8
        self.buf = torch.zeros(self.cap_max // 4 + 1, dtype=torch.float32, device="cuda")
        self.stream = torch.cuda.current_stream().cuda_stream

    def write(self, levels, k):
        """hsb_update_level_by_scan on `levels` of the owner: a scan family around a point of each level."""
        for l in levels:
            L = self.lv[l]
            c = (L.sx // 3 + 7 * k) % L.sx, (L.sy // 2 + 5 * k) % L.sy
            pose = mw.pose_for_cell(L, c[0], c[1], 0.3 * k)
            pts = mw.points_for_targets(L, pose, mw.family_targets(L, c, self.rng, 16))
            self.owner.update_level_by_scan(l, pts, pose)

    def cells(self, rects):
        return sum(0 if r is None else (r[2] - r[0] + 1) * (r[3] - r[1] + 1) for r in rects)

    def header(self):
        import torch

        return self.buf[:HEADER_WORDS].view(torch.int32).cpu().numpy()

    def pack_unpack(self, capacity, reset):
        """One-shot transport; returns the owner's rectangles before the pack."""
        rects = self.owner.get_dirty_rects()
        self.owner.pack_dirty_device(self.buf.data_ptr(), capacity, reset, self.stream)
        self.replica.unpack_dirty_device(self.buf.data_ptr(), capacity, self.stream)
        return rects

    def shipped_from_owner(self, rects):
        owner = [self.owner.download_level(l) for l in range(self.levels)]
        for l, r in enumerate(rects):
            if r is not None:
                x0, y0, x1, y1 = r
                self.want[l][y0:y1 + 1, x0:x1 + 1] = owner[l][y0:y1 + 1, x0:x1 + 1]
                self.shipped[l].append(r)

    def check(self, what):
        rep = self.replica
        for l, L in enumerate(self.lv):
            got = rep.download_level(l)
            bad = bits(got) != bits(self.want[l])
            assert not bad.any(), (what, l, int(bad.sum()), np.argwhere(bad)[:5].tolist())          # (a)
            assert same(rep.download_prob(l), mw.prob(got)), (what, l)                               # (b)
            probe_twin(rep, l, L, got, union(self.shipped[l]), what, max_cells=20000)                # (c)
            assert rep.get_mirror_dirty_rect(l) == union(self.shipped[l]), (what, l)                 # (d)
        assert rep.get_dirty_rects() == [None] * self.levels, what                                   # (e)

    def close(self):
        self.owner.close()
        self.replica.close()


@MODES
@pytest.mark.parametrize("geom", REPL_MAPS, ids=mc.geom_id)
def test_one_shot_replication(hsb_lib, geom, mode):
    t = Replication(geom, mode, seed=geom[0] + mode)
    levels = t.levels
    schedule = [[0, levels - 1], list(range(levels)), [levels - 1]]
    for k, lv in enumerate(schedule):
        t.write(lv, k)
        if k == 2:
            t.owner.upload_level(0, mw.preload((t.lv[0].sy, t.lv[0].sx), t.rng))   # a whole-level rectangle
        rects = t.owner.get_dirty_rects()
        if k == 0 and levels == 3:
            assert rects[1] is None and rects[0] is not None and rects[2] is not None   # a clean level between two
        cells = t.cells(rects)
        exact = 4 * (HEADER_WORDS + cells)
        # short by one byte and by one word: overflow, nothing shipped, rectangles kept even with reset, counted once
        for cap in (exact - 1, exact - 4):
            before = [t.replica.download_level(l) for l in range(levels)]
            t.pack_unpack(cap, True)
            h = t.header()
            assert (h[0], h[1], h[2], h[3]) == (MAGIC, levels, 1, cells), (k, cap, h[:4])
            assert t.owner.get_dirty_rects() == rects
            assert t.replica.replication_overflows(reset=True) == 1
            assert all(same(t.replica.download_level(l), before[l]) for l in range(levels))
        # exactly the size: ships; reset=False keeps the rectangles
        t.pack_unpack(exact, False)
        assert t.owner.get_dirty_rects() == rects
        h = t.header()
        want_hdr = [MAGIC, levels, 0, cells] + sum([list(r) if r else [INT_MAX, INT_MAX, -1, -1] for r in rects], [])
        assert list(h[:4 + 4 * levels]) == want_hdr, (k, h[:4 + 4 * levels])
        t.shipped_from_owner(rects)
        t.check(f"{geom} mode {mode} write {k} exact capacity")
        # three bytes more (not a multiple of 4): ships; reset=True clears the rectangles
        t.pack_unpack(exact + 3, True)
        assert t.owner.get_dirty_rects() == [None] * levels
        assert t.replica.replication_overflows() == 0
        t.shipped_from_owner(rects)
        t.check(f"{geom} mode {mode} write {k} capacity + 3")
        if k == 1:   # the replica's host mirror syncs: its rectangle starts again
            for l in range(levels):
                t.replica.get_mirror_dirty_rect(l, reset=True)
                t.shipped[l] = []
    # a buffer from a handle with another level count is counted, not applied
    other = handle((geom[0], geom[1], levels - 1, geom[3]), mode)
    other.upload_level(0, mw.preload((t.lv[0].sy, t.lv[0].sx), t.rng))
    other.pack_dirty_device(t.buf.data_ptr(), t.cap_max, True, t.stream)
    t.replica.unpack_dirty_device(t.buf.data_ptr(), t.cap_max, t.stream)
    assert t.replica.replication_overflows(reset=True) == 1
    t.check(f"{geom} mode {mode} foreign level count")
    other.close()
    t.close()


@MODES
@pytest.mark.parametrize("geom", REPL_MAPS, ids=mc.geom_id)
def test_two_step_replication(hsb_lib, geom, mode):
    """hsb_get_dirty_rects + hsb_pack_rect_device + hsb_unpack_rect_device: the owner's dirty rectangles after writes
    that leave a level clean, then arbitrary rectangles of a re-uploaded owner plane (the corners as single cells, a
    row and a column strip) that only those rectangles may carry to the replica."""
    t = Replication(geom, mode, seed=3 * geom[0] + mode)
    levels = t.levels
    for k, lv in enumerate([[0, levels - 1], list(range(levels))]):
        t.write(lv, k)
        rects = t.owner.get_dirty_rects(reset=True)
        assert t.owner.get_dirty_rects() == [None] * levels
        for l, r in enumerate(rects):
            if r is not None:
                t.owner.pack_rect_device(l, r, t.buf.data_ptr(), t.stream)
                t.replica.unpack_rect_device(l, r, t.buf.data_ptr(), t.stream)
        t.shipped_from_owner(rects)
        t.check(f"{geom} mode {mode} two-step write {k}")
    for l, L in enumerate(t.lv):
        t.owner.upload_level(l, mw.preload((L.sy, L.sx), t.rng))
        sx, sy = L.sx, L.sy
        rects = [(0, 0, 0, 0), (sx - 1, 0, sx - 1, 0), (0, sy - 1, 0, sy - 1), (sx - 1, sy - 1, sx - 1, sy - 1),
                 (0, sy // 2, sx - 1, sy // 2), (sx // 3, 0, sx // 3, sy - 1), (sx - 1, 1, sx - 1, sy - 2)]
        for r in rects:
            t.owner.pack_rect_device(l, r, t.buf.data_ptr(), t.stream)
            t.replica.unpack_rect_device(l, r, t.buf.data_ptr(), t.stream)
            t.shipped_from_owner([r if m == l else None for m in range(levels)])
        t.check(f"{geom} mode {mode} two-step rectangles level {l}")
    t.close()


@MODES
def test_refresh_level_after_a_plane_written_on_a_caller_stream(hsb_lib, mode):
    """parallel.replicate_map's receive side: a plane written into hsb_level_logodds_device_ptr on a caller's stream,
    hsb_refresh_level on that stream: P equals libm's on every cell, the texture twin follows, and the mirror
    rectangle covers the level (a host mirror that had synced must re-read it) while the replication rectangle stays
    clean (the replica must not ship the plane back)."""
    import torch

    from hector_slam_b200 import parallel

    geom = REPL_MAPS[1]
    t = Replication(geom, mode, seed=5 + mode)
    rep = t.replica
    dev = torch.device("cuda", 0)
    side = torch.cuda.Stream(device=dev)
    for l, L in enumerate(t.lv):
        rep.get_mirror_dirty_rect(l, reset=True)
        new = mw.preload((L.sy, L.sx), t.rng)
        new[0, 0], new[-1, -1], new[-1, 0] = np.float32(50.0), np.float32(-60.0), np.float32(0.0)
        view = parallel.level_plane_tensor(rep, l, dev)
        with torch.cuda.stream(side):
            view.copy_(torch.from_numpy(new).to(dev, non_blocking=False))
            rep.refresh_level(l, side.cuda_stream)
        side.synchronize()
        assert same(rep.download_level(l), new)
        assert same(rep.download_prob(l), mw.prob(new)), (mode, l)
        probe_twin(rep, l, L, new, (0, 0, L.sx - 1, L.sy - 1), f"refresh mode {mode} level {l}", max_cells=20000)
        assert rep.get_mirror_dirty_rect(l) == (0, 0, L.sx - 1, L.sy - 1), (mode, l)
        assert rep.get_dirty_rect(l) is None
    t.close()
