"""GPU: the N3 kernels — likelihood_kernel (the device entry points), likelihood_group_kernel and covariance_kernel (the
host-buffer ones, hsb_likelihood_batch and hsb_covariance_batch) and the arg-max of hsb_best_hypothesis_device — against
the float64 reference of the pose likelihood (oracle/likelihood64.py), tightly enough to see ONE endpoint lost or counted
twice, in both scan layouts, both gather modes, around both grid caps and on the map's edges.

Probe.  Resolution 0.25 and start = (0, 0): world <-> map is exact on every level (a power-of-two scale, no offset), so
the reference gets the kernel's own map state.  The planes are a smooth probability field with a saturated and a flat
patch; the reference reads the plane the device holds (download_prob).  Two 3-level maps: 256 x 256 and 404 x 300,
whose coarse levels (202 x 150, 101 x 75) have widths that are not multiples of 4.

Bound.  A pose's likelihood is summed by one warp: each lane adds k = ceil(n / 32) funval sequentially, the butterfly
adds 5 levels, then one division by (float)n and one subtraction.  funval >= 0, so with u = 2^-24

    |lh_gpu - lh64| <= 1.01 ((k + 6) u R64 / n + u |lh64|)          (R64 = sum funval in float64)

Power.  The endpoints where a lane or pass boundary falls — 0, 1, n-2, n-1, every 32j-1 and 32j — are out of the map
(funval = 1), and each case asserts that each of them moves the likelihood by more than 4 tol.  The 40 000-point scans
are held to the bound only (it exceeds one endpoint's share there); their test ids say so.

Bitwise.  The summation order depends on the scan only, so a pose's likelihood has the same bits in any batch, at any
index, in either layout (one shared scan or per-pose offsets), through the host or the device entry point, as the
d_out_likelihood of hsb_best_hypothesis_device and in either gather mode.  The covariance is then pinned bit for bit:
hsb_covariance_batch equals likelihood64.covariance_fp32 of the seven hsb_likelihood_batch values at the sigma points.

Arg-max.  The winner of hsb_best_hypothesis_device is the lowest-index maximum of the hsb_likelihood_batch scores, where
a non-finite pose and a NaN likelihood (an empty scan: 1 - 0/0) both rank as -1.
"""
import math

import numpy as np
import pytest

from conftest import report
from oracle import likelihood64

pytestmark = pytest.mark.gpu

F32 = np.float32
RES = 0.25
MODES = (1, 2)                                  # LDG, TEX
MAPS = {"sq": (256, 256), "odd": (404, 300)}
LENGTHS = [0, 1, 2, 31, 32, 33, 63, 64, 65, 1081, 2049]
LONG = 40000
_WORST = {}


def sm_count():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def lh_cap():
    """poses the likelihood grid covers in one pass: sm_count * 16 CTAs of 4 warps (hsb_api.cu likelihood_device and
    score_query)"""
    return sm_count() * 16 * 4


def cov_cap():
    """poses the covariance grid covers in one pass: sm_count * 8 CTAs (hsb_covariance_batch)"""
    return sm_count() * 8


def bits(a):
    return np.ascontiguousarray(a, F32).view(np.uint32)


def field_logodds(sx, sy):
    yy, xx = np.mgrid[0:sy, 0:sx].astype(np.float64)
    lo = (1.5 * np.sin(2 * np.pi * xx / 37.0) + 1.5 * np.sin(2 * np.pi * yy / 29.0)
          + 0.8 * np.sin(2 * np.pi * (xx + 0.6 * yy) / 53.0) + 0.02 * np.clip(xx - yy, -64, 64)).astype(F32)
    lo[sy // 3: sy // 3 + 6, sx // 2: sx // 2 + 8] = 60.0      # saturated: p == 1
    lo[sy // 2: sy // 2 + 6, sx // 8: sx // 8 + 8] = 0.0       # flat: p == 0.5
    return lo


def boundary_indices(n):
    if n <= 0:
        return np.zeros(0, np.int64)
    ks = np.arange(1, n // 32 + 2) * 32
    idx = {0, 1, n - 2, n - 1} | set(ks.tolist()) | set((ks - 1).tolist())
    return np.array(sorted(i for i in idx if 0 <= i < n), np.int64)


class Ref:
    """One (scan, pose) on one level, with its float64 reference."""

    def __init__(self, lv, pts, pose_map):
        self.lv = lv
        self.pts = np.ascontiguousarray(pts, F32).reshape(-1, 2)
        self.n = self.pts.shape[0]
        self.pose_map = np.asarray(pose_map, F32)
        self.pose = (self.pose_map * F32([lv.cell, lv.cell, 1.0])).astype(F32)      # exact: power of two
        self.ev = likelihood64.evaluate(lv.prob, self.pts, self.pose_map, lv.pt_scale)
        self.tol = self.ev.tol(-(-self.n // 32) + 5)

    def check(self, got, what):
        """the bound (NaN for an empty scan); returns err / tol"""
        got = F32(got)
        if self.n == 0:
            assert np.isnan(got), (what, "empty scan", got)
            return 0.0
        err = abs(float(got) - self.ev.lh64)
        assert err <= self.tol, (what, self.n, float(got), self.ev.lh64, err, self.tol)
        return err / self.tol if self.tol else 0.0

    def power(self):
        """min over the boundary endpoints of |funval| / n / tol"""
        idx = boundary_indices(self.n)
        return float(self.ev.funval[idx].min()) / self.n / self.tol if len(idx) else math.inf


class Level:
    def __init__(self, reps, l):
        self.l = l
        self.sx, self.sy, self.cell = reps[1].level_info(l)
        self.pt_scale = F32(2.0 ** -l)
        self.prob = reps[1].download_prob(l)
        assert np.array_equal(self.prob, reps[2].download_prob(l))
        assert self.cell == RES * 2 ** l

    def scan(self, n, rng, pose_map, extras=()):
        """n endpoints (level-0 cells) for pose_map: the boundary endpoints out of the map (funval 1), `extras` (level
        cells, exact q for psi = 0) and a few non-finite / far endpoints at other indices, the rest inside the map."""
        x, y, psi = (float(v) for v in pose_map)
        c, s = math.cos(psi), math.sin(psi)

        def to_pts(q):                                  # level cells q -> endpoint in the scan frame, level-0 cells
            d = q - np.float64([x, y])
            p = np.stack([c * d[:, 0] + s * d[:, 1], -s * d[:, 0] + c * d[:, 1]], axis=1)
            return (p.astype(F32) / self.pt_scale).astype(F32)

        q = np.stack([rng.uniform(1.0, self.sx - 3.0, n), rng.uniform(1.0, self.sy - 3.0, n)], axis=1)
        pts = to_pts(q)
        heavy = np.zeros(n, bool)
        heavy[boundary_indices(n)] = True
        far = np.stack([rng.choice([-30.0, self.sx + 30.0], n), rng.uniform(-40.0, self.sy + 40.0, n)], axis=1)
        pts[heavy] = to_pts(far[heavy])
        free = [i for i in range(2, n) if not heavy[i]]
        extras = [np.float32(e) for e in extras] + [np.float32([np.nan, 3.0]), np.float32([np.inf, 1.0]),
                                                    np.float32([2.0, -np.inf]), np.float32([np.nan, np.nan])]
        for i, e in zip(free, extras):
            pts[i] = e / self.pt_scale if np.all(np.isfinite(e)) else e
        return pts.astype(F32)

    def edge_extras(self, pose_map):
        """level-cell endpoints for a psi = 0 integer pose: q on 0 and on S-2, one ulp past each, on integers, -0.0"""
        lx, ly, up = F32(self.sx - 2), F32(self.sy - 2), F32(1e9)
        x, y = pose_map[0], pose_map[1]
        return [(0.0 - x, 0.0 - y), (lx - x, ly - y), (0.0 - x, ly - y), (lx - x, 0.0 - y),
                (np.nextafter(lx, up) - x, 5.0), (5.0, np.nextafter(ly, up) - y),
                (np.nextafter(F32(-x), -up), 3.0), (3.0, np.nextafter(F32(-y), -up)),
                (-0.0, 2.0), (2.0, -0.0), (-0.0, -0.0), (1.0 - x, 1.0 - y), (7.0 - x, 3.0 - y)]


class MapSetup:
    def __init__(self, capi, name):
        sx, sy = MAPS[name]
        self.name = name
        self.reps = {}
        for mode in MODES:
            rep = capi.MapRepB200(RES, sx, sy, levels=3, start=(0.0, 0.0), gather_mode=mode)
            assert rep.gather_mode == mode
            for l in range(3):
                rep.upload_level(l, field_logodds(sx >> l, sy >> l))
            self.reps[mode] = rep
        self.levels = [Level(self.reps, l) for l in range(3)]
        self._refs = {}

    def random_pose(self, lv, rng):
        return F32([rng.uniform(lv.sx / 4, 3 * lv.sx / 4), rng.uniform(lv.sy / 4, 3 * lv.sy / 4), rng.uniform(-3.1, 3.1)])

    def length_refs(self, l):
        """every length in LENGTHS and LONG with its own pose, plus an edge scan (psi = 0, integer pose)"""
        if l not in self._refs:
            lv = self.levels[l]
            rng = np.random.default_rng(1000 * l + len(self.name))
            refs = [Ref(lv, lv.scan(n, rng, p), p) for n in LENGTHS + [LONG] for p in [self.random_pose(lv, rng)]]
            ep = F32([5.0, 7.0, 0.0])
            refs.append(Ref(lv, lv.scan(300, rng, ep, lv.edge_extras(ep)), ep))
            e = refs[-1].ev
            # the edges: q == 0 / S-2 in, one ulp past out, -0.0 in (the scan's extras start at index 2)
            free = [i for i in range(2, 300) if i not in set(boundary_indices(300).tolist())]
            assert e.inside[free[:4]].all() and not e.inside[free[4:8]].any() and e.inside[free[8:13]].all()
            assert not e.inside[free[13:17]].any()
            self._refs[l] = refs
        return self._refs[l]

    def close(self):
        for r in self.reps.values():
            r.close()


@pytest.fixture(scope="module")
def M(hsb_lib):
    from hector_slam_b200 import capi

    maps = {name: MapSetup(capi, name) for name in MAPS}
    yield maps
    for m in maps.values():
        m.close()
    for fam in sorted(_WORST):
        report(f"likelihood sums [{fam}]: max err / tol = {_WORST[fam]:.3f}")


_BITS = {}       # (map, level, id(ref)) -> the likelihood's bits, from the first result seen


def record(fam, worst):
    _WORST[fam] = max(_WORST.get(fam, 0.0), worst)


def same_bits(key, value, what):
    v = bits(F32(value))
    if key not in _BITS:
        _BITS[key] = (v, what)
    else:
        assert v == _BITS[key][0], (what, "differs from", _BITS[key][1])


def pack(refs):
    pts = np.concatenate([r.pts for r in refs]).astype(F32) if refs else np.zeros((0, 2), F32)
    offs = np.concatenate([[0], np.cumsum([r.n for r in refs])]).astype(np.int32)
    poses = np.stack([r.pose for r in refs]).astype(F32)
    return poses, pts, offs


def expected_winner(scores, poses):
    """lowest-index maximum with non-finite poses and NaN likelihoods ranked -1 -> (index, ranked score)"""
    rank = np.where(np.all(np.isfinite(poses), axis=1) & ~np.isnan(scores), scores, F32(-1.0)).astype(F32)
    k = int(np.argmax(rank))
    return k, rank[k]


def best_on_device(rep, l, poses, pts, offs, n_shared=0, want_out=False):
    """hsb_best_hypothesis_device on device copies -> (best4, d_out_likelihood or None)"""
    import torch

    B = poses.shape[0]
    d_poses = torch.from_numpy(np.ascontiguousarray(poses, F32)).cuda()
    d_pts = torch.from_numpy(np.ascontiguousarray(pts, F32).reshape(-1)).cuda() if pts.size else torch.zeros(2, device="cuda")
    d_offs = torch.from_numpy(offs).cuda() if offs is not None else None
    d_best = torch.full((4,), 7.0, dtype=torch.float32, device="cuda")
    d_out = torch.full((max(B, 1),), 7.0, dtype=torch.float32, device="cuda") if want_out else None
    rep.best_hypothesis_device(l, B, d_poses.data_ptr(), d_pts.data_ptr(),
                               d_offs.data_ptr() if d_offs is not None else None, n_shared, d_best.data_ptr(),
                               d_out.data_ptr() if want_out else None, 0)
    torch.cuda.synchronize()
    return d_best.cpu().numpy(), (d_out.cpu().numpy()[:B] if want_out else None)


def check_winner(best4, scores, poses, what):
    k, sc = expected_winner(scores, poses)
    got_k = np.flatnonzero(np.all(bits(poses) == bits(best4[1:]), axis=1))[:1].tolist()
    assert bits(best4[0]) == bits(sc) and np.array_equal(bits(best4[1:]), bits(poses[k])), \
        (what, "want index", k, float(sc), "device returned", best4.tolist(), "= the pose at index", got_k)


# ---- 1. scan lengths, edges, layouts, entry points, gather modes ----------------------------------------------------
CASES = [(name, l, mode) for name in MAPS for l in range(3) for mode in MODES]


@pytest.mark.parametrize("name,l,mode", CASES, ids=[f"{n}-L{l}-{'LDG' if m == 1 else 'TEX'}-40k-bound-only"
                                                     for n, l, m in CASES])
def test_lengths_edges_layouts(M, name, l, mode):
    import torch

    S = M[name]
    rep = S.reps[mode]
    refs = S.length_refs(l)
    worst = 0.0
    rng = np.random.default_rng(7)
    for order in ("given", "ragged"):
        batch = refs if order == "given" else [refs[i] for i in rng.permutation(len(refs))] + refs[:3]
        poses, pts, offs = pack(batch)
        got = rep.likelihood_batch(l, poses, pts, offs)
        for b, r in enumerate(batch):
            what = f"{name} L{l} mode{mode} {order} offsets b{b} n{r.n}"
            worst = max(worst, r.check(got[b], what))
            same_bits((name, l, id(r)), got[b], what)
    for r in refs:
        if r.n and r.n < LONG:
            assert r.power() > 4.0, (name, l, r.n, "a lost / doubled boundary endpoint would go unseen", r.power())
    # one shared scan (offsets == NULL): the scan's own pose among absurd ones, and the replicated-offsets layout
    absurd = F32([[np.nan, 1.0, 0.1], [np.inf, 1.0, 0.1], [1.0, -np.inf, 0.1], [1e30, 1.0, 0.1], [1.0, -1e30, 0.1],
                  [1.0, 1.0, np.nan], [-np.inf, np.nan, np.inf]])
    for r in refs:
        poses = np.concatenate([absurd[:3], r.pose[None], absurd[3:], r.pose[None]]).astype(F32)
        got = rep.likelihood_batch(l, poses, r.pts, None)
        what = f"{name} L{l} mode{mode} shared n{r.n}"
        same_bits((name, l, id(r)), got[3], what)
        same_bits((name, l, id(r)), got[-1], what + " (last)")
        other = np.delete(got, [3, len(got) - 1])
        if r.n:
            assert np.all(bits(other) == 0), (what, other)          # every endpoint out of the map: exactly +0.0
        else:
            assert np.all(np.isnan(got)), (what, got)
        rep_offs = (np.arange(len(poses) + 1) * r.n).astype(np.int32)
        got2 = rep.likelihood_batch(l, poses, np.tile(r.pts, (len(poses), 1)), rep_offs)
        assert np.array_equal(bits(got2), bits(got)), (what, "replicated offsets")
    # the device entry point on a side stream, and d_out_likelihood of the arg-max launch
    poses, pts, offs = pack(refs)
    want = rep.likelihood_batch(l, poses, pts, offs)
    dev = torch.device("cuda", 0)
    side = torch.cuda.Stream(device=dev)
    d_poses, d_pts, d_offs = (torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (poses, pts, offs))
    d_out = torch.full((len(refs),), -7.0, dtype=torch.float32, device=dev)
    with torch.cuda.stream(side):
        rep.likelihood_batch_device(l, len(refs), d_poses.data_ptr(), d_pts.data_ptr(), d_offs.data_ptr(), 0,
                                    d_out.data_ptr(), side.cuda_stream)
    side.synchronize()
    assert np.array_equal(bits(d_out.cpu().numpy()), bits(want))
    best4, out = best_on_device(rep, l, poses, pts, offs, want_out=True)
    assert np.array_equal(bits(out), bits(want))
    # the batch holds an empty scan (refs[0]): its NaN must not win
    assert refs[0].n == 0 and np.isnan(want[0])
    check_winner(best4, want, poses, f"{name} L{l} mode{mode} lengths batch with an empty scan")
    record("lengths, edges, layouts", worst)


# ---- 2. grid-stride passes -----------------------------------------------------------------------------------------
P = 61


def pool(S):
    """P short-scan refs on the square map's level 0 (lengths 0 ... 2049), plus BEST and BEST2: scans whose every
    endpoint sits on a saturated cell at an integer q (funval exactly 0: likelihood exactly 1, above every pool entry),
    seen from two different poses."""
    if not hasattr(S, "_pool"):
        lv = S.levels[0]
        rng = np.random.default_rng(61)
        lens = LENGTHS + rng.integers(3, 120, P - len(LENGTHS)).tolist()
        refs = [Ref(lv, lv.scan(int(n), rng, p), p) for n in lens for p in [S.random_pose(lv, rng)]]
        sat_y, sat_x = lv.sy // 3, lv.sx // 2
        bp = F32([sat_x + 1.0, sat_y + 1.0, 0.0])
        q = np.stack(np.meshgrid(np.arange(sat_x, sat_x + 7), np.arange(sat_y, sat_y + 5)), axis=-1).reshape(-1, 2)
        bp2 = bp + F32([2.0, 1.0, 0.0])
        best = [Ref(lv, (q - b[:2]).astype(F32), b) for b in (bp, bp2)]
        assert best[0].ev.lh64 == 1.0 and best[1].ev.lh64 == 1.0
        assert all(r.n == 0 or r.ev.lh64 < 0.99 for r in refs)
        S._pool = refs + best
    return S._pool


def pool_batch(refs, sel):
    lens = np.array([r.n for r in refs])[sel]
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    pts = np.concatenate([refs[j].pts for j in sel]).astype(F32)
    poses = np.stack([r.pose for r in refs])[sel].astype(F32)
    return poses, pts, offs


@pytest.mark.parametrize("mode", MODES)
def test_grid_stride_and_best_hypothesis(M, mode):
    S = M["sq"]
    rep = S.reps[mode]
    refs = pool(S)
    BEST, BEST2 = P, P + 1
    nref = len(refs)
    cap = lh_cap()
    # the pool alone: reference bound, power, and the bits every later batch has to reproduce
    poses, pts, offs = pool_batch(refs, np.arange(nref))
    base = rep.likelihood_batch(0, poses, pts, offs)
    worst = max(r.check(base[j], f"mode{mode} pool {j}") for j, r in enumerate(refs))
    assert all(r.power() > 4.0 for r in refs[:P] if r.n), "a lost / doubled boundary endpoint would go unseen"
    lh64 = np.array([r.ev.lh64 for r in refs])
    tol = np.array([r.tol for r in refs])
    for B in (1, cap - 1, cap, cap + 1, 65536):
        base_sel = (np.arange(B) * 7 + B) % P
        sel = base_sel.copy()
        if B > 2 * cap:
            sel[B - 1], sel[cap + 5] = BEST, BEST2       # equal best scores at the last index and in the second pass
        poses, pts, offs = pool_batch(refs, sel)
        got = rep.likelihood_batch(0, poses, pts, offs)
        assert np.array_equal(bits(got), bits(base[sel])), (mode, B, "a pose's bits depend on its batch / index")
        sample = np.unique(np.concatenate([np.arange(cap, B), np.arange(0, B, 100)]))
        ok = np.isnan(lh64[sel[sample]]) & np.isnan(got[sample]) | (np.abs(got[sample] - lh64[sel[sample]]) <= tol[sel[sample]])
        assert ok.all(), (mode, B, sample[~ok][:5])
        best4, out = best_on_device(rep, 0, poses, pts, offs, want_out=True)
        assert np.array_equal(bits(out), bits(got))
        check_winner(best4, got, poses, f"mode{mode} B{B}")
        if B > 2 * cap:
            assert np.array_equal(bits(best4), bits(np.concatenate([[1.0], refs[BEST2].pose]))), (mode, best4)
            # the unique best at the last index, and in a later pass
            for k in (B - 1, 3 * cap + 17):
                sel2 = base_sel.copy()
                sel2[k] = BEST
                p2, x2, o2 = pool_batch(refs, sel2)
                best4, _ = best_on_device(rep, 0, p2, x2, o2)
                assert np.array_equal(bits(best4), bits(np.concatenate([[1.0], p2[k]]))), (mode, B, k, best4)
            # equal best scores in two later passes, either way round: the lower index wins
            for lo_ref, hi_ref in ((BEST, BEST2), (BEST2, BEST)):
                sel2 = base_sel.copy()
                sel2[2 * cap + 3], sel2[4 * cap + 1] = lo_ref, hi_ref
                p2, x2, o2 = pool_batch(refs, sel2)
                best4, _ = best_on_device(rep, 0, p2, x2, o2)
                assert np.array_equal(bits(best4), bits(np.concatenate([[1.0], refs[lo_ref].pose]))), (mode, best4)
        # the shared layout: one 1081-point scan against B poses, against its replicated offsets (B up to cap + 1)
        if B <= cap + 1:
            scan = refs[LENGTHS.index(1081)].pts
            shp = np.stack([r.pose for r in refs])[sel].astype(F32)
            g1 = rep.likelihood_batch(0, shp, scan, None)
            if B == cap + 1:
                g2 = rep.likelihood_batch(0, shp, np.tile(scan, (B, 1)), (np.arange(B + 1) * len(scan)).astype(np.int32))
                assert np.array_equal(bits(g1), bits(g2)), (mode, B)
                sh = [Ref(S.levels[0], scan, refs[j].pose_map) for j in range(P)]
                for b in np.concatenate([np.arange(cap - 3, B), np.arange(0, B, 100)]):
                    worst = max(worst, sh[sel[b]].check(g1[b], f"mode{mode} shared B{B} b{b}"))
                best4, _ = best_on_device(rep, 0, shp, scan, None, n_shared=len(scan))
                check_winner(best4, g1, shp, f"mode{mode} shared B{B}")
    record("grid stride", worst)


@pytest.mark.parametrize("mode", MODES)
def test_best_hypothesis_edge_cases(M, mode):
    S = M["sq"]
    rep = S.reps[mode]
    refs = pool(S)
    cap = lh_cap()
    # one empty scan among per-hypothesis offsets: 1 - 0/0 is NaN and ranks -1; the best real score wins
    sel = np.arange(40) + 1
    sel[7] = 0                                           # LENGTHS[0] == 0
    assert refs[0].n == 0
    poses, pts, offs = pool_batch(refs, sel)
    got = rep.likelihood_batch(0, poses, pts, offs)
    assert np.isnan(got[7])
    best4, out = best_on_device(rep, 0, poses, pts, offs, want_out=True)
    assert np.isnan(out[7])                              # d_out_likelihood keeps the reference's NaN
    check_winner(best4, got, poses, f"mode{mode} an empty scan among per-hypothesis offsets")
    # only empty scans: every hypothesis ranks -1, index 0 wins with -1
    sel0 = np.zeros(cap + 3, np.int64)
    p0, x0, o0 = pool_batch(refs, sel0)
    best4, _ = best_on_device(rep, 0, p0, x0, o0)
    assert np.array_equal(bits(best4), bits(np.concatenate([[-1.0], p0[0]]))), (mode, "all empty", best4)
    # a shared scan with n_shared == 0
    best4, out = best_on_device(rep, 0, poses, np.zeros((0, 2), F32), None, n_shared=0, want_out=True)
    assert np.all(np.isnan(out))
    assert np.array_equal(bits(best4), bits(np.concatenate([[-1.0], poses[0]]))), (mode, "n_shared == 0", best4)
    # every hypothesis non-finite, across grid-stride passes: index 0 wins with -1
    B = 2 * cap + 5
    bad = np.tile(F32([[np.nan, 1.0, 0.0], [np.inf, 0.0, 0.0], [0.0, -np.inf, 0.0], [1.0, 1.0, np.nan]]), (B // 4 + 1, 1))[:B]
    scan = refs[LENGTHS.index(1081)].pts
    best4, out = best_on_device(rep, 0, bad, scan, None, n_shared=len(scan), want_out=True)
    assert np.array_equal(bits(best4), bits(np.concatenate([[-1.0], bad[0]]))), (mode, "all non-finite", best4)
    assert np.all(bits(out) == 0), out                   # every endpoint out of the map: exactly +0.0
    # consecutive calls re-arm the accumulator: a high-scoring batch, then a lower one, then an empty one
    hi = pool_batch(refs, np.array([1, len(refs) - 1, 2]))
    lo = pool_batch(refs, np.array([3, 4, 5, 6]))
    b_hi, _ = best_on_device(rep, 0, *hi)
    assert b_hi[0] == 1.0
    b_lo, _ = best_on_device(rep, 0, *lo)
    check_winner(b_lo, rep.likelihood_batch(0, *lo), lo[0], f"mode{mode} after a higher batch")
    b_0, _ = best_on_device(rep, 0, np.zeros((0, 3), F32), np.zeros((0, 2), F32), None, n_shared=0)
    assert b_0[0] == -1.0, b_0
    b_lo2, _ = best_on_device(rep, 0, *lo)
    assert np.array_equal(bits(b_lo2), bits(b_lo))


@pytest.mark.parametrize("mode", MODES)
def test_best_hypothesis_largest_finite_poses(M, mode):
    """A finite pose keeps its score however large its coordinates: FLT_MAX (what hsb_reset stores as a pose), the
    largest negative value and the rest of (3.4e38, FLT_MAX] are finite.  Through hsb_best_hypothesis_device,
    hsb_group_best_hypothesis and its _subset form."""
    from hector_slam_b200 import capi

    S = M["sq"]
    rep = S.reps[mode]
    lv = S.levels[0]
    fmax = np.finfo(F32).max
    big = np.nextafter(F32(3.4e38), F32(np.inf))
    rng = np.random.default_rng(77)
    g = capi.SlamGroup([rep])
    try:
        def all_calls(poses, scan, what):
            """(best4, index) of the three entry points, which must agree bit for bit"""
            best4, out = best_on_device(rep, 0, poses, scan, None, n_shared=len(scan), want_out=True)
            lh = rep.likelihood_batch(0, poses, scan)
            assert np.array_equal(bits(out), bits(lh)), what
            check_winner(best4, lh, poses, what)
            k = int(np.flatnonzero(np.all(bits(poses) == bits(best4[1:]), axis=1))[0])
            for members in (None, [0]):
                out_g, b4, idx = g.best_hypothesis(0, [poses], [scan], members=members)
                assert np.array_equal(bits(out_g), bits(lh)), (what, members)
                assert np.array_equal(bits(b4[0]), bits(best4)) and idx[0] == k, (what, members, b4[0], idx[0], best4, k)
            return best4, k, lh

        # (FLT_MAX, 0, 0), then a far-off finite pose: every endpoint of both is out of the map, both score exactly 0,
        # and the lower index wins the tie
        pose_map = S.random_pose(lv, rng)
        scan = lv.scan(300, rng, pose_map)
        poses = F32([[fmax, 0.0, 0.0], [1e6, -1e6, 0.5]])
        best4, k, lh = all_calls(poses, scan, f"mode{mode} FLT_MAX then far off")
        assert np.all(bits(lh) == 0) and k == 0, (lh, best4)
        # poses made only of largest-finite coordinates: x, y far out of the map score 0; a psi of FLT_MAX, -FLT_MAX or
        # just above 3.4e38 with x, y on the map scores a real likelihood, pinned to the float64 reference
        xy = pose_map[:2] * F32(lv.cell)
        psis = F32([fmax, -fmax, big, -big])
        poses = np.concatenate([F32([[fmax, fmax, fmax], [-fmax, big, 0.0]]),
                                np.stack([np.full(4, xy[0]), np.full(4, xy[1]), psis], 1)]).astype(F32)
        scan = lv.scan(500, rng, F32([pose_map[0], pose_map[1], fmax]))
        best4, k, lh = all_calls(poses, scan, f"mode{mode} largest finite coordinates")
        assert np.all(bits(lh[:2]) == 0)
        for j in range(2, poses.shape[0]):
            Ref(lv, scan, F32([pose_map[0], pose_map[1], poses[j, 2]])).check(lh[j], f"mode{mode} psi {poses[j, 2]}")
        assert k >= 2 and best4[0] > 0, (k, best4)
    finally:
        g.close()


# ---- 3. covariance -------------------------------------------------------------------------------------------------
def sigma_world(r):
    sp = likelihood64.sigma_points(r.pose_map)
    return (sp * F32([r.lv.cell, r.lv.cell, 1.0])).astype(F32), sp


def cov_check(rep, l, refs, cm, cw, what, worst_fam="covariance sigma points"):
    """cm / cw (B, 3, 3) of hsb_covariance_batch against covariance_fp32 of the seven hsb_likelihood_batch values"""
    worst = 0.0
    for b, r in enumerate(refs):
        spw, sp = sigma_world(r)
        lhs = rep.likelihood_batch(l, spw, r.pts, None)
        for i in range(7):
            worst = max(worst, Ref(r.lv, r.pts, sp[i]).check(lhs[i], f"{what} b{b} sigma {i}"))
        wm, ww = likelihood64.covariance_fp32(lhs, r.pose_map, r.lv.cell)
        assert likelihood64.same_bits_or_nan(cm[b], wm), (what, b, r.n, cm[b], wm)
        assert likelihood64.same_bits_or_nan(cw[b], ww), (what, b, r.n, cw[b], ww)
    record(worst_fam, worst)


@pytest.mark.parametrize("name,l,mode", CASES, ids=[f"{n}-L{l}-{'LDG' if m == 1 else 'TEX'}-40k-bound-only"
                                                     for n, l, m in CASES])
def test_covariance(M, name, l, mode):
    S = M[name]
    rep = S.reps[mode]
    lv = S.levels[l]
    refs = list(S.length_refs(l))
    far = F32([lv.sx + 500.0, lv.sy + 500.0, 0.3])        # all seven sigma points out of the map: sum 0, NaNs
    refs.append(Ref(lv, refs[LENGTHS.index(65)].pts, far))
    assert refs[-1].ev.lh64 == 0.0
    poses, pts, offs = pack(refs)
    cm, cw = rep.covariance_batch(l, poses, pts, offs)
    cov_check(rep, l, refs, cm, cw, f"{name} L{l} mode{mode} offsets")
    assert np.isnan(cm[-1]).any() and np.all(np.isnan(cm[0]))          # the out-of-map pose, the empty scan
    assert np.all(cm[[i for i, r in enumerate(refs) if r.n >= 31 and r is not refs[-1]], 0, 0] > 0)
    # the shared layout: one scan, the poses of all refs; the scan's own pose must give its offsets result
    r = refs[LENGTHS.index(1081)]
    cm1, cw1 = rep.covariance_batch(l, poses, r.pts, None)
    k = refs.index(r)
    assert np.array_equal(bits(cm1[k]), bits(cm[k])) and np.array_equal(bits(cw1[k]), bits(cw[k]))
    cov_check(rep, l, [Ref(lv, r.pts, q.pose_map) for q in refs[:6]], cm1[:6], cw1[:6], f"{name} L{l} mode{mode} shared")
    # an empty shared scan: every entry NaN
    cm0, _ = rep.covariance_batch(l, poses[:3], np.zeros((0, 2), F32), None)
    assert np.all(np.isnan(cm0))


@pytest.mark.parametrize("mode", MODES)
def test_covariance_past_the_grid_cap(M, mode):
    S = M["sq"]
    rep = S.reps[mode]
    refs = pool(S)[:P]
    poses, pts, offs = pool_batch(refs, np.arange(P))
    cm0, cw0 = rep.covariance_batch(0, poses, pts, offs)
    cov_check(rep, 0, refs, cm0, cw0, f"mode{mode} pool")
    cap = cov_cap()
    for B in (cap - 1, cap, cap + 1, 2 * cap + 3):
        sel = (np.arange(B) * 5 + B) % P
        p, x, o = pool_batch(refs, sel)
        cm, cw = rep.covariance_batch(0, p, x, o)
        assert np.array_equal(bits(cm), bits(cm0[sel])) and np.array_equal(bits(cw), bits(cw0[sel])), (mode, B)
