"""Non-square, odd-sized and off-centre multi-level maps for the match kernel, shared by the CPU test of the record
oracles (tests/test_match_record_oracle.py) and the GPU test of the kernel (tests/test_gpu_match_geometry.py).

The geometries are tests/maptools_cases.py's (resolution 0.05, not a power of two, so world <-> map is inexact) with the
levels the reference's integer halving gives them (MapRepMultiMap.h:67: a 243 x 200 map has a 121 x 100 level 1 whose
extent ends short of level 0's), plus one at the node's default resolution 0.025.  Each has a 1-level companion whose
map origin is world (-0, -0): only there can a pose coordinate, and so an endpoint's map coordinate, be -0.

Everything the tests assert about an edge is built exactly here, from a level's input pose: endpoints whose fp32 map
coordinate q (oracle/hessian64.py's arithmetic, bit for bit the kernel's) is lim = S - 2, the first value past it, +0,
the first value below 0, and -0.  Every set is built from a seed, so the CPU and the GPU tests see the same scans.
"""
import math

import numpy as np

import maptools_cases as mc
from oracle import hessian64

f32 = np.float32
RES = mc.RES
# (sx, sy, levels, start, resolution)
GEOMS = [(404, 300, 3, (0.5, 0.5), RES), (150, 404, 2, (0.3, 0.7), RES), (243, 200, 2, (0.5, 0.5), RES),
         (257, 131, 3, (0.5, 0.5), RES), (404, 300, 3, (0.3, 0.7), 0.025), (6000, 100, 1, (0.3, 0.7), RES),
         (7, 4, 1, (0.5, 0.5), RES)]
CORNER = (-0.0, -0.0)          # the 1-level companions' start
LONG = 40000                   # longer than one CTA can stage
LENGTHS = [0, 1, 31, 32, 33, 1081, 2049, LONG]
ANGLES = [0.3, 1.9, -2.6, -0.8, 3.5, -3.6, 2.9, -1.4]   # every quadrant, and past +-pi
SCHEDULES = {"default": None, "random": [-1, 2, 4]}
PLACEHOLDER = (1.0e5, 1.0e5)   # an endpoint out of every map at any pose: one of its q has magnitude >= 1e5
SLOTS = 32                     # placeholders an edge scan reserves


def edge_iterations(levels):
    """the schedule edge scans are built and classified with: level 0's default, one evaluation on each coarse level"""
    return [0] + [-1] * (levels - 1)


def geom_id(g):
    return f"{g[0]}x{g[1]}x{g[2]}" + (f"-res{g[4]}" if g[4] != RES else "")


def companion(g):
    """the 1-level handle of a geometry: level 0's size and resolution, origin at world (-0, -0)"""
    return (g[0], g[1], 1, CORNER, g[4])


def schedule(name, levels):
    s = SCHEDULES[name]
    return None if s is None else s[:levels]


def level_sizes(g):
    return [(g[0] >> l, g[1] >> l) for l in range(g[2])]


def lims(prob):
    sy, sx = prob.shape
    return f32(sx) - f32(2.0), f32(sy) - f32(2.0)


def field(sx, sy, level):
    """A smooth log-odds plane with a gradient everywhere, also across the first and last two rows and columns (so that
    endpoints on the edges contribute), a saturated patch (p == 1, no gradient) and a flat one.  Every level samples
    the same function of level-0 cells, as a real map's levels see the same world: the levels' Gauss-Newton optima lie
    close together, and a level's evaluations stay near the pose the finer level takes over."""
    yy, xx = np.mgrid[0:sy, 0:sx].astype(np.float64) * 2.0 ** level
    lo = (1.5 * np.sin(2 * np.pi * xx / 37.0) + 1.5 * np.sin(2 * np.pi * yy / 29.0)
          + 0.8 * np.sin(2 * np.pi * (xx + 0.6 * yy) / 53.0) + 0.02 * np.clip(xx - yy, -64, 64))
    if sx >= 4:
        lo[:, 0] = lo[:, 1] - 0.7
        lo[:, -1] = lo[:, -2] + 0.9
    if sy >= 4:
        lo[0, :] = lo[1, :] + 0.7
        lo[-1, :] = lo[-2, :] - 0.9
    if sx >= 24 and sy >= 16:
        y0, x0 = sy * 5 // 8, sx * 5 // 8
        lo[y0:y0 + 4, x0:x0 + 6] = 60.0
        y1, x1 = sy // 4, sx // 8
        lo[y1:y1 + 4, x1:x1 + 6] = 0.0
    return lo.astype(np.float32)


def q_map(pts, pose, level):
    """fp32 map coordinates of level-0 endpoints on `level` at the level's map pose (hessian64.evaluate's arithmetic)"""
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 2)
    pose = np.asarray(pose, np.float32)
    s, c = hessian64.sinf(pose[2]), hessian64.cosf(pose[2])
    with np.errstate(invalid="ignore", over="ignore"):
        px, py = pts[:, 0] * f32(2.0 ** -level), pts[:, 1] * f32(2.0 ** -level)
        return c * px + ((-s) * py + pose[0]), s * px + (c * py + pose[1])


def split_record(rec, levels, iters=None):
    """a record in the layout of include/hector_slam_b200.h -> one dict per level, indexed by level (as
    MapRepB200.split_record)"""
    from oracle.record_oracle import level_iterations

    evals = [m + 1 for m in level_iterations(levels, iters)]
    out, off = [None] * levels, 0
    for l in range(levels - 1, -1, -1):
        E = evals[l]
        ev = np.asarray(rec[off + 3:off + 3 + 15 * E], np.float32).reshape(E, 15)
        out[l] = dict(start=np.asarray(rec[off:off + 3], np.float32), H=ev[:, :9].reshape(E, 3, 3), dTr=ev[:, 9:12],
                      est=ev[:, 12:15])
        off += 3 + 15 * E
    return out


class Cases:
    """A geometry's designed endpoints: a pool of map points (level-0 cells) ranked by how much each moves H on every
    level, the scans drawn from it, and the edge constructions.  conv: map_coords_pose / world_coords_pose of the
    geometry (the port's or the device's: tests/test_gpu_match_geometry.py asserts they agree)."""

    def __init__(self, g, probs, conv, seed):
        self.g, self.probs, self.conv = g, probs, conv
        self.L = len(probs)
        sx, sy = g[0], g[1]
        rng = np.random.default_rng(seed)
        self.rng = rng
        self.base = conv.world_coords_pose(0, f32([0.42 * sx, 0.45 * sy, 0.0]))
        poses = [conv.map_coords_pose(l, self.base) for l in range(self.L)]
        Q = np.stack([rng.uniform(0.0, sx - 2.0, 20000), rng.uniform(0.0, sy - 2.0, 20000)], axis=1)
        p = (Q - np.float64(poses[0][:2])).astype(np.float32)
        score, light = np.full(len(Q), np.inf), np.zeros(len(Q))
        for l in range(self.L):
            ev = hessian64.evaluate(probs[l], p, f32([poses[l][0], poses[l][1], 0.0]), 2.0 ** -l)
            mean = ev.A[:6] / max(1, int(ev.inside.sum()))
            r = np.where(ev.inside, (np.abs(ev.contrib[:, :6]) / np.maximum(mean, 1e-300)).max(axis=1), 0.0)
            score = np.minimum(score, r)
            light = np.maximum(light, r)
        # heavy endpoints keep clear of the edges, where the pose a level hands on may push them out
        m = np.minimum(8.0, np.float64([sx, sy]) / 8.0)
        score[np.any((Q < m) | (Q > np.float64([sx, sy]) - 2.0 - 2.0 ** (self.L - 1) * m), axis=1)] = 0.0
        order = np.argsort(score, kind="stable")
        self.heavy = Q[order[-max(8, len(Q) // 200):]]     # the 0.5 % that move H most on the level that moves them least
        self.bulk = Q[np.argsort(light, kind="stable")[: len(Q) * 6 // 10]]   # the 60 % that move H least on any level

    # ---- scans -------------------------------------------------------------------------------------------------------
    def hint(self, k):
        j = self.rng.integers(-2, 3, 2) * self.g[4]
        return f32([self.base[0] + j[0], self.base[1] + j[1], ANGLES[k % len(ANGLES)]])

    def endpoints(self, Q, hint):
        """level-0 endpoints, seen from `hint`, of map points Q (level-0 cells)"""
        pm = self.conv.map_coords_pose(0, hint)
        c, s = math.cos(float(pm[2])), math.sin(float(pm[2]))
        d = np.asarray(Q, np.float64).reshape(-1, 2) - np.float64(pm[:2])
        return np.stack([c * d[:, 0] + s * d[:, 1], -s * d[:, 0] + c * d[:, 1]], axis=1).astype(np.float32)

    def scan(self, n, hint, nonfinite=True, slots=0):
        """heavy endpoints where lane, warp-group and CTA boundaries fall, ones far outside the map and (nonfinite)
        NaN / inf ones elsewhere.  The reference indexes the map with a NaN endpoint's cell (SURVEY.md Q4), so a scan
        that the C port or the compiled reference matches has none."""
        rng = self.rng
        idx = np.arange(n)
        Q = self.bulk[rng.integers(0, len(self.bulk), n)].copy()
        heavy = (idx % 32 == 0) | (idx % 32 == 31) | (idx < 3) | (idx >= n - 2)
        Q[heavy] = self.heavy[rng.integers(0, len(self.heavy), int(heavy.sum()))]
        pts = self.endpoints(Q, hint)
        free = np.flatnonzero(~heavy)
        if slots:
            # placeholders for the edge endpoints (build_edge_scan): out of the map at any pose, away from every
            # boundary and from the endpoints below
            self.slots = free[40:40 + slots]
            assert len(self.slots) == slots
            pts[self.slots] = PLACEHOLDER
        if len(free) > 8:
            big = 3.0 * max(self.g[0], self.g[1])
            pts[free[5]] = (-big, -big)
            pts[free[7]] = (big, 10.0)
            if nonfinite:
                pts[free[1]] = (np.nan, 3.0)
                pts[free[3]] = (np.inf, 1.0)
                pts[free[-2]] = (np.nan, np.nan)
        return pts

    def strip_scan(self, n, hint):
        """endpoints in level 0's strips beyond every coarse level's extent (x or y past 2^l (S_l - 2) + 1/4)"""
        sx, sy = self.g[0], self.g[1]
        ex = max(2 ** l * ((sx >> l) - 2) for l in range(1, self.L)) + 0.25
        ey = max(2 ** l * ((sy >> l) - 2) for l in range(1, self.L)) + 0.25
        rng = self.rng
        half = n // 2
        Q = np.concatenate([np.stack([rng.uniform(ex, sx - 2.0, half), rng.uniform(0.0, sy - 2.0, half)], axis=1),
                            np.stack([rng.uniform(0.0, sx - 2.0, n - half), rng.uniform(ey, sy - 2.0, n - half)], axis=1)])
        return self.endpoints(Q, hint)

    def outside_scan(self, n, hint):
        sx, sy = self.g[0], self.g[1]
        Q = np.stack([self.rng.uniform(sx + 1.0, sx + 60.0, n), self.rng.uniform(-30.0, sy + 30.0, n)], axis=1)
        return self.endpoints(Q, hint)

    # ---- exact edges ---------------------------------------------------------------------------------------------------
    def edge_points(self, level, pose, near, mean, coarse=()):
        """Endpoints on `level` at its map pose: q == lim and the first q past it on each axis, and (near) q == +0 and the
        first q below 0 and, on a non-square level, endpoints whose long-axis q lies between the two limits (inside) and
        whose short-axis q does (outside).  The free coordinate of each is the candidate that moves H most relative to
        `mean` (6,) among those out of every coarser level at its pose (`coarse`, see outside_coarser).
        -> (pts (k, 2), [(axis, target q or None, inside)])"""
        prob = self.probs[level]
        lx, ly = lims(prob)
        lim = (lx, ly)
        cand = np.linspace(0.5, 1.0, 40)
        out, kinds = [], []

        def by_power(axis, q_axis):
            """candidate endpoints on the line q[axis] == q_axis, the one that moves H most first"""
            free = cand * (float(lim[1 - axis]) - 0.5)
            Q = np.zeros((len(free), 2))
            Q[:, axis] = q_axis
            Q[:, 1 - axis] = free
            pts = self.level_endpoints(Q, pose, level)
            ev = hessian64.evaluate(prob, pts, pose, 2.0 ** -level)
            r = np.where(ev.inside, (np.abs(ev.contrib[:, :6]) / np.maximum(mean, 1e-300)).max(axis=1), -1.0)
            return pts[np.argsort(-r, kind="stable")]

        def best_free(axis, q_axis):
            return by_power(axis, q_axis)[0]

        targets = [(0, lx), (1, ly)] + ([(0, f32(0.0)), (1, f32(0.0))] if near else [])
        for axis, t in targets:
            cand_pts = by_power(axis, float(t) + (1e-3 if t == 0 else -1e-3))
            if coarse:
                cand_pts = cand_pts[outside_coarser(self, cand_pts, coarse)]
            p = past = None
            for p0 in cand_pts[:16]:
                p = solve_q(p0, pose, level, axis, t)
                if p is not None:
                    past = step_past(p, pose, level, axis, up=(t != 0))
                    if not coarse or outside_coarser(self, np.stack([p, past]), coarse).all():
                        break
                    p = None
            assert p is not None, ("no endpoint with q ==", axis, t, pose, coarse)
            out.append(p)
            kinds.append((axis, t, True))
            q = q_map(past, pose, level)[axis][0]
            assert (q > t) if t != 0 else (q < 0), (axis, t, q)
            out.append(past)
            kinds.append((axis, q, False))
        if near and lx != ly:                          # (inside the coarser levels too: built where the near edges are)
            a = 0 if lx > ly else 1                    # the long axis
            lo_, hi_ = float(min(lx, ly)), float(max(lx, ly))
            if hi_ - lo_ >= 1.5:
                for k, v in enumerate(np.linspace(lo_ + 0.5, hi_ - 0.25, 3)):
                    out.append(best_free(a, v))
                    kinds.append((a, None, True))
                    Q = np.zeros((1, 2))
                    Q[0, 1 - a] = v                    # the short axis past its limit, the long one inside
                    Q[0, a] = 0.3 * lo_ + k
                    out.append(self.level_endpoints(Q, pose, level)[0])
                    kinds.append((1 - a, None, False))
        return np.stack(out).astype(np.float32), kinds

    @staticmethod
    def level_endpoints(Q, pose, level):
        """level-0 endpoints that land near map points Q (the level's cells) from the level's map pose"""
        c, s = math.cos(float(pose[2])), math.sin(float(pose[2]))
        d = np.asarray(Q, np.float64).reshape(-1, 2) - np.float64(pose[:2])
        p = np.stack([c * d[:, 0] + s * d[:, 1], -s * d[:, 0] + c * d[:, 1]], axis=1) * 2.0 ** level
        return p.astype(np.float32)

    def zero_points(self, pose, mean, axis):
        """On a companion at a pose whose coordinates are -0 and whose angle is +0 (axis 0) or -0 (axis 1): an endpoint
        with q[axis] == -0 and the other q inside, the candidate that moves H most."""
        assert np.signbit(pose[0]) and np.signbit(pose[1]) and pose[0] == 0 and pose[1] == 0, pose
        assert bool(np.signbit(pose[2])) == (axis == 1) and pose[2] == 0, pose
        prob = self.probs[0]
        lim = lims(prob)
        free = np.linspace(0.5, float(lim[1 - axis]) - 0.5, 40).astype(np.float32)
        pts = np.zeros((len(free), 2), np.float32)
        pts[:, axis] = -0.0
        pts[:, 1 - axis] = free
        q = q_map(pts, pose, 0)[axis]
        assert np.all(q == 0) and np.all(np.signbit(q)), q
        ev = hessian64.evaluate(prob, pts, pose)
        r = np.where(ev.inside, (np.abs(ev.contrib[:, :6]) / np.maximum(mean, 1e-300)).max(axis=1), -1.0)
        return pts[int(np.argmax(r))]


def solve_q(p0, pose, level, axis, target, max_steps=20000):
    """Step one fp32 coordinate of the endpoint p0 by nextafter until its q[axis] on `level` is `target` exactly (+0 is
    not -0).  The coordinate with the larger weight in q[axis] is stepped; if a step jumps over the target, the other
    coordinate moves one ulp and the search starts again.  -> the endpoint, or None"""
    s, c = hessian64.sinf(f32(pose[2])), hessian64.cosf(f32(pose[2]))
    coef = (float(c), -float(s)) if axis == 0 else (float(s), float(c))
    j0 = 0 if abs(coef[0]) >= abs(coef[1]) else 1
    p = np.asarray(p0, np.float32).copy()

    def q_of(pp):
        return q_map(pp, pose, level)[axis][0]

    def hit(q):
        return q == target and bool(np.signbit(q)) == bool(np.signbit(target))

    for attempt in range(256):
        j = j0 if attempt % 4 != 3 or coef[1 - j0] == 0 else 1 - j0
        up = coef[j] > 0
        q = q_of(p)
        for _ in range(max_steps):
            if hit(q):
                return p
            inc = (q < target) or (q == target)       # +0 wanted, -0 got: go up
            nxt = p.copy()
            nxt[j] = np.nextafter(p[j], f32(np.inf) if inc == up else f32(-np.inf))
            qn = q_of(nxt)
            if hit(qn):
                return nxt
            if (qn > target) != (q > target) and (qn < target) != (q < target):
                break                                 # jumped over the target
            p, q = nxt, qn
        p[1 - j0] = np.nextafter(p[1 - j0], f32(np.inf))
    return None


def step_past(p, pose, level, axis, up):
    """From an endpoint with q[axis] == t, nextafter steps of the coordinate with the larger weight until q[axis] passes
    t (up: above it; else below it): the first value past t that the endpoint can reach."""
    s, c = hessian64.sinf(f32(pose[2])), hessian64.cosf(f32(pose[2]))
    coef = (float(c), -float(s)) if axis == 0 else (float(s), float(c))
    j = 0 if abs(coef[0]) >= abs(coef[1]) else 1
    t = q_map(p, pose, level)[axis][0]
    d = f32(np.inf) if (coef[j] > 0) == up else f32(-np.inf)
    p = np.asarray(p, np.float32).copy()
    for _ in range(20000):
        p[j] = np.nextafter(p[j], d)
        q = q_map(p, pose, level)[axis][0]
        if (q > t) if up else (q < 0):
            return p
    raise AssertionError(("no endpoint past", t, pose))


def matched_pose(cases, rec):
    """the world pose a record returns: level 0's last estimate, angle normalised"""
    from oracle import pose32

    last = rec[0]["est"][-1]
    return cases.conv.world_coords_pose(0, f32([last[0], last[1], pose32.normalize_angle(last[2])]))


def settle(cases, runner, hint, pts, rounds=3):
    """the hint moved to where matching `pts` from it ends, `rounds` times: Gauss-Newton steps from there are small"""
    for _ in range(rounds):
        hint = matched_pose(cases, runner(hint, pts))
    return hint


def outside_coarser(cases, pts, coarse):
    """every endpoint out of every coarser level at the pose that level evaluates at: coarse [(level, map pose)]"""
    ok = np.ones(len(pts), bool)
    for l, pose in coarse:
        ev = hessian64.evaluate(cases.probs[l], pts, pose, 2.0 ** -l)
        ok &= ~ev.inside
    return ok


def build_edge_scan(cases, runner, hint, base, slots):
    """The edge endpoints of every level written into the placeholder `slots` of `base` (so that the boundary endpoints
    stay heavy), coarsest level first: level l's are built at the input pose the coarser levels hand it
    (runner(hint, pts) -> split record), and adding them must leave the coarser levels' records unchanged bit for bit.
    The coarsest level (input pose: the hint) also gets the near edges.  The runner matches with EDGE_ITERATIONS, so
    that a coarse level's one evaluation is at the pose it starts from and hands on: a finer level's far edges, one
    cell or more past the coarse level's extent, stay outside it (with Gauss-Newton steps on a scan unrelated to the
    map a coarse level can move further than that).
    -> (pts, designed: [(level, index, axis, target q or None, inside)], the final record)"""
    L = cases.L
    pts = np.asarray(base, np.float32).copy()
    slots = list(slots)
    if L > 1:
        hint = settle(cases, runner, hint, pts)
    designed, prev = [], None
    for l in range(L - 1, -1, -1):
        if l == L - 1:
            pose = cases.conv.map_coords_pose(l, hint)
        else:
            rec = runner(hint, pts)
            if prev is not None:
                assert_levels_equal(rec, prev, range(l + 2, L), "coarser levels changed by level %d's edges" % (l + 1))
            prev = rec
            pose = cases.conv.map_coords_pose(l, rec[l]["start"])
        coarse = [] if l == L - 1 else [(c, cases.conv.map_coords_pose(c, rec[c]["start"])) for c in range(l + 1, L)]
        ev = hessian64.evaluate(cases.probs[l], pts, pose, 2.0 ** -l)
        mean = ev.A[:6] / max(1, int(ev.inside.sum()))
        new, kinds = cases.edge_points(l, pose, l == L - 1, mean, coarse)
        assert len(new) <= len(slots), (len(new), len(slots))
        for i, (a, t, inside) in enumerate(kinds):
            k = slots.pop(0)
            pts[k] = new[i]
            designed.append((l, k, a, t, inside))
    rec = runner(hint, pts)
    if prev is not None:
        assert_levels_equal(rec, prev, range(1, L), "coarser levels changed by level 0's edges")
    return hint, pts, designed, rec


def assert_levels_equal(a, b, levels, msg):
    for l in levels:
        for k in ("start", "H", "dTr", "est"):
            assert np.array_equal(np.asarray(a[l][k], np.float32).view(np.uint32),
                                  np.asarray(b[l][k], np.float32).view(np.uint32)), (msg, l, k)


def check_edges(cases, rec, pts, designed):
    """At each level's recorded input pose, hessian64 classifies every designed endpoint as designed and an exact
    one's q is its target bit for bit.  -> {level: evaluation at the input pose}"""
    evs = {}
    for l in range(cases.L):
        pin = cases.conv.map_coords_pose(l, rec[l]["start"])
        evs[l] = (pin, hessian64.evaluate(cases.probs[l], pts, pin, 2.0 ** -l))
    for l, i, axis, t, inside in designed:
        pin, ev = evs[l]
        assert bool(ev.inside[i]) == inside, (l, i, axis, t, inside)
        if t is not None:
            q = q_map(pts[i], pin, l)[axis][0]
            assert q == t and np.signbit(q) == np.signbit(t), (l, i, axis, q, t)
    return evs
