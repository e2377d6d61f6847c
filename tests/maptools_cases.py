"""Maps and rays for hector_map_tools' ray cast and getDist (checkOccupancyBresenhami / getDist, HectorMapTools.h:133-237)
and for the occupancy export, shared by the CPU test of the C port and the GPU test of the device.

The geometries are the map writer's (every width residue mod 4, square and not, wide and tall), two of them with a
non-default start, and two long single-level maps, 6000 x 100 and 100 x 6000, on which rays run longer than
bresenham2D's 5000-step cap in both dominant directions.  The long maps are 100 cells across because the first offsets
whose fp32 distance sum lands on the other side of a perfect square than the exact sum have a minor component of 91.

Every ray set is built from a seed, so the CPU and the GPU test see the same rays.
"""
from dataclasses import dataclass

import numpy as np

from oracle import mapwrite as mw

f32 = np.float32
RES = 0.05
MIN_DENORMAL = np.nextafter(f32(0), f32(1))
# (sx, sy, levels, start)
GEOMS = [(404, 300, 3, (0.5, 0.5)), (150, 404, 2, (0.3, 0.7)), (243, 200, 2, (0.5, 0.5)), (257, 131, 1, (0.5, 0.5)),
         (5, 7, 1, (0.3, 0.7)), (7, 4, 1, (0.5, 0.5)), (6000, 100, 1, (0.3, 0.7)), (100, 6000, 1, (0.7, 0.2))]
LONG = [g for g in GEOMS if max(g[0], g[1]) > 5000]
CAP = 5000   # bresenham2D's max_length as checkOccupancyBresenhami passes it (HectorMapTools.h:173-179)
# the values the occupancy export and the ray cast have to classify: isFree / isOccupied are strict comparisons with 0
SPECIAL = f32([-0.0, 0.0, MIN_DENORMAL, -MIN_DENORMAL, np.inf, -np.inf, np.nan, 50.0])


def geom_id(g):
    return f"{g[0]}x{g[1]}x{g[2]}"


def level_sizes(g):
    sx, sy, levels, _ = g
    return [(sx >> l, sy >> l) for l in range(levels)]


def occupancy(plane):
    """HectorMappingRos::publishMap's cell values (HectorMappingRos.cpp:448-468): 0 free (l < 0), 100 occupied
    (l > 0), -1 otherwise (0, -0 and NaN)."""
    p = np.asarray(plane, np.float32)
    out = np.full(p.shape, -1, np.int8)
    with np.errstate(invalid="ignore"):
        out[p < 0] = 0
        out[p > 0] = 100
    return out


def plane(sx, sy, seed, occupied=None):
    """A log-odds plane: mapwrite.PRELOAD values and uniform draws, a fraction `occupied` of the cells made positive
    and the rest negative, the SPECIAL values planted at the four corners, along the last row and column and at
    random cells."""
    rng = np.random.default_rng(seed)
    if occupied is None:
        occupied = 0.3 if sx * sy < 100 else 0.03
    base = np.abs(mw.preload((sy, sx), rng))
    p = np.where(rng.random((sy, sx)) < occupied, base, -base).astype(np.float32)
    corners = [(0, 0), (0, sx - 1), (sy - 1, 0), (sy - 1, sx - 1)]
    for k, (y, x) in enumerate(corners):
        p[y, x] = SPECIAL[(k + seed) % SPECIAL.size]
    p[sy - 1, ::7] = np.resize(SPECIAL, p[sy - 1, ::7].shape)
    p[::5, sx - 1] = np.resize(SPECIAL[::-1], p[::5, sx - 1].shape)
    n = max(8, sx * sy // 200)
    p[rng.integers(0, sy, n), rng.integers(0, sx, n)] = rng.choice(SPECIAL, n)
    return p


def cell_rays(sx, sy, occ, seed, n_random=1500):
    """(begin, end) int32 (B, 2) cell rays on one level with occupancy `occ`: random rays in and around the level,
    begins on occupied cells (distance 0), begin == end, ends and begins on and one past every edge, coordinates in
    [min(sx, sy), max(sx, sy)) on both axes (inside along the long axis, outside along the short one).  A level of
    fewer than 100 cells gets every ray between the cells of the level and its one-cell border."""
    rng = np.random.default_rng(seed)
    if sx * sy < 100:
        ys, xs = np.mgrid[-1:sy + 1, -1:sx + 1]
        c = np.stack([xs.reshape(-1), ys.reshape(-1)], axis=1)
        i, j = np.meshgrid(np.arange(c.shape[0]), np.arange(c.shape[0]), indexing="ij")
        return c[i.reshape(-1)].astype(np.int32), c[j.reshape(-1)].astype(np.int32)

    def inside(n):
        return np.stack([rng.integers(0, sx, n), rng.integers(0, sy, n)], axis=1)

    b, e = [], []
    b.append(np.stack([rng.integers(-2, sx + 2, n_random), rng.integers(-2, sy + 2, n_random)], axis=1))
    e.append(np.stack([rng.integers(-2, sx + 2, n_random), rng.integers(-2, sy + 2, n_random)], axis=1))
    occ_cells = np.argwhere(occ == 100)[:, ::-1]
    k = occ_cells[rng.choice(occ_cells.shape[0], 24)]
    b.append(k)
    e.append(inside(24))
    s = inside(24)
    s[:8] = k[:8]
    b.append(s)
    e.append(s)
    edges = []
    for y in (rng.integers(0, sy), 0, sy - 1):
        edges += [(-1, y), (0, y), (sx - 1, y), (sx, y)]
    for x in (rng.integers(0, sx), 0, sx - 1):
        edges += [(x, -1), (x, 0), (x, sy - 1), (x, sy)]
    edges += [(-1, -1), (sx, sy), (-1, sy), (sx, -1), (0, 0), (sx - 1, sy - 1), (sx - 1, 0), (0, sy - 1)]
    edges = np.asarray(edges)
    m = edges.shape[0]
    b += [inside(m), edges]
    e += [edges, inside(m)]
    lo, hi = min(sx, sy), max(sx, sy)
    if hi > lo:
        n = 64
        t = rng.integers(lo, hi, n)
        u = np.stack([rng.integers(0, lo, n), t], axis=1)     # (short-axis coordinate, long-axis coordinate)
        along_long = u if sy > sx else u[:, ::-1]             # inside: the long coordinate on the long axis
        across = along_long[:, ::-1]                          # the transposed cells: outside
        b += [inside(n), along_long, inside(n), across]
        e += [along_long, inside(n), across, inside(n)]
    return np.concatenate(b).astype(np.int32), np.concatenate(e).astype(np.int32)


def world_rays(sx, sy, origin, cell, seed, n_random=600):
    """(begin, end) float32 (B, 2) world points for getDist: random points in and around the level, begins whose cell
    coordinate lies in (-1, 0) (truncated to 0: inside), and NaN begins and ends.  -> (begin, end, mask of the NaN
    rays)"""
    rng = np.random.default_rng(seed)
    o = np.asarray(origin, np.float32)
    c = f32(cell)

    def world(cx, cy):
        return (o + np.stack([cx, cy], axis=1).astype(np.float32) * c).astype(np.float32)

    b = [world(rng.uniform(-3, sx + 3, n_random), rng.uniform(-3, sy + 3, n_random))]
    e = [world(rng.uniform(-3, sx + 3, n_random), rng.uniform(-3, sy + 3, n_random))]
    n = 48
    frac = -rng.uniform(0.05, 0.95, n)
    b.append(world(frac, rng.uniform(0, sy, n)))
    b.append(world(rng.uniform(0, sx, n), frac))
    b.append(world(frac, frac))
    e += [world(rng.uniform(0, sx, n), rng.uniform(0, sy, n)) for _ in range(3)]
    nb = world(rng.uniform(0, sx, 4), rng.uniform(0, sy, 4))
    ne = world(rng.uniform(0, sx, 4), rng.uniform(0, sy, 4))
    nb[0, 0] = nb[2] = np.nan
    ne[1, 1] = ne[3, 0] = np.nan
    b.append(nb)
    e.append(ne)
    b, e = np.concatenate(b).astype(np.float32), np.concatenate(e).astype(np.float32)
    is_nan = np.isnan(b).any(axis=1) | np.isnan(e).any(axis=1)
    assert is_nan.sum() == 4
    return b, e, is_nan


def fp32_dist(dx, dy):
    """int distMap = (float vector).norm() (HectorMapTools.h:194): fl(fl(dx^2) + fl(dy^2)), sqrtf, truncation."""
    fx, fy = f32(dx), f32(dy)
    return int(np.sqrt(f32(fx * fx + fy * fy)))


def near_square_offsets(minor_max):
    """(major, minor) hit offsets, 4096 < major < CAP, 0 <= minor <= minor_max, where the fp32 sum of squares and the
    exact one fall on different sides of a perfect square, or where a fused multiply-add on the major axis' square
    (one rounding instead of two) does: the truncated distance differs from the exact one, or from the fused one."""
    major = np.arange(4097, CAP, dtype=np.int64)[:, None]
    minor = np.arange(0, minor_max + 1, dtype=np.int64)[None, :]
    fa, fb = major.astype(np.float32), minor.astype(np.float32)
    ref = np.sqrt(fa * fa + fb * fb).astype(np.int64)
    exact = np.floor(np.sqrt((major * major + minor * minor).astype(np.float64))).astype(np.int64)
    fused = np.sqrt((major * major + (fb * fb).astype(np.int64)).astype(np.float64).astype(np.float32)).astype(np.int64)
    out = []
    for kind, other in (("exact", exact), ("fused", fused)):
        for a, b in np.argwhere(ref != other):
            out.append((int(major[a, 0]), int(minor[0, b]), kind, int(ref[a, b]), int(other[a, b])))
    return out


@dataclass
class LoneCase:
    """One ray over a level whose only occupied cell is `cell`; `hit`: the ray must stop there."""
    name: str
    cell: tuple
    begin: tuple
    end: tuple
    hit: bool
    dist: int = -1


def line_cell(begin, end, i):
    """Cell i of bresenham2D's walk from begin towards end (closed form: carries after i steps)."""
    dx, dy = end[0] - begin[0], end[1] - begin[1]
    adx, ady = abs(dx), abs(dy)
    sx, sy = (1 if dx > 0 else -1), (1 if dy > 0 else -1)
    ada, adb = (adx, ady) if adx >= ady else (ady, adx)
    q = (ada // 2 + i * adb) // ada
    a, b = (i, q) if adx >= ady else (q, i)
    return begin[0] + sx * a, begin[1] + sy * b


def lone_cases(sx, sy):
    """Constructed rays on a long level: the 5000-step cap, the last step before the end cell, and hit offsets whose
    distance is near a perfect square, in all four octant mirrors."""
    wide = sx > sy
    W, S = (sx, sy) if wide else (sy, sx)

    def orient(p):                        # (long-axis, short-axis) -> (x, y)
        return (p[0], p[1]) if wide else (p[1], p[0])

    out = []

    def add(name, begin, end, i, hit):
        b, e = orient(begin), orient(end)
        c = line_cell(b, e, i)
        out.append(LoneCase(name, c, b, e, hit, fp32_dist(b[0] - c[0], b[1] - c[1]) if hit else -1))

    rows = [(0, S - 1), (S // 3, S // 3), (S - 1, 0), (S // 2, S - 1)]   # begin / end short-axis coordinates
    for k, (r0, r1) in enumerate(rows):
        for fwd in (True, False):
            b, e = ((0, r0), (W - 1, r1)) if fwd else ((W - 1, r0), (0, r1))
            d = "fwd" if fwd else "back"
            add(f"cap step {CAP - 1} {d} {k}", b, e, CAP - 1, True)
            add(f"cap step {CAP} {d} {k}", b, e, CAP, False)
            add(f"cap step {CAP + 1} {d} {k}", b, e, CAP + 1, False)
    for k, (b, e) in enumerate([((3, 5), (2000, S - 7)), ((W - 2, S - 1), (W - 1800, 0)), ((10, 0), (10 + CAP, S - 1))]):
        ada = max(abs(e[0] - b[0]), abs(e[1] - b[1]))
        add(f"step ada-1 {k}", b, e, ada - 1, True)
        add(f"step ada (the end cell) {k}", b, e, ada, False)
    for major, minor, kind, _, _ in near_square_offsets(S - 1):
        for gx in (1, -1):
            for gy in (1, -1):
                x0 = 0 if gx > 0 else W - 1
                y0 = 0 if gy > 0 else S - 1
                b = (x0, y0)
                e = (x0 + gx * (major + 1), y0 + gy * minor)
                add(f"near square {kind} {major},{minor} {gx:+d}{gy:+d}", b, e, major, True)
                assert out[-1].cell == orient((x0 + gx * major, y0 + gy * minor))
    return out


def lone_plane(sx, sy, cell, seed):
    """A level with one occupied cell: the rest free, unknown, -0, NaN, -inf or a negative denormal."""
    rng = np.random.default_rng(seed)
    p = rng.choice(f32([-2.0, -0.4, 0.0, -0.0, np.nan, -np.inf, -MIN_DENORMAL]), size=(sy, sx)).astype(np.float32)
    p[cell[1], cell[0]] = f32(0.75)
    return p
