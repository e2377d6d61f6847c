"""One map write in fp32, as the reference and as the device — TEST INFRASTRUCTURE, not product code.

OccGridMapBase::updateByScan (OccGridMapBase.h:121-168) for one level, restated in numpy operation for operation after
oracle/hs_oracle.c grid_update_by_scan / update_line / bresenham2d (paths relative to
hector_mapping/include/hector_slam_lib/):

  * getMapCoordsPose (GridMapBase.h:235-239): the level's mapTworld applied to the world pose, every product and sum
    rounded, a0 + (a1 + a2);
  * getTransformForState (OccGridMapUtil.h:349-352): Translation(x, y) * Rotation2Df(psi) with libm sinf / cosf;
  * the start cell (int)(T * origo + 0.5f) (:134-137) and each end cell (int)(T * p + 0.5f) (:148-155), truncated
    toward zero, so a coordinate in (-1, 0) after the + 0.5 lands in cell 0;
  * the start == end drop (:158) and the bounds tests of the start and the end cell (:176, :186), x against size_x
    and y against size_y;
  * cell i (0 <= i < ada) of a line in closed form: q(i) = floor((err0 + i * adb) / ada) carries after i steps of
    bresenham2D (:243-260), err0 = ada / 2; the end cell is marked occupied (:211-212).

Per cell the first freeing beam F and the first hitting beam H decide the reference's result (bresenhamCellFree /
bresenhamCellOcc :216-241 with the updateIndex stamps, GridMapLogOdds.h:135-156):

  free only           l + lf
  hit, F < H          fl(fl(l + lf) - lf), then `< 50` decides, then + lo (the free is undone first)
  hit, no F < H       l < 50 ? l + lo : l (a later free is skipped: the cell already carries the occupied stamp)

The device's two-phase writer (update_kernel.cuh) is order-free: every hit cell takes the last rule (SURVEY.md Q10).
`write` returns both planes from the same input, so the two can differ only on freed-then-hit cells where
fl(fl(l + lf) - lf) != l, and `Write.deviation` says where.

A non-finite endpoint (or one beyond 1e9 cells) is dropped by the device; the reference casts it with undefined
behaviour, so `Write.ref_defined` is False for such a scan and its `ref` plane must not be compared with anything.
"""
from __future__ import annotations

import ctypes as C
import ctypes.util
from dataclasses import dataclass

import numpy as np

from oracle.hessian64 import cosf, sinf

f32 = np.float32
FREE, HIT, FREED_THEN_HIT = 1, 2, 3   # Write.cls values; 0 = untouched

_libm = C.CDLL(ctypes.util.find_library("m") or "libm.so.6")
_libm.expf.restype = C.c_float
_libm.expf.argtypes = [C.c_float]


def expf(x) -> np.float32:
    return f32(_libm.expf(float(f32(x))))


def prob(logodds) -> np.ndarray:
    """getGridProbability (GridMapLogOdds.h:163-166): expf(l) / (expf(l) + 1) in fp32 with libm expf, per cell."""
    a = np.asarray(logodds, np.float32)
    vals, inv = np.unique(a.reshape(-1), return_inverse=True)
    out = np.empty(vals.shape, np.float32)
    with np.errstate(invalid="ignore"):
        for k, v in enumerate(vals):
            e = expf(v)
            out[k] = e / (e + f32(1.0))
    return out[inv].reshape(a.shape)


@dataclass
class Level:
    """One level's geometry: size and mapTworld (row-major 2 x 3: [s 0 tx; 0 s ty])."""
    sx: int
    sy: int
    mtw: np.ndarray


def geometry(res: float, sx: int, sy: int, levels: int, start=(0.5, 0.5)) -> list[Level]:
    """MapRepMultiMap's levels (MapRepMultiMap.h:48-72, GridMapBase.h:265-280) in fp32, as hs_oracle.c hso_create."""
    total_x, total_y = f32(res) * f32(sx), f32(res) * f32(sy)
    mid_x, mid_y = total_x * f32(start[0]), total_y * f32(start[1])
    out, r, dx, dy = [], f32(res), int(sx), int(sy)
    for _ in range(levels):
        s = f32(1.0) / r
        out.append(Level(dx, dy, np.array([s, 0.0, s * mid_x, 0.0, s, s * mid_y], np.float32)))
        dx //= 2
        dy //= 2
        r = r * f32(2.0)
    return out


def _affine(m, vx, vy):
    """shim Transform * vector: m0*vx + (m1*vy + m2*1), every operation rounded (hs_oracle.c affine2_apply)."""
    m = [f32(v) for v in m]
    with np.errstate(invalid="ignore", over="ignore"):
        return m[0] * vx + (m[1] * vy + m[2] * f32(1.0)), m[3] * vx + (m[4] * vy + m[5] * f32(1.0))


def _cell(v):
    """(int)(v + 0.5f) for an array of fp32 coordinates; ok = the cast is defined and the device keeps the value."""
    with np.errstate(invalid="ignore", over="ignore"):
        h = np.asarray(v, np.float32) + f32(0.5)
        ok = np.abs(h) < f32(1.0e9)          # the device's sanity test (update_kernel.cuh beam_frame / beam_end)
        defined = np.abs(h) < f32(2.0 ** 31)  # C's float -> int cast (the reference) is defined here
        return np.where(ok, h, f32(0)).astype(np.int64), ok, defined


@dataclass
class Beams:
    """One updateByScan call on one level: the start cell and every beam's end cell and fate."""
    x0: int
    y0: int
    start_ok: bool      # the start cell is a valid cast and inside the level
    x1: np.ndarray
    y1: np.ndarray
    kept: np.ndarray    # (n,) bool: the beam is drawn
    ref_defined: bool


def beams(L: Level, pts, pose_world, origo=(0.0, 0.0), pt_scale: float = 1.0) -> Beams:
    """Start and end cells of a scan (container points in level-0 cells, scaled by pt_scale as setFrom does)."""
    pts = np.asarray(pts, np.float32).reshape(-1, 2)
    pw = np.asarray(pose_world, np.float32).reshape(3)
    mx, my = _affine(L.mtw, pw[0], pw[1])                        # getMapCoordsPose :127
    c, s = cosf(pw[2]), sinf(pw[2])                              # Rotation2Df :130-131
    ps = f32(pt_scale)
    with np.errstate(invalid="ignore", over="ignore"):
        ox, oy = f32(origo[0]) * ps, f32(origo[1]) * ps          # DataPointContainer setFrom (MapRepMultiMap.h:127)
        px, py = pts[:, 0] * ps, pts[:, 1] * ps
        T = (c, -s, mx, s, c, my)
        bx, by = _affine(T, ox, oy)                              # :134
        ex, ey = _affine(T, px, py)                              # :148
    sc, sok, sdef = _cell(np.float32([bx, by]))
    x0, y0 = int(sc[0]), int(sc[1])
    start_ok = bool(sok.all()) and 0 <= x0 < L.sx and 0 <= y0 < L.sy   # :176
    x1, okx, defx = _cell(ex)
    y1, oky, defy = _cell(ey)
    kept = okx & oky & ~((x1 == x0) & (y1 == y0))                # :158
    kept &= (x1 >= 0) & (x1 < L.sx) & (y1 >= 0) & (y1 < L.sy)    # :186
    kept &= start_ok
    ref_defined = bool(sdef.all()) and bool(np.all(defx & defy))
    return Beams(x0, y0, start_ok, x1, y1, kept, ref_defined)


def line_cells(L: Level, b: Beams):
    """Free cells of every kept beam: (flat cell index, beam index), all lines at once (bresenham2D :243-260)."""
    idx = np.nonzero(b.kept)[0]
    if idx.size == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    dx, dy = b.x1[idx] - b.x0, b.y1[idx] - b.y0
    adx, ady = np.abs(dx), np.abs(dy)
    sgx, sgy = np.where(dx > 0, 1, -1), np.where(dy > 0, 1, -1)   # util::sign (UtilFunctions.h:56-59)
    xmaj = adx >= ady                                             # :202
    ada, adb = np.where(xmaj, adx, ady), np.where(xmaj, ady, adx)
    err0 = ada // 2
    beam = np.repeat(np.arange(idx.size), ada)
    i = np.arange(beam.size) - np.repeat(np.cumsum(ada) - ada, ada)
    q = (err0[beam] + i * adb[beam]) // ada[beam]
    xm = xmaj[beam]
    x = b.x0 + sgx[beam] * np.where(xm, i, q)
    y = b.y0 + sgy[beam] * np.where(xm, q, i)
    return y * L.sx + x, idx[beam]


@dataclass
class Write:
    ref: np.ndarray        # the reference's plane after the write
    dev: np.ndarray        # the order-free plane the device is specified to produce
    cls: np.ndarray        # 0 untouched, FREE, HIT, FREED_THEN_HIT
    box: tuple | None      # (x0, y0, x1, y1) inclusive: the start cell and the kept end cells
    deviation: np.ndarray  # bool: freed-then-hit cells where fl(fl(l + lf) - lf) != l
    ref_defined: bool


def write(plane, L: Level, b: Beams, lf, lo) -> Write:
    """The planes after drawing `b` into `plane` (sy, sx) with the increments lf (free) and lo (occupied)."""
    lf, lo = f32(lf), f32(lo)
    l = np.asarray(plane, np.float32).reshape(-1)
    n_cells = L.sx * L.sy
    big = np.iinfo(np.int64).max
    F = np.full(n_cells, big, np.int64)
    H = np.full(n_cells, big, np.int64)
    cells, beam = line_cells(L, b)
    np.minimum.at(F, cells, beam)
    kept = np.nonzero(b.kept)[0]
    np.minimum.at(H, b.y1[kept] * L.sx + b.x1[kept], kept)
    free = (F < big) & (H == big)
    hit = H < big
    fth = hit & (F < H)
    with np.errstate(over="ignore", invalid="ignore"):
        occ = np.where(l < f32(50.0), l + lo, l)                 # updateSetOccupied (GridMapLogOdds.h:135-140)
        back = (l + lf) - lf                                     # updateUnsetFree after updateSetFree (:146-156)
        occ_back = np.where(back < f32(50.0), back + lo, back)
        dev = np.where(free, l + lf, np.where(hit, occ, l)).astype(np.float32)
        ref = np.where(fth, occ_back, dev).astype(np.float32)
    cls = np.zeros(n_cells, np.int8)
    cls[free] = FREE
    cls[hit] = HIT
    cls[fth] = FREED_THEN_HIT
    box = None
    if kept.size:
        box = (int(min(b.x0, b.x1[kept].min())), int(min(b.y0, b.y1[kept].min())),
               int(max(b.x0, b.x1[kept].max())), int(max(b.y0, b.y1[kept].max())))
    shape = (L.sy, L.sx)
    return Write(ref.reshape(shape), dev.reshape(shape), cls.reshape(shape), box, (fth & (back != l)).reshape(shape),
                 b.ref_defined)


def union(a, b):
    if a is None:
        return b
    if b is None:
        return a
    return (min(a[0], b[0]), min(a[1], b[1]), max(a[2], b[2]), max(a[3], b[3]))


class MultiMap:
    """MapRepMultiMap's planes on the CPU (MapRepMultiMap.h:116-147).  `follow` picks which result the planes carry
    from one write to the next: "ref" (the reference's sequence) or "dev" (the device's)."""

    def __init__(self, res, sx, sy, levels, lf, lo, start=(0.5, 0.5), follow="dev"):
        self.lv = geometry(res, sx, sy, levels, start)
        self.planes = [np.zeros((L.sy, L.sx), np.float32) for L in self.lv]
        self.lf, self.lo = f32(lf), f32(lo)
        self.follow = follow
        self.container = None          # the last matched scan and its origo (MapRepMultiMap.h:127)
        self.dirty = [None] * levels   # the union of the boxes since the last reset

    def set_plane(self, level, plane):
        self.planes[level] = np.array(plane, np.float32).reshape(self.planes[level].shape)

    def update_level(self, level, pts_level, pose_world, origo_level=(0.0, 0.0)) -> Write:
        """OccGridMapBase::updateByScan on one level, points already in that level's cells."""
        L = self.lv[level]
        w = write(self.planes[level], L, beams(L, pts_level, pose_world, origo_level), self.lf, self.lo)
        self.planes[level] = w.ref if self.follow == "ref" else w.dev
        self.dirty[level] = union(self.dirty[level], w.box)
        return w

    def match(self, pts, origo=(0.0, 0.0)):
        """What matchData leaves behind for the map write: the scan becomes the coarse levels' container."""
        pts = np.asarray(pts, np.float32).reshape(-1, 2)
        if pts.shape[0]:
            self.container = (pts.copy(), (f32(origo[0]), f32(origo[1])))
        else:
            self.container = (pts.copy(), (f32(0), f32(0)))

    def update_by_scan(self, pts, pose_world, origo=(0.0, 0.0)) -> list:
        """MapRepMultiMap::updateByScan (:134-147): level 0 from `pts`, level l > 0 from the last matched scan scaled by
        1 / 2^l with its origo (SURVEY.md Q11).  Returns one Write per level (None where there is nothing to draw)."""
        out = []
        for l, L in enumerate(self.lv):
            if l == 0:
                src, og = np.asarray(pts, np.float32).reshape(-1, 2), origo
            elif self.container is None:
                out.append(None)
                continue
            else:
                src, og = self.container
            scale = float(f32(1.0 / 2.0 ** l))
            w = write(self.planes[l], L, beams(L, src, pose_world, og, scale), self.lf, self.lo)
            self.planes[l] = w.ref if self.follow == "ref" else w.dev
            self.dirty[l] = union(self.dirty[l], w.box)
            out.append(w)
        return out


# ---- scan families in a level's cells ------------------------------------------------------------------------------
# TL = 64 lanes per team and U * TL = 256 cells per pass are the boundaries of the device's mark loop
LENGTHS = (1, 2, 63, 64, 65, 255, 256, 257)
DIRS = ((1, 0), (0, 1), (-1, 0), (0, -1), (1, 1), (1, -1), (-1, 1), (-1, -1),
        (2, 1), (1, 2), (-1, 2), (-2, 1), (-2, -1), (-1, -2), (1, -2), (2, -1))


def pose_for_cell(L: Level, cx, cy, psi=0.0) -> np.ndarray:
    """A world pose whose map coordinates on level L are (cx, cy) up to rounding."""
    m = L.mtw.astype(np.float64)
    return np.float32([(cx - m[2]) / m[0], (cy - m[5]) / m[4], psi])


def points_for_targets(L: Level, pose_world, targets, pt_scale: float = 1.0) -> np.ndarray:
    """Container points (level-0 cells when pt_scale = 2^-l) whose end cells on level L are near `targets` (level cells,
    an integer target c ends in cell c: c + 0.5 truncates to c with half a cell to spare)."""
    pw = np.asarray(pose_world, np.float32).astype(np.float64)
    mx, my = _affine(L.mtw, f32(pw[0]), f32(pw[1]))
    c, s = float(cosf(pw[2])), float(sinf(pw[2]))
    t = np.asarray(targets, np.float64).reshape(-1, 2)
    dx, dy = t[:, 0] - float(mx), t[:, 1] - float(my)
    px, py = c * dx + s * dy, -s * dx + c * dy
    return (np.stack([px, py], axis=1) / pt_scale).astype(np.float32)


def family_targets(L: Level, start, rng, n_random: int = 48) -> np.ndarray:
    """End-cell targets around the start cell: lines in all eight octants (and the axes and exact diagonals) of every
    length in LENGTHS and one longer than the level; end cells on 0, sx-1, sy-1, one past each edge, in (-1, 0) (cell
    0 by truncation) and just beyond it; end == start; several beams ending in one cell; a cell freed by an earlier
    beam and hit by a later one and the reverse order; random ends in and around the level."""
    x0, y0 = float(start[0]), float(start[1])
    t = []
    for a, b in DIRS:
        m = max(abs(a), abs(b))
        for n in LENGTHS + (max(L.sx, L.sy) + 3,):
            t.append((x0 + (a * n) // m, y0 + (b * n) // m))
    xs = (0.0, 1.0, L.sx - 2.0, L.sx - 1.0, float(L.sx), -1.0, -0.7, -1.6)
    ys = (0.0, 1.0, L.sy - 2.0, L.sy - 1.0, float(L.sy), -1.0, -0.7, -1.6)
    for x in xs:
        for y in (ys + (y0,)):
            t.append((x, y))
    for y in ys:
        t.append((x0, y))
    t += [(x0, y0), (x0 + 0.3, y0 - 0.4)]                               # end == start
    t += [(x0 + 5, y0 + 3)] * 3 + [(x0 - 4, y0 + 7)] * 2                # several beams, one end cell
    t += [(x0 + 40, y0), (x0 + 20, y0)]                                 # freed by the earlier beam, hit by the later
    t += [(x0 + 17, y0 + 17), (x0 + 33, y0 + 33)]                       # hit first, the later beam's free is skipped
    t += [(x0 - 30, y0 + 15), (x0 - 10, y0 + 5), (x0 - 12, y0 + 6)]
    t += list(zip(rng.uniform(-3, L.sx + 3, n_random), rng.uniform(-3, L.sy + 3, n_random)))
    return np.asarray(t, np.float64)


# log-odds the preloaded planes draw from: around 0, straddling +-0.5, 1, 2 and 32 (where l and l + lf sit in
# different binades), just below, at and above the `< 50` clamp, and very negative
_N = np.nextafter


def _around(v):
    v = f32(v)
    return [_N(v, f32(-np.inf)), v, _N(v, f32(np.inf))]


PRELOAD = np.float32(sum((_around(v) + _around(-v) for v in (0.5, 1.0, 2.0, 32.0)), [])
                     + _around(50.0) + [0.0, 1e-3, -1e-3, 0.49, 0.51, 0.3, -0.3, 0.8, 1.3, 2.2, 31.7, 32.3,
                                        49.0, 49.5, 49.99, 50.3, 51.0, 60.0, -60.0, -1000.0, -1e4])


def preload(shape, rng, uniform: bool = True) -> np.ndarray:
    """A plane of PRELOAD values and (uniform) as many uniform draws in [-60, 50]."""
    a = rng.choice(PRELOAD, size=shape).astype(np.float32)
    if not uniform:
        return a
    u = rng.uniform(-60, 50, size=shape).astype(np.float32)
    return np.where(rng.random(shape) < 0.5, a, u).astype(np.float32)
