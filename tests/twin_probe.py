"""The one-texel likelihood probe of a level's probability plane, shared by the GPU map tests.

A one-endpoint likelihood at an integer cell (x <= sx-2, y <= sy-2: the interpolation's bounds) has bilinear weights 1
and 0, so it reads exactly that cell's P and returns 1 - (1 - P): in TEX mode the texture twin, in LDG mode the
probability plane.  Any addressing error of the twin, or a twin that was not rewritten, shows.
"""
import numpy as np

from oracle import mapwrite as mw


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def probe_points(rep, level, cells):
    """One container point per cell (level-0 cells) whose likelihood endpoint at world pose (0, 0, 0) is exactly the
    integer cell: qx = fl(2^-l * px + tx) (match_kernel.cuh point_address with psi = 0)."""
    t = rep.map_coords_pose(level, [0.0, 0.0, 0.0])
    sc = np.float32(2.0 ** -level)
    out = np.zeros((cells.shape[0], 2), np.float32)
    for k in range(2):
        want = cells[:, k].astype(np.float32)
        p = ((want.astype(np.float64) - float(t[k])) / float(sc)).astype(np.float32)
        for _ in range(4):
            q = p * sc + t[k]
            p = np.where(q < want, np.nextafter(p, np.float32(np.inf)), np.where(q > want, np.nextafter(p, np.float32(-np.inf)), p))
        assert np.array_equal(p * sc + t[k], want)
        out[:, k] = p
    return out


def probe_twin(rep, level, L, plane, rect, what, max_cells=60000):
    """The probe at every integer cell of `rect` (the box's border and a sample of its inside when it is large):
    the likelihood must be 1 - (1 - P) of mapwrite.prob(plane) bit for bit."""
    if rect is None:
        return
    x0, y0, x1, y1 = rect
    x1, y1 = min(x1, L.sx - 2), min(y1, L.sy - 2)
    if x1 < x0 or y1 < y0:
        return
    ys, xs = np.mgrid[y0:y1 + 1, x0:x1 + 1]
    cells = np.stack([xs.reshape(-1), ys.reshape(-1)], axis=1)
    if cells.shape[0] > max_cells:   # the box's border and a sample of its inside
        rng = np.random.default_rng(cells.shape[0])
        border = (cells[:, 0] == x0) | (cells[:, 0] == x1) | (cells[:, 1] == y0) | (cells[:, 1] == y1)
        inner = np.nonzero(~border)[0]
        cells = np.concatenate([cells[border], cells[rng.choice(inner, min(max_cells, inner.size), replace=False)]])
    pts = probe_points(rep, level, cells)
    B = cells.shape[0]
    lh = rep.likelihood_batch(level, np.zeros((B, 3), np.float32), pts, np.arange(B + 1, dtype=np.int32))
    P = mw.prob(plane)[cells[:, 1], cells[:, 0]]
    want = np.float32(1.0) - (np.float32(1.0) - P)
    bad = bits(lh) != bits(want)
    assert not bad.any(), (what, level, int(bad.sum()), cells[bad][:5].tolist())
