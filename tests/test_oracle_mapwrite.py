"""CPU: oracle/mapwrite.py's reference plane (the map write in fp32, beam order included) is the compiled reference's
and the C port's bit for bit — OccGridMapBase::updateByScan on one level and MapRepMultiMap::updateByScan on all
levels, square and non-square maps with every width residue mod 4, several consecutive scans on preloaded planes —
and its probability is getGridProbability's."""
import numpy as np
import pytest

from oracle import mapwrite as mw

# (size_x, size_y, levels): the widths written cover every residue mod 4 (404 / 202 / 101, 150 / 75, 243 / 121, 7, 5)
MAPS = [(64, 64, 2), (404, 300, 3), (150, 404, 2), (243, 200, 2), (257, 131, 2), (5, 7, 1), (7, 4, 1)]


def _oracle(pyoracle, kind, res, sx, sy, levels, ffree=0.4, focc=0.9):
    if not pyoracle.available(kind):
        pytest.skip(f"{kind} oracle not built")
    orc = pyoracle.Oracle(kind, res, sx, levels, size_y=sy)
    orc.set_update_factors(ffree, focc)
    return orc


def _same(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


def _scan(L, start_cell, psi, rng, origo=(0.0, 0.0), pt_scale=1.0):
    pose = mw.pose_for_cell(L, start_cell[0], start_cell[1], psi)
    return pose, mw.points_for_targets(L, pose, mw.family_targets(L, start_cell, rng), pt_scale)


def _starts(L):
    """start cells: the middle, near a corner, on the first and the last column, outside the level"""
    return [(L.sx // 2, L.sy // 2), (min(3, L.sx - 1), min(2, L.sy - 1)), (0, L.sy // 2), (L.sx - 1, L.sy - 1),
            (L.sx // 2, L.sy - 1), (-3, L.sy // 2)]


@pytest.mark.parametrize("kind", ["port", "reference"])
@pytest.mark.parametrize("geom", MAPS, ids=lambda g: "x".join(map(str, g)))
def test_update_level_matches_oracle(pyoracle, kind, geom):
    sx, sy, levels = geom
    orc = _oracle(pyoracle, kind, 0.05, sx, sy, levels)
    lf, lo = orc.logodds_increments()
    model = mw.MultiMap(0.05, sx, sy, levels, lf, lo, follow="ref")
    rng = np.random.default_rng(sx * 1000 + sy)
    counts = np.zeros(4, np.int64)
    for l, L in enumerate(model.lv):
        assert (orc.level_size(l)) == (L.sx, L.sy)
        plane = mw.preload((L.sy, L.sx), rng)
        orc.set_logodds(l, plane)
        model.set_plane(l, plane)
        for k, st in enumerate(_starts(L)):
            psi = (0.0, 0.3, -2.0, 1.5707964)[k % 4]
            pose, pts = _scan(L, st, psi, rng)
            origo = (0.0, 0.0) if k % 2 == 0 else (0.25, -0.5)
            w = model.update_level(l, pts, pose, origo)
            orc.update_level(l, pts, pose, origo)
            assert w.ref_defined
            assert _same(orc.get_logodds(l), model.planes[l]), (kind, geom, l, k)
            counts += np.bincount(w.cls.reshape(-1), minlength=4)
        assert _same(orc.get_prob(l), mw.prob(model.planes[l])), (kind, geom, l)
    assert counts[mw.FREED_THEN_HIT] > 0 and counts[mw.HIT] > 0 and counts[mw.FREE] > 0
    orc.close()


@pytest.mark.parametrize("kind", ["port", "reference"])
@pytest.mark.parametrize("geom", [(404, 300, 3), (243, 200, 2), (150, 404, 2)], ids=lambda g: "x".join(map(str, g)))
def test_update_by_scan_matches_oracle(pyoracle, kind, geom):
    """MapRepMultiMap::updateByScan: level 0 from the given scan, the coarse levels from the last matched scan (scaled by
    1 / 2^l, with its origo), which need not be the written one (SURVEY.md Q11)."""
    sx, sy, levels = geom
    orc = _oracle(pyoracle, kind, 0.05, sx, sy, levels, 0.35, 0.8)
    lf, lo = orc.logodds_increments()
    model = mw.MultiMap(0.05, sx, sy, levels, lf, lo, follow="ref")
    rng = np.random.default_rng(7 + sx)
    for l, L in enumerate(model.lv):
        plane = mw.preload((L.sy, L.sx), rng)
        orc.set_logodds(l, plane)
        model.set_plane(l, plane)
    L0 = model.lv[0]
    for k in range(4):
        pose_a, scan_a = _scan(L0, (sx // 2 + 3 * k, sy // 2 - 2 * k), 0.2 * k, rng)
        origo_a = np.float32([0.5 * k, -0.25 * k])
        orc.match(pose_a, scan_a, origo_a)           # fills the coarse containers; the map is not touched
        model.match(scan_a, origo_a)
        if k % 2:
            pose_b, scan_b, origo_b = pose_a, scan_a, origo_a
        else:                                         # written: another scan at another pose
            pose_b, scan_b = _scan(L0, (sx // 3, sy // 3 + k), -0.7, rng)
            origo_b = np.float32([-1.0, 0.5])
        ws = model.update_by_scan(scan_b, pose_b, origo_b)
        orc.update_by_scan(scan_b, pose_b, origo_b)
        for l in range(levels):
            assert ws[l].ref_defined
            assert _same(orc.get_logodds(l), model.planes[l]), (kind, geom, k, l)
    orc.close()


def test_prob_is_libm_expf():
    """mapwrite.prob against the float64 formula, within a few fp32 roundings (expf overflows beyond 88.7, where the
    reference's probability is inf / inf; the log-odds written here stay far below)."""
    v = np.concatenate([mw.PRELOAD, np.linspace(-80, 80, 2001, dtype=np.float32)]).astype(np.float32)
    p = mw.prob(v).astype(np.float64)
    e = np.exp(v.astype(np.float64))
    want = e / (e + 1.0)
    assert np.all(np.abs(p - want) <= 4 * np.spacing(np.float32(1.0)) * np.maximum(want, 1e-30) + 1e-45)
    assert mw.prob(np.float32([50.0]))[0] == np.float32(1.0) and mw.prob(np.float32([0.0]))[0] == np.float32(0.5)


def test_q10_deviation_is_exactly_the_round_trip():
    """The ref and dev planes of one write differ only on freed-then-hit cells whose l does not survive
    fl(fl(l + lf) - lf) (the final + lo may round both back together), by at most 2 ulp of |l| + |lf| (SURVEY.md
    Q10: l and l + lf straddle a power of two), for the default increments."""
    rng = np.random.default_rng(3)
    L = mw.geometry(0.05, 300, 300, 1)[0]
    lf, lo = mw.f32(np.log(np.float32(0.4) / np.float32(0.6))), mw.f32(np.log(np.float32(0.6) / np.float32(0.4)))
    n_fth = n_dev = 0
    for k in range(6):
        plane = mw.preload((L.sy, L.sx), rng)
        st = (150 + 7 * k, 150 - 5 * k)
        pose = mw.pose_for_cell(L, st[0], st[1], 0.4 * k)
        pts = mw.points_for_targets(L, pose, mw.family_targets(L, st, rng, 400))
        w = mw.write(plane, L, mw.beams(L, pts, pose), lf, lo)
        diff = w.ref.view(np.uint32) != w.dev.view(np.uint32)
        assert not np.any(diff & ~w.deviation)
        assert np.all(w.cls[diff] == mw.FREED_THEN_HIT)
        err = np.abs(w.ref.astype(np.float64) - w.dev.astype(np.float64))[diff]
        assert np.all(err <= 2 * np.spacing(np.abs(plane[diff]) + np.abs(lf)).astype(np.float64))
        n_fth += int((w.cls == mw.FREED_THEN_HIT).sum())
        n_dev += int(diff.sum())
    assert n_fth > 0 and n_dev > 0
