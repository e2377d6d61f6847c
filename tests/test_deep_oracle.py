"""CPU: the oracles on maps of four to eight levels (tests/deep_cases.py) against the compiled reference, so that what
the device is compared with at depth is itself pinned: oracle/hs_oracle.c (its per-level containers, indexed level - 1),
oracle/port_record.c, oracle/record_oracle.py and oracle/mapwrite.py::MultiMap.

  * The port's record reduced to the hooks' view equals what the reference's ScanMatcher reports to its hooks bit for
    bit, on every geometry, under every schedule (all eight max_iterations entries in use) and the edge scans' own, and
    every recorded H / dTr equals getCompleteHessianDerivs at the recorded pose on every level.
  * A 14-step HectorSlamProcessor::update run from an empty map with three map_without_matching steps (the coarse
    levels then write from the stale containers, levels - 1 of them): poses, covariances and every plane of the port
    equal MapRepMultiMap's bit for bit, and mapwrite.MultiMap's `ref` planes equal both on every level.
  * tests/golden/deep.npz is reproduced bit-exactly by the port everywhere (tests/test_oracle_golden.py) and by the
    compiled reference where it is built (here).

Skipped where oracle/_ref is absent, apart from the geometry facts.
"""
import numpy as np
import pytest

import deep_cases as dc
import match_cases as mcs
from conftest import load_golden
from oracle import gen_golden, mapwrite as mw
from test_match_record_oracle import bits, rec_oracle  # noqa: F401 (rec_oracle: a fixture)


def test_geometries_are_what_the_halving_gives():
    w = [s[0] for s in mcs.level_sizes(dc.GEOMS[0])]
    assert w == [1000, 500, 250, 125, 62, 31, 15, 7] and {v % 4 for v in w[1:]} == {0, 1, 2, 3}
    assert [s[1] for s in mcs.level_sizes(dc.GEOMS[0])][-1] == 5
    assert [s[0] for s in mcs.level_sizes(dc.GEOMS[1])] == [515, 257, 128, 64, 32, 16, 8]
    for g in dc.GEOMS[3:]:
        assert min(mcs.level_sizes(g)[-1]) == 4
    for sx, sy, L in dc.REJECTED:
        assert min(sx >> (L - 1), sy >> (L - 1)) == 3
    assert dc.record_floats(8) == 8 * 3 + 15 * (6 + 7 * 4)
    assert dc.record_floats(8, dc.schedule("mixed", 8)) == 8 * 3 + 15 * (6 + 1 + 3 + 8 + 1 + 2 + 4 + 5)
    assert dc.record_floats(5, dc.schedule("single", 5)) == 5 * 18


def oracles(rec_oracle, g):
    sx, sy, L, start, res = g
    out = [rec_oracle.RecordOracle(k, res, sx, L, start=start, size_y=sy) for k in ("port", "reference")]
    for o in out:
        for l, size in enumerate(mcs.level_sizes(g)):
            assert o.level_size(l) == size
    return out


@pytest.mark.parametrize("gi", range(len(dc.GEOMS)), ids=dc.IDS)
def test_deep_port_record_equals_reference(rec_oracle, gi):
    if not rec_oracle.available("reference"):
        pytest.skip("compiled reference not built")
    g = dc.GEOMS[gi]
    L = g[2]
    po, ro = oracles(rec_oracle, g)
    dc.set_fields(g, po, ro)
    for l in range(L):
        assert np.array_equal(bits(po.get_prob(l)), bits(ro.get_prob(l))), l
    cases = mcs.Cases(g, [po.get_prob(l) for l in range(L)], po, seed=300 + gi)
    it = mcs.edge_iterations(L)
    scans, designed, _ = dc.designed_scans(
        g, cases, lambda h, p: mcs.split_record(po.match_record(h, p, it)[2], L, it))
    for l in range(L):   # the conversions the hand-offs use, on every level
        for h, _, _ in scans:
            m = po.map_coords_pose(l, h)
            assert np.array_equal(bits(m), bits(ro.map_coords_pose(l, h))), l
            assert np.array_equal(bits(po.world_coords_pose(l, m)), bits(ro.world_coords_pose(l, m))), l
    undefined = []
    for iters in [dc.schedule(s, L) for s in dc.SCHEDULES] + [it]:
        mis = po.level_iterations(iters)
        for hint, scan, tag in scans:
            pp, cp, rec = po.match_record(hint, scan, iters)
            assert rec.size == dc.record_floats(L, iters)
            if not np.all(np.isfinite(rec)):
                # a singular solve on a 4-cell level made the pose NaN: the reference would index the map with a NaN
                # endpoint's cell (SURVEY.md Q4), which is undefined
                assert not dc.has_edges(g), (tag, iters)
                undefined.append((tag, iters))
                continue
            pr, cr, hooks, _ = ro.match_record(hint, scan, iters)
            assert np.array_equal(bits(pp), bits(pr)) and np.array_equal(bits(cp), bits(cr)), (tag, iters)
            assert np.array_equal(bits(rec_oracle.port_hooks(po, rec, scan.shape[0], iters)), bits(hooks)), (tag, iters)
            if scan.shape[0] == 0:
                continue
            off = 0
            for l in range(L - 1, -1, -1):
                E = mis[l] + 1
                ev = rec[off + 3:off + 3 + 15 * E].reshape(E, 15)
                pin = ro.map_coords_pose(l, rec[off:off + 3])
                pl = (scan * np.float32(2.0 ** -l)).astype(np.float32)
                for e in range(E):
                    H, d = ro.hessian_derivs(l, pin, pl)
                    assert np.array_equal(bits(H.reshape(9)), bits(ev[e, :9])), (tag, iters, l, e)
                    assert np.array_equal(bits(d), bits(ev[e, 9:12])), (tag, iters, l, e)
                    pin = ev[e, 12:15]
                off += 3 + 15 * E
    assert len(undefined) <= 4, undefined
    po.close()
    ro.close()


@pytest.mark.parametrize("gi", range(len(dc.GEOMS)), ids=dc.IDS)
def test_deep_slam_run_port_reference_and_mapwrite(rec_oracle, gi):
    if not rec_oracle.available("reference"):
        pytest.skip("compiled reference not built")
    g = dc.GEOMS[gi]
    sx, sy, L, start, res = g
    po, ro = oracles(rec_oracle, g)
    for o in (po, ro):
        o.set_update_factors(0.4, 0.9)
        o.set_map_update_thresholds(0.0, 0.0)
    lf, lo = po.logodds_increments()
    assert np.array_equal(bits(po.logodds_increments()), bits(ro.logodds_increments()))
    model = mw.MultiMap(res, sx, sy, L, lf, lo, start=start, follow="ref")
    scans, mwm, hints, _ = gen_golden.deep_run(g)
    assert len(scans) >= 12 and mwm.any() and not mwm[0]
    written = np.zeros(L, bool)
    for k in range(len(scans)):
        hint = hints[k]
        pp, cp = po.update(scans[k], hint, map_without_matching=bool(mwm[k]))
        pr, cr = ro.update(scans[k], hint, map_without_matching=bool(mwm[k]))
        assert np.array_equal(bits(pp), bits(pr)) and np.array_equal(bits(cp), bits(cr)), k
        if mwm[k]:
            assert np.array_equal(bits(pp), bits(hint)), k
        else:
            model.match(scans[k])
        ws = model.update_by_scan(scans[k], pp)
        assert all(w.ref_defined for w in ws)
        for l in range(L):
            a, b = po.get_logodds(l), ro.get_logodds(l)
            assert np.array_equal(bits(a), bits(b)), (k, l)
            assert np.array_equal(bits(model.planes[l]), bits(b)), (k, l)
            if mwm[k]:
                written[l] |= bool(ws[l].box is not None)
    # where the map holds the scans at all, the stale containers wrote every coarse level
    if min(sx, sy) >= 500:
        assert written.all(), written
    for l in range(L):
        assert np.array_equal(bits(po.get_prob(l)), bits(ro.get_prob(l))), l
    po.close()
    ro.close()


def test_deep_golden_reproduced_by_the_reference(rec_oracle):
    if not rec_oracle.available("reference"):
        pytest.skip("compiled reference not built")
    want, got = load_golden("deep.npz"), gen_golden.deep_arrays("reference")
    assert sorted(want.files) == sorted(got)
    for k in want.files:
        a, b = want[k], np.asarray(got[k])
        assert a.shape == b.shape and a.dtype == b.dtype, k
        assert np.array_equal(bits(a), bits(b)) if a.dtype == np.float32 else np.array_equal(a, b), k
