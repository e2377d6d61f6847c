"""CPU: the per-evaluation record of matchData in the C port (oracle/port_record.c hso_match_record) against what the
compiled reference's ScanMatcher reports to recording DrawInterface / HectorDebugInfoInterface hooks
(oracle/ref_record_driver.cpp hsref_match_record), and tests/golden/record.npz.

  * The port's record reduced to the hooks' view — the start arrow, then for evaluations 1 .. maxIterations the
    Hessian and the world arrow — equals the reference's hooks bit for bit on every level.
  * The port's evaluation 0 and every dTr equal getCompleteHessianDerivs (hsref_hessian_derivs) at the recorded input
    pose of that evaluation.
  * record.npz is reproduced bit-exactly: by the port everywhere, by the compiled reference where it is built.
"""
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT, load_golden
from oracle import gen_record_golden as gen_golden
from oracle import record_oracle


@pytest.fixture(scope="module")
def rec_oracle():
    """oracle.record_oracle, with the port's record library built if it is missing"""
    if not record_oracle.available("port"):
        subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "-f", "record.mk", "port"], check=True,
                       capture_output=True)
    return record_oracle


def maps(rec_oracle, kind):
    out = {}
    for name in ("match3", "match1"):
        g = load_golden(name + ".npz")
        size, levels = int(g["size"]), int(g["levels"])
        orc = rec_oracle.RecordOracle(kind, float(g["res"]), size, levels)
        for l in range(levels):
            p = np.zeros((size >> l) ** 2, np.float32)
            p[g[f"map_idx{l}"]] = g[f"map_val{l}"]
            orc.set_logodds(l, p.reshape(size >> l, size >> l))
        out[name] = (g, orc)
    return out


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("kind", ["port", "reference"])
def test_record_golden_reproduced(rec_oracle, kind):
    if not rec_oracle.available(kind):
        pytest.skip(f"oracle {kind} not built")
    want = load_golden("record.npz")
    got = gen_golden.record_arrays(kind)
    for k in want.files:
        if k.endswith("_points") and kind == "port":   # drawn points are counted by the reference's hooks only
            continue
        a, b = want[k], got[k]
        if a.dtype.kind == "f":
            assert np.array_equal(bits(a), bits(b)), k
        else:
            assert np.array_equal(a, b), k


def test_port_record_equals_reference_hooks(rec_oracle):
    if not rec_oracle.available("reference"):
        pytest.skip("compiled reference not built")
    port, ref = maps(rec_oracle, "port"), maps(rec_oracle, "reference")
    rng = np.random.default_rng(8)
    cases = list(gen_golden.RECORD_CASES)
    for k in range(16):   # every golden scan of both maps, default iteration counts and a random schedule
        iters = None if k % 2 == 0 else [int(v) for v in rng.integers(-1, 5, 3)]
        cases.append((f"scan{k}", "match3" if k < 12 else "match1", k, (0, 0, 0), iters))
    for name, mp, src, offset, iters in cases:
        g, po = port[mp]
        ro = ref[mp][1]
        scan, hint = gen_golden.record_inputs(g, src, offset)
        pp, cp, rec = po.match_record(hint, scan, iters)
        pr, cr, hooks, npts = ro.match_record(hint, scan, iters)
        assert np.array_equal(bits(pp), bits(pr)) and np.array_equal(bits(cp), bits(cr)), name
        assert np.array_equal(bits(rec_oracle.port_hooks(po, rec, scan.shape[0], iters)), bits(hooks)), name
        # drawScan twice per level for a scan, once (start pose) for an empty one
        assert np.all(npts == (2 * scan.shape[0])), (name, npts)
        # the plain matchData path is unchanged by the record
        if iters is None:
            assert np.array_equal(bits(pp), bits(ro.match(hint, scan)[0])), name


def geometry_cases(rec_oracle, kind, gi):
    """tests/match_cases.py's geometry gi on the oracle `kind`: its finite scans and the edge scan, built with the
    port as the matcher"""
    import match_cases as mcs

    g = (mcs.GEOMS + [mcs.companion(x) for x in mcs.GEOMS])[gi]
    sx, sy, L, start, res = g
    orcs = {}
    for k in ("port", kind):
        o = rec_oracle.RecordOracle(k, res, sx, L, start=start, size_y=sy)
        for l, (a, b) in enumerate(mcs.level_sizes(g)):
            o.set_logodds(l, mcs.field(a, b, l))
        orcs[k] = o
    po = orcs["port"]
    cases = mcs.Cases(g, [po.get_prob(l) for l in range(L)], po, seed=100 + gi)
    scans = []
    for k, n in enumerate((33, 1081, 2049)):
        h = cases.hint(k)
        scans.append((h, cases.scan(n, h, nonfinite=False)))
    if L > 1:
        h = cases.hint(5)
        scans.append((h, cases.strip_scan(700, h)))
    h = cases.hint(3)
    base = cases.scan(1081, h, nonfinite=False, slots=mcs.SLOTS)
    it = mcs.edge_iterations(L)
    h, pts, designed, rec = mcs.build_edge_scan(
        cases, lambda hh, p: mcs.split_record(po.match_record(hh, p, it)[2], L, it), h, base, cases.slots)
    mcs.check_edges(cases, rec, pts, designed)
    scans.append((h, pts))
    return orcs, scans


def _geom_params():
    import match_cases as mcs

    allg = mcs.GEOMS + [mcs.companion(x) for x in mcs.GEOMS]
    return list(range(len(allg))), [mcs.geom_id(g) + ("-corner" if g[3] is mcs.CORNER else "") for g in allg]


@pytest.mark.parametrize("gi", _geom_params()[0], ids=_geom_params()[1])
def test_geometry_port_record_equals_reference(rec_oracle, gi):
    """Non-square, odd-sized and off-centre multi-level maps (tests/match_cases.py), edge endpoints built exactly: the
    port's record reduced to the hooks' view equals the reference's hooks bit for bit, with the default iteration
    schedule, [-1, 2, 4] and the edge scans' schedule, and its every evaluation equals getCompleteHessianDerivs at the recorded input pose on
    every level."""
    if not rec_oracle.available("reference"):
        pytest.skip("compiled reference not built")
    import match_cases as mcs

    orcs, scans = geometry_cases(rec_oracle, "reference", gi)
    po, ro = orcs["port"], orcs["reference"]
    for iters in (None, [-1, 2, 4][:po.levels], mcs.edge_iterations(po.levels)):
        for k, (hint, scan) in enumerate(scans):
            pp, cp, rec = po.match_record(hint, scan, iters)
            pr, cr, hooks, _ = ro.match_record(hint, scan, iters)
            assert np.array_equal(bits(pp), bits(pr)) and np.array_equal(bits(cp), bits(cr)), (k, iters)
            assert np.array_equal(bits(rec_oracle.port_hooks(po, rec, scan.shape[0], iters)), bits(hooks)), (k, iters)
            mis = po.level_iterations(iters)
            off = 0
            for l in range(po.levels - 1, -1, -1):
                E = mis[l] + 1
                ev = rec[off + 3:off + 3 + 15 * E].reshape(E, 15)
                pin = ro.map_coords_pose(l, rec[off:off + 3])
                pl = (scan * np.float32(2.0 ** -l)).astype(np.float32)
                for e in range(E):
                    H, d = ro.hessian_derivs(l, pin, pl)
                    assert np.array_equal(bits(H.reshape(9)), bits(ev[e, :9])), (k, l, e)
                    assert np.array_equal(bits(d), bits(ev[e, 9:12])), (k, l, e)
                    pin = ev[e, 12:15]
                off += 3 + 15 * E
    for o in orcs.values():
        o.close()


def test_port_record_sums_equal_reference_derivs(rec_oracle):
    if not rec_oracle.available("reference"):
        pytest.skip("compiled reference not built")
    port, ref = maps(rec_oracle, "port"), maps(rec_oracle, "reference")
    for name, mp, src, offset, iters in gen_golden.RECORD_CASES:
        g, po = port[mp]
        ro = ref[mp][1]
        scan, hint = gen_golden.record_inputs(g, src, offset)
        if scan.shape[0] == 0:
            continue
        _, _, rec = po.match_record(hint, scan, iters)
        mis = po.level_iterations(iters)
        off = 0
        for l in range(po.levels - 1, -1, -1):
            E = mis[l] + 1
            start = rec[off:off + 3]
            ev = rec[off + 3:off + 3 + 15 * E].reshape(E, 15)
            pin = ro.map_coords_pose(l, start)
            pl = (scan * np.float32(2.0 ** -l)).astype(np.float32)   # DataContainer::setFrom, MapRepMultiMap.h:127
            for e in range(E):
                H, d = ro.hessian_derivs(l, pin, pl)
                assert np.array_equal(bits(H.reshape(9)), bits(ev[e, :9])), (name, l, e)
                assert np.array_equal(bits(d), bits(ev[e, 9:12])), (name, l, e)
                pin = ev[e, 12:15]
            off += 3 + 15 * E
