"""CPU: oracle/pose32.py, the fp32 restatement of the matcher's per-scan pose arithmetic, against the C port and the
compiled reference.

  * pose32.step reproduces every estimate of the C port's match record (oracle/port_record.c) bit for bit, NaN as NaN:
    the goldens, scans of 1, 2 and 3 endpoints, planes constant along y (H(1,1) exactly 0) and along x (H(0,0) exactly
    0), hints 0.3 rad off (the clamp), the golden clamp case, scans entirely out of the map and non-finite endpoints.
  * pose32.normalize_angle and pose32.pose_difference_larger_than equal the reference's util:: functions
    (oracle/_ref/libhsref_util.so, where it is built) and the C port's on edge tables and 1e5 random arguments; the gate also equals the
    host façade's (hsbp_pose_difference_larger_than).
"""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT, golden_planes, load_golden
from oracle import gen_record_golden, likelihood64, pose32, record_oracle

F32 = np.float32
FMAX = np.finfo(F32).max
same = likelihood64.same_bits_or_nan


@pytest.fixture(scope="module")
def port_record():
    if not record_oracle.available("port"):
        subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "-f", "record.mk", "port"], check=True,
                       capture_output=True)


def up(x, k=1):
    x = F32(x)
    for _ in range(k):
        x = np.nextafter(x, F32(np.inf))
    return x


def down(x, k=1):
    x = F32(x)
    for _ in range(k):
        x = np.nextafter(x, F32(-np.inf))
    return x


# ---- 1. the Gauss-Newton step against every estimate of the port's record ---------------------------------------------
def check_record(orc, hint, scan):
    """every evaluation of orc's record for (hint, scan): pose32.step(previous estimate, H, dTr) == the estimate.
    -> (evaluations checked, steps taken, steps clamped)"""
    _, _, rec = orc.match_record(hint, scan)
    mis = orc.level_iterations()
    off, checked, moved, clamped = 0, 0, 0, 0
    for l in range(orc.levels - 1, -1, -1):
        E = mis[l] + 1
        start = rec[off:off + 3]
        ev = rec[off + 3:off + 3 + 15 * E].reshape(E, 15)
        off += 3 + 15 * E
        if scan.shape[0] == 0:
            assert np.all(ev == 0)
            continue
        prev = orc.map_coords_pose(l, start)
        for e in range(E):
            H, d, est = ev[e, :9].reshape(3, 3), ev[e, 9:12], ev[e, 12:15]
            want = pose32.step(prev, H, d)
            assert same(want, est), (l, e, prev, H, d, est, want)
            if H[0, 0] != 0 and H[1, 1] != 0:
                moved += 1
                with np.errstate(all="ignore"):
                    clamped += int(abs(float(pose32.solve3(H, d)[2])) > 0.2)
            checked += 1
            prev = est
        # the level's normalisation and conversion: the next level starts there
        nxt = orc.world_coords_pose(l, F32([prev[0], prev[1], pose32.normalize_angle(prev[2])]))
        if l > 0:
            assert same(rec[off:off + 3], nxt), (l, rec[off:off + 3], nxt)
    return checked, moved, clamped


def golden_port(name):
    g = load_golden(name + ".npz")
    size, levels = int(g["size"]), int(g["levels"])
    orc = record_oracle.RecordOracle("port", float(g["res"]), size, levels)
    for l, p in enumerate(golden_planes(g)):
        orc.set_logodds(l, p)
    return g, orc


def test_step_goldens(port_record):
    totals = np.zeros(3, int)
    for name in ("match3", "match1"):
        g, orc = golden_port(name)
        scans, hints = g["scans"], g["hints"]
        for k in range(scans.shape[0]):
            s, h = scans[k], hints[k]
            cases = [(h, s), (h + F32([0, 0, 0.3]), s), (h - F32([0, 0, 0.3]), s),
                     (h, s[:1]), (h, s[:2]), (h, s[:3]), (h, s[5:8]),
                     (h, np.zeros((0, 2), F32)), (h, (s + F32(1e5)).astype(F32))]
            # non-finite endpoints: out of the map, and the 0 * inf of rotDeriv makes H and dTr NaN, so the step is NaN
            bad = s[:40].copy()
            bad[3] = [np.nan, 1.0]
            bad[7] = [np.inf, -np.inf]
            bad[9] = [1e30, -1e30]
            cases.append((h, bad))
            for hint, scan in cases:
                totals += check_record(orc, F32(hint), np.ascontiguousarray(scan, F32))
        for cname, mp, src, offset, iters in gen_record_golden.RECORD_CASES:
            if mp == name and iters is None:
                scan, hint = gen_record_golden.record_inputs(g, src, offset)
                totals += check_record(orc, hint, scan)
        orc.close()
    checked, moved, clamped = totals
    assert moved > 100 and clamped > 0 and checked > moved, totals


@pytest.mark.parametrize("axis", ["x", "y"])
def test_step_degenerate_planes(port_record, axis):
    """a plane constant along one axis: the map gradient across it is exactly zero, so H(1,1) (varying in x only) or
    H(0,0) (varying in y only) is exactly 0 and the step is gated off; the other entries are not"""
    size = 128
    t = np.arange(size, dtype=np.float64)
    prof = (2.0 * np.sin(2 * np.pi * t / 23.0)).astype(F32)
    plane = np.tile(prof, (size, 1)) if axis == "x" else np.tile(prof[:, None], (1, size))
    orc = record_oracle.RecordOracle("port", 0.05, size, 2)
    orc.set_logodds(0, plane)
    orc.set_logodds(1, plane[::2, ::2].copy())
    rng = np.random.default_rng(5)
    zero_gate = 0
    for k in range(12):
        scan = rng.uniform(-25, 25, (1 + 7 * k, 2)).astype(F32)
        hint = F32([rng.uniform(2.5, 3.9), rng.uniform(2.5, 3.9), rng.uniform(-3, 3)])
        check_record(orc, hint, scan)
        _, _, rec = orc.match_record(hint, scan)
        H = rec[3:12].reshape(3, 3)
        zero_gate += int(H[1, 1] == 0 if axis == "x" else H[0, 0] == 0)
    orc.close()
    assert zero_gate > 0


# ---- 2. normalize_angle and the gate against the reference's util:: functions ------------------------------------------
def kinds():
    from oracle import pyoracle

    if not pyoracle.available("port"):
        subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "port"], check=True, capture_output=True)
    return ["port"] + (["reference"] if pyoracle.util_available("reference") else [])


def angle_edges():
    pi = F32(math.pi)
    out = [0.0, -0.0, pi, -pi, up(pi), down(pi), -up(pi), -down(pi), 1e3, -1e3, 1e6, -1e6, 3.4e38, -3.4e38, FMAX, -FMAX,
           1e-45, -1e-45, 1e-40, -1e-40, -1e-30, 1e-30, np.inf, -np.inf, np.nan, 0.2, -0.2, 120.0, -120.0]
    for k in range(1, 40):
        m = F32(2 * math.pi * k)
        out += [m, up(m), down(m), -m, -up(m), -down(m), F32(math.pi * (2 * k + 1)), -F32(math.pi * (2 * k + 1))]
    return np.array(out, F32)


def test_normalize_angle_tables():
    rng = np.random.default_rng(11)
    bits = rng.integers(0, 2 ** 32, 100000, dtype=np.uint64).astype(np.uint32)
    args = np.concatenate([angle_edges(), bits.view(F32), rng.uniform(-20, 20, 100000).astype(F32)])
    want = np.array([pose32.normalize_angle(a) for a in args], F32)
    from oracle import pyoracle

    for kind in kinds():
        got = pyoracle.normalize_angle(args, kind)
        bad = [i for i in range(args.size) if not same(got[i], want[i])]
        assert not bad, (kind, [(float(args[i]), float(got[i]), float(want[i])) for i in bad[:8]])


def gate_edges():
    """(p1, p2, dist, ang, expected) rows: the threshold boundaries of poseDifferenceLargerThan"""
    rows = []
    for k in range(0, 40, 3):   # a 3-4-5 triangle scaled by 2^-k: the norm is exactly the threshold
        s = F32(2.0 ** -k)
        p1, p2 = F32([3 * s, 4 * s, 0.0]), F32([0.0, 0.0, 0.0])
        rows += [(p1, p2, 5 * s, 1.0, False), (p1, p2, down(5 * s), 1.0, True)]
        rows += [(p1 + F32([1.5, -2.0, 0.25]), F32([1.5, -2.0, 0.25]), 5 * s, 1.0, None)]
    pi = F32(math.pi)
    for a, b in ((pi, -pi), (-pi, pi), (3.1, -3.1), (-3.1, 3.1), (10.0, 0.0), (-10.0, 0.0), (0.0, 10.0), (20.0, -1.0),
                 (up(pi), 0.0), (down(pi), 0.0), (-up(pi), 0.0), (0.0, up(pi)), (1e6, 0.0), (np.inf, 0.0)):
        for ang in (0.0, 0.05, 0.9, 3.0, 4.0):
            rows.append((F32([1.0, 1.0, a]), F32([1.0, 1.0, b]), 0.4, ang, None))
    for t in (F32(0.25), F32(0.05), F32(1.0)):   # |a| exactly the threshold, and one ulp either side
        for a in (t, -t):
            rows += [(F32([0, 0, a]), F32([0, 0, 0]), 0.4, t, False), (F32([0, 0, a]), F32([0, 0, 0]), 0.4, down(t), True),
                     (F32([0, 0, a]), F32([0, 0, 0]), 0.4, up(t), False)]
    z = F32([0.5, -0.5, 0.1])
    rows += [(z, z, 0.0, 0.0, False), (z, z, -1.0, 0.0, True), (z, z, 0.0, -1.0, True), (z, z, -0.0, -0.0, False),
             (z, F32([0.5, -0.5, up(F32(0.1))]), 0.0, 0.0, True),
             (z, F32([FMAX] * 3), 0.4, 0.9, True), (F32([0, 0, 0]), F32([FMAX] * 3), 0.4, 0.9, True),
             (F32([np.nan, 0, 0]), z, 0.4, 0.9, False), (z, F32([np.nan] * 3), 0.4, 0.9, False),
             (z, F32([np.nan] * 3), -1.0, -1.0, False), (F32([0.5, -0.5, np.nan]), z, 0.4, 0.9, False),
             (z, z, np.nan, np.nan, False)]
    return rows


def gate_random(n, seed):
    rng = np.random.default_rng(seed)
    p2 = np.stack([rng.uniform(-50, 50, n), rng.uniform(-50, 50, n), rng.uniform(-40, 40, n)], 1).astype(F32)
    d = np.stack([rng.normal(0, 0.3, n), rng.normal(0, 0.3, n), rng.normal(0, 3.0, n)], 1).astype(F32)
    p1 = (p2 + d).astype(F32)
    dist = np.abs(rng.normal(0, 0.4, n)).astype(F32)
    ang = np.abs(rng.normal(0, 1.0, n)).astype(F32)
    return p1, p2, dist, ang


def gate_table():
    rows = gate_edges()
    p1, p2, dist, ang = gate_random(100000, 13)
    P1 = np.concatenate([np.stack([r[0] for r in rows]), p1]).astype(F32)
    P2 = np.concatenate([np.stack([r[1] for r in rows]), p2]).astype(F32)
    D = np.concatenate([F32([r[2] for r in rows]), dist]).astype(F32)
    A = np.concatenate([F32([r[3] for r in rows]), ang]).astype(F32)
    want = np.array([pose32.pose_difference_larger_than(P1[i], P2[i], D[i], A[i]) for i in range(P1.shape[0])])
    for i, r in enumerate(rows):
        if r[4] is not None:
            assert want[i] == r[4], (i, r)
    assert 0.05 < want[len(rows):].mean() < 0.95   # both outcomes, in bulk
    return P1, P2, D, A, want


def test_pose_difference_tables():
    from oracle import pyoracle

    P1, P2, D, A, want = gate_table()
    for kind in kinds():
        got = pyoracle.pose_difference_larger_than(P1, P2, D, A, kind)
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, (kind, [(P1[i], P2[i], D[i], A[i], want[i]) for i in bad[:8]])


def test_pose_difference_facade(hsb_lib):
    """the host façade's gate (SlamProcessorB200.hpp poseDifferenceLargerThan) on the same table"""
    from hector_slam_b200 import build

    L = C.CDLL(build.HOST_LIB)
    L.hsbp_pose_difference_larger_than.argtypes = [C.c_void_p, C.c_void_p, C.c_float, C.c_float]
    P1, P2, D, A, want = gate_table()
    P1, P2 = np.ascontiguousarray(P1), np.ascontiguousarray(P2)
    row = P1.strides[0]
    got = np.array([bool(L.hsbp_pose_difference_larger_than(P1.ctypes.data + i * row, P2.ctypes.data + i * row,
                                                             float(D[i]), float(A[i]))) for i in range(P1.shape[0])])
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, [(P1[i], P2[i], D[i], A[i], want[i]) for i in bad[:8]]
