"""The fused and group SLAM steps' per-evaluation record (hsb_set_step_record, hsb_get_step_record,
hsb_get_last_match_scan): the matcher's draw and debug hooks for robots that keep stepping with their fleet.

GPU.
  - test_group_records: same-geometry, mixed and heterogeneous groups (1 to 8 levels, both gather modes, a non-default
    iteration schedule).  Each fleet has a recording group, a twin group that records nothing and single-step twins
    that record.  Seeded ticks of all four input kinds, full steps and permuted subsets, nowait, map_without_matching,
    recording and non-recording members in one step, and an empty scan from every member.  The recording group
    equals the plain one bit for bit in every output, launch count, end state and last-match container; each recording
    member's record equals its twin's single fused-step record; a member with recording off, or a session without
    matching, reports no record; the container equals the conversion entry points' endpoints, also straight after a
    nowait step.
  - test_single_step_record: the single fused steps' record equals hsb_match_data_record's on a twin holding the
    same map with the same endpoints, for all four input kinds, nowait or not, an empty scan and steps that reach a
    fixed point early.
  - test_fleet_300_records: a 300-member heterogeneous group with recording members across the 32- and 128-session
    boundaries, full steps and subsets of K = 129.
  - test_rejections: every bad argument's status and message.
  - test_fleet_hooks_against_reference: oracle/_ref/fleet_hooks_check (built where the reference headers are), the
    hook call sequences of hsb200::SlamProcessor::updateMany* with the shared replay against unmodified
    HectorSlamProcessors."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT, report
from test_gpu_group_score import thinned
from test_gpu_group_subset import KINDS, assert_same_state, bits, close_all, geometry, scan_of, session_data

pytestmark = pytest.mark.gpu

F32 = np.float32
TEX, LDG = 2, 1   # capi.GATHER_TEX, capi.GATHER_LDG
HSB_ERR_INVALID_ARG = -1


def flavour(name, M):
    """M members of a group of `name`: (make_rep(s), member_data(s), levels(s), SlamGroup keyword arguments)"""
    import test_gpu_group_heterogeneous as het
    import test_gpu_group_mixed as mixed
    import test_gpu_group_subset as sub

    if name == "same":
        return (lambda s: sub.make_rep(s, TEX), lambda s: session_data(700 + s, 20, geometry(s)), lambda s: sub.LEVELS,
                {})
    if name == "mixed":
        return (lambda s: mixed.make_rep(s % mixed.M, LDG), lambda s: mixed.member_data(s % mixed.M),
                lambda s: mixed.LEVELS, {"mixed": True})
    return het.make_rep, het.member_data, lambda s: het.LEVELS[s], {"heterogeneous": True}


def container_of(rep, kind, x):
    """the endpoints (and origo) the node's conversion gives for input x of `kind`, by the stand-alone entry points"""
    if kind == "endpoints":
        return np.ascontiguousarray(x, F32).reshape(-1, 2), np.zeros(2, F32)
    if kind == "ranges":
        return rep.scan_to_points(x), np.zeros(2, F32)
    pts, origo = rep.cloud_to_points(x) if kind == "cloud" else rep.projected_scan_to_points(x)
    return pts, np.asarray(origo, F32).reshape(2)


def empty_like(kind, scan):
    """an input of `kind` that leaves no endpoint: no points, or every beam beyond range_max"""
    if kind in ("endpoints", "cloud"):
        return np.zeros((0, 3 if kind == "cloud" else 2), F32)
    return np.full_like(scan, 1000.0)


def single_step_nowait(rep, kind, hint, scan, without, cov, nowait):
    """The single fused step of `kind` -> (pose, cov, updated, kept or None)"""
    kw = dict(map_without_matching=without, cov_inout=cov, nowait=nowait)
    if kind == "endpoints":
        return rep.slam_update(hint, scan, **kw) + (None,)
    return {"cloud": rep.slam_update_cloud, "ranges": rep.slam_update_ranges,
            "projected": rep.slam_update_projected}[kind](hint, scan, **kw)


def group_step(group, kind, hints, scans, mwm, members, nowait, cov):
    kw = dict(map_without_matching=mwm, nowait=nowait, cov_inout=cov, members=members)
    if kind == "endpoints":
        return group.slam_update(hints, scans, **kw) + (None,)
    return {"cloud": group.slam_update_cloud, "ranges": group.slam_update_ranges,
            "projected": group.slam_update_projected}[kind](hints, scans, **kw)


def assert_same_record(a, b, tag):
    ra, rb = a.step_record(raw=True), b.step_record(raw=True)
    assert (ra is None) == (rb is None), (tag, ra is None, rb is None)
    if ra is not None:
        assert np.array_equal(bits(ra), bits(rb)), (tag, int(np.argmax(bits(ra) != bits(rb))))


def assert_container(rep, want, tag):
    pts, origo = rep.last_match_scan()
    assert np.array_equal(bits(pts), bits(want[0])), (tag, pts.shape, want[0].shape)
    assert np.array_equal(bits(origo), bits(want[1])), (tag, origo, want[1])


@pytest.mark.parametrize("name", ["same", "mixed", "het"])
def test_group_records(hsb_lib, name):
    from hector_slam_b200 import capi

    M = 6
    make_rep, member_data, levels, kw = flavour(name, M)
    rec = [make_rep(s) for s in range(M)]     # the recording group
    plain = [make_rep(s) for s in range(M)]   # its twin that records nothing
    one = [make_rep(s) for s in range(M)]     # single fused steps, recording
    conv = [make_rep(s) for s in range(M)]    # never stepped: the conversion entry points
    data = [member_data(s) for s in range(M)]
    g_rec, g_plain = capi.SlamGroup(rec, **kw), capi.SlamGroup(plain, **kw)
    recording = [s % 3 != 1 for s in range(M)]   # members 1 and 4 record nothing
    for s in range(M):
        if recording[s]:
            rec[s].set_step_record(True)
            one[s].set_step_record(True)
    # a member whose switch was on and is off again: its buffer exists, it reports nothing
    rec[4].set_step_record(True)
    rec[4].set_step_record(False)
    rng = np.random.default_rng(31 + len(name))
    at = [0] * M
    covs = [np.full((3, 3), 5.0, F32) for _ in range(M)]
    last = [None] * M
    ticks = 14
    try:
        for t in range(ticks):
            kind = KINDS[t % 4]
            members = None if t % 2 == 0 else [int(j) for j in rng.permutation(M)[:int(rng.integers(1, M + 1))]]
            sel = list(range(M)) if members is None else members
            without = [bool(rng.random() < 0.25) and at[j] > 0 for j in sel]
            nowait = t % 3 == 1
            hints = np.asarray([data[j]["truth" if w else "hints"][at[j]] for j, w in zip(sel, without)],
                               F32).reshape(len(sel), 3)
            scans = [thinned(kind, scan_of(kind, data[j], at[j])) for j in sel]
            if t == ticks - 2:   # an empty scan from every session (every member of the heterogeneous fleet: 1-8 levels)
                scans = [empty_like(kind, x) for x in scans]
            cov = np.stack([covs[j] for j in sel])
            l_rec, l_plain = rec[0].launch_count, plain[0].launch_count
            out_r = group_step(g_rec, kind, hints, scans, without, members, nowait, cov.copy())
            out_p = group_step(g_plain, kind, hints, scans, without, members, nowait, cov.copy())
            assert rec[0].launch_count - l_rec == plain[0].launch_count - l_plain == 3, (name, t)
            for x, y in zip(out_r, out_p):
                if x is not None:
                    assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8)), (name, t, kind)
            for i, j in enumerate(sel):
                tag = (name, t, kind, i, j)
                ref = single_step_nowait(one[j], kind, hints[i], scans[i], without[i], covs[j].copy(), nowait)
                assert np.array_equal(bits(out_r[0][i]), bits(ref[0])), tag
                if without[i] or not recording[j]:
                    assert rec[j].step_record() is None, tag
                else:
                    r = rec[j].step_record(raw=True)
                    assert r is not None, tag
                    assert_same_record(rec[j], one[j], tag)
                    if scans[i].size == 0 or (out_r[3] is not None and out_r[3][i] == 0):
                        lv = rec[j].split_record(r)   # an empty scan: every level starts at the hint, no evaluation
                        for d in lv:
                            assert np.array_equal(bits(d["start"]), bits(hints[i])) and not d["H"].any(), tag
                assert plain[j].step_record() is None, tag
                if not without[i]:
                    last[j] = container_of(conv[j], kind, scans[i])
                if last[j] is not None:
                    assert_container(rec[j], last[j], tag)   # (straight after a nowait step too)
                covs[j] = out_r[1][i].copy()
                at[j] += 1
        for j in range(M):
            assert_same_state(rec[j], plain[j], (name, j), probe=False, levels=levels(j))
            assert_same_state(rec[j], one[j], (name, j), probe=False, levels=levels(j))
            if last[j] is not None:
                assert_container(plain[j], last[j], (name, j))
                assert_container(one[j], last[j], (name, j))
        # turning the switch on again: no record until the next step
        rec[0].set_step_record(False)
        rec[0].set_step_record(True)
        assert rec[0].step_record() is None
    finally:
        g_rec.close()
        g_plain.close()
        close_all(rec, plain, one, conv)


def copy_maps(src, dst):
    for l in range(src.levels):
        dst.upload_level(l, src.download_level(l))
        assert np.array_equal(bits(dst.download_prob(l)), bits(src.download_prob(l))), l


def test_single_step_record(hsb_lib):
    """Each fused step's record against hsb_match_data_record on a twin holding the step's map, with the endpoints the
    step converts (the stand-alone conversion of the same input)"""
    import test_gpu_group_heterogeneous as het

    for s in (het.A, het.C, het.D, het.F):   # 1, 3 (LDG), 3 (iterations [6, 0, -1]) and 8 levels
        rep, twin = het.make_rep(s), het.make_rep(s)
        d = het.member_data(s)
        rep.set_step_record(True)
        fixpoints = 0
        try:
            for t in range(12):
                kind = KINDS[t % 4]
                without = t == 5
                nowait = t % 3 == 2
                # a repeat of the previous scan from the pose it was matched at: Gauss-Newton reaches a fixed point early
                k = t - 1 if t in (7, 11) else t
                hint = d["truth"][k] if t in (7, 11) else d["hints"][k]
                scan = scan_of(kind, d, k)
                if t == 9:
                    scan = empty_like(kind, scan)   # an empty scan
                copy_maps(rep, twin)
                pose, cov, _, kept = single_step_nowait(rep, kind, hint, scan, without, None, nowait)
                r = rep.step_record(raw=True)
                if without:
                    assert r is None, t
                    continue
                pts, origo = container_of(twin, kind, scan)
                if kept is not None:
                    assert kept == pts.shape[0], (s, t)
                tp, _, tr = twin.matchData(hint, pts, origo=origo, record=True)
                assert np.array_equal(bits(pose), bits(tp)), (s, t)
                want = np.concatenate([np.concatenate([lv["start"].reshape(-1), np.concatenate(
                    [lv["H"].reshape(-1, 9), lv["dTr"], lv["est"]], axis=1).reshape(-1)]) for lv in tr[::-1]])
                assert np.array_equal(bits(r), bits(want)), (s, t, kind)
                assert_container(rep, (pts, origo), (s, t))
                for lv in rep.split_record(r):
                    est = lv["est"]
                    if est.shape[0] > 1 and pts.shape[0] and np.array_equal(bits(est[-1]), bits(est[-2])):
                        fixpoints += 1
            assert fixpoints > 0, s
        finally:
            close_all(rep, twin)


def test_fleet_300_records(hsb_lib):
    from test_gpu_group_heterogeneous_fleet import HetFleet, fleet_spec

    M = 300
    f = HetFleet([fleet_spec(s) for s in range(M)], 6)
    recording = {0, 31, 32, 33, 127, 128, 129, 200, 255, 256, 299}
    for j in recording:
        f.grp[j].set_step_record(True)
        f.one[j].set_step_record(True)
    rng = np.random.default_rng(5)
    try:
        for t, (kind, K) in enumerate([("endpoints", None), ("cloud", 129), ("ranges", None), ("projected", 129),
                                       ("endpoints", 129), ("ranges", 121)]):
            members = None if K is None else [int(j) for j in rng.permutation(M)[:K]]
            f.tick(kind, members, t % 2 == 1, rng)
            sel = range(M) if members is None else members
            stepped = 0
            for j in sel:
                if j in recording:
                    assert_same_record(f.grp[j], f.one[j], (t, kind, j))
                    stepped += f.grp[j].step_record() is not None
                else:
                    assert f.grp[j].step_record() is None, (t, j)
            assert stepped > 0, t
    finally:
        f.close()


def test_rejections(hsb_lib):
    from hector_slam_b200 import capi

    lib = capi.load_library()
    rep = capi.MapRepB200(0.05, 256, levels=2)
    try:
        def err():
            return (lib.hsb_last_error(rep.h) or b"").decode()

        R = rep.record_floats
        assert rep.level_evals() == [6, 4]
        assert lib.hsb_get_level_evals(rep.h, 2) == HSB_ERR_INVALID_ARG
        rec, matched, n, origo = np.zeros(R, F32), C.c_int(7), C.c_int(-1), np.zeros(2, F32)
        assert lib.hsb_set_step_record(None, 1) == HSB_ERR_INVALID_ARG
        assert lib.hsb_get_step_record(rep.h, rec.ctypes.data, C.byref(matched)) == HSB_ERR_INVALID_ARG
        assert "no fused SLAM step" in err()
        assert lib.hsb_get_last_match_scan(rep.h, None, 0, C.byref(n), origo.ctypes.data) == HSB_ERR_INVALID_ARG
        assert "matched no scan" in err()
        rep.set_step_record(True)
        pts = (np.random.default_rng(0).uniform(-40, 40, (50, 2))).astype(F32)
        rep.slam_update([0, 0, 0], pts)
        assert lib.hsb_get_step_record(rep.h, None, C.byref(matched)) == HSB_ERR_INVALID_ARG
        assert "record_out is NULL" in err()
        assert lib.hsb_get_step_record(rep.h, rec.ctypes.data, None) == HSB_ERR_INVALID_ARG
        assert "matched is NULL" in err()
        assert lib.hsb_get_step_record(rep.h, rec.ctypes.data, C.byref(matched)) == 0 and matched.value == 1
        out = np.zeros((50, 2), F32)
        assert lib.hsb_get_last_match_scan(rep.h, out.ctypes.data, 49, C.byref(n), origo.ctypes.data) == \
            HSB_ERR_INVALID_ARG
        assert n.value == 50 and "capacity 49 is below the container's 50 endpoints" in err()
        assert lib.hsb_get_last_match_scan(rep.h, None, 50, C.byref(n), origo.ctypes.data) == HSB_ERR_INVALID_ARG
        assert "points_xy_out is NULL" in err()
        assert lib.hsb_get_last_match_scan(rep.h, out.ctypes.data, 50, None, origo.ctypes.data) == HSB_ERR_INVALID_ARG
        assert "n_out is NULL" in err()
        assert lib.hsb_get_last_match_scan(rep.h, out.ctypes.data, 50, C.byref(n), None) == HSB_ERR_INVALID_ARG
        assert "origo_out is NULL" in err()
        assert lib.hsb_get_last_match_scan(rep.h, out.ctypes.data, 50, C.byref(n), origo.ctypes.data) == 0
        assert np.array_equal(bits(out), bits(pts))
        rep.slam_update([0, 0, 0], pts, map_without_matching=True)
        assert lib.hsb_get_step_record(rep.h, rec.ctypes.data, C.byref(matched)) == 0 and matched.value == 0
    finally:
        rep.close()


BIN = os.path.join(ROOT, "oracle", "_ref", "fleet_hooks_check")


def test_fleet_hooks_against_reference(hsb_lib):
    if not os.path.exists(BIN):
        pytest.skip("oracle/_ref/fleet_hooks_check not built (needs the reference headers at build time)")
    out = subprocess.run([BIN, "40"], capture_output=True, text=True, timeout=900)
    print(out.stdout, out.stderr)
    for line in out.stdout.splitlines():
        report("fleet_hooks_check: " + line.strip())
    assert out.returncode == 0 and "FLEET HOOKS OK" in out.stdout, out.stdout + out.stderr
