"""Which status every batch-match and single-SLAM-step entry point returns for arguments it must reject, which of two
failing checks wins, and that a rejected call queues no kernel.

Each row calls one C-ABI entry point with one argument changed from a valid call and names the status and, where the
entry point sets one, a piece of the message.  The host-buffer, submit and device forms of the four batch input kinds
(endpoints, LaserScan ranges, point clouds, projected ranges), the match-record batch and the five single SLAM steps
are all covered.  A row with B == 0 pins where the empty batch returns: after the argument and format checks, before
anything is queued."""
import ctypes as C
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

F32 = np.float32
INVALID, UNSUPPORTED = -1, -5
NB = 32          # beams of the scan format and of the laser projection
LONG = 40000     # beams / points past what the fused conversion can stage in shared memory (28 749 at 8 warps)
B = 2
PTS = 8          # endpoints or cloud points per scan


def _fmt(n):
    return dict(n_beams=n, angle_min=float(F32(-math.pi / 2)), angle_increment=float(F32(math.pi / n)), range_min=0.1,
                range_max=30.0)


def _rep(scan=None, cloud=False, proj=None):
    from hector_slam_b200 import capi, synth

    rep = capi.MapRepB200(0.05, 128, levels=2, gather_mode=capi.GATHER_LDG)
    if scan:
        rep.set_scan_format(**_fmt(scan))
    if cloud:
        rep.set_cloud_format(synth.laser_transform(), **synth.CLOUD_FORMAT)
    if proj:
        rep.set_laser_projection(**_fmt(proj))
    return rep


@pytest.fixture(scope="module")
def reps(hsb_lib):
    import torch

    r = {"full": _rep(NB, True, NB), "bare": _rep(), "no_cloud": _rep(NB, False, NB), "long": _rep(LONG, True, LONG)}
    # every device pointer of a device-form call points here (a rejected call reads none of it)
    r["dev"] = torch.zeros(3 * B * LONG + 64, dtype=torch.float32, device="cuda")
    yield r
    for k, v in r.items():
        if k != "dev":
            v.close()


def _host(n_per_scan=NB, width=1):
    return np.zeros((B * n_per_scan, width), F32)


def _args(reps, kind, form, over):
    """A valid call's arguments for (kind, form), with `over` applied; the rep it runs on."""
    a = dict(rep="full", B=B, hints=np.zeros((B, 3), F32), out=np.zeros((B, 3), F32), cov=np.zeros((B, 9), F32),
             origo=np.zeros((B, 2), F32), tf=None, ticket=C.c_int(5))
    n = LONG if over.get("rep") == "long" else NB
    if kind == "endpoints":
        a.update(inp=_host(PTS, 2), offsets=np.array([0, PTS, 2 * PTS], np.int32), n_shared=0, max_n=PTS)
    elif kind == "cloud":
        n = LONG if over.get("rep") == "long" else PTS
        a.update(inp=_host(n, 3), offsets=np.array([0, n, 2 * n], np.int32), max_n=n)
    else:
        a.update(inp=_host(n))
    a.update(over)
    if form == "device":
        d = reps["dev"].data_ptr()
        for k in ("hints", "out", "cov", "origo", "inp", "offsets", "record"):
            if k in a and a[k] is not None and not isinstance(a[k], int):
                a[k] = d
    return reps[a["rep"]] if isinstance(a["rep"], str) else a["rep"], a


def _p(x):
    if x is None or isinstance(x, int):
        return x
    return x.ctypes.data


def _call_batch(lib, rep, kind, form, a):
    h = None if a.get("null_handle") else rep.h
    P = _p
    if kind == "endpoints":
        if form == "device":
            return lib.hsb_match_batch_device(h, a["B"], P(a["hints"]), P(a["inp"]), P(a["offsets"]), a["n_shared"],
                                              a["max_n"], P(a["out"]), P(a["cov"]), None)
        if form == "record_device":
            return lib.hsb_match_batch_record_device(h, a["B"], P(a["hints"]), P(a["inp"]), P(a["offsets"]),
                                                     a["n_shared"], a["max_n"], P(a["out"]), P(a["cov"]),
                                                     P(a["record"]), None)
        if form == "submit":
            return lib.hsb_match_batch_submit(h, a["B"], P(a["hints"]), P(a["inp"]), P(a["offsets"]), a["n_shared"],
                                              P(a["out"]), P(a["cov"]), C.byref(a["ticket"]))
        return lib.hsb_match_batch(h, a["B"], P(a["hints"]), P(a["inp"]), P(a["offsets"]), a["n_shared"], P(a["out"]),
                                   P(a["cov"]))
    if kind == "ranges":
        if form == "device":
            return lib.hsb_match_batch_ranges_device(h, a["B"], P(a["hints"]), P(a["inp"]), P(a["out"]), P(a["cov"]),
                                                     None)
        if form == "submit":
            return lib.hsb_match_batch_ranges_submit(h, a["B"], P(a["hints"]), P(a["inp"]), P(a["out"]), P(a["cov"]),
                                                     C.byref(a["ticket"]))
        return lib.hsb_match_batch_ranges(h, a["B"], P(a["hints"]), P(a["inp"]), P(a["out"]), P(a["cov"]))
    if kind == "cloud":
        if form == "device":
            return lib.hsb_match_batch_cloud_device(h, a["B"], P(a["hints"]), P(a["inp"]), P(a["offsets"]), a["max_n"],
                                                    P(a["tf"]), P(a["out"]), P(a["cov"]), P(a["origo"]), None)
        if form == "submit":
            return lib.hsb_match_batch_cloud_submit(h, a["B"], P(a["hints"]), P(a["inp"]), P(a["offsets"]), P(a["tf"]),
                                                    P(a["out"]), P(a["cov"]), P(a["origo"]), C.byref(a["ticket"]))
        return lib.hsb_match_batch_cloud(h, a["B"], P(a["hints"]), P(a["inp"]), P(a["offsets"]), P(a["tf"]),
                                         P(a["out"]), P(a["cov"]), P(a["origo"]))
    if form == "device":
        return lib.hsb_match_batch_projected_device(h, a["B"], P(a["hints"]), P(a["inp"]), P(a["tf"]), P(a["out"]),
                                                    P(a["cov"]), P(a["origo"]), None)
    if form == "submit":
        return lib.hsb_match_batch_projected_submit(h, a["B"], P(a["hints"]), P(a["inp"]), P(a["tf"]), P(a["out"]),
                                                    P(a["cov"]), P(a["origo"]), C.byref(a["ticket"]))
    return lib.hsb_match_batch_projected(h, a["B"], P(a["hints"]), P(a["inp"]), P(a["tf"]), P(a["out"]), P(a["cov"]),
                                         P(a["origo"]))


# (override, status, message piece or None) — the rows every form of a kind shares
NULLS = [(dict(null_handle=True), INVALID, None), (dict(hints=None), INVALID, None), (dict(out=None), INVALID, None),
         (dict(B=-1), INVALID, None)]
BATCH_ROWS = {
    "endpoints": NULLS + [
        (dict(inp=None), INVALID, "points pointer is NULL"),
        (dict(offsets=None, n_shared=-1), INVALID, "n_shared >= 0"),
        (dict(B=0, inp=None, offsets=None, n_shared=-1), 0, None),
    ],
    "ranges": NULLS + [
        (dict(inp=None), INVALID, None),
        (dict(B=0, inp=None), INVALID, None),
        (dict(rep="bare"), INVALID, "hsb_set_scan_format has not been called"),
        (dict(rep="bare", B=0), INVALID, "hsb_set_scan_format has not been called"),
        (dict(rep="long"), UNSUPPORTED, "scan too long for the fused conversion"),
        (dict(B=0), 0, None),
    ],
    "cloud": NULLS + [
        (dict(offsets=None), INVALID, None),
        (dict(B=0, offsets=None), INVALID, None),
        (dict(rep="bare"), INVALID, "hsb_set_cloud_format has not been called"),
        (dict(rep="bare", B=0), INVALID, "hsb_set_cloud_format has not been called"),
        (dict(inp=None), INVALID, "points pointer is NULL"),
        (dict(rep="long"), UNSUPPORTED, "scan too long for the fused conversion"),
        (dict(B=0, inp=None), 0, None),
    ],
    "projected": NULLS + [
        (dict(inp=None), INVALID, None),
        (dict(B=0, inp=None), INVALID, None),
        (dict(rep="bare"), INVALID, "hsb_set_laser_projection has not been called"),
        (dict(rep="bare", B=0), INVALID, "hsb_set_laser_projection has not been called"),
        (dict(rep="no_cloud"), INVALID, "hsb_set_cloud_format has not been called"),
        (dict(rep="no_cloud", B=0), INVALID, "hsb_set_cloud_format has not been called"),
        (dict(rep="long"), UNSUPPORTED, "scan too long for the fused conversion (%d points)" % LONG),
        (dict(rep="long", B=0), UNSUPPORTED, "scan too long for the fused conversion (%d points)" % LONG),
        (dict(tune=dict(warps_per_scan=16)), UNSUPPORTED, "no projected-scan kernel for tuning"),
        (dict(tune=dict(scans_per_block=7), B=0), UNSUPPORTED, "no projected-scan kernel for tuning"),
        (dict(B=0), 0, None),
    ],
}
# rows of one form only
FORM_ROWS = {
    ("endpoints", "device"): [(dict(B=0, hints=None), INVALID, None)],
    ("endpoints", "record_device"): [(dict(record=None), INVALID, None),
                                     (dict(record=None, B=0, null_handle=True), INVALID, None)],
    ("endpoints", "host"): [(dict(B=0, hints=None), INVALID, None),
                            (dict(offsets=np.array([0, PTS, PTS - 1], np.int32)), INVALID, "non-decreasing")],
    ("endpoints", "submit"): [(dict(offsets=np.array([0, PTS, PTS - 1], np.int32)), INVALID, "non-decreasing")],
    ("cloud", "device"): [(dict(max_n=-1), INVALID, None), (dict(max_n=-1, B=0), INVALID, None),
                          (dict(B=0, inp=None, max_n=PTS), 0, None)],
    ("cloud", "host"): [(dict(offsets=np.array([0, PTS, PTS - 1], np.int32)), INVALID, "non-decreasing")],
}
FORMS = {"endpoints": ["host", "submit", "device", "record_device"], "ranges": ["host", "submit", "device"],
         "cloud": ["host", "submit", "device"], "projected": ["host", "submit", "device"]}
CASES = [(kind, form, i, row) for kind, forms in FORMS.items() for form in forms
         for i, row in enumerate(BATCH_ROWS[kind] + FORM_ROWS.get((kind, form), []))]


def _run(rep, lib, fn, tune):
    if tune:
        rep.set_tuning(**tune)
    try:
        before = lib.hsb_get_launch_count(rep.h)
        status = fn()
        return status, (lib.hsb_last_error(rep.h) or b"").decode(), lib.hsb_get_launch_count(rep.h) - before
    finally:
        if tune:
            rep.set_tuning(**{k: 0 for k in tune})


@pytest.mark.parametrize("kind,form,i,row", CASES, ids=[f"{k}-{f}-{i}" for k, f, i, _ in CASES])
def test_batch_rejection(reps, hsb_lib, kind, form, i, row):
    over, want, text = row
    over = dict(over)
    tune = over.pop("tune", None)
    if form == "record_device":
        over.setdefault("record", 0)
    if "record" in over and over["record"] == 0:
        over["record"] = reps["dev"].data_ptr()
    rep, a = _args(reps, kind, "device" if form in ("device", "record_device") else form, over)
    if "record" in over and over["record"] is None:
        a["record"] = None
    status, msg, launched = _run(rep, hsb_lib, lambda: _call_batch(hsb_lib, rep, kind, form, a), tune)
    assert status == want, (status, msg)
    if text is not None:
        assert text in msg, msg
    assert launched == 0
    if form == "submit" and status == 0:
        assert a["ticket"].value == -1


# ---- single SLAM steps ----------------------------------------------------------------------------------------------
def _call_step(lib, rep, kind, a):
    h = None if a.get("null_handle") else rep.h
    P = _p
    upd, kept = C.c_int(0), C.c_int(0)
    if kind in ("endpoints", "endpoints_nowait"):
        fn = lib.hsb_slam_update_nowait if kind == "endpoints_nowait" else lib.hsb_slam_update
        return fn(h, P(a["hint"]), P(a["inp"]), a["n"], None, a["mwm"], P(a["out"]), P(a["cov"]), C.byref(upd))
    if kind == "cloud":
        return lib.hsb_slam_update_cloud(h, P(a["hint"]), P(a["inp"]), a["n"], None, a["mwm"], 0, P(a["out"]),
                                         P(a["cov"]), C.byref(upd), C.byref(kept))
    if kind == "ranges":
        return lib.hsb_slam_update_ranges(h, P(a["hint"]), P(a["inp"]), a["n"], a["mwm"], 0, P(a["out"]), P(a["cov"]),
                                          C.byref(upd), C.byref(kept))
    return lib.hsb_slam_update_projected(h, P(a["hint"]), P(a["inp"]), a["n"], None, a["mwm"], 0, P(a["out"]),
                                         P(a["cov"]), C.byref(upd), C.byref(kept))


STEP_NULLS = [(dict(null_handle=True), INVALID, None), (dict(hint=None), INVALID, None), (dict(out=None), INVALID, None),
              (dict(inp=None), INVALID, None)]
STEP_ROWS = {
    "endpoints": STEP_NULLS + [(dict(n=-1), INVALID, None), (dict(inp=None, n=-1), INVALID, None)],
    "cloud": STEP_NULLS + [
        (dict(n=-1), INVALID, None),
        (dict(rep="bare"), INVALID, "hsb_slam_update_cloud: hsb_set_cloud_format has not been called"),
        (dict(rep="long"), UNSUPPORTED, "scan too long for the fused conversion (%d points)" % LONG),
    ],
    "ranges": STEP_NULLS + [
        (dict(rep="bare"), INVALID, "hsb_slam_update_ranges: hsb_set_scan_format has not been called"),
        (dict(n=NB - 1), INVALID, "hsb_slam_update_ranges: n is %d, the scan format has %d beams" % (NB - 1, NB)),
        (dict(n=NB - 1, rep="bare"), INVALID, "hsb_set_scan_format has not been called"),
        (dict(rep="long"), UNSUPPORTED, "scan too long for the fused conversion (%d points)" % LONG),
    ],
    "projected": STEP_NULLS + [
        (dict(rep="bare"), INVALID, "hsb_slam_update_projected: hsb_set_laser_projection has not been called"),
        (dict(rep="no_cloud"), INVALID, "hsb_slam_update_projected: hsb_set_cloud_format has not been called"),
        (dict(n=NB + 1), INVALID,
         "hsb_slam_update_projected: n is %d, the laser projection has %d beams" % (NB + 1, NB)),
        (dict(rep="long"), UNSUPPORTED, "scan too long for the fused conversion (%d points)" % LONG),
        (dict(rep="long", mwm=1), UNSUPPORTED, "scan too long for the fused conversion (%d points)" % LONG),
        (dict(n=NB + 1, tune=dict(warps_per_scan=4)), INVALID, "n is %d" % (NB + 1)),
        (dict(tune=dict(warps_per_scan=4)), UNSUPPORTED, "hsb_slam_update_projected: no projected-scan kernel"),
        (dict(tune=dict(unroll=8), mwm=1), UNSUPPORTED, "hsb_slam_update_projected: no projected-scan kernel"),
    ],
}
STEP_ROWS["endpoints_nowait"] = STEP_ROWS["endpoints"]
STEP_CASES = [(kind, i, row) for kind, rows in STEP_ROWS.items() for i, row in enumerate(rows)]


@pytest.mark.parametrize("kind,i,row", STEP_CASES, ids=[f"{k}-{i}" for k, i, _ in STEP_CASES])
def test_step_rejection(reps, hsb_lib, kind, i, row):
    over = dict(row[0])
    want, text = row[1], row[2]
    tune = over.pop("tune", None)
    long = over.get("rep") == "long"
    n = LONG if long else (PTS if kind.startswith("endpoints") or kind == "cloud" else NB)
    width = 2 if kind.startswith("endpoints") else 3 if kind == "cloud" else 1
    a = dict(rep="full", hint=np.zeros(3, F32), out=np.zeros(3, F32), cov=np.zeros(9, F32), mwm=0, n=n,
             inp=np.zeros((n, width), F32))
    a.update(over)
    rep = reps[a["rep"]]
    status, msg, launched = _run(rep, hsb_lib, lambda: _call_step(hsb_lib, rep, kind, a), tune)
    assert status == want, (status, msg)
    if text is not None:
        assert text in msg, msg
    assert launched == 0
