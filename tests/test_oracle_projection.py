"""CPU: the oracle of the projected SLAM step — laser_geometry's projection (tests/laser_projection.py) followed by the
node's cloud conversion — checked on its own.  The vectorised projection equals a beam-by-beam restatement, the
plain-C port of the cloud conversion equals the node's compiled converter on projected scans bit for bit, and the edge
values land on the side of each window the contract says."""
import ctypes as C
import ctypes.util
import math
import struct

import numpy as np
import pytest

from laser_projection import container, cutoff_of, edge_ranges, kept_beams, project, tilted_transform, unit_vectors

F32 = np.float32
SCALE = 20.0

# n_beams, angle_min (deg), angle_increment (deg), range_min, range_max, range_cutoff
PROJECTIONS = [(1081, -135.0, 0.25, 0.1, 30.0, 30.0),    # the node's call, range_max == cutoff
               (720, -180.0, 0.5, 0.3, 12.0, 30.0),      # range_max < cutoff: the cutoff is the projector's, not range_max
               (360, -120.0, 0.75, 0.5, 20.0, -1.0),     # negative cutoff: range_max
               (1440, -180.0, 0.25, 0.2, 8.0, 6.5)]      # cutoff < range_max


def proj_of(k):
    n, a0, da, rmin, rmax, cut = PROJECTIONS[k]
    return dict(n_beams=n, angle_min=float(F32(math.radians(a0))), angle_increment=float(F32(math.radians(da))),
                range_min=float(F32(rmin)), range_max=float(F32(rmax)), range_cutoff=cut)


def cloud_format(k):
    from hector_slam_b200 import synth

    fmt = dict(synth.CLOUD_FORMAT)
    if k == 3:   # the tilted mount's z window removes far points
        fmt.update(laser_z_min_value=-0.5, laser_z_max_value=0.5)
    return fmt


def transform_of(k):
    from hector_slam_b200 import synth

    return tilted_transform() if k == 3 else synth.laser_transform(xyz=(0.1 + 0.02 * k, -0.03, 0.3),
                                                                   rpy=(0.02, -0.03 * k, 0.05 * k))


def scalar_project(ranges, proj):
    """Beam by beam in Python doubles, float32 rounding through struct (C's (float) cast)."""
    a0, da = float(F32(proj["angle_min"])), float(F32(proj["angle_increment"]))
    cut, rmin = cutoff_of(proj), float(F32(proj["range_min"]))
    out = []
    for i, r in enumerate(np.asarray(ranges, F32).tolist()):
        if not (r < cut and r >= rmin):
            continue
        a = a0 + i * da
        fx = struct.unpack("f", struct.pack("f", r * math.cos(a)))[0]
        fy = struct.unpack("f", struct.pack("f", r * math.sin(a)))[0]
        out.append((fx, fy, 0.0))
    return np.asarray(out, F32).reshape(-1, 3)


def same(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def test_unit_vectors_are_libm_of_the_once_rounded_angle():
    """The table's two claims, each checked another way: the angle angle_min + i * angle_increment is the exact value
    rounded ONCE to double (i * increment is exact: a 24-bit float times i < 2^20), and its cos / sin are the C library's
    double functions (called through ctypes, as the library's host code calls them)."""
    from fractions import Fraction

    libm = C.CDLL(ctypes.util.find_library("m") or "libm.so.6")
    libm.cos.restype = libm.sin.restype = C.c_double
    libm.cos.argtypes = libm.sin.argtypes = [C.c_double]
    for k in range(len(PROJECTIONS)):
        p = proj_of(k)
        u = unit_vectors(p["n_beams"], p["angle_min"], p["angle_increment"])
        a0, da = Fraction(float(F32(p["angle_min"]))), Fraction(float(F32(p["angle_increment"])))
        for i in range(0, p["n_beams"], 7):
            a = float(a0 + i * da)   # exact sum, one rounding
            assert u[i, 0] == libm.cos(a) and u[i, 1] == libm.sin(a), (k, i)


@pytest.mark.parametrize("k", range(len(PROJECTIONS)))
def test_projection_equals_beam_by_beam_restatement(k):
    p = proj_of(k)
    for seed in range(3):
        r = edge_ranges(p["n_beams"], p, 100 * k + seed)
        assert same(project(r, p), scalar_project(r, p)), (k, seed)


def test_edge_values_fall_where_the_contract_says():
    p = proj_of(0)   # cutoff 30.0 and range_max 30.0 are floats: the edges are exact
    rmin, cut = F32(p["range_min"]), F32(30.0)
    r = np.array([np.nan, np.inf, -np.inf, -1.0, 0.0, rmin, np.nextafter(rmin, F32(0)), cut, np.nextafter(cut, F32(0)), 5.0],
                 F32)
    p1 = dict(p, n_beams=r.size)
    assert kept_beams(r, p1).tolist() == [False, False, False, False, False, True, False, False, True, True]
    p2 = dict(p1, range_cutoff=-1.0, range_max=float(F32(4.0)))   # negative cutoff: range_max = 4 drops the 5 m return
    assert kept_beams(r, p2).tolist()[-1] is False and kept_beams(r, p2).tolist()[5] is True
    assert project(np.full(r.size, np.nan, F32), p1).shape == (0, 3)


@pytest.mark.parametrize("k", range(len(PROJECTIONS)))
def test_port_equals_compiled_reference_on_projected_scans(pyoracle, oracle_kinds, k):
    """The cloud conversion of projected edge scans: port == the node's compiled converter, bit for bit (endpoints,
    count, origo).  Rear-close returns and (k = 3) the tilted mount's z window remove points the projector kept."""
    if "reference" not in oracle_kinds:
        pytest.skip("oracle/_ref is not built here")
    p, fmt, T = proj_of(k), cloud_format(k), transform_of(k)
    removed = 0
    for seed in range(4):
        r = edge_ranges(p["n_beams"], p, 10 * k + seed)
        a, oa = container(r, p, fmt, T, SCALE, pyoracle, kind="port")
        b, ob = container(r, p, fmt, T, SCALE, pyoracle, kind="reference")
        assert same(a, b) and same(oa, ob), (k, seed)
        removed += project(r, p).shape[0] - a.shape[0]
    assert removed > 0
    r = np.full(p["n_beams"], np.nan, F32)   # an all-dropped scan
    assert container(r, p, fmt, T, SCALE, pyoracle, kind="reference")[0].shape == (0, 2)


def test_tilted_mount_and_rear_close_zone_remove_points(pyoracle):
    p, fmt, T = proj_of(3), cloud_format(3), transform_of(3)
    r = np.full(p["n_beams"], F32(9.0), F32)
    r[: p["n_beams"] // 2] = F32(1.0)
    pts = project(r, p)
    assert pts.shape[0] == p["n_beams"] // 2   # 9 m is past the 6.5 m cutoff
    got, _ = container(r, p, fmt, T, SCALE, pyoracle)
    near = np.full(p["n_beams"], F32(3.0), F32)
    far_got, _ = container(near, p, fmt, T, SCALE, pyoracle)
    assert far_got.shape[0] < p["n_beams"]   # z window: 3 m at 0.3 rad pitch is ~0.9 m below the laser
    back = np.full(p["n_beams"], F32(0.55), F32)   # every beam 0.55 m: the backward ones are rear-close
    b, _ = container(back, proj_of(0) | {"n_beams": p["n_beams"]}, cloud_format(0), transform_of(0), SCALE, pyoracle)
    assert 0 < b.shape[0] < p["n_beams"]
    assert got.shape[0] <= pts.shape[0]
