"""CPU: the scan -> DataContainer converters of the node (SURVEY.md §8f N2).  Where oracle/_ref is present the C
port is compared bit for bit with the node's own source text compiled by oracle/ros_conv_driver.cpp
(HectorMappingRos.cpp:483-542 cut out at build time); everywhere it is checked against a numpy statement of the
same formulas and on the edge cases (rear-close reject, z window, distance window)."""
import numpy as np
import pytest


def make_cloud(seed, n=1081):
    from hector_slam_b200 import synth

    rng = np.random.default_rng(seed)
    world = synth.World(1, seed=3)
    pose = world.sample_free_poses(1, rng)[0]
    r = world.cast(pose) + rng.normal(0, 0.01, n)
    cloud = synth.ranges_to_cloud(r)
    # sprinkle the cases the function tests for
    cloud[5] = (-0.5, 0.3, 0.0)          # x < 0 and d^2 = 0.34 < 0.5 -> rejected        (:528)
    cloud[6] = (-0.7, 0.3, 0.0)          # x < 0 but d^2 = 0.58 -> kept
    cloud[7] = (0.3, 0.2, 0.0)           # d^2 = 0.13 < 0.16 -> rejected                 (:526)
    cloud[8] = (25.0, 20.0, 0.0)         # d^2 = 1025 > 900 -> rejected
    cloud[9, 2] = 1.5                    # z window                                      (:536)
    cloud[10, 2] = -1.5
    cloud[11, 2] = 0.97
    return r.astype(np.float32), cloud


def numpy_cloud(cloud, T, fmt, scale):
    x, y, z = cloud[:, 0], cloud[:, 1], cloud[:, 2]
    d2 = (x * x + y * y).astype(np.float32)
    keep = (d2 > np.float32(fmt["sqr_laser_min_dist"])) & (d2 < np.float32(fmt["sqr_laser_max_dist"]))
    keep &= ~((x < 0) & (d2 < np.float32(0.5)))
    T = T.reshape(3, 4)
    v = cloud.astype(np.float64)
    b = np.stack([(T[r, 0] * v[:, 0] + T[r, 1] * v[:, 1] + T[r, 2] * v[:, 2]) + T[r, 3] for r in range(3)], axis=1)
    zl = (b[:, 2] - T[2, 3]).astype(np.float32)
    keep &= (zl > np.float32(fmt["laser_z_min_value"])) & (zl < np.float32(fmt["laser_z_max_value"]))
    out = (b[keep, :2].astype(np.float32) * np.float32(scale)).astype(np.float32)
    origo = (T[:2, 3].astype(np.float32) * np.float32(scale)).astype(np.float32)
    return out, origo


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_cloud_to_points_port(pyoracle, oracle_kinds, seed):
    from hector_slam_b200 import synth

    _, cloud = make_cloud(seed)
    T = synth.laser_transform()
    fmt = synth.CLOUD_FORMAT
    got, origo = pyoracle.cloud_to_points(cloud, T, fmt["sqr_laser_min_dist"], fmt["sqr_laser_max_dist"],
                                          fmt["laser_z_min_value"], fmt["laser_z_max_value"], 20.0)
    want, want_origo = numpy_cloud(cloud, T, fmt, 20.0)
    assert got.shape == want.shape and np.array_equal(got, want) and np.array_equal(origo, want_origo)
    assert got.shape[0] < cloud.shape[0] - 4          # the sprinkled rejects are gone
    if "reference" in oracle_kinds:
        ref, ref_origo = pyoracle.cloud_to_points(cloud, T, fmt["sqr_laser_min_dist"], fmt["sqr_laser_max_dist"],
                                                  fmt["laser_z_min_value"], fmt["laser_z_max_value"], 20.0,
                                                  kind="reference")
        assert np.array_equal(got, ref) and np.array_equal(origo, ref_origo)
    # empty cloud
    e, _ = pyoracle.cloud_to_points(np.zeros((0, 3), np.float32), T, 0.16, 900.0, -1.0, 1.0, 20.0)
    assert e.shape == (0, 2)


def test_scan_to_points_port_equals_node_source(pyoracle, oracle_kinds):
    from hector_slam_b200 import synth

    if "reference" not in oracle_kinds:
        pytest.skip("oracle/_ref not built here")
    for seed in range(3):
        r, _ = make_cloud(seed)
        r[::97] = 45.0      # beyond range_max - 0.1
        r[3::131] = 0.05    # below range_min
        f = synth.SCAN_FORMAT
        a = pyoracle.scan_to_points(r, f["angle_min"], f["angle_increment"], f["range_min"], f["range_max"], 20.0)
        b = pyoracle.scan_to_points(r, f["angle_min"], f["angle_increment"], f["range_min"], f["range_max"], 20.0,
                                    kind="reference")
        assert a.shape == b.shape and np.array_equal(a, b)
        assert np.allclose(a, synth.ranges_to_points(r, 20.0), rtol=1e-6, atol=1e-5)  # numpy cos is not glibc cosf


@pytest.mark.parametrize("angle_min,angle_increment", [(-3.14159, 1.0e-6), (0.5, 3.0e-6),
                                                       (-3.1415927, float(np.float32(2 * np.pi / (1 << 20)))),
                                                       (1.0e3, 1.0e-6)])
def test_scan_to_points_port_equals_node_source_on_long_formats(pyoracle, oracle_kinds, angle_min, angle_increment):
    """2^20 beams (the longest scan format the library accepts) with increments down to 1e-6 rad: both accumulate the
    beam angle in fp32 (`angle += angle_increment`), so the port equals the node's converter bit for bit, endpoints
    at the far end of the accumulation included."""
    if "reference" not in oracle_kinds:
        pytest.skip("oracle/_ref not built here")
    rng = np.random.default_rng(7)
    r = rng.uniform(0.05, 32.0, 1 << 20).astype(np.float32)
    r[::11] = np.nan
    a = pyoracle.scan_to_points(r, angle_min, angle_increment, 0.1, 30.0, 20.0)
    b = pyoracle.scan_to_points(r, angle_min, angle_increment, 0.1, 30.0, 20.0, kind="reference")
    assert a.shape == b.shape and a.shape[0] > (1 << 19)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
