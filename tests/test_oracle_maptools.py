"""CPU: the C port's hector_map_tools rows (hso_raycast, hso_get_dist, hso_map_origin in oracle/hs_oracle.c) against
the unmodified HectorMapTools.h compiled in oracle/_ref, on the geometries the 512^2 golden map cannot reach: non-square
levels, rays longer than bresenham2D's 5000-step cap in both dominant directions, hit offsets whose distance sits next to
a perfect square, and world points that truncate into the map from (-1, 0).  The GPU tests fall back to the port where
oracle/_ref is absent, so the port is pinned here first.  Integer work: every result must be identical."""
import numpy as np
import pytest

import maptools_cases as mc


@pytest.fixture(scope="module")
def ref_available(pyoracle):
    if not pyoracle.available("reference"):
        pytest.skip("compiled reference (oracle/_ref/libhsref.so) not present")


def ref_origin(ref, level, cell):
    """HectorMappingRos::setServiceGetMapData's origin (HectorMappingRos.cpp:546-550) from the compiled GridMap:
    getWorldCoords(0) - cellLength * 0.5f, in fp32."""
    w = ref.world_coords_pose(level, [0.0, 0.0, 0.0])[:2]
    return (w - np.float32(cell) * np.float32(0.5)).astype(np.float32)


def same_bits(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


@pytest.mark.parametrize("geom", mc.GEOMS, ids=mc.geom_id)
def test_raycast_get_dist_and_origin_port_equals_header(pyoracle, ref_available, geom):
    sx, sy, levels, start = geom
    port = pyoracle.Oracle("port", mc.RES, sx, levels, start=start, size_y=sy)
    ref = pyoracle.Oracle("reference", mc.RES, sx, levels, start=start, size_y=sy)
    for l, (lx, ly) in enumerate(mc.level_sizes(geom)):
        assert port.level_size(l) == ref.level_size(l) == (lx, ly)
        cell = port.cell_length(l)
        origin = port.map_origin(l)
        assert same_bits(origin, ref_origin(ref, l, cell)), (l, origin, ref_origin(ref, l, cell))
        p = mc.plane(lx, ly, seed=lx * 31 + ly + l)
        port.set_logodds(l, p)
        mt = pyoracle.RefMapTools(mc.occupancy(p), cell, origin)
        begin, end = mc.cell_rays(lx, ly, mc.occupancy(p), seed=lx + 7 * ly)
        hits = zero = 0
        for b, e in zip(begin, end):
            want = mt.raycast(b, e)
            assert port.raycast(l, b, e) == want, (geom, l, b, e, want)
            hits += want[0] >= 0
            zero += want[0] == 0
        assert hits > 200 and zero >= 8, (hits, zero)
        bw, ew, is_nan = mc.world_rays(lx, ly, origin, cell, seed=lx + 3 * ly)
        found = 0
        for b, e, nan in zip(bw, ew, is_nan):
            d, hw, f = port.get_dist(l, b, e)
            if nan:             # the reference's cast of NaN is undefined: the port, like the device, misses
                assert not f and np.float32(d) == np.float32(-cell)
                continue
            rd, rhw, rf = mt.get_dist(b, e)
            assert (np.float32(d), f) == (np.float32(rd), rf) and same_bits(hw, rhw), (geom, l, b, e, d, rd)
            found += f
        assert found > 100, found
        mt.close()
    port.close()
    ref.close()


@pytest.mark.parametrize("geom", mc.LONG, ids=mc.geom_id)
def test_constructed_long_rays_port_equals_header(pyoracle, ref_available, geom):
    """One occupied cell per ray: at step 4999 (hit) and 5000 / 5001 (beyond the cap: miss) of 6000-cell rays, at the
    last step before the end cell (hit) and on the end cell (excluded: miss), and at hit offsets next to a perfect
    square in all four mirrors, where the fp32 distance differs from the exact or the fused one."""
    sx, sy, _, start = geom
    port = pyoracle.Oracle("port", mc.RES, sx, 1, start=start, size_y=sy)
    cell = port.cell_length(0)
    origin = port.map_origin(0)
    cases = mc.lone_cases(sx, sy)
    assert sum(c.name.startswith("near square") for c in cases) == 4 * 9
    for k, c in enumerate(cases):
        p = mc.lone_plane(sx, sy, c.cell, seed=k)
        port.set_logodds(0, p)
        mt = pyoracle.RefMapTools(mc.occupancy(p), cell, origin)
        want = (float(c.dist), c.cell) if c.hit else (-1.0, (-1, -1))
        assert mt.raycast(c.begin, c.end) == want, (c, mt.raycast(c.begin, c.end))
        assert port.raycast(0, c.begin, c.end) == want, c
        mt.close()
    port.close()
