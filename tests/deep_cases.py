"""Maps of four to eight levels, shared by the CPU test of the oracles (tests/test_deep_oracle.py) and the GPU test of
the device (tests/test_gpu_deep_levels.py).  HSB_MAX_LEVELS is 8 and hector_mapping exposes the depth as
map_multi_res_levels; every per-level array of the library and of the oracles has entries 3..7 that only these
geometries reach.

The sizes are chosen so that the reference's integer halving (MapRepMultiMap.h:67) gives awkward coarse levels:

  1000 x 640 x 8, start (0.3, 0.7)   widths 1000 500 250 125 62 31 15 7, heights 640 .. 5: every width residue mod 4
                                     (the map writer's scalar and uint4 apply paths in one handle), levels 3+ end
                                     short of level 0's extent, the coarsest is near the 4-cell minimum
  515 x 900 x 7                      taller than wide, level 0 odd: 515 257 128 64 32 16 8
  2048 x 2048 x 5 at 0.025 m         the node's default size with two more levels than its default 3
  512 x 512 x 8, 1024 x 64 x 5,      the smallest maps hsb_create accepts at those depths: a 4-cell coarsest side
  64 x 1024 x 5

and one cell below the last three hsb_create refuses (REJECTED).  The iteration schedules fill all eight entries of
hsb_config::max_iterations in every encoding.  The designed scans are tests/match_cases.py's, built per level coarsest
first; the SLAM run and the golden matches are oracle/gen_golden.py's (deep.npz holds them for the two GOLDEN
geometries from the compiled reference).
"""
import numpy as np

import match_cases as mcs
from oracle import gen_golden
from oracle.record_oracle import level_iterations

f32 = np.float32
RES = mcs.RES
GOLDEN = gen_golden.DEEP_GEOMS                     # tag -> geometry, in tests/golden/deep.npz
# (sx, sy, levels, start, resolution), as match_cases.GEOMS
GEOMS = [GOLDEN["g8"], (515, 900, 7, (0.5, 0.5), RES), GOLDEN["g5"], (512, 512, 8, (0.5, 0.5), RES),
         (1024, 64, 5, (0.5, 0.5), RES), (64, 1024, 5, (0.5, 0.5), RES)]
REJECTED = [(511, 512, 8), (1024, 63, 5)]          # the coarsest level would have 3 cells on one side
SCHEDULES = gen_golden.DEEP_SCHEDULES
SLOTS = 64                                         # placeholders of an edge scan: 4 endpoints per level, 14 on the coarsest
IDS = [mcs.geom_id(g) for g in GEOMS]
GS = [(gi, s) for gi in range(len(GEOMS)) for s in SCHEDULES]
GS_IDS = [f"{IDS[gi]}-{s}" for gi, s in GS]


def schedule(name, levels):
    s = SCHEDULES[name]
    return None if s is None else s[:levels]


def record_floats(levels, iters=None):
    """hsb_get_match_record_floats: sum over the levels of 3 + 15 * evaluations"""
    return sum(3 + 15 * (m + 1) for m in level_iterations(levels, iters))


def set_fields(g, *maps):
    """match_cases.field on every level of each map (an oracle: set_logodds, a device handle: upload_level)"""
    for l, (a, b) in enumerate(mcs.level_sizes(g)):
        plane = mcs.field(a, b, l)
        for m in maps:
            (m.set_logodds if hasattr(m, "set_logodds") else m.upload_level)(l, plane)


def has_edges(g):
    """The edge scan is built where the coarsest level is larger than the 4-cell minimum.  On a 4-cell side the
    interpolation's range is [0, 2]: the one-evaluation hand-offs of such levels leave the finer levels' poses outside
    their maps, where no endpoint can sit on one level's limit and outside every coarser level."""
    return min(mcs.level_sizes(g)[-1]) > 4


def designed_scans(g, cases, runner):
    """The scans every match check uses on geometry g: finite ones of three lengths, one in level 0's strip beyond the
    coarse levels, one outside the map, an empty one, and the edge scan (match_cases.build_edge_scan with `runner`, a
    matcher under match_cases.edge_iterations: endpoints on each level's q = S - 2, the first value past it, +0 and
    the first value below 0, coarsest level first; see has_edges).
    -> (scans [(hint, pts, tag)], designed [(level, index, axis, q, inside)], index of the edge scan or None)"""
    scans = []
    # (33 endpoints leave a 4-cell level's H singular: the solve makes the pose NaN, and the reference then indexes the
    # map with a NaN endpoint's cell, SURVEY.md Q4)
    for k, n in enumerate((33 if has_edges(g) else 257, 1081, 2049)):
        h = cases.hint(k)
        scans.append((h, cases.scan(n, h, nonfinite=False), f"finite{n}"))
    h = cases.hint(5)
    scans.append((h, cases.strip_scan(700, h), "strip"))
    h = cases.hint(6)
    scans.append((h, cases.outside_scan(300, h), "outside"))
    scans.append((cases.hint(7), np.zeros((0, 2), np.float32), "empty"))
    if not has_edges(g):
        return scans, [], None
    h = cases.hint(3)
    base = cases.scan(1081, h, nonfinite=False, slots=SLOTS)
    h, pts, designed, rec = mcs.build_edge_scan(cases, runner, h, base, cases.slots)
    mcs.check_edges(cases, rec, pts, designed)
    assert {d[0] for d in designed} == set(range(g[2])), "every level has edge endpoints"
    scans.append((h, pts, "edges"))
    return scans, designed, len(scans) - 1


def golden_geometry(d, tag):
    sx, sy, L, s0, s1, res = d[f"{tag}_geom"]
    g = (int(sx), int(sy), int(L), (float(s0), float(s1)), float(res))
    assert g == GOLDEN[tag], (g, GOLDEN[tag])
    return g
