"""GPU: the node's three scan -> DataContainer conversions bit for bit, stand-alone and fused into the match kernel's
staging step in every launch shape that compiles one.

  * LaserScan ranges (rosLaserScanToDataContainer, stage_from_ranges), point clouds (rosPointCloudToDataContainer,
    stage_from_cloud) and projected ranges (laser_geometry's projection, then the cloud rule: stage_from_projected).
  * Each is a compaction: warp w of W converts the chunk [w * ceil(n / W), ...), a counting pass feeds the cross-warp
    prefix (W > 1), and a point's rank in its warp is popc(ballot & lanemask_lt).  A wrong chunk end, prefix or rank
    drops, duplicates or reorders endpoints; Gauss-Newton and the map writer would not object, so every comparison
    here is bitwise: the endpoints, their order, their number and the origo.
  * The reference is the node's own converter compiled in oracle/_ref where it is built, the C port otherwise
    (oracle.pyoracle.scan_to_points / cloud_to_points; tests/laser_projection.py for the projection).
  * Kept patterns are chosen against the chunks of the shape that converts them: all, none, one point at a chunk's
    first or last index, only the chunk and 32-lane pass boundaries, alternating points, random, and a staircase in
    which warp w's chunk keeps w mod 32 points (every warp a distinct prefix).  The window-edge values of each
    conversion sit on those same boundary indices.
  * Staging limit: a fused conversion stages the whole scan in the match kernel's shared memory, 227 KB of dynamic
    shared memory less the shape's header, shared by the G scans of a CTA.  An explicit scans_per_block = G tuning
    reserves G whole scans even when the batch has fewer scans than G (the CTA is launched with all G groups), so its
    limit is that of G scans whatever the batch size.  Projected input is checked against the single step's shape
    (8 warps, one scan per CTA) at every entry point, so its limit is that shape's in every batch shape.
  * A refused single step leaves the handle as it was: the last match's endpoints, the planes and the step record.
"""
import numpy as np
import pytest

from conftest import golden_planes, load_golden
import laser_projection as lp

pytestmark = pytest.mark.gpu

F32 = np.float32
MAX_DYN_SMEM = 232448   # dynamic shared memory one CTA may ask for (227 KB)
# every HSB_CASE launch shape: (warps per scan W, scans per CTA G, gathers in flight U)
SHAPES = [(1, 1, 4), (1, 2, 4), (2, 1, 4), (2, 2, 4), (4, 1, 4), (8, 1, 4), (16, 1, 4), (1, 7, 4), (1, 14, 4),
          (1, 28, 4), (1, 32, 4), (1, 1, 8), (2, 1, 8), (8, 1, 5), (16, 1, 3)]
PROJ_W = (1, 2, 4, 8)
RESET = dict(warps_per_scan=0, scans_per_block=0, unroll=0)
# lengths around the lane (32), warp-split (8 x 32) and chunk boundaries
LENGTHS = [1, 2, 7, 8, 9, 15, 16, 17, 31, 32, 33, 255, 256, 257, 511, 513, 1279, 1281, 4351, 4353, 1081, 4097, 65537,
           1 << 20]
FUSED_LENGTHS = [1, 7, 9, 33, 257, 513, 1081, 4097]
STANDALONE_W = 8        # conv_to_points_kernel's warps

ANGLE_MIN = float(F32(-2.3561945))
SPAN = 4.712389


def header_bytes(W, G):
    """MatchSmem<W, G>::kHeaderBytes: mbarriers, reduction rows and per-warp counts (W > 1), pacing slots (G > 1)."""
    bar = (G * 8 + 15) // 16 * 16
    red = G * 2 * 9 * 32 * 4 if W > 1 else 0
    cnt = G * 32 * 4 if W > 1 else 0
    prog = 32 * 4 if G > 1 else 0
    return (bar + red + cnt + prog + 15) // 16 * 16


def staged_limit(W, G):
    """The longest scan whose whole_scan_slots(n) = (n + 2) & ~1 slots fit G times beside the header."""
    slots = ((MAX_DYN_SMEM - header_bytes(W, G)) // (8 * G)) & ~1
    return slots - 1


SINGLE_LIMIT = staged_limit(8, 1)   # single steps, group steps and every projected entry point


def proj_limit(W):
    return min(staged_limit(W, 1), SINGLE_LIMIT)


def test_staging_limits_match_the_documented_budget():
    assert SINGLE_LIMIT == 28749
    assert staged_limit(1, 1) == 29053 and staged_limit(1, 32) == 905 and staged_limit(16, 1) == 28749


def conv_kind(oracle_kinds):
    return "reference" if "reference" in oracle_kinds else "port"


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def same(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(bits(a), bits(b))


# ---- kept patterns -----------------------------------------------------------------------------------------------
def chunks(n, W):
    c = -(-n // W)
    return [(w * c, min(n, w * c + c)) for w in range(W) if w * c < n]


def boundary_index(n, W):
    """chunk starts and ends, and every 32-lane pass's first and last index inside a chunk"""
    idx = []
    for b0, b1 in chunks(n, W):
        s = np.arange(b0, b1, 32)
        idx += [s, np.minimum(s + 31, b1 - 1), [b1 - 1]]
    return np.unique(np.concatenate(idx)) if idx else np.zeros(0, np.int64)


def patterns(n, W, seed, singles=True):
    """(name, keep mask) pairs for a scan of n inputs converted by W warps"""
    rng = np.random.default_rng(seed)
    out = [("all", np.ones(n, bool)), ("none", np.zeros(n, bool))]
    ch = chunks(n, W)
    if singles:
        pick = range(len(ch)) if n <= 4353 else sorted({0, len(ch) // 2, len(ch) - 1})
        for w in pick:
            for end, i in (("first", ch[w][0]), ("last", ch[w][1] - 1)):
                m = np.zeros(n, bool)
                m[i] = True
                out.append((f"one@w{w}{end}", m))
    m = np.zeros(n, bool)
    m[boundary_index(n, W)] = True
    out.append(("boundaries", m))
    out.append(("even", np.arange(n) % 2 == 0))
    out.append(("odd", np.arange(n) % 2 == 1))
    out.append(("random", rng.random(n) < 0.5))
    m = np.zeros(n, bool)
    for w, (b0, b1) in enumerate(ch):
        k = min(w % 32, b1 - b0)
        m[b1 - k:b1] = True
    out.append(("staircase", m))
    return out


def place_edges(vals, keep, n, W, kept_edges, dropped_edges, dropped_fill):
    """kept / dropped window-edge values on the boundary indices; dropped values everywhere else a point is dropped"""
    drop = np.nonzero(~keep)[0]
    if drop.size:
        vals[drop] = dropped_fill[np.arange(drop.size) % len(dropped_fill)]
    b = boundary_index(n, W)
    kb, db = b[keep[b]], b[~keep[b]]
    vals[kb] = kept_edges[np.arange(kb.size) % len(kept_edges)]
    vals[db] = dropped_edges[np.arange(db.size) % len(dropped_edges)]
    return vals


# ---- ranges ------------------------------------------------------------------------------------------------------
def scan_format(n, angle_min=ANGLE_MIN, inc=None):
    inc = float(F32(SPAN / max(n - 1, 1))) if inc is None else inc
    return dict(n_beams=n, angle_min=angle_min, angle_increment=inc, range_min=float(F32(0.1)), range_max=30.0)


def range_edges(fmt):
    rmin = F32(fmt["range_min"])
    rmaxc = F32(F32(fmt["range_max"]) - F32(0.1))
    kept = np.array([np.nextafter(rmin, F32(np.inf)), np.nextafter(rmaxc, F32(0)), 1.0, 12.5], F32)
    dropped = np.array([rmin, rmaxc, np.nan, np.inf, -np.inf, -0.0, np.float32(1e-40), 0.0, F32(fmt["range_max"]),
                        45.0], F32)
    return kept, dropped


def ranges_for(keep, fmt, W, base=None, seed=0):
    n = keep.size
    r = (np.random.default_rng(seed).uniform(0.5, 25.0, n) if base is None else np.array(base, np.float64)).astype(F32)
    kept, dropped = range_edges(fmt)
    rmaxc = F32(F32(fmt["range_max"]) - F32(0.1))
    r[keep & ~((r > F32(fmt["range_min"])) & (r < rmaxc))] = F32(5.0)
    return place_edges(r, keep, n, W, kept, dropped, dropped)


def ref_ranges(pyoracle, r, fmt, scale, kind):
    return pyoracle.scan_to_points(r, fmt["angle_min"], fmt["angle_increment"], fmt["range_min"], fmt["range_max"], scale,
                                   kind=kind)


# ---- clouds ------------------------------------------------------------------------------------------------------
CLOUD_FMT = dict(sqr_laser_min_dist=float(F32(0.4) * F32(0.4)), sqr_laser_max_dist=float(F32(30.0) * F32(30.0)),
                 laser_z_min_value=-1.0, laser_z_max_value=1.0)


def flat_transform(xyz=(0.12, -0.03, 0.31), yaw=0.05):
    """a laser mounted level: z_laser = z exactly, so the distance window alone decides"""
    from hector_slam_b200 import synth

    return synth.laser_transform(xyz=xyz, rpy=(0.0, 0.0, yaw))


CLOUD_KEPT = np.array([(-0.0, 0.6, 0.0),              # x = -0 is not < 0: kept though d2 < 0.5
                       (-0.5, 0.5, 0.0),              # x < 0, d2 = 0.5 exactly: not < 0.5, kept
                       (0.41, 0.0, 0.0),              # just inside sqr_min
                       (float(np.nextafter(F32(30.0), F32(0))), 0.0, 0.0),   # just inside sqr_max
                       (3.0, -2.0, 0.5)], F32)
CLOUD_DROPPED = np.array([(0.4, 0.0, 0.0),            # d2 == sqr_min: strict >
                          (30.0, 0.0, 0.0),           # d2 == sqr_max: strict <
                          (-0.5, 0.3, 0.0),           # x < 0 and d2 < 0.5
                          (-0.7, 0.1, 0.0),           # x < 0 and d2 = 0.49999997, the float under 0.5
                          (np.nan, 1.0, 0.0), (1.0, np.inf, 0.0), (2.0, 1.0, np.nan),
                          (2.0, 1.0, 1.0),            # z_laser == z_max: strict <
                          (2.0, 1.0, -1.0),           # z_laser == z_min: strict >
                          (0.1, 0.1, 0.0)], F32)


def cloud_for(keep, W, base=None, seed=0):
    n = keep.size
    rng = np.random.default_rng(seed)
    if base is None:
        r = rng.uniform(0.8, 25.0, n)
        a = rng.uniform(-np.pi, np.pi, n)
        base = np.stack([r * np.cos(a), r * np.sin(a), rng.uniform(-0.5, 0.5, n)], axis=1)
    c = np.array(base, F32).reshape(n, 3)
    return place_edges(c, keep, n, W, CLOUD_KEPT, CLOUD_DROPPED, CLOUD_DROPPED)


def ref_cloud(pyoracle, cloud, T, scale, kind, fmt=CLOUD_FMT):
    return pyoracle.cloud_to_points(cloud, T, fmt["sqr_laser_min_dist"], fmt["sqr_laser_max_dist"],
                                    fmt["laser_z_min_value"], fmt["laser_z_max_value"], scale, kind=kind)


# ---- projected ranges --------------------------------------------------------------------------------------------
PROJ_CLOUD_FMT = CLOUD_FMT   # kept ranges lie in [1, 29.5]: the cloud rule keeps all of them
CUT_F = F32(29.5)
CUTOFF = float(CUT_F) + 2.0 ** -21   # a quarter ulp above a float: r == 29.5 is kept in double, not in float


def projection(n, angle_min=ANGLE_MIN, inc=None):
    inc = float(F32(SPAN / max(n - 1, 1))) if inc is None else inc
    return dict(n_beams=n, angle_min=angle_min, angle_increment=inc, range_min=1.0, range_max=30.0,
                range_cutoff=CUTOFF)


PROJ_KEPT = np.array([1.0, CUT_F, np.nextafter(CUT_F, F32(0)), 7.25], F32)            # r == range_min is kept (>=)
PROJ_DROPPED = np.array([np.nextafter(F32(1.0), F32(0)), np.nextafter(CUT_F, F32(np.inf)), np.nan, np.inf, -np.inf,
                         -1.5, 0.0, -0.0, 30.0], F32)


def projected_for(keep, W, base=None, seed=0):
    n = keep.size
    r = (np.random.default_rng(seed).uniform(1.5, 25.0, n) if base is None else np.array(base, np.float64)).astype(F32)
    r[keep & ~((r >= F32(1.0)) & (r < CUT_F))] = F32(5.0)
    return place_edges(r, keep, n, W, PROJ_KEPT, PROJ_DROPPED, PROJ_DROPPED)


def ref_projected(pyoracle, r, proj, T, scale, kind, unit=None):
    return pyoracle.cloud_to_points(lp.project(r, proj, unit), T, PROJ_CLOUD_FMT["sqr_laser_min_dist"],
                                    PROJ_CLOUD_FMT["sqr_laser_max_dist"], PROJ_CLOUD_FMT["laser_z_min_value"],
                                    PROJ_CLOUD_FMT["laser_z_max_value"], scale, kind=kind)


# ---- 1. stand-alone conversions ----------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [1, 2])
def test_standalone_conversions_every_length_and_pattern(hsb_lib, pyoracle, oracle_kinds, mode):
    from hector_slam_b200 import capi

    kind = conv_kind(oracle_kinds)
    rep = capi.MapRepB200(0.05, 512, levels=1, gather_mode=mode)
    scale = rep.getScaleToMap()
    T = flat_transform()
    rep.set_cloud_format(T, **CLOUD_FMT)
    cases = 0
    for n in LENGTHS:
        fmt = scan_format(n)
        rep.set_scan_format(**fmt)
        for name, keep in patterns(n, STANDALONE_W, seed=n):
            r = ranges_for(keep, fmt, STANDALONE_W, seed=n)
            want = ref_ranges(pyoracle, r, fmt, scale, kind)
            assert want.shape[0] == keep.sum(), ("ranges pattern not realised", n, name)
            got = rep.scan_to_points(r)
            assert same(got, want), ("ranges", n, name, got.shape, want.shape)
            cloud = cloud_for(keep, STANDALONE_W, seed=n)
            want, want_origo = ref_cloud(pyoracle, cloud, T, scale, kind)
            assert want.shape[0] == keep.sum(), ("cloud pattern not realised", n, name)
            got, origo = rep.cloud_to_points(cloud)
            assert same(got, want) and same(origo, want_origo), ("cloud", n, name, got.shape, want.shape)
            cases += 1
    # projected: every length its entry point accepts
    rep.set_cloud_format(T, **PROJ_CLOUD_FMT)
    for n in sorted({m for m in LENGTHS if m <= SINGLE_LIMIT} | {SINGLE_LIMIT}):
        proj = projection(n)
        rep.set_laser_projection(**proj)
        unit = lp.unit_vectors(n, proj["angle_min"], proj["angle_increment"])
        for name, keep in patterns(n, STANDALONE_W, seed=n + 1):
            r = projected_for(keep, STANDALONE_W, seed=n)
            want, want_origo = ref_projected(pyoracle, r, proj, T, scale, kind, unit)
            assert want.shape[0] == keep.sum(), ("projected pattern not realised", n, name)
            got, origo = rep.projected_scan_to_points(r)
            assert same(got, want) and same(origo, want_origo), ("projected", n, name, got.shape, want.shape)
    assert cases > 300
    rep.close()


def z_laser(T, x, y, z):
    """float((T8 x + T9 y + T10 z) + T11 - T11), every double operation rounded (the cloud rule's z test)"""
    return F32((((T[8] * float(x) + T[9] * float(y)) + T[10] * float(z)) + T[11]) - T[11])


def find_z(T, x, y, edge, inside):
    """(y', z) near (y, the plane's z) whose z_laser is exactly `edge` (inside=False) or the float next to it inside
    the window: the z window's edges under a tilted transform.  Where the floats of z step over the edge, y moves by
    2e-6 and the search runs again."""
    want = F32(edge) if not inside else np.nextafter(F32(edge), F32(0))
    y = F32(y)
    for _ in range(400):
        z = F32((float(edge) - T[8] * float(x) - T[9] * float(y)) / T[10])
        up = z_laser(T, x, y, z) < want
        for _ in range(64):
            zl = z_laser(T, x, y, z)
            if zl == want:
                return y, z
            if (zl < want) != up:
                break
            z2 = F32(z + F32(2e-8 if up else -2e-8))   # a third of z_laser's float spacing below 1, or one ulp of z
            z = z2 if z2 != z else np.nextafter(z, F32(np.inf) if up else F32(-np.inf))
        y = F32(y + F32(2e-6))
    raise AssertionError(("no z found", edge, inside))


@pytest.mark.parametrize("mode", [1, 2])
def test_cloud_edges_under_tilted_and_translated_transforms(hsb_lib, pyoracle, oracle_kinds, mode):
    """z exactly on each edge of the window (and the float inside it) under a tilted transform, at chunk and lane
    boundaries; a transform with a large translation (origo and endpoints far from the map's start)."""
    from hector_slam_b200 import capi, synth

    kind = conv_kind(oracle_kinds)
    rep = capi.MapRepB200(0.05, 512, levels=1, gather_mode=mode)
    scale = rep.getScaleToMap()
    tilted = lp.tilted_transform()
    far = synth.laser_transform(xyz=(1.0e4 + 0.3, -3.0e3 - 0.7, 0.4), rpy=(0.03, -0.05, 2.9))
    for T in (tilted, far):
        rep.set_cloud_format(T, **CLOUD_FMT)
        for n in (33, 257, 1081, 4353):
            rng = np.random.default_rng(n)
            r = rng.uniform(0.8, 6.0, n)
            a = rng.uniform(-np.pi, np.pi, n)
            cloud = np.stack([r * np.cos(a), r * np.sin(a), np.zeros(n)], axis=1).astype(F32)
            b = boundary_index(n, STANDALONE_W)
            for j, i in enumerate(b):   # z_max, z_min, the float inside z_max, the float inside z_min, ...
                cloud[i, 1:] = find_z(T, cloud[i, 0], cloud[i, 1], (1.0, -1.0)[j % 2], inside=(j // 2) % 2 == 1)
                assert z_laser(T, cloud[i, 0], cloud[i, 1], cloud[i, 2]) != 0
            want, want_origo = ref_cloud(pyoracle, cloud, T, scale, kind)
            got, origo = rep.cloud_to_points(cloud)
            assert same(got, want) and same(origo, want_origo), (n, got.shape, want.shape)
            assert 0 < want.shape[0] < n
    rep.close()


@pytest.mark.parametrize("mode", [1, 2])
def test_long_formats_build_their_tables_like_the_reference(hsb_lib, pyoracle, oracle_kinds, mode):
    """2^20-beam scan formats with angle increments down to 1e-6 rad: the host's fp32 angle accumulation in
    hsb_set_scan_format against the reference converter; the double unit vectors of hsb_set_laser_projection against
    tests/laser_projection.py on the longest scan the projected entry point accepts."""
    from hector_slam_b200 import capi

    kind = conv_kind(oracle_kinds)
    rep = capi.MapRepB200(0.05, 512, levels=1, gather_mode=mode)
    scale = rep.getScaleToMap()
    T = flat_transform()
    rep.set_cloud_format(T, **PROJ_CLOUD_FMT)
    rng = np.random.default_rng(5)
    for a0, inc in ((-3.14159, 1.0e-6), (0.5, 3.0e-6), (-3.1415927, float(F32(2 * np.pi / (1 << 20)))),
                    (1.0e3, 1.0e-6)):
        fmt = scan_format(1 << 20, angle_min=a0, inc=inc)
        rep.set_scan_format(**fmt)
        r = rng.uniform(0.5, 25.0, 1 << 20).astype(F32)
        r[::7] = np.nan
        want = ref_ranges(pyoracle, r, fmt, scale, kind)
        assert same(rep.scan_to_points(r), want), (a0, inc)
        proj = projection(SINGLE_LIMIT, angle_min=a0, inc=inc)
        rep.set_laser_projection(**proj)
        rp = rng.uniform(1.5, 25.0, SINGLE_LIMIT).astype(F32)
        want, want_origo = ref_projected(pyoracle, rp, proj, T, scale, kind)
        got, origo = rep.projected_scan_to_points(rp)
        assert same(got, want) and same(origo, want_origo), (a0, inc)
    rep.close()


# ---- 2. fused conversions in every shape -------------------------------------------------------------------------
def golden_rep(mode):
    from hector_slam_b200 import capi

    g = load_golden("match3.npz")
    rep = capi.MapRepB200(float(g["res"]), int(g["size"]), levels=3, update_factor_free=0.4, update_factor_occupied=0.9,
                          gather_mode=mode)
    for l, p in enumerate(golden_planes(g)):
        rep.upload_level(l, p)
    return rep


def beam_angles(fmt):
    out = np.empty(fmt["n_beams"], F32)
    a = F32(fmt["angle_min"])
    for i in range(fmt["n_beams"]):
        out[i] = a
        a = F32(a + F32(fmt["angle_increment"]))
    return out


def world_scans(n, B, seed):
    """B scans of n beams spread over the full circle, taken in the synthetic world, and their poses"""
    from hector_slam_b200 import synth

    world = synth.World(1, seed=1234)
    poses = world.sample_free_poses(B, np.random.default_rng(seed), margin=0.8)
    ang = np.linspace(-np.pi, np.pi, n, endpoint=False)
    return poses, [world.cast(p, ang) for p in poses], ang


def shape_lengths(limit):
    return [n for n in FUSED_LENGTHS if n <= limit] + [limit]


def assert_shape(rep, W, G, U):
    s = rep.last_launch_shape()
    assert (s["warps_per_scan"], s["scans_per_block"], s["unroll"]) == (W, G, U), s


def offsets_of(chunks_):
    return np.concatenate([[0], np.cumsum([c.shape[0] for c in chunks_])]).astype(np.int32)


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("shape", SHAPES, ids=[f"W{w}G{g}U{u}" for w, g, u in SHAPES])
def test_fused_batch_ranges_and_cloud_every_shape(hsb_lib, pyoracle, oracle_kinds, shape, mode):
    """hsb_match_batch_ranges / _cloud in the shape == hsb_match_batch in the same shape on the reference converter's
    endpoints, poses and covariances bit for bit; patterns against the shape's own chunks; lengths up to the limit."""
    from hector_slam_b200 import synth

    W, G, U = shape
    kind = conv_kind(oracle_kinds)
    rep = golden_rep(mode)
    scale = rep.getScaleToMap()
    rep.set_tuning(**{**RESET, "warps_per_scan": W, "scans_per_block": G, "unroll": U})
    limit = staged_limit(W, G)
    for n in shape_lengths(limit):
        fmt = dict(scan_format(n), angle_min=float(F32(-np.pi)), angle_increment=float(F32(2 * np.pi / n)))
        rep.set_scan_format(**fmt)
        pats = patterns(n, W, seed=n, singles=n <= 1081)
        poses, casts, _ = world_scans(n, len(pats), seed=n)
        ranges = np.stack([ranges_for(k, fmt, W, base=c) for (_, k), c in zip(pats, casts)])
        refs = [ref_ranges(pyoracle, r, fmt, scale, kind) for r in ranges]
        for (name, k), e in zip(pats, refs):
            assert e.shape[0] == k.sum(), (n, name)
        hints = synth.perturb_hints(poses, seed=n)
        got, cov = rep.match_batch_ranges(hints, ranges)
        assert_shape(rep, W, G, U)
        want, wcov = rep.match_batch(hints, np.concatenate(refs).reshape(-1, 2), offsets_of(refs))
        assert_shape(rep, W, G, U)
        assert same(got, want) and same(cov, wcov), ("ranges", shape, n)
    # clouds: ragged lengths in one batch, every pattern of every length class, one transform per scan
    rep.set_cloud_format(flat_transform(), **CLOUD_FMT)
    clouds, refs, Ts, origos = [], [], [], []
    for n in shape_lengths(limit):
        pats = patterns(n, W, seed=n + 7, singles=n <= 257)
        _, casts, ang = world_scans(n, len(pats), seed=n + 7)
        for j, ((name, k), c) in enumerate(zip(pats, casts)):
            base = np.stack([c * np.cos(ang), c * np.sin(ang), np.zeros(n)], axis=1)
            cl = cloud_for(k, W, base=base)
            T = flat_transform(xyz=(0.1 * (j % 3), -0.05, 0.3), yaw=0.01 * j)
            e, og = ref_cloud(pyoracle, cl, T, scale, kind)
            assert e.shape[0] == k.sum(), (n, name)
            clouds.append(cl), refs.append(e), Ts.append(T), origos.append(og)
    B = len(clouds)
    hints = synth.perturb_hints(synth.World(1, seed=1234).sample_free_poses(B, np.random.default_rng(3), margin=0.8))
    got, cov, og = rep.match_batch_cloud(hints, np.concatenate(clouds), offsets_of(clouds), transforms=np.stack(Ts))
    assert_shape(rep, W, G, U)
    want, wcov = rep.match_batch(hints, np.concatenate(refs).reshape(-1, 2), offsets_of(refs))
    assert same(got, want) and same(cov, wcov) and same(og, np.stack(origos)), ("cloud", shape)
    rep.close()


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("W", PROJ_W)
def test_fused_batch_projected_every_shape(hsb_lib, pyoracle, oracle_kinds, W, mode):
    from hector_slam_b200 import synth

    kind = conv_kind(oracle_kinds)
    rep = golden_rep(mode)
    scale = rep.getScaleToMap()
    rep.set_tuning(**{**RESET, "warps_per_scan": W, "scans_per_block": 1, "unroll": 4})
    rep.set_cloud_format(flat_transform(), **PROJ_CLOUD_FMT)
    for n in shape_lengths(proj_limit(W)):
        proj = dict(projection(n), angle_min=float(F32(-np.pi)), angle_increment=float(F32(2 * np.pi / n)))
        rep.set_laser_projection(**proj)
        unit = lp.unit_vectors(n, proj["angle_min"], proj["angle_increment"])
        pats = patterns(n, W, seed=n + 3, singles=n <= 1081)
        poses, casts, _ = world_scans(n, len(pats), seed=n + 3)
        ranges = np.stack([projected_for(k, W, base=c) for (_, k), c in zip(pats, casts)])
        Ts = np.stack([flat_transform(xyz=(0.05 * (b % 4), 0.02, 0.3), yaw=-0.02 * b) for b in range(len(pats))])
        refs, origos = [], []
        for (name, k), r, T in zip(pats, ranges, Ts):
            e, og = ref_projected(pyoracle, r, proj, T, scale, kind, unit)
            assert e.shape[0] == k.sum(), (n, name)
            refs.append(e), origos.append(og)
        hints = synth.perturb_hints(poses, seed=n)
        got, cov, og = rep.match_batch_projected(hints, ranges, transforms=Ts)
        assert_shape(rep, W, 1, 4)
        want, wcov = rep.match_batch(hints, np.concatenate(refs).reshape(-1, 2), offsets_of(refs))
        assert same(got, want) and same(cov, wcov) and same(og, np.stack(origos)), ("projected", W, n)
    rep.close()


class Steps:
    """One scan in each input kind, with its reference container: ranges (scan format), cloud, projected."""

    def __init__(self, pyoracle, kind, n, keep, seed, scale):
        _, casts, ang = world_scans(n, 1, seed)
        c = casts[0]
        self.fmt = dict(scan_format(n), angle_min=float(F32(-np.pi)), angle_increment=float(F32(2 * np.pi / n)))
        self.proj = dict(projection(n), angle_min=float(F32(-np.pi)), angle_increment=float(F32(2 * np.pi / n)))
        self.T = flat_transform(xyz=(0.2, -0.1, 0.3), yaw=0.03)
        self.ranges = ranges_for(keep, self.fmt, 8, base=c)
        self.cloud = cloud_for(keep, 8, base=np.stack([c * np.cos(ang), c * np.sin(ang), np.zeros(n)], axis=1))
        self.projected = projected_for(keep, 8, base=c)
        self.want = {"ranges": (ref_ranges(pyoracle, self.ranges, self.fmt, scale, kind), np.zeros(2, F32)),
                     "cloud": ref_cloud(pyoracle, self.cloud, self.T, scale, kind),
                     "projected": ref_projected(pyoracle, self.projected, self.proj, self.T, scale, kind)}
        for k, (e, _) in self.want.items():
            assert e.shape[0] == keep.sum(), k

    def configure(self, rep):
        rep.set_scan_format(**self.fmt)
        rep.set_cloud_format(self.T, **PROJ_CLOUD_FMT)
        rep.set_laser_projection(**self.proj)

    def step(self, rep, what, hint, without=False):
        if what == "ranges":
            return rep.slam_update_ranges(hint, self.ranges, map_without_matching=without)
        if what == "cloud":
            return rep.slam_update_cloud(hint, self.cloud, map_without_matching=without)
        return rep.slam_update_projected(hint, self.projected, map_without_matching=without)

    def group_step(self, grp, what, hints, members):
        scans = {"ranges": self.ranges, "cloud": self.cloud, "projected": self.projected}[what]
        fn = getattr(grp, f"slam_update_{what}")
        return fn(hints, [scans] * len(members), members=members)


KINDS = ("ranges", "cloud", "projected")


def fresh_rep(mode, levels=2):
    from hector_slam_b200 import capi

    rep = capi.MapRepB200(0.05, 1024, levels=levels, update_factor_free=0.4, update_factor_occupied=0.9,
                          gather_mode=mode)
    rep.setMapUpdateMinDistDiff(0.0)
    rep.setMapUpdateMinAngleDiff(0.0)
    return rep


@pytest.mark.parametrize("mode", [1, 2])
def test_fused_single_and_group_steps_stage_the_reference_container(hsb_lib, pyoracle, oracle_kinds, mode):
    """slam_update_ranges / _cloud / _projected and the group steps of all three kinds, full and subset: the kept count
    and last_match_scan() (endpoints and origo) equal the reference converter; a map_without_matching step's level-0
    plane equals oracle/mapwrite.py's `dev` plane written from the converter's endpoints."""
    from hector_slam_b200 import capi
    from oracle import mapwrite as mw

    kind = conv_kind(oracle_kinds)
    M = 4
    hint = np.float32([0.3, -0.2, 0.1])
    for n in [1, 9, 33, 257, 1081, 4097, SINGLE_LIMIT]:
        for pname, keep in patterns(n, 8, seed=n, singles=False):
            if pname in ("even", "odd") and n > 1081:
                continue
            reps = [fresh_rep(mode) for _ in range(M)]
            S = Steps(pyoracle, kind, n, keep, seed=n, scale=reps[0].getScaleToMap())
            for r in reps:
                S.configure(r)
            for what in KINDS:
                want, want_origo = S.want[what]
                _, _, _, kept = S.step(reps[0], what, hint)
                pts, origo = reps[0].last_match_scan()
                assert kept == want.shape[0] and same(pts, want) and same(origo, want_origo), (what, n, pname)
                grp = capi.SlamGroup(reps)
                for members in (list(range(M)), [2, 0]):
                    hints = np.tile(hint, (len(members), 1))
                    _, _, _, kept = S.group_step(grp, what, hints, members)
                    assert list(kept) == [want.shape[0]] * len(members), (what, n, pname, members)
                    for m in members:
                        pts, origo = reps[m].last_match_scan()
                        assert same(pts, want) and same(origo, want_origo), (what, n, pname, members, m)
                grp.close()
            if pname in ("random", "boundaries") and n <= 4097:
                for what in KINDS:
                    rep = fresh_rep(mode, levels=1)
                    S.configure(rep)
                    _, _, upd, kept = S.step(rep, what, hint, without=True)
                    want, want_origo = S.want[what]
                    assert upd and kept == want.shape[0], (what, n, pname)
                    L = mw.geometry(0.05, 1024, 1024, 1)[0]
                    lf, lo = rep.logodds_increments()
                    w = mw.write(np.zeros((1024, 1024), F32), L, mw.beams(L, want, hint, want_origo), lf, lo)
                    assert np.array_equal(bits(rep.download_level(0)), bits(w.dev)), (what, n, pname)
                    rep.close()
            for r in reps:
                r.close()


# ---- 3. staging limits --------------------------------------------------------------------------------------------
def too_long(excinfo):
    return "scan too long" in str(excinfo.value)


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("shape", SHAPES, ids=[f"W{w}G{g}U{u}" for w, g, u in SHAPES])
def test_batch_staging_limit_per_shape(hsb_lib, pyoracle, oracle_kinds, shape, mode):
    """The longest scan a shape stages is accepted, every point kept (the last slot written), and matches like its
    reference endpoints; one point more is refused with "scan too long", and the batch after it is unaffected."""
    from hector_slam_b200 import capi, synth

    W, G, U = shape
    kind = conv_kind(oracle_kinds)
    rep = golden_rep(mode)
    scale = rep.getScaleToMap()
    rep.set_tuning(**{**RESET, "warps_per_scan": W, "scans_per_block": G, "unroll": U})
    limit = staged_limit(W, G)
    poses, casts, ang = world_scans(limit + 1, 3, seed=W * 100 + G)
    hints = synth.perturb_hints(poses, seed=G)
    fmt = dict(scan_format(limit), angle_min=float(F32(-np.pi)), angle_increment=float(F32(2 * np.pi / limit)))
    rep.set_scan_format(**fmt)
    keep = np.ones(limit, bool)
    ranges = np.stack([ranges_for(keep, fmt, W, base=c[:limit]) for c in casts])
    refs = [ref_ranges(pyoracle, r, fmt, scale, kind) for r in ranges]
    assert all(e.shape[0] == limit for e in refs)
    got, cov = rep.match_batch_ranges(hints, ranges)
    assert_shape(rep, W, G, U)
    want, wcov = rep.match_batch(hints, np.concatenate(refs), offsets_of(refs))
    assert same(got, want) and same(cov, wcov)
    rep.set_scan_format(**dict(fmt, n_beams=limit + 1))
    with pytest.raises(capi.HsbError) as e:
        rep.match_batch_ranges(hints, np.stack([c.astype(F32) for c in casts]))
    assert too_long(e), str(e.value)
    rep.set_scan_format(**fmt)
    again, again_cov = rep.match_batch_ranges(hints, ranges)
    assert same(again, got) and same(again_cov, cov)
    # clouds: the longest accepted beside shorter ones, then one point more
    rep.set_cloud_format(flat_transform(), **CLOUD_FMT)
    T = flat_transform()
    full = [np.stack([c * np.cos(ang), c * np.sin(ang), np.zeros(limit + 1)], axis=1).astype(F32) for c in casts]
    clouds = [full[0][:limit], full[1][:limit // 2], full[2][:limit]]
    refs = [ref_cloud(pyoracle, c, T, scale, kind)[0] for c in clouds]
    assert refs[0].shape[0] == limit and refs[2].shape[0] == limit
    got, cov, _ = rep.match_batch_cloud(hints, np.concatenate(clouds), offsets_of(clouds))
    assert_shape(rep, W, G, U)
    want, wcov = rep.match_batch(hints, np.concatenate(refs), offsets_of(refs))
    assert same(got, want) and same(cov, wcov)
    longer = [clouds[0], full[1], clouds[2]]
    with pytest.raises(capi.HsbError) as e:
        rep.match_batch_cloud(hints, np.concatenate(longer), offsets_of(longer))
    assert too_long(e), str(e.value)
    again, again_cov, _ = rep.match_batch_cloud(hints, np.concatenate(clouds), offsets_of(clouds))
    assert same(again, got) and same(again_cov, cov)
    rep.close()


@pytest.mark.parametrize("mode", [1, 2])
def test_projected_batch_staging_limit(hsb_lib, pyoracle, oracle_kinds, mode):
    """every projected batch shape accepts the single step's limit (the entry point checks that shape) and refuses one
    beam more"""
    from hector_slam_b200 import capi, synth

    kind = conv_kind(oracle_kinds)
    rep = golden_rep(mode)
    scale = rep.getScaleToMap()
    T = flat_transform()
    rep.set_cloud_format(T, **PROJ_CLOUD_FMT)
    n = SINGLE_LIMIT
    poses, casts, _ = world_scans(n, 2, seed=11)
    hints = synth.perturb_hints(poses, seed=4)
    proj = dict(projection(n), angle_min=float(F32(-np.pi)), angle_increment=float(F32(2 * np.pi / n)))
    ranges = np.stack([projected_for(np.ones(n, bool), 8, base=c) for c in casts])
    unit = lp.unit_vectors(n, proj["angle_min"], proj["angle_increment"])
    refs = [ref_projected(pyoracle, r, proj, T, scale, kind, unit)[0] for r in ranges]
    assert all(e.shape[0] == n for e in refs)
    for W in PROJ_W:
        assert proj_limit(W) == n
        rep.set_tuning(**{**RESET, "warps_per_scan": W, "scans_per_block": 1, "unroll": 4})
        rep.set_laser_projection(**proj)
        got, cov, _ = rep.match_batch_projected(hints, ranges)
        assert_shape(rep, W, 1, 4)
        want, wcov = rep.match_batch(hints, np.concatenate(refs), offsets_of(refs))
        assert same(got, want) and same(cov, wcov), W
        rep.set_laser_projection(**dict(proj, n_beams=n + 1))
        with pytest.raises(capi.HsbError) as e:
            rep.match_batch_projected(hints, np.concatenate([ranges, ranges[:, :1]], axis=1))
        assert too_long(e), str(e.value)
    rep.close()


def handle_state(rep):
    pts, origo = rep.last_match_scan()
    return (pts, origo, [rep.download_level(l) for l in range(rep.levels)], rep.last_map_update_pose())


def assert_same_state(a, b):
    assert same(a[0], b[0]) and same(a[1], b[1]), "last match container changed"
    for l, (p, q) in enumerate(zip(a[2], b[2])):
        assert np.array_equal(bits(p), bits(q)), ("plane changed", l)
    assert same(a[3], b[3])


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("what", KINDS)
def test_single_and_group_step_staging_limit(hsb_lib, pyoracle, oracle_kinds, what, mode):
    """A single or group step of SINGLE_LIMIT inputs, every one kept, stages all of them (last_match_scan equals the
    reference converter's, its last endpoint included); one input more is refused with "scan too long" and leaves the
    handle as it was: the last match's endpoints and origo, every plane, the gate pose, and no step record where no
    step ran."""
    from hector_slam_b200 import capi

    kind = conv_kind(oracle_kinds)
    n = SINGLE_LIMIT
    hint = np.float32([0.1, 0.2, -0.05])
    rep, twin = fresh_rep(mode), fresh_rep(mode)
    S = Steps(pyoracle, kind, n, np.ones(n, bool), seed=21, scale=rep.getScaleToMap())
    Sl = Steps(pyoracle, kind, n + 1, np.ones(n + 1, bool), seed=22, scale=rep.getScaleToMap())
    # a refused first step: the handle has taken no fused step
    Sl.configure(rep)
    rep.set_step_record(True)
    with pytest.raises(capi.HsbError) as e:
        Sl.step(rep, what, hint)
    assert too_long(e), str(e.value)
    with pytest.raises(capi.HsbError):
        rep.step_record()
    # accepted at the limit
    S.configure(rep)
    _, _, _, kept = S.step(rep, what, hint)
    want, want_origo = S.want[what]
    pts, origo = rep.last_match_scan()
    assert kept == n and same(pts, want) and same(origo, want_origo)
    rec = rep.step_record(raw=True)
    before = handle_state(rep)
    Sl.configure(rep)
    with pytest.raises(capi.HsbError) as e:
        Sl.step(rep, what, hint)
    assert too_long(e), str(e.value)
    assert_same_state(handle_state(rep), before)
    assert same(rep.step_record(raw=True), rec)
    # the next step draws the coarse level from the kept container: it equals a twin's that was never refused
    S.configure(rep)
    S.configure(twin)
    S.step(twin, what, hint)
    a = S.step(rep, what, hint, without=True)
    b = S.step(twin, what, hint, without=True)
    assert same(a[0], b[0]) and a[2:] == b[2:]
    assert_same_state(handle_state(rep), handle_state(twin))
    # group steps: the limit of their one-scan-per-CTA 8-warp shape
    grp = capi.SlamGroup([rep, twin])
    _, _, _, kept = S.group_step(grp, what, np.tile(hint, (2, 1)), [0, 1])
    assert list(kept) == [n, n]
    for r in (rep, twin):
        pts, origo = r.last_match_scan()
        assert same(pts, want) and same(origo, want_origo)
    before = handle_state(rep)
    Sl.configure(rep)
    Sl.configure(twin)
    with pytest.raises(capi.HsbError) as e:
        Sl.group_step(grp, what, np.tile(hint, (2, 1)), [1, 0])
    assert too_long(e), str(e.value)
    assert_same_state(handle_state(rep), before)
    grp.close()
    rep.close()
    twin.close()
