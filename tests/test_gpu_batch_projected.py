"""hsb_match_batch_projected (host buffers, submit / wait) and hsb_match_batch_projected_device — a default node's
LaserScans matched in one batch: laser_geometry's projection and the cloud conversion in the match kernel's staging step.

Every scan's pose, covariance and origo must equal hsb_match_batch_cloud on the cloud tests/laser_projection.py projects
from it and hsb_match_batch on the endpoints hsb_projected_scan_to_points returns, bit for bit, in every launch shape the
projection is compiled into; and the poses must agree with the node's compiled converter + the reference's matcher."""
import math

import numpy as np
import pytest

from conftest import golden_planes, load_golden, pose_err, report
from laser_projection import edge_ranges, project, tilted_transform, unit_vectors

pytestmark = pytest.mark.gpu

F32 = np.float32
B = 48
# n_beams, angle_min (deg), angle_increment (deg), range_min, range_max, range_cutoff (< 0: range_max)
GEOMS = [(1081, -135.0, 0.25, 0.1, 30.0, 30.0), (720, -180.0, 0.5, 0.3, 12.0, 30.0), (360, -120.0, 0.75, 0.5, 20.0, -1.0),
         (1440, -180.0, 0.25, 0.2, 8.0, 6.5)]
DROPPED = 11   # the all-dropped scan
# the staging limit of the fused conversion (8-warp shape): 2448 B of header + whole_scan_slots(n) * 8 B <= 227 KB
LIMIT = 28749


def geometry(k):
    n, a0, da, rmin, rmax, cut = GEOMS[k]
    return dict(n_beams=n, angle_min=float(F32(math.radians(a0))), angle_increment=float(F32(math.radians(da))),
                range_min=rmin, range_max=rmax, range_cutoff=cut)


def golden_rep(gather, proj=None, with_cloud=True, T0=None):
    from hector_slam_b200 import capi, synth

    g = load_golden("match3.npz")
    rep = capi.MapRepB200(float(g["res"]), int(g["size"]), levels=3, update_factor_free=0.4, update_factor_occupied=0.9,
                          gather_mode=gather)
    for l, p in enumerate(golden_planes(g)):
        rep.upload_level(l, p)
    if proj is not None:
        rep.set_laser_projection(**proj)
    if with_cloud:
        rep.set_cloud_format(synth.laser_transform() if T0 is None else T0, **synth.CLOUD_FORMAT)
    return rep


def scans(k):
    """B scans of geometry k in the golden map's world with the projector's edge values, one all-dropped scan, hints,
    and per-scan transforms (every third one tilted, its own)."""
    from hector_slam_b200 import synth

    p = geometry(k)
    world = synth.World(1, seed=1234)
    rng = np.random.default_rng(78 + k)
    poses = world.sample_free_poses(B, rng, margin=0.8)
    angles = (float(F32(p["angle_min"])) + np.arange(p["n_beams"]) * float(F32(p["angle_increment"]))).astype(F32)
    ranges = np.empty((B, p["n_beams"]), F32)
    for b in range(B):
        r = (world.cast(poses[b], angles) + rng.normal(0.0, 0.01, p["n_beams"])).astype(F32)
        ranges[b] = edge_ranges(p["n_beams"], p, 100 * k + b, base=r)
    ranges[DROPPED] = np.nan
    T0 = synth.laser_transform()
    Ts = np.tile(T0, (B, 1))
    for b in range(0, B, 3):
        Ts[b] = tilted_transform(pitch=0.01 * (b % 7), yaw=0.03 * (b % 5), z=0.3)
    return p, ranges, synth.perturb_hints(poses, seed=2 + k), T0, Ts


def by_cloud(rep, p, ranges, hints, Ts):
    u = unit_vectors(p["n_beams"], p["angle_min"], p["angle_increment"])
    clouds = [project(ranges[b], p, u) for b in range(B)]
    offs = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int32)
    return rep.match_batch_cloud(hints, np.concatenate(clouds), offs, transforms=Ts)


def by_endpoints(rep, ranges, hints, Ts):
    conv = [rep.projected_scan_to_points(ranges[b], Ts[b]) for b in range(B)]
    offs = np.concatenate([[0], np.cumsum([c[0].shape[0] for c in conv])]).astype(np.int32)
    poses, cov = rep.match_batch(hints, np.concatenate([c[0] for c in conv]), offs)
    return poses, cov, np.stack([c[1] for c in conv]), offs


@pytest.mark.parametrize("gather", ["ldg", "tex"])
@pytest.mark.parametrize("k", range(4))
def test_bitwise_equal_to_cloud_and_endpoint_batches(hsb_lib, gather, k):
    from hector_slam_b200 import capi

    p, ranges, hints, T0, Ts = scans(k)
    rep = golden_rep(capi.GATHER_LDG if gather == "ldg" else capi.GATHER_TEX, p, T0=T0)
    for w in (0, 1, 2, 4, 8):
        rep.set_tuning(warps_per_scan=w)
        got, cov, og = rep.match_batch_projected(hints, ranges, transforms=Ts)
        if w:
            shape = rep.last_launch_shape()
            assert (shape["warps_per_scan"], shape["scans_per_block"], shape["unroll"]) == (w, 1, 4), shape
        c_p, c_cov, c_og = by_cloud(rep, p, ranges, hints, Ts)
        e_p, e_cov, e_og, offs = by_endpoints(rep, ranges, hints, Ts)
        for want, want_cov, want_og in ((c_p, c_cov, c_og), (e_p, e_cov, e_og)):
            assert np.array_equal(got, want), (w, np.abs(got - want).max())
            assert np.array_equal(cov, want_cov), w
            assert np.array_equal(og, want_og), w
    assert offs[DROPPED + 1] == offs[DROPPED] and (np.diff(offs) > 0).sum() == B - 1
    assert np.array_equal(got[DROPPED], hints[DROPPED]) and not cov[DROPPED].any()
    # NULL transforms == B copies of the cloud format's
    rep.set_tuning(warps_per_scan=0)
    a, ca, oa = rep.match_batch_projected(hints, ranges)
    b_, cb, ob = rep.match_batch_projected(hints, ranges, transforms=np.tile(T0, (B, 1)))
    assert np.array_equal(a, b_) and np.array_equal(ca, cb) and np.array_equal(oa, ob)
    rep.close()


def test_against_the_reference_converter_and_matcher(hsb_lib, pyoracle, oracle_kinds):
    """The same scans through the node's compiled converter (laser_projection.container) and the oracle's match_batch."""
    from hector_slam_b200 import capi, synth

    from laser_projection import container

    kind = "reference" if "reference" in oracle_kinds else "port"
    g = load_golden("match3.npz")
    orc = pyoracle.Oracle(kind, float(g["res"]), int(g["size"]), 3)
    orc.set_update_factors(0.4, 0.9)
    for l, plane in enumerate(golden_planes(g)):
        orc.set_logodds(l, plane)
    worst = 0.0
    for k in range(4):
        p, ranges, hints, T0, Ts = scans(k)
        rep = golden_rep(capi.GATHER_LDG, p, T0=T0)
        got, _, og = rep.match_batch_projected(hints, ranges, transforms=Ts)
        conts = [container(ranges[b], p, synth.CLOUD_FORMAT, Ts[b], rep.getScaleToMap(), pyoracle, kind=kind)
                 for b in range(B)]
        offs = np.concatenate([[0], np.cumsum([c[0].shape[0] for c in conts])]).astype(np.int32)
        want, _, _ = orc.match_batch(hints, np.concatenate([c[0] for c in conts]).astype(F32), offs)
        assert np.array_equal(og, np.stack([c[1] for c in conts])), k
        ex, ey, ea = pose_err(got, want)
        worst = max(worst, ex, ey, ea)
        assert max(ex, ey) <= 1e-4 and ea <= 1e-4, (k, ex, ey, ea)
        rep.close()
    orc.close()
    report(f"projected batch vs {kind} converter + match_batch, 4 x {B} scans: worst pose difference {worst:.2e}")


# ---- the bench-sized map: auto shapes, the two-half host pipeline, submit / wait, launch counts -------------------
@pytest.fixture(scope="module")
def bench_rep(hsb_lib):
    import bench
    from hector_slam_b200 import capi, synth

    world, _, _, _, hints = bench.make_workload(0, bench.BATCH)
    ranges = np.ascontiguousarray(bench.make_workload.ranges)
    rep = capi.MapRepB200(bench.RES, bench.MAP_SIZE, levels=bench.LEVELS, update_factor_free=0.4,
                          update_factor_occupied=0.9)
    bench.build_map_on_gpu(rep, world)
    rep.set_laser_projection(**synth.SCAN_FORMAT, range_cutoff=30.0)
    rep.set_scan_format(**synth.SCAN_FORMAT)
    T0 = synth.laser_transform()
    rep.set_cloud_format(T0, **synth.CLOUD_FORMAT)
    Ts = np.tile(T0, (bench.BATCH, 1))
    Ts[::3] = tilted_transform(pitch=0.02, z=0.3)
    yield dict(rep=rep, hints=hints, ranges=ranges, Ts=Ts, B=bench.BATCH)
    rep.close()


def device_projected(rep, hints, ranges, Ts):
    import torch

    dev = torch.device("cuda", 0)
    n = hints.shape[0]
    d_h, d_r, d_t = (torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (hints, ranges, Ts))
    d_p = torch.empty((n, 3), dtype=torch.float32, device=dev)
    d_c = torch.empty((n, 9), dtype=torch.float32, device=dev)
    d_o = torch.empty((n, 2), dtype=torch.float32, device=dev)
    rep.match_batch_projected_device(n, d_h.data_ptr(), d_r.data_ptr(), d_t.data_ptr(), d_p.data_ptr(), d_c.data_ptr(),
                                     d_o.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return d_p.cpu().numpy(), d_c.cpu().numpy().reshape(n, 3, 3), d_o.cpu().numpy()


def test_auto_shapes_and_host_pipeline(bench_rep):
    """Auto shapes on an H100 (132 SMs): 8, 4, 2, 1 warps per scan at B = 256 .. 4096, one scan per CTA.  The host call
    of 4096 scans travels in two halves matched in the shape of a 2048-scan batch (one warp per scan, as the device call
    of 4096 takes): it equals the device call bit for bit.  One match launch per chunk."""
    w = bench_rep
    rep = w["rep"]
    for n, warps in ((256, 8), (512, 4), (1024, 2), (4096, 1)):
        before = rep.launch_count
        dev = device_projected(rep, w["hints"][:n], w["ranges"][:n], w["Ts"][:n])
        shape = rep.last_launch_shape()
        assert (shape["warps_per_scan"], shape["scans_per_block"]) == (warps, 1), (n, shape)
        assert rep.launch_count - before == 1
    before = rep.launch_count
    host = rep.match_batch_projected(w["hints"], w["ranges"], transforms=w["Ts"])
    assert rep.launch_count - before == 2
    assert rep.last_launch_shape()["warps_per_scan"] == 1
    for a, b in zip(host, dev):
        assert np.array_equal(a, b)
    before = rep.launch_count
    rep.match_batch_projected(w["hints"][:1000], w["ranges"][:1000])
    assert rep.launch_count - before == 1


def test_submit_wait_interleaved_with_ranges_and_cloud(bench_rep):
    from hector_slam_b200 import capi, synth

    w = bench_rep
    rep = w["rep"]
    n = 2048
    hints, ranges, Ts = w["hints"][:n], w["ranges"][:n], w["Ts"][:n]
    p = dict(synth.SCAN_FORMAT, range_cutoff=30.0)
    u = unit_vectors(p["n_beams"], p["angle_min"], p["angle_increment"])
    clouds = [project(ranges[b], p, u) for b in range(n)]
    c_offs = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int32)
    cloud_all = np.ascontiguousarray(np.concatenate(clouds), F32)
    want_p = rep.match_batch_projected(hints, ranges, transforms=Ts)
    want_q = rep.match_batch_projected(hints[::-1].copy(), ranges[::-1].copy())
    want_r = rep.match_batch_ranges(hints, ranges)
    want_c = rep.match_batch_cloud(hints, cloud_all, c_offs, transforms=Ts)
    assert np.array_equal(want_c[0], want_p[0])

    def outs():
        return capi.PinnedArray((n, 3)), capi.PinnedArray((n, 9)), capi.PinnedArray((n, 2))

    hp, rp, tp = capi.pinned_copy(hints), capi.pinned_copy(ranges), capi.pinned_copy(Ts)
    hq, rq = capi.pinned_copy(hints[::-1].copy()), capi.pinned_copy(ranges[::-1].copy())
    cp = capi.pinned_copy(cloud_all)
    o = [outs() for _ in range(5)]
    t0 = rep.match_batch_projected_submit(hp.array, rp.array, o[0][0].array, o[0][1].array, o[0][2].array, tp.array)
    t1 = rep.match_batch_projected_submit(hq.array, rq.array, o[1][0].array, o[1][1].array, o[1][2].array)
    assert {t0, t1} == {0, 1}
    rep.match_batch_wait(t0)
    t2 = rep.match_batch_ranges_submit(hp.array, rp.array, o[2][0].array, o[2][1].array)
    rep.match_batch_wait(t1)
    t3 = rep.match_batch_cloud_submit(hp.array, cp.array, c_offs, o[3][0].array, o[3][1].array, o[3][2].array, tp.array)
    rep.match_batch_wait(t2)
    t4 = rep.match_batch_projected_submit(hp.array, rp.array, o[4][0].array, None, None, tp.array)
    rep.match_batch_wait(t3)
    rep.match_batch_wait(t4)

    def same(got, want, with_origo=True):
        assert np.array_equal(got[0].array, want[0])
        assert np.array_equal(got[1].array.reshape(n, 3, 3), want[1])
        if with_origo:
            assert np.array_equal(got[2].array, want[2])

    same(o[0], want_p)
    same(o[1], want_q)
    same(o[2], want_r, with_origo=False)
    same(o[3], want_c)
    assert np.array_equal(o[4][0].array, want_p[0])
    for a in [hp, rp, tp, hq, rq, cp] + [x for t in o for x in t]:
        a.free()


# ---- validation ---------------------------------------------------------------------------------------------------
def test_rejections_queue_nothing(hsb_lib):
    import ctypes as C

    from hector_slam_b200 import capi

    p, ranges, hints, T0, Ts = scans(0)
    lib = hsb_lib
    out = np.zeros((B, 3), F32)

    def rejected(rep, status, texts, r=ranges, h=hints, device=False):
        before = rep.launch_count
        with pytest.raises(capi.HsbError) as e:
            if device:
                import torch

                d = torch.zeros(max(r.size, 1), dtype=torch.float32, device="cuda")
                rep.match_batch_projected_device(h.shape[0], d.data_ptr(), d.data_ptr(), None, d.data_ptr(), None, None)
            else:
                rep.match_batch_projected(h, r)
        assert e.value.status == status and all(t in str(e.value) for t in texts), str(e.value)
        assert rep.launch_count == before
        return str(e.value)

    no_proj = golden_rep(capi.GATHER_LDG)
    rejected(no_proj, -1, ["hsb_match_batch_projected", "hsb_set_laser_projection"])
    rejected(no_proj, -1, ["hsb_match_batch_projected_device", "hsb_set_laser_projection"], device=True)
    no_cloud = golden_rep(capi.GATHER_LDG, p, with_cloud=False)
    rejected(no_cloud, -1, ["hsb_match_batch_projected", "hsb_set_cloud_format"])
    big = dict(p, n_beams=LIMIT + 1, angle_increment=float(F32(1e-4)))
    long_rep = golden_rep(capi.GATHER_LDG, big)
    rejected(long_rep, -5, ["scan too long for the fused conversion (%d points)" % (LIMIT + 1)],
             r=np.full((2, LIMIT + 1), 3.0, F32), h=hints[:2])
    long_rep.close()

    reps = {m: golden_rep(m, p, T0=T0) for m in (capi.GATHER_LDG, capi.GATHER_TEX)}
    twins = {m: golden_rep(m, p, T0=T0) for m in (capi.GATHER_LDG, capi.GATHER_TEX)}
    bad = [(capi.GATHER_LDG, dict(warps_per_scan=16)), (capi.GATHER_LDG, dict(scans_per_block=7)),
           (capi.GATHER_TEX, dict(unroll=8)), (capi.GATHER_TEX, dict(packed=1))]
    for m, tune in bad:
        rep = reps[m]
        rep.set_tuning(**tune)
        rejected(rep, -5, ["hsb_match_batch_projected", "tuning"])
        rejected(rep, -5, ["hsb_match_batch_projected_device", "tuning"], device=True)
        rep.set_tuning(warps_per_scan=0, scans_per_block=0, unroll=0, packed=0)
        got = rep.match_batch_projected(hints, ranges, transforms=Ts)
        want = twins[m].match_batch_projected(hints, ranges, transforms=Ts)
        assert all(np.array_equal(a, b) for a, b in zip(got, want)), tune
    # LDG ignores "packed": the unpacked kernel runs
    reps[capi.GATHER_LDG].set_tuning(packed=1)
    got = reps[capi.GATHER_LDG].match_batch_projected(hints, ranges, transforms=Ts)
    assert np.array_equal(got[0], twins[capi.GATHER_LDG].match_batch_projected(hints, ranges, transforms=Ts)[0])

    rep = reps[capi.GATHER_LDG]
    before = rep.launch_count
    h, r = hints.ctypes.data, ranges.ctypes.data
    assert lib.hsb_match_batch_projected(rep.h, B, h, None, None, out.ctypes.data, None, None) == -1
    assert lib.hsb_match_batch_projected(rep.h, B, None, r, None, out.ctypes.data, None, None) == -1
    assert lib.hsb_match_batch_projected(rep.h, B, h, r, None, None, None, None) == -1
    assert lib.hsb_match_batch_projected(rep.h, -1, h, r, None, out.ctypes.data, None, None) == -1
    assert lib.hsb_match_batch_projected_device(rep.h, -1, h, r, None, out.ctypes.data, None, None, None) == -1
    assert lib.hsb_match_batch_projected(None, B, h, r, None, out.ctypes.data, None, None) == -1
    t = C.c_int(5)
    assert lib.hsb_match_batch_projected_submit(rep.h, 0, h, r, None, out.ctypes.data, None, None, C.byref(t)) == 0
    assert t.value == -1
    assert lib.hsb_match_batch_projected(rep.h, 0, h, r, None, out.ctypes.data, None, None) == 0
    assert lib.hsb_match_batch_projected_device(rep.h, 0, h, r, None, out.ctypes.data, None, None, None) == 0
    assert rep.launch_count == before
    got = rep.match_batch_projected(hints, ranges, transforms=Ts)
    want = twins[capi.GATHER_LDG].match_batch_projected(hints, ranges, transforms=Ts)
    assert all(np.array_equal(a, b) for a, b in zip(got, want))
    for x in [no_proj, no_cloud] + list(reps.values()) + list(twins.values()):
        x.close()
