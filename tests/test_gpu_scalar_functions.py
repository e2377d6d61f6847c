"""GPU: the kernels' scalar device functions on their own, through the probe library (tests/device/hsb_probe.cu, built by
hector_slam_b200/build.py build_probe with the product library's nvcc flags), against host references bit for bit.

  * Every fp32 argument (2^32 bit patterns, in chunks): sinf_glibc, cosf_glibc and both outputs of sincosf_glibc against
    the running libm and sincosf_glibc against the separate calls; expf_glibc against libm expf; normalize_angle against
    the C port (oracle/hs_oracle.c hso_normalize_angle), itself tied to the compiled reference by test_pose32_oracle.py,
    and on a 2^24-argument sample against the compiled reference (oracle/_ref/libhsref_util.so) where it is built.
    Power: the number of arguments whose libm sinf / cosf or expf is not the correctly rounded value (float64 libm
    rounded to fp32) is reported and must be nonzero — a correctly rounded device implementation would fail here.
  * best_pack / best_unpack on every fp32 score with a finite pose, for indices 0, 1 and 2^32 - 1: the round trip gives
    the score's bits (NaN gives -1) and the index back, no packed value is 0 (the empty-accumulator sentinel), and the
    packed order is strictly monotone in the score.  Then poses: every finite coordinate keeps the score — FLT_MAX, the
    largest negative value and all of (3.4e38, FLT_MAX] — and +-inf or NaN in any coordinate scores -1.
  * solve3 against the port's inverse3_times (hso_inverse3_times) on 2^24 symmetric H / dTr cases: well-conditioned,
    rank-deficient and nearly singular, entries over 1e-30 .. 1e30 with subnormals, +-0, +-inf and NaN, det underflowing
    to 0 and overflowing to inf.  Power: fused cofactors (fmaf(a, b, -c*d)) change the port's output on some of them.
  * pose_difference_larger_than against the port's (and the reference's, where built) on 2^24 cases: distances at the
    threshold +- a few ulp (3-4-5 triangles scaled by 2^k), angle differences at +-pi and +-2pi +- ulp and past one
    wrap, zero / negative / inf / NaN thresholds, FLT_MAX^3 as the stored pose.

Every test reports its counts and wall time through conftest.report.
"""
import ctypes as C
import os
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import libm_sweep
from conftest import report

pytestmark = pytest.mark.gpu

F32 = np.float32
U32 = np.uint32
FMAX = np.finfo(F32).max
CHUNK = 1 << 26
SAMPLE = 1 << 24
_vp, _ll, _u32 = C.c_void_p, C.c_longlong, C.c_uint32


@pytest.fixture(scope="module")
def probe(hsb_lib):
    from hector_slam_b200 import build

    L = C.CDLL(build.PROBE_LIB)
    L.hsb_probe_trig_sweep.argtypes = [_u32, _ll, _vp, _vp, _vp, _vp]
    L.hsb_probe_exp_sweep.argtypes = [_u32, _ll, _vp]
    L.hsb_probe_normalize_angle_sweep.argtypes = [_u32, _ll, _vp]
    L.hsb_probe_normalize_angle.argtypes = [_vp, _ll, _vp]
    L.hsb_probe_solve3.argtypes = [_vp, _vp, _ll, _vp]
    L.hsb_probe_pose_difference_larger_than.argtypes = [_vp, _vp, _vp, _vp, _ll, _vp]
    L.hsb_probe_best_pack.argtypes = [_vp, _vp, _vp, _ll, _vp]
    L.hsb_probe_best_pack_sweep.argtypes = [_u32, _ll, _vp, _u32, _vp, _vp, _vp]
    return L


@pytest.fixture(scope="module")
def helper(tmp_path_factory):
    import shutil

    if not shutil.which("g++"):
        pytest.skip("no g++")
    return libm_sweep.build(tmp_path_factory.mktemp("libm_sweep"))


@pytest.fixture(scope="module")
def libm(helper):
    why = libm_sweep.skip_reason()
    if why:
        pytest.skip(why)
    return helper


@pytest.fixture(scope="module")
def port():
    from oracle import pyoracle

    if not pyoracle.available("port"):
        import subprocess

        from conftest import ROOT
        subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "port"], check=True, capture_output=True)
    L = C.CDLL(pyoracle.PORT_LIB)
    L.hso_normalize_angle.argtypes = [_vp, C.c_int, _vp]
    L.hso_inverse3_times.argtypes = [_vp, _vp, C.c_int, _vp]
    L.hso_pose_difference_larger_than.argtypes = [_vp, _vp, _vp, _vp, C.c_int, _vp]
    return L


def ref_util():
    from oracle import pyoracle

    if not pyoracle.util_available("reference"):
        return None
    L = C.CDLL(pyoracle.REF_UTIL_LIB)
    L.hsref_normalize_angle.argtypes = [_vp, C.c_int, _vp]
    L.hsref_pose_difference_larger_than.argtypes = [_vp, _vp, _vp, _vp, C.c_int, _vp]
    return L


def pinned(n, dtype):
    """a page-locked host array (the probe's copies run at full bus speed into it)"""
    import torch

    t = torch.empty(n * np.dtype(dtype).itemsize, dtype=torch.uint8, pin_memory=True)
    return t.numpy().view(dtype)


def ptr(a):
    return a.ctypes.data


def threaded(fn, n, *spec):
    """a single-threaded port function fn(pointers..., count, pointers...) over n items, split over every CPU: ctypes
    releases the GIL while each piece runs.  spec: fn's arguments in order, (array, items per row) for an array and "n"
    for the count."""
    T = libm_sweep.threads()
    bounds = [n * w // T for w in range(T + 1)]

    def piece(w):
        b, cnt = bounds[w], bounds[w + 1] - bounds[w]
        if cnt > 0:
            fn(*[cnt if a == "n" else ptr(a[0]) + b * a[1] * a[0].dtype.itemsize for a in spec])

    with ThreadPoolExecutor(T) as ex:
        list(ex.map(piece, range(T)))


class Tally:
    """mismatch counts of one sweep and the lowest mismatching arguments of each"""

    def __init__(self, names):
        self.names = names
        self.counts = np.zeros(len(names), np.int64)
        self.first = [[] for _ in names]
        self.n = 0

    def add(self, counts, bad):
        for k in range(len(self.names)):
            room = min(int(counts[k]), libm_sweep.MAX_BAD) - len(self.first[k])
            self.first[k] += bad[k][:max(0, room)].tolist()
        self.counts += counts

    def message(self):
        bad = np.array([(b + [0] * libm_sweep.MAX_BAD)[:libm_sweep.MAX_BAD] for b in self.first], np.uint32)
        return libm_sweep.report_bad(self.names, self.counts, bad)

    def summary(self):
        return ", ".join(f"{n} {int(c)}" for n, c in zip(self.names, self.counts))


# ---- 1. every fp32 argument ------------------------------------------------------------------------------------------
def test_trig_exp_every_argument(probe, libm):
    t0 = time.perf_counter()
    names = ["sinf", "cosf", "sincosf sin", "sincosf cos", "sincosf sin vs sinf", "sincosf cos vs cosf", "expf"]
    tally = Tally(names)
    power = np.zeros(2, np.int64)
    stride, sampled = 64, 0
    s, c, ss, sc, e = (pinned(CHUNK, F32) for _ in range(5))
    for first, n in libm_sweep.chunks(CHUNK):
        assert probe.hsb_probe_trig_sweep(first, n, ptr(s), ptr(c), ptr(ss), ptr(sc)) == 0
        assert probe.hsb_probe_exp_sweep(first, n, ptr(e)) == 0
        ct, bt = libm.check_trig(first, s[:n], c[:n], ss[:n], sc[:n])
        ce, be = libm.check_exp(first, e[:n])
        tally.add(np.concatenate([ct, ce]), np.concatenate([bt, be]))
        p, _ = libm.power(first, n, stride)
        power += p
        sampled += -(-n // stride)
        tally.n += n
    dt = time.perf_counter() - t0
    report(f"scalar functions: sinf/cosf/sincosf/expf on {tally.n} arguments each, mismatches: {tally.summary()}; "
           f"power: libm sinf/cosf not correctly rounded on {int(power[0])}, expf on {int(power[1])} of {sampled} sampled "
           f"(every {stride}th pattern); {dt:.1f} s")
    assert tally.n == libm_sweep.ALL
    assert not tally.counts.any(), tally.message()
    assert power[0] > 0 and power[1] > 0, power


def test_normalize_angle_every_argument(probe, helper, port):
    t0 = time.perf_counter()
    tally = Tally(["normalize_angle"])
    na = pinned(CHUNK, F32)
    want = np.empty(CHUNK, F32)
    for first, n in libm_sweep.chunks(CHUNK):
        assert probe.hsb_probe_normalize_angle_sweep(first, n, ptr(na)) == 0
        args = np.arange(first, first + n, dtype=np.uint64).astype(U32).view(F32)
        threaded(port.hso_normalize_angle, n, (args, 1), "n", (want, 1))
        tally.add(*helper.compare(first, na[:n], want[:n]))
        tally.n += n
    msg = f"scalar functions: normalize_angle on {tally.n} arguments vs the port, mismatches: {tally.summary()}"
    # the compiled reference on a sample of bit patterns
    ref = ref_util()
    if ref is not None:
        rng = np.random.default_rng(31)
        args = rng.integers(0, 1 << 32, SAMPLE, dtype=np.uint64).astype(U32).view(F32)
        got, want = np.empty(SAMPLE, F32), np.empty(SAMPLE, F32)
        assert probe.hsb_probe_normalize_angle(ptr(args), SAMPLE, ptr(got)) == 0
        threaded(ref.hsref_normalize_angle, SAMPLE, (args, 1), "n", (want, 1))
        bad = np.flatnonzero((got.view(U32) != want.view(U32)) & ~(np.isnan(got) & np.isnan(want)))
        msg += f"; {SAMPLE} sampled vs the reference: {bad.size} mismatches"
        assert bad.size == 0, [(hex(int(args.view(U32)[i])), got[i], want[i]) for i in bad[:8]]
    report(msg + f"; {time.perf_counter() - t0:.1f} s")
    assert tally.n == libm_sweep.ALL
    assert not tally.counts.any(), tally.message()


# ---- 2. best-hypothesis ranking ----------------------------------------------------------------------------------------
def test_best_pack_every_score(probe, helper):
    t0 = time.perf_counter()
    pose = F32([0.5, -2.0, 0.25])
    packed, score, idx = pinned(CHUNK, np.uint64), pinned(CHUNK, F32), pinned(CHUNK, U32)
    zero = {}
    for index in (0, 1, 0xffffffff):
        tally = Tally(["round trip score", "round trip index", "packed 0", "order"])
        prev = None
        for first, n in libm_sweep.chunks(CHUNK):
            assert probe.hsb_probe_best_pack_sweep(first, n, ptr(pose), index, ptr(packed), ptr(score), ptr(idx)) == 0
            tally.add(*helper.check_pack(first, packed[:n], score[:n], idx[:n], index, prev))
            prev = int(packed[n - 1])
            if first in (0, 0x80000000):
                zero[(index, first)] = int(packed[0])
            tally.n += n
        assert tally.n == libm_sweep.ALL
        assert not tally.counts.any(), (index, tally.message())
        # -0 ranks strictly below +0 (recorded: the order is by bits there, not by value)
        assert zero[(index, 0x80000000)] < zero[(index, 0)], (index, zero)
    report(f"scalar functions: best_pack/best_unpack on every score for indices 0, 1, 2^32-1: round trip, no 0, strictly "
           f"monotone; -0 packs below +0; {time.perf_counter() - t0:.1f} s")


def pack(probe, lh, poses, index):
    lh, poses = np.ascontiguousarray(lh, F32), np.ascontiguousarray(poses, F32).reshape(-1, 3)
    index = np.ascontiguousarray(np.broadcast_to(np.asarray(index, U32), lh.shape))
    out = np.zeros(lh.size, np.uint64)
    assert probe.hsb_probe_best_pack(ptr(lh), ptr(poses), ptr(index), lh.size, ptr(out)) == 0
    return out


def packed_model(score, index):
    """the packing best_pack documents, restated on the host: the score's bits mapped to an unsigned order (negative:
    all bits flipped, else the sign bit set) in the high word, 2^32 - 1 - index in the low word.  Independent of the
    device; test_best_pack_every_score pins the device's round trip and order on every score."""
    u = np.asarray(score, F32).reshape(-1).view(U32).astype(np.uint64)
    u = np.where(u & 0x80000000, ~u & 0xffffffff, u | 0x80000000).astype(np.uint64)
    return (u << np.uint64(32)) | np.uint64(0xffffffff - int(index))


def test_best_pack_poses(probe):
    """the pose part of best_pack: a pose with every coordinate finite keeps its score, one with +-inf or NaN anywhere
    scores -1 (as does a NaN score), against the host model of the packing"""
    top = np.arange(np.float32(3.4e38).view(U32), FMAX.view(U32) + 1, dtype=np.uint64).astype(U32).view(F32)
    assert top[0] == F32(3.4e38) and top[-1] == FMAX and top.size == 13922
    finite = np.concatenate([top, -top, F32([0.0, -0.0, 1e-45, -1e-45, 1.0, -7.5, 1e38, -1e38])])
    nonfinite = F32([np.inf, -np.inf, np.nan, -np.nan])
    scores = F32([0.0, 0.75, 1.0, -0.0, 1e-30, np.nan])
    base = F32([1.5, -2.5, 0.3])
    for vals, keeps in ((finite, True), (nonfinite, False)):
        for coord in range(3):
            poses = np.tile(base, (vals.size, 1))
            poses[:, coord] = vals
            for s in scores:
                lh = np.full(vals.size, s, F32)
                got = pack(probe, lh, poses, 7)
                ranked = s if keeps and not np.isnan(s) else F32(-1.0)
                want = packed_model(ranked, 7)[0]
                bad = np.flatnonzero(got != want)
                assert bad.size == 0, (coord, float(s), keeps, [float(vals[i]) for i in bad[:8]])


# ---- 3. solve3 ---------------------------------------------------------------------------------------------------------
def wide(rng, shape):
    """sign * 10^U(-30, 30) with subnormals, +-0, +-inf and NaN sprinkled in"""
    v = np.sign(rng.uniform(-1, 1, shape)) * 10.0 ** rng.uniform(-30, 30, shape)
    r = rng.uniform(0, 1, shape)
    v = np.where(r < 0.02, rng.uniform(-1, 1, shape) * 1e-39, v)
    v = np.where((r >= 0.02) & (r < 0.03), np.where(rng.uniform(0, 1, shape) < 0.5, 0.0, -0.0), v)
    v = np.where((r >= 0.03) & (r < 0.034), np.where(rng.uniform(0, 1, shape) < 0.5, np.inf, -np.inf), v)
    v = np.where((r >= 0.034) & (r < 0.038), np.nan, v)
    with np.errstate(over="ignore"):
        return v.astype(F32)


def sym6(Hf):
    """(n, 3, 3) float64 -> (n, 6) float32 (h00, h11, h22, h01, h02, h12)"""
    with np.errstate(over="ignore", under="ignore"):
        return np.stack([Hf[:, 0, 0], Hf[:, 1, 1], Hf[:, 2, 2], Hf[:, 0, 1], Hf[:, 0, 2], Hf[:, 1, 2]], 1).astype(F32)


def solve3_family(k, rng, n):
    """family k of n cases -> (h6 (n, 6), d3 (n, 3)) float32"""
    A = rng.normal(size=(n, 3, 3))
    eye = np.eye(3)[None]
    d = (rng.normal(size=(n, 3)) * 10.0 ** rng.uniform(-5, 5, (n, 1))).astype(F32)
    if k == 0:     # well-conditioned, over nine decades of scale
        H = (A @ A.transpose(0, 2, 1) + 0.5 * eye) * 10.0 ** rng.uniform(-3, 6, (n, 1, 1))
        return sym6(H), d
    if k == 1:     # rank 1 and 2, nearly singular, and a map constant along one axis (a zero row and column)
        u, v, w = rng.normal(size=(n, 3)), rng.normal(size=(n, 3)), rng.normal(size=(n, 3))
        eps = rng.choice([0.0, 1e-7, 1e-5, 1e-3], n)[:, None, None]
        rank = rng.integers(1, 3, n)[:, None, None]
        H = u[:, :, None] * u[:, None, :] + (rank == 2) * v[:, :, None] * v[:, None, :] + eps * w[:, :, None] * w[:, None, :]
        H *= 10.0 ** rng.uniform(-2, 5, (n, 1, 1))
        h = sym6(H)
        axis = rng.integers(0, 4, n)          # 0: constant along x, 1: along y, else as drawn
        h[np.ix_(axis == 0, [0, 3, 4])] = 0.0
        h[np.ix_(axis == 1, [1, 3, 5])] = 0.0
        return h, d
    if k == 2:     # every entry over 1e-30 .. 1e30 with subnormals, +-0, +-inf, NaN
        return wide(rng, (n, 6)), wide(rng, (n, 3))
    # det underflowing to 0 and overflowing to inf: well-conditioned H scaled to 1e-20 .. 1e-13 and 1e13 .. 1e20
    H = A @ A.transpose(0, 2, 1) + 0.5 * eye
    e = np.where(rng.uniform(0, 1, n) < 0.5, rng.uniform(-20, -13, n), rng.uniform(13, 20, n))
    return sym6(H * 10.0 ** e[:, None, None]), d


def full9(h6):
    h00, h11, h22, h01, h02, h12 = (h6[:, i] for i in range(6))
    return np.ascontiguousarray(np.stack([h00, h01, h02, h01, h11, h12, h02, h12, h22], 1), F32)


def same_rows(a, b):
    eq = (a.view(U32) == b.view(U32)) | (np.isnan(a) & np.isnan(b))
    return eq.all(axis=1)


def test_solve3_sweep(probe, helper, port):
    t0 = time.perf_counter()
    rng = np.random.default_rng(41)
    n = SAMPLE // 4
    total, fused, special = 0, 0, {"det 0": 0, "det inf": 0, "nan out": 0}
    for k in range(4):
        h6, d3 = solve3_family(k, rng, n)
        got = np.empty((n, 3), F32)
        assert probe.hsb_probe_solve3(ptr(h6), ptr(d3), n, ptr(got)) == 0
        m9 = full9(h6)
        want = np.empty((n, 3), F32)
        threaded(port.hso_inverse3_times, n, (m9, 9), (d3, 3), "n", (want, 3))
        ok = same_rows(got, want)
        bad = np.flatnonzero(~ok)
        assert bad.size == 0, (k, bad.size, [(h6[i].tolist(), d3[i].tolist(), got[i].tolist(), want[i].tolist())
                                             for i in bad[:4]])
        fused += helper.inverse3_fma(m9, d3, want)
        with np.errstate(all="ignore"):
            m = m9.reshape(n, 3, 3).astype(np.float64)
            det = np.linalg.det(np.where(np.isfinite(m), m, 0.0))
        special["det 0"] += int(((np.abs(det) < 1e-45) & np.isfinite(m9).all(1)).sum())
        special["det inf"] += int((np.abs(det) > 3.5e38).sum())
        special["nan out"] += int(np.isnan(want).any(1).sum())
        total += n
    report(f"scalar functions: solve3 on {total} cases vs the port's inverse3_times, 0 mismatches ({special}); fused "
           f"cofactors change {fused}; {time.perf_counter() - t0:.1f} s")
    assert total >= SAMPLE
    assert all(v > 0 for v in special.values()), special
    assert fused > 0


# ---- 4. pose_difference_larger_than -------------------------------------------------------------------------------------
def ulps(x, j):
    """x moved by j ulp (x > 0 finite, |j| small)"""
    return (np.asarray(x, F32).view(np.int32) + np.asarray(j, np.int32)).view(F32)


def gate_family(k, rng, n):
    """family k of n cases -> (p1 (n, 3), p2 (n, 3), dist (n,), ang (n,)) float32"""
    p2 = np.stack([rng.uniform(-100, 100, n), rng.uniform(-100, 100, n), rng.uniform(-20, 20, n)], 1).astype(F32)
    p2[rng.uniform(0, 1, n) < 0.5, :2] = 0.0
    ang = np.abs(rng.normal(0, 1, n)).astype(F32)
    dist = np.abs(rng.normal(0, 0.5, n)).astype(F32)
    p1 = p2.copy()
    if k == 0:     # a 3-4-5 triangle scaled by 2^k: the norm at the threshold +- a few ulp
        s = 2.0 ** rng.integers(-40, 40, n)
        sx, sy = rng.choice([-1.0, 1.0], n), rng.choice([-1.0, 1.0], n)
        swap = rng.uniform(0, 1, n) < 0.5
        dx, dy = np.where(swap, 4.0, 3.0) * s * sx, np.where(swap, 3.0, 4.0) * s * sy
        p1[:, 0], p1[:, 1] = (p2[:, 0] + dx).astype(F32), (p2[:, 1] + dy).astype(F32)
        dist = ulps((5.0 * s).astype(F32), rng.integers(-3, 4, n))
        p1[:, 2] = p2[:, 2]
    elif k == 1:   # angle differences at +-pi, +-2pi, +-3pi, +-4pi +- a few ulp; the threshold at the result +- ulp
        t = rng.choice([np.pi, 2 * np.pi, 3 * np.pi, 4 * np.pi, 1.5 * np.pi], n) * rng.choice([-1.0, 1.0], n)
        tt = ulps(np.abs(t).astype(F32), rng.integers(-3, 4, n)) * np.sign(t).astype(F32)
        p2[:, 2] = np.where(rng.uniform(0, 1, n) < 0.5, F32(0.0), p2[:, 2])
        p1[:, 2] = (p2[:, 2] + tt).astype(F32)
        a = (p1[:, 2].astype(np.float64) - p2[:, 2].astype(np.float64))
        a = np.where(a > np.pi, a - 2 * np.pi, np.where(a < -np.pi, a + 2 * np.pi, a))
        mag = np.maximum(np.abs(a), 1e-30).astype(F32)
        ang = ulps(mag, rng.integers(-2, 3, n))
        dist = F32(0.4) * np.ones(n, F32)
    elif k == 2:   # zero, negative, inf and NaN thresholds on nearby poses
        p1 = (p2 + rng.normal(0, 0.3, (n, 3)) * rng.choice([0.0, 1.0], (n, 1))).astype(F32)
        special = F32([0.0, -0.0, -1.0, -1e-30, np.inf, -np.inf, np.nan, 1e-45, 0.4])
        dist = rng.choice(special, n)
        ang = rng.choice(special, n)
    else:          # FLT_MAX^3 as the stored pose (hsb_reset), against ordinary, huge and non-finite poses
        p2[:] = FMAX
        pick = rng.uniform(0, 1, (n, 3))
        p1 = np.where(pick < 0.6, p1, np.where(pick < 0.8, FMAX, np.where(pick < 0.9, -FMAX, rng.choice(
            F32([np.inf, -np.inf, np.nan, 3.4e38, 0.0]), (n, 3))))).astype(F32)
    return np.ascontiguousarray(p1, F32), np.ascontiguousarray(p2, F32), np.ascontiguousarray(dist, F32), \
        np.ascontiguousarray(ang, F32)


def test_pose_difference_sweep(probe, port):
    t0 = time.perf_counter()
    rng = np.random.default_rng(43)
    ref = ref_util()
    n = SAMPLE // 4
    total, trues = 0, []
    for k in range(4):
        p1, p2, dist, ang = gate_family(k, rng, n)
        got = np.empty(n, np.int32)
        assert probe.hsb_probe_pose_difference_larger_than(ptr(p1), ptr(p2), ptr(dist), ptr(ang), n, ptr(got)) == 0
        for lib, fn in ((port, "hso_pose_difference_larger_than"), (ref, "hsref_pose_difference_larger_than")):
            if lib is None:
                continue
            want = np.empty(n, np.int32)
            threaded(getattr(lib, fn), n, (p1, 3), (p2, 3), (dist, 1), (ang, 1), "n", (want, 1))
            bad = np.flatnonzero((got != 0) != (want != 0))
            assert bad.size == 0, (fn, k, bad.size, [(p1[i].tolist(), p2[i].tolist(), float(dist[i]), float(ang[i]),
                                                      int(got[i])) for i in bad[:6]])
        trues.append(float((got != 0).mean()))
        total += n
    report(f"scalar functions: pose_difference_larger_than on {total} cases vs the port"
           f"{' and the reference' if ref is not None else ''}, 0 mismatches (share true per family "
           f"{[round(t, 3) for t in trues]}); {time.perf_counter() - t0:.1f} s")
    assert total >= SAMPLE
    assert all(0.02 < t < 0.98 for t in trues[:3]), trues   # both outcomes in every boundary family
