"""Every stream-ordering promise of include/hector_slam_b200.h with the earlier work held back on the device.

The library runs its work on private non-blocking streams (the handle's stream, its two copy streams, each group's
stream) and on the caller's streams of the "_device" entry points, and orders them with events.  A test that issues a
consumer a few microseconds after a producer that runs a few microseconds cannot tell a missing event from the host's
own call overhead.  Here the producer is slow on purpose:

- held: a bounded torch.cuda._sleep (about 100 ms, calibrated once) on a caller stream, with the map-changing
  "_device" producer (an unpack, a group unpack, a plane write and refresh_level) queued behind it.  Every consumer is
  issued while the hold still runs: an event recorded right after the hold must still be pending when the last
  asynchronous consumer has been issued and before a blocking one is called (the window check), otherwise the case
  tested nothing and fails;
- slow: a nowait SLAM step (single, from endpoints, ranges or a cloud, or group) whose map write is a long scan on a 4096^2 map; its
  device time, measured once on the identical synchronous step (tuning "time_update"), must be far longer than
  the host time taken to issue the consumers.

Each case runs twice: held / slow without any synchronisation, and on twin handles with torch.cuda.synchronize() and
hsb_on_map_updated on every handle between any two calls.  Every output and the end state (log-odds and P of every
level, the texture twin through the one-texel likelihood probe, both dirty rectangles, the gate pose and the last-match
container) must agree bit for bit.  A missing dependency lets the consumer read the map before the producer wrote it.
"""
import time

import numpy as np
import pytest

from twin_probe import probe_points

pytestmark = pytest.mark.gpu

MODES = pytest.mark.parametrize("mode", [2, 1], ids=["tex", "ldg"])   # capi.GATHER_TEX, capi.GATHER_LDG
RES, SIZE, LEVELS, M = 0.05, 512, 3, 3
SCALE = 1.0 / RES
B = 6                      # scans / poses of a batch consumer
CAP = 4 << 20              # tile buffer bytes
HOLD_MS = 100.0            # calibrated hold; every hold is bounded by HOLD_MAX_MS
HOLD_MAX_MS = 400.0
BIG = 4096                 # map size of the slow (nowait) producers
LONG_R = 1900.0            # long rays: level-0 cells from the robot (95 m), inside the 4096^2 map
WRITE_MIN_MS = 40.0        # the long write's device time aimed at ...
MAX_BEAMS = 1 << 22        # ... with at most this many endpoints (a scan format's ranges: at most 2^20)
MARGINS = []               # (case, ms left of the hold or of the write when the last consumer was issued)


# ---- fixtures: hold calibration, owner maps, long-write calibration ----------------------------------------------

@pytest.fixture(scope="module")
def hold_cycles(hsb_lib):
    """Sleep cycles of a HOLD_MS hold, measured with CUDA events on a fresh stream."""
    import torch

    s = torch.cuda.Stream()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    probe = 20_000_000
    try:
        with torch.cuda.stream(s):
            torch.cuda._sleep(1000)
            a.record(s)
            torch.cuda._sleep(probe)
            b.record(s)
        b.synchronize()
        cycles = int(probe * HOLD_MS / a.elapsed_time(b))
        with torch.cuda.stream(s):
            a.record(s)
            torch.cuda._sleep(cycles)
            b.record(s)
        b.synchronize()
        ms = a.elapsed_time(b)
    finally:
        torch.cuda.synchronize()
    assert 0.5 * HOLD_MS < ms < HOLD_MAX_MS, ms
    print(f"\nhold: {cycles} cycles = {ms:.1f} ms")
    yield cycles
    if MARGINS:
        worst = min(MARGINS, key=lambda x: x[1])
        print(f"\nsmallest window margin: {worst[1]:.1f} ms ({worst[0]}), {len(MARGINS)} windows")


def session_data(seed, steps):
    from hector_slam_b200 import synth

    rng = np.random.default_rng(seed)
    world = synth.World(1, seed=1000 + seed)
    x, y, a = rng.uniform(-2, 2), rng.uniform(-1.5, 1.5), rng.uniform(-3, 3)
    truth, ranges = [], []
    for _ in range(steps):
        p = np.array([x, y, a], np.float32)
        truth.append(p)
        ranges.append((world.cast(p) + rng.normal(0.0, 0.01, synth.N_BEAMS)).astype(np.float32))
        a += rng.uniform(-0.08, 0.08)
        step = rng.uniform(0.05, 0.15)
        x = float(np.clip(x + step * np.cos(a), -6.0, 6.0))
        y = float(np.clip(y + step * np.sin(a), -4.0, 4.0))
    truth = np.asarray(truth, np.float32)
    hints = (truth + rng.uniform(-1, 1, truth.shape).astype(np.float32) * np.float32([0.04, 0.04, 0.02])).astype(np.float32)
    scans = [synth.ranges_to_points(r, SCALE) for r in ranges]
    return dict(truth=truth, hints=hints, ranges=np.asarray(ranges, np.float32), scans=scans)


def make_rep(m, mode, size=SIZE):
    from hector_slam_b200 import capi, synth

    rep = capi.MapRepB200(RES, size, levels=LEVELS, update_factor_free=0.4 + 0.02 * m,
                          update_factor_occupied=0.7 + 0.05 * m, gather_mode=mode)
    rep.set_scan_format(**synth.SCAN_FORMAT)
    rep.setMapUpdateMinDistDiff(0.0)
    rep.setMapUpdateMinAngleDiff(0.0)
    return rep


@pytest.fixture(scope="module")
def world(hsb_lib):
    """Owner maps of M sessions (sync steps) and the buffers packed from them: one handle's tiles, one level-0
    rectangle, the same two of a second owner, the group's tiles (every member and members 0, 2); the consumers' inputs on
    host and device."""
    import torch

    from hector_slam_b200 import capi

    data = [session_data(m, 14) for m in range(M + 1)]
    owners = [make_rep(m, 1) for m in range(M)]
    for m in range(M):
        for k in range(8):
            owners[m].slam_update(data[m]["hints"][k], data[m]["scans"][k])
    og = capi.SlamGroup(owners)
    dev = torch.device("cuda", 0)
    W = dict(data=data)
    s = torch.cuda.Stream()
    W["sbuf"] = torch.zeros(CAP // 4, dtype=torch.float32, device=dev)
    W["gbuf"] = torch.zeros(CAP // 4, dtype=torch.float32, device=dev)
    W["gsub"] = torch.zeros(CAP // 4, dtype=torch.float32, device=dev)
    W["rect"] = owners[0].get_dirty_rect(0)
    x0, y0, x1, y1 = W["rect"]
    W["rbuf"] = torch.zeros((y1 - y0 + 1) * (x1 - x0 + 1), dtype=torch.float32, device=dev)
    torch.cuda.synchronize()
    owners[0].pack_dirty_device(W["sbuf"].data_ptr(), CAP, False, s.cuda_stream)
    owners[0].pack_rect_device(0, W["rect"], W["rbuf"].data_ptr(), s.cuda_stream)
    W["sbuf2"] = torch.zeros(CAP // 4, dtype=torch.float32, device=dev)
    W["rbuf2"] = torch.zeros_like(W["rbuf"])
    torch.cuda.synchronize()
    owners[1].pack_dirty_device(W["sbuf2"].data_ptr(), CAP, False, s.cuda_stream)
    owners[1].pack_rect_device(0, W["rect"], W["rbuf2"].data_ptr(), s.cuda_stream)
    og.pack_dirty_device(W["gbuf"].data_ptr(), CAP, False, s.cuda_stream)
    og.pack_dirty_device(W["gsub"].data_ptr(), CAP, False, s.cuda_stream, members=[0, 2])
    torch.cuda.synchronize()
    W["owner_planes"] = [owners[0].download_level(l) for l in range(LEVELS)]
    # consumer inputs: member m's scans 8.. (B of them), hints near its truth
    for m in range(M + 1):
        d = data[m]
        sc = d["scans"][8:8 + B]
        d["bh"] = np.ascontiguousarray(d["hints"][8:8 + B])
        d["bp"] = np.ascontiguousarray(np.concatenate(sc))
        d["bo"] = np.zeros(B + 1, np.int32)
        d["bo"][1:] = np.cumsum([x.shape[0] for x in sc])
        d["br"] = np.ascontiguousarray(d["ranges"][8:8 + B])
        d["maxn"] = int(np.diff(d["bo"]).max())
    d = data[0]
    W["d_hints"] = torch.from_numpy(d["bh"]).to(dev)
    W["d_pts"] = torch.from_numpy(d["bp"]).to(dev)
    W["d_offs"] = torch.from_numpy(d["bo"]).to(dev)
    W["d_ranges"] = torch.from_numpy(d["br"]).to(dev)
    W["d_truth"] = torch.from_numpy(np.ascontiguousarray(d["truth"][8:8 + B])).to(dev)
    torch.cuda.synchronize()
    og.close()
    for o in owners:
        o.close()
    return W


def long_scan(n):
    """n endpoints on a circle of LONG_R level-0 cells: every ray crosses the map's middle."""
    a = (np.arange(n, dtype=np.float64) * (2 * np.pi / n) - np.pi)
    return np.ascontiguousarray(np.stack([LONG_R * np.cos(a), LONG_R * np.sin(a)], 1).astype(np.float32))


@pytest.fixture(scope="module")
def long_write(hsb_lib):
    """(beams, device ms): the beam count whose map write takes at least WRITE_MIN_MS on the device (a few doublings
    from 2^16, at most 2^20) and that write's time, measured with "time_update" on the identical synchronous
    map_without_matching step.  A group step writes that scan on each of its members."""
    n, ms = 1 << 16, {}
    while True:
        rep = make_rep(0, 1, BIG)
        rep.set_tuning(time_update=1)
        rep.slam_update([0.0, 0.0, 0.0], long_scan(n), map_without_matching=True)
        ms[n] = rep.last_update_device_ms()
        rep.close()
        if ms[n] >= WRITE_MIN_MS or n >= MAX_BEAMS:
            break
        n *= 2
    print(f"\nlong write: {n} beams, {ms[n]:.1f} ms; " + ", ".join(f"{k}: {v:.1f} ms" for k, v in ms.items()))
    return n, ms


@pytest.fixture(autouse=True)
def synchronise_everything(hsb_lib):
    """Every stream a case used is synchronised before it returns, whether or not it passed."""
    import torch

    yield
    torch.cuda.synchronize()


# ---- the two runs of a case ------------------------------------------------------------------------------------

class Env:
    """M replica handles in group G, one more handle sharing member 0 in group H, a producer stream, a second caller
    stream and pre-allocated device outputs (nothing is allocated once a run has started)."""

    def __init__(self, W, mode, size=SIZE):
        import torch

        from hector_slam_b200 import capi

        self.W, self.size = W, size
        self.reps = [make_rep(m, mode, size) for m in range(M)]
        self.extra = make_rep(M, mode, size)
        self.all = self.reps + [self.extra]
        self.G = capi.SlamGroup(self.reps)
        self.H = capi.SlamGroup([self.reps[0], self.extra])
        # the producer's stream, and a caller stream of each asynchronous consumer of its own (e.s2 while it is issued):
        # one consumer's wait must not order the next one
        self.sp = torch.cuda.Stream()
        self.cstream = {name: torch.cuda.Stream() for name, (blocking, _) in CONSUMERS.items() if not blocking}
        self.s2 = self.cstream["match_batch_device"]
        dev = torch.device("cuda", 0)
        R = self.reps[0].record_floats
        z = lambda *sh: torch.zeros(sh, dtype=torch.float32, device=dev)   # noqa: E731
        self.o = dict(mbd=(z(B, 3), z(B, 9)), mbr=(z(B, 3), z(B, 9)), rec=(z(B, 3), z(B, 9), z(B, R)), lh=z(B),
                      best=(z(B), z(4)), prect=z(size * size), pdirty=z(CAP // 4), gpack=z(CAP // 4), hpack=z(CAP // 4),
                      plane=z(size * size))
        # the submit form's host buffers are pinned: a copy from pageable memory would wait for the copy stream
        d = W["data"][0]
        self.pinned = [capi.pinned_copy(a) for a in (d["bh"], d["bp"], d["bo"], np.zeros((B, 3), np.float32),
                                                      np.zeros((B, 9), np.float32))]
        self.rpinned = [capi.pinned_copy(a) for a in (d["bh"], d["br"], np.zeros((B, 3), np.float32),
                                                       np.zeros((B, 9), np.float32))]
        self.ticket = -1
        self.issue_t0 = None
        torch.cuda.synchronize()

    def warm(self):
        """Every asynchronous consumer once on the empty maps, so that no first call allocates while a case runs."""
        import torch

        for name, (blocking, fn) in CONSUMERS.items():
            if not blocking and name not in ("pack_dirty_device", "group_pack_dirty_device", "second_group_pack",
                                             "match_batch_submit", "match_batch_ranges_submit", "second_unpack_dirty",
                                             "second_unpack_rect", "group_reset"):
                self.s2 = self.cstream[name]
                fn(self)
        torch.cuda.synchronize()
        self.reps[0].match_batch_wait(self.reps[0].match_batch_submit(*self._sub_args()))
        self.reps[0].match_batch_wait(self.reps[0].match_batch_ranges_submit(*(p.array for p in self.rpinned)))
        torch.cuda.synchronize()

    def _sub_args(self):
        return tuple(p.array for p in self.pinned)

    def sync(self):
        import torch

        torch.cuda.synchronize()
        for r in self.all:
            r.onMapUpdated()
        torch.cuda.synchronize()

    def close(self):
        for p in self.pinned + self.rpinned:
            p.free()
        self.H.close()
        self.G.close()
        for r in self.all:
            r.close()


def to_np(x):
    import torch

    if isinstance(x, torch.Tensor):
        return x.cpu().numpy()
    if isinstance(x, (tuple, list)):
        return [to_np(v) for v in x]
    if isinstance(x, dict):
        return {k: to_np(v) for k, v in x.items()}
    return np.asarray(x) if x is not None else None


def flat(x):
    """A nested output as one list of arrays."""
    if isinstance(x, dict):
        return [a for k in sorted(x) for a in flat(x[k])]
    if isinstance(x, (list, tuple)):
        return [a for v in x for a in flat(v)]
    return [np.asarray(x)] if x is not None else [np.zeros(0)]


def end_state(e):
    """Planes, texture twin (probe), dirty rectangles, gate pose, last-match container of every handle."""
    out = []
    rng = np.random.default_rng(5)
    for r in e.all:
        for l in range(LEVELS):
            sx, sy, _ = r.level_info(l)
            out += [r.download_level(l), r.download_prob(l)]
            cells = np.stack([rng.integers(0, sx - 1, 3000), rng.integers(0, sy - 1, 3000)], 1)
            pts = probe_points(r, l, cells)
            out.append(r.likelihood_batch(l, np.zeros((cells.shape[0], 3), np.float32), pts,
                                          np.arange(cells.shape[0] + 1, dtype=np.int32)))
            out.append(np.asarray(r.get_mirror_dirty_rect(l) or (-1,) * 4))
        out.append(np.asarray([x or (-1,) * 4 for x in r.get_dirty_rects()]))
        out.append(r.last_map_update_pose())
        try:
            out += list(r.last_match_scan())
        except Exception:   # (no scan matched yet: the same status on both twins)
            out.append(np.asarray([-1]))
    return out


class Window:
    """The hold: a bounded sleep on the producer stream and the event recorded right after it."""

    def __init__(self, e, cycles):
        import torch

        self.ev = torch.cuda.Event()
        with torch.cuda.stream(e.sp):
            torch.cuda._sleep(cycles)
            self.ev.record(e.sp)
        self.t0 = time.perf_counter()

    def check(self, case, what):
        left = HOLD_MS - 1e3 * (time.perf_counter() - self.t0)
        assert not self.ev.query(), f"{case}: the hold ended before {what} was issued: the case tested nothing"
        MARGINS.append((case, left))


def run_case(W, mode, cycles, case, producer, consumers, prepare=None, size=SIZE, write_ms=None, produced=None):
    """The held / slow run and the synchronised twin run of one case -> both runs' outputs and end states.
    produced(e): what a reading producer wrote (a pack's buffer), compared once every stream has finished."""
    results = []
    for held in (True, False):
        e = None
        try:
            e = Env(W, mode, size)
            e.warm()
            if prepare:
                prepare(e)
                e.sync()
            outs = []
            win = Window(e, cycles) if held and cycles else None
            t0 = None
            producer(e)
            if held and not cycles:
                t0 = time.perf_counter()
            for name in consumers:
                blocking, fn = CONSUMERS[name]
                if not held:
                    e.sync()
                elif blocking:
                    check(case, win, t0, write_ms, f"{name} (blocking)")
                if not blocking:
                    e.s2 = e.cstream[name]
                outs.append(fn(e))
                if held and not blocking:
                    check(case, win, t0, write_ms, name)
            e.sync()
            if produced:
                outs.append(produced(e))
            results.append((flat(to_np(outs)), end_state(e)))
        finally:
            import torch

            torch.cuda.synchronize()
            if e is not None:
                e.close()
    (go, gs), (wo, ws) = results
    assert len(go) == len(wo)
    for i, (a, b) in enumerate(zip(go, wo)):
        a, b = np.ascontiguousarray(np.atleast_1d(a)), np.ascontiguousarray(np.atleast_1d(b))
        assert a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8)), \
            f"{case}: output {i} ({consumers}) differs from the synchronised twin"
    for i, (a, b) in enumerate(zip(gs, ws)):
        a, b = np.ascontiguousarray(np.atleast_1d(a)), np.ascontiguousarray(np.atleast_1d(b))
        assert a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8)), \
            f"{case}: end state item {i} differs from the synchronised twin"


def check(case, win, t0, write_ms, what):
    if win is not None:
        win.check(case, what)
    else:
        issue = 1e3 * (time.perf_counter() - t0)
        assert issue * 5 < write_ms, f"{case}: {issue:.2f} ms to issue up to {what}, the write takes {write_ms:.1f} ms"
        MARGINS.append((case, write_ms - issue))


# ---- consumers: (blocking, fn(env) -> output) ------------------------------------------------------------------

def _dev(e):
    W = e.W
    return W["d_hints"].data_ptr(), W["d_pts"].data_ptr(), W["d_offs"].data_ptr(), W["data"][0]["maxn"]


def c_match_batch_device(e):
    h, p, o, n = _dev(e)
    po, co = e.o["mbd"]
    e.reps[0].match_batch_device(B, h, p, o, 0, n, po.data_ptr(), co.data_ptr(), e.s2.cuda_stream)
    return e.o["mbd"]


def c_match_batch_ranges_device(e):
    po, co = e.o["mbr"]
    e.reps[0].match_batch_ranges_device(B, e.W["d_hints"].data_ptr(), e.W["d_ranges"].data_ptr(), po.data_ptr(),
                                        co.data_ptr(), e.s2.cuda_stream)
    return e.o["mbr"]


def c_match_batch_record_device(e):
    h, p, o, n = _dev(e)
    po, co, ro = e.o["rec"]
    e.reps[0].match_batch_record_device(B, h, p, o, 0, n, po.data_ptr(), co.data_ptr(), ro.data_ptr(), e.s2.cuda_stream)
    return e.o["rec"]


def c_likelihood_batch_device(e):
    _, p, o, _ = _dev(e)
    e.reps[0].likelihood_batch_device(0, B, e.W["d_truth"].data_ptr(), p, o, 0, e.o["lh"].data_ptr(), e.s2.cuda_stream)
    return e.o["lh"]


def c_best_hypothesis_device(e):
    _, p, o, _ = _dev(e)
    lh, b4 = e.o["best"]
    e.reps[0].best_hypothesis_device(1, B, e.W["d_truth"].data_ptr(), p, o, 0, b4.data_ptr(), lh.data_ptr(),
                                     e.s2.cuda_stream)
    return e.o["best"]


def c_pack_rect_device(e):
    e.reps[0].pack_rect_device(0, (0, 0, e.size - 1, e.size - 1), e.o["prect"].data_ptr(), e.s2.cuda_stream)
    return e.o["prect"]


def c_pack_dirty_device(e):
    e.reps[0].pack_dirty_device(e.o["pdirty"].data_ptr(), CAP, False, e.s2.cuda_stream)
    return e.o["pdirty"]


def c_group_pack_dirty_device(e):
    e.G.pack_dirty_device(e.o["gpack"].data_ptr(), CAP, False, e.s2.cuda_stream)
    return e.o["gpack"]


def c_match_batch_submit(e):
    e.ticket = e.reps[0].match_batch_submit(*e._sub_args())
    return None


def c_match_batch_wait(e):
    e.reps[0].match_batch_wait(e.ticket)
    return [p.array.copy() for p in e.pinned[3:]]


def c_match_batch_ranges_submit(e):
    e.ticket = e.reps[0].match_batch_ranges_submit(*(p.array for p in e.rpinned))
    return None


def c_match_batch_ranges_wait(e):
    e.reps[0].match_batch_wait(e.ticket)
    return [p.array.copy() for p in e.rpinned[2:]]


def c_second_unpack_dirty(e):
    """another owner's tiles into member 0, on a stream that nothing held"""
    e.reps[0].unpack_dirty_device(e.W["sbuf2"].data_ptr(), CAP, e.s2.cuda_stream)
    return None


def c_second_unpack_rect(e):
    e.reps[0].unpack_rect_device(0, e.W["rect"], e.W["rbuf2"].data_ptr(), e.s2.cuda_stream)
    return None


def c_group_reset(e):
    e.G.reset()
    return None


def c_match_batch(e):
    d = e.W["data"][0]
    return e.reps[0].match_batch(d["bh"], d["bp"], d["bo"])


def c_match_data(e):
    d = e.W["data"][0]
    return e.reps[0].matchData(d["bh"][0], d["scans"][8])


def c_match_data_record(e):
    d = e.W["data"][0]
    pose, cov, rec = e.reps[0].matchData(d["bh"][1], d["scans"][9], record=True)
    return pose, cov, rec


def c_slam_update(e):
    d = e.W["data"][0]
    return e.reps[0].slam_update(d["bh"][2], d["scans"][10])


def _gq(e):
    data = e.W["data"]
    return [data[m]["truth"][8:10] for m in range(M)], [data[m]["scans"][8] for m in range(M)]


def c_group_step(e):
    data = e.W["data"]
    return e.G.slam_update(np.stack([data[m]["hints"][11] for m in range(M)]), [data[m]["scans"][11] for m in range(M)])


def c_group_match_batch(e):
    poses, scans = _gq(e)
    return e.G.match_batch(poses, points=scans)


def c_group_match_batch_ranges(e):
    data = e.W["data"]
    return e.G.match_batch_ranges([data[m]["hints"][12:13] for m in range(M)], [data[m]["ranges"][12] for m in range(M)],
                                  score=True)


def c_group_likelihood(e):
    poses, scans = _gq(e)
    return e.G.likelihood(0, poses, points=scans)


def c_group_covariance(e):
    poses, scans = _gq(e)
    return e.G.covariance(1, poses, points=scans)


def c_group_best_hypothesis(e):
    poses, scans = _gq(e)
    return e.G.best_hypothesis(0, poses, points=scans)


def _rays(e):
    b = [np.float32([[0.0, 0.0], [0.3, -0.2], [-1.0, 0.5]]) for _ in range(M)]
    en = [np.float32([[8.0, 1.0], [-7.0, 6.0], [5.0, -9.0]]) for _ in range(M)]
    return b, en


def c_group_get_dist(e):
    return e.G.get_dist(0, *_rays(e))


def c_group_raycast(e):
    c = e.size // 2
    b = [np.int32([[c, c], [c + 3, c - 2]]) for _ in range(M)]
    en = [np.int32([[c + 200, c + 17], [c - 150, c + 90]]) for _ in range(M)]
    return e.G.raycast(0, b, en)


def c_group_sync_occupancy(e):
    grids = []
    for r in e.reps:
        sx, sy, _ = r.level_info(0)
        grids.append(np.full((sy, sx), 7, np.int8))
    rects = e.G.sync_occupancy(0, grids, reset=False)
    return [np.asarray([x or (-1,) * 4 for x in rects])] + grids


def c_second_group_likelihood(e):
    data = e.W["data"]
    return e.H.likelihood(0, [data[0]["truth"][8:10], data[M]["truth"][8:10]], points=[data[0]["scans"][8], data[M]["scans"][8]])


def c_download_level(e):
    return [e.reps[0].download_level(l) for l in range(LEVELS)]


def c_download_prob(e):
    return [e.reps[0].download_prob(l) for l in range(LEVELS)]


def c_download_occupancy(e):
    return e.reps[0].download_occupancy(0)


def c_get_dirty_rects(e):
    return np.asarray([x or (-1,) * 4 for x in e.reps[0].get_dirty_rects()])


def c_get_mirror_dirty_rect(e):
    return np.asarray([e.reps[0].get_mirror_dirty_rect(l) or (-1,) * 4 for l in range(LEVELS)])


def c_last_match_scan(e):
    return e.reps[0].last_match_scan()


def c_second_group_pack(e):
    e.H.pack_dirty_device(e.o["hpack"].data_ptr(), CAP, False, e.s2.cuda_stream)
    return e.o["hpack"]


CONSUMERS = {
    # a second caller stream
    "match_batch_device": (False, c_match_batch_device),
    "match_batch_ranges_device": (False, c_match_batch_ranges_device),
    "match_batch_record_device": (False, c_match_batch_record_device),
    "likelihood_batch_device": (False, c_likelihood_batch_device),
    "best_hypothesis_device": (False, c_best_hypothesis_device),
    "pack_rect_device": (False, c_pack_rect_device),
    "pack_dirty_device": (False, c_pack_dirty_device),
    "group_pack_dirty_device": (False, c_group_pack_dirty_device),
    # the copy streams
    "match_batch_submit": (False, c_match_batch_submit),
    "match_batch_wait": (True, c_match_batch_wait),
    "match_batch": (True, c_match_batch),
    "match_batch_ranges_submit": (False, c_match_batch_ranges_submit),
    "match_batch_ranges_wait": (True, c_match_batch_ranges_wait),
    # map writes behind a held read
    "second_unpack_dirty": (False, c_second_unpack_dirty),
    "second_unpack_rect": (False, c_second_unpack_rect),
    "group_reset": (False, c_group_reset),
    # the handle's stream
    "match_data": (True, c_match_data),
    "match_data_record": (True, c_match_data_record),
    "slam_update": (True, c_slam_update),
    # the group's stream, and a second group sharing member 0
    "group_step": (True, c_group_step),
    "group_match_batch": (True, c_group_match_batch),
    "group_match_batch_ranges": (True, c_group_match_batch_ranges),
    "group_likelihood": (True, c_group_likelihood),
    "group_covariance": (True, c_group_covariance),
    "group_best_hypothesis": (True, c_group_best_hypothesis),
    "group_get_dist": (True, c_group_get_dist),
    "group_raycast": (True, c_group_raycast),
    "group_sync_occupancy": (True, c_group_sync_occupancy),
    "second_group_likelihood": (True, c_second_group_likelihood),
    "second_group_pack": (False, c_second_group_pack),
    # host reads
    "download_level": (True, c_download_level),
    "download_prob": (True, c_download_prob),
    "download_occupancy": (True, c_download_occupancy),
    "get_dirty_rects": (True, c_get_dirty_rects),
    "get_mirror_dirty_rect": (True, c_get_mirror_dirty_rect),
    "last_match_scan": (True, c_last_match_scan),
}

# every asynchronous consumer on a second caller stream, then the copy streams' submit
SECOND_STREAM = ["match_batch_device", "match_batch_ranges_device", "match_batch_record_device", "likelihood_batch_device",
                 "best_hypothesis_device", "pack_rect_device", "pack_dirty_device", "group_pack_dirty_device",
                 "match_batch_submit", "match_batch_wait"]


# ---- held producers ------------------------------------------------------------------------------------------

def p_unpack_dirty(e):
    e.reps[0].unpack_dirty_device(e.W["sbuf"].data_ptr(), CAP, e.sp.cuda_stream)


def p_unpack_rect(e):
    e.reps[0].unpack_rect_device(0, e.W["rect"], e.W["rbuf"].data_ptr(), e.sp.cuda_stream)


def p_group_unpack(e):
    e.G.unpack_dirty_device(e.W["gbuf"].data_ptr(), CAP, e.sp.cuda_stream)


def p_group_unpack_subset(e):
    e.G.unpack_dirty_device(e.W["gsub"].data_ptr(), CAP, e.sp.cuda_stream)


def p_refresh_level(e):
    """The owner's level-0 plane written through the device pointer on the caller's stream, then refresh_level."""
    import torch

    dst = torch.as_tensor(DevicePlane(e.reps[0].level_logodds_device_ptr(0), e.size * e.size), device="cuda")
    with torch.cuda.stream(e.sp):
        dst.copy_(e.o["plane"])   # (staged before the hold: a device-to-device copy behind it)
    e.reps[0].refresh_level(0, e.sp.cuda_stream)


class DevicePlane:
    """A level's log-odds plane (hsb_level_logodds_device_ptr) as a torch tensor, without a stream of its own."""

    def __init__(self, ptr, n):
        assert ptr
        self.__cuda_array_interface__ = dict(shape=(n,), typestr="<f4", data=(ptr, False), version=3, stream=None)


def prep_plane(e):
    import torch

    e.o["plane"].copy_(torch.from_numpy(np.ascontiguousarray(e.W["owner_planes"][0]).reshape(-1)))


def p_group_reset(e, members=None):
    """A held unpack of every member's tiles, then the group reset behind it on the group's stream."""
    e.G.unpack_dirty_device(e.W["gbuf"].data_ptr(), CAP, e.sp.cuda_stream)
    e.G.reset(members=members)


def prep_mapped(e):
    """Maps on every replica before a reset: the owner's tiles, synchronously."""
    import torch

    s = torch.cuda.Stream()
    e.G.unpack_dirty_device(e.W["gbuf"].data_ptr(), CAP, s.cuda_stream)
    e.H.slam_update(np.stack([e.W["data"][0]["hints"][0], e.W["data"][M]["hints"][0]]),
                    [e.W["data"][0]["scans"][0], e.W["data"][M]["scans"][0]])


HELD = {
    "unpack_dirty": (p_unpack_dirty, None),
    "unpack_rect": (p_unpack_rect, None),
    "group_unpack": (p_group_unpack, None),
    "group_unpack_subset": (p_group_unpack_subset, None),
    "refresh_level": (p_refresh_level, prep_plane),
    "group_reset": (p_group_reset, prep_mapped),
    "group_reset_subset": (lambda e: p_group_reset(e, [0, 2]), prep_mapped),
}

# Each producer: every asynchronous consumer on a second caller stream and the copy streams, then one blocking consumer
# of each kind of stream -- the handle's, two of the group's, the second group's, a host read -- taken in turn from
# these lists, so that every consumer meets at least one held producer.
ON_HANDLE = ["match_data", "match_data_record", "slam_update", "match_batch"]
ON_GROUP = ["group_step", "group_match_batch", "group_match_batch_ranges", "group_likelihood", "group_covariance",
            "group_best_hypothesis", "group_get_dist", "group_raycast", "group_sync_occupancy"]
HOST_READS = ["download_level", "download_prob", "download_occupancy", "get_dirty_rects", "get_mirror_dirty_rect",
              "last_match_scan"]
HELD_CASES = []
for _i, _p in enumerate(HELD):
    HELD_CASES += [(_p, SECOND_STREAM), (_p, [ON_HANDLE[_i % len(ON_HANDLE)]]), (_p, [ON_GROUP[(2 * _i) % len(ON_GROUP)]]),
                   (_p, [ON_GROUP[(2 * _i + 1) % len(ON_GROUP)]]), (_p, ["second_group_likelihood"]),
                   (_p, [HOST_READS[_i % len(HOST_READS)]])]


@MODES
@pytest.mark.parametrize("producer,consumers", HELD_CASES,
                         ids=[f"{p}-{'second_stream' if len(c) > 1 else c[0]}" for p, c in HELD_CASES])
def test_held_producer(world, hold_cycles, mode, producer, consumers):
    """A map-changing call queued behind a hold on a caller stream; each consumer is issued while the hold runs and
    must see the map the producer wrote, as on the synchronised twin."""
    fn, prep = HELD[producer]
    run_case(world, mode, hold_cycles, f"{producer}/{consumers[0]}", fn, consumers, prepare=prep)


# ---- write after read: a held read, then a map write that must not overtake it -------------------------------------

def prep_stepped(e):
    """Two synchronous steps on member 0 and one group step: written maps and dirty rectangles for the packs."""
    d = e.W["data"]
    for k in range(2):
        e.reps[0].slam_update(d[0]["hints"][k], d[0]["scans"][k])
    e.G.slam_update(np.stack([d[m]["hints"][2] for m in range(M)]), [d[m]["scans"][2] for m in range(M)])


def p_pack_dirty(e):
    e.reps[0].pack_dirty_device(e.o["pdirty"].data_ptr(), CAP, False, e.sp.cuda_stream)


def p_pack_rect(e):
    e.reps[0].pack_rect_device(0, (0, 0, e.size - 1, e.size - 1), e.o["prect"].data_ptr(), e.sp.cuda_stream)


def p_group_pack(e):
    e.G.pack_dirty_device(e.o["gpack"].data_ptr(), CAP, False, e.sp.cuda_stream)


# (producer, its output, prepare, consumers).  "pack waits for the map writes the handle has queued and the handle's next
# map write waits for pack": a sync step right behind a held pack; the group pack's members' next map write, a group
# step or a group reset, likewise ("their next map write waits for it").  "unpack waits for everything the handle has
# queued (matches still reading the planes)": a submitted match behind a held unpack, then a second unpack on a stream
# nothing held -- the match must see the first buffer's map.  (The group queries block until their result is on the
# host, so a map write issued after one cannot overtake it; reads a "_device" call queued on a caller stream are the
# caller's to order before a map write.)
WAR = {
    "pack_dirty-slam_update": (p_pack_dirty, lambda e: e.o["pdirty"], prep_stepped, ["slam_update"]),
    "pack_rect-slam_update": (p_pack_rect, lambda e: e.o["prect"], prep_stepped, ["slam_update"]),
    "group_pack-group_step": (p_group_pack, lambda e: e.o["gpack"], prep_stepped, ["group_step"]),
    "group_pack-group_reset": (p_group_pack, lambda e: e.o["gpack"], prep_stepped, ["group_reset"]),
    "unpack_dirty-submit-second_unpack": (p_unpack_dirty, None, None,
                                          ["match_batch_ranges_submit", "second_unpack_dirty", "match_batch_ranges_wait"]),
    "unpack_rect-submit-second_unpack": (p_unpack_rect, None, None,
                                         ["match_batch_ranges_submit", "second_unpack_rect", "match_batch_ranges_wait"]),
}


@MODES
@pytest.mark.parametrize("case", list(WAR))
def test_write_after_held_read(world, hold_cycles, mode, case):
    """A read queued behind a hold (a pack), or a match queued behind a held unpack; the map write issued right after
    it must wait: the pack ships, and the match sees, the map from before that write, as on the synchronised twin."""
    fn, produced, prep, consumers = WAR[case]
    run_case(world, mode, hold_cycles, case, fn, consumers, prepare=prep, produced=produced)


# ---- slow producers: nowait steps with a long map write ----------------------------------------------------------

def _long_inputs(e, n):
    from hector_slam_b200 import synth

    for r in e.all:
        nr = min(n, 1 << 20)
        r.set_scan_format(nr, -np.pi, 2 * np.pi / nr, 0.1, 200.0)
        r.set_cloud_format(synth.laser_transform(xyz=(0.0, 0.0, 0.0), rpy=(0.0, 0.0, 0.0)), 0.16, 200.0 ** 2, -1.0, 1.0)


def nowait_single(kind, n):
    def producer(e):
        r = e.reps[0]
        pts = long_scan(n)
        hint = [0.0, 0.0, 0.0]
        if kind == "endpoints":
            r.slam_update(hint, pts, map_without_matching=True, nowait=True)
        elif kind == "ranges":
            r.slam_update_ranges(hint, np.full(n, LONG_R * RES, np.float32), map_without_matching=True, nowait=True)
        else:
            xyz = np.zeros((n, 3), np.float32)
            xyz[:, :2] = pts * np.float32(RES)
            r.slam_update_cloud(hint, xyz, map_without_matching=True, nowait=True)
    return producer


def nowait_group(n, members):
    def producer(e):
        pts = long_scan(n)
        K = M if members is None else len(members)
        e.G.slam_update(np.zeros((K, 3), np.float32), [pts] * K, map_without_matching=[1] * K, nowait=True,
                        members=members)
    return producer


def nowait_mixed(n):
    """A nowait step of G on members 0 and 1; its consumers start with a call of H (member 0 and a handle of its own),
    which leaves H's event in member 0's one group-event slot: member 0's next single-handle call must still wait for
    G's write."""
    def producer(e):
        pts = long_scan(n)
        e.G.slam_update(np.zeros((2, 3), np.float32), [pts, pts], map_without_matching=[1, 1], nowait=True, members=[0, 1])
    return producer


SLOW_CONSUMERS = {
    "second_stream": ["match_batch_device", "likelihood_batch_device", "best_hypothesis_device", "pack_dirty_device",
                      "match_batch_record_device", "pack_rect_device", "match_batch_submit", "match_batch_wait"],
    "match_batch": ["match_batch"],
    "group_likelihood": ["group_likelihood"],
    "second_group": ["second_group_likelihood"],
    "match_data": ["match_data"],
    "download_level": ["download_level"],
    "group_pack": ["group_pack_dirty_device", "group_get_dist"],
    "second_group_then_member": ["second_group_pack", "match_data"],
}
# (a single step's write is on the handle's own stream: the handle's stream and host reads are ordered by the stream)
# (the LaserScan-projection kind converts its whole scan in shared memory, so its write cannot be made long: its nowait
# step runs the same host body as the other three kinds)
SLOW_CASES = ([(p, c) for p in ("endpoints", "ranges", "cloud") for c in ("second_stream", "group_likelihood")]
              + [("endpoints", c) for c in ("match_batch", "second_group", "group_pack")]
              + [("group", c) for c in ("second_stream", "match_batch", "second_group", "match_data", "download_level",
                                         "group_pack")]
              + [("group_subset", c) for c in ("second_stream", "match_data", "second_group")]
              + [("mixed", c) for c in ("second_group_then_member", "second_stream")])


@MODES
@pytest.mark.parametrize("producer,consumers", SLOW_CASES, ids=[f"{p}-{c}" for p, c in SLOW_CASES])
def test_nowait_producer(world, long_write, mode, producer, consumers):
    """A nowait step whose map write takes tens of ms on the device; every consumer is issued while it runs and must
    see the written map, as on the synchronised twin."""
    n, ms = long_write
    if producer == "ranges":
        n = min(n, 1 << 20)
    write_ms = ms[n]
    fn = {"group": nowait_group(n, None), "group_subset": nowait_group(n, [0, 2]), "mixed": nowait_mixed(n)}.get(
        producer) or nowait_single(producer, n)

    def prep(e):
        _long_inputs(e, n)
        prep_base(e)
    run_case(world, mode, 0, f"nowait {producer}/{consumers}", fn, SLOW_CONSUMERS[consumers], prepare=prep, size=BIG,
             write_ms=write_ms)


def prep_base(e):
    """A matched step on every handle (the last-match containers, a written map) before the slow producer."""
    for m, r in enumerate(e.all):
        d = e.W["data"][m]
        r.slam_update(d["hints"][0] + np.float32([1.0, 0.0, 0.0]), d["scans"][0])
