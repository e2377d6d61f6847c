"""What scoring a fleet's poses in one pass buys a server of robots.

Workload: M robots (--sizes), each a handle with a 3-level 2048^2 map, stepped as in scripts/group_step_subset.py: 40 Hz
lidars with seeded random phases, a tick every --window-ms (5 ms) steps the robots whose scan falls into it with one
hsb_group_slam_update_projected_subset(nowait = 1).  Right after every step the server scores the poses the step
returned, at level 0, against the scans it just stepped: getLikelihoodForState (is the match plausible?) and
getCovarianceForPose (the reference's own covariance).

Three twin fleets get the same scans, one per arm:
  last      one hsb_group_likelihood_subset / hsb_group_covariance_subset without points: each robot's last matched scan
            as it lies on the device
  resent    the same group call with the scans' endpoints sent along
  loop      per stepped robot one hsb_likelihood_batch / hsb_covariance_batch (the per-member C-ABI path, driven from
            Python through ctypes)
(The endpoints of `resent` and `loop` are converted before the timed loop; a server would pay for that conversion too.)
Every fleet is stepped every tick and scored right after its step, first the likelihood, then the covariance; the
order of the arms rotates from tick to tick, in each of --rounds rounds of --ticks ticks after a warm-up round.
Reported per arm: the time of the likelihood round and of the covariance round (host clock around the round, which
ends in a synchronise) and of the tick (step + likelihood round), p50 / p99, and the host-to-device bytes of a mean
round computed from its inputs.  Every round's results of the three arms are compared bit for bit.

Relocalisation (--reloc, members x --hypotheses): one hsb_group_best_hypothesis_subset with the robots' scans against
per member hsb_best_hypothesis_device on device tensors plus the read-back of each winner; the winners are compared bit
for bit.

Prints one JSON line per M and per relocalisation size, with the card and power limit read in the same run.  Needs a
GPU; there is no fall-back.

    python scripts/group_score.py [--sizes 16,128] [--rounds 3] [--ticks 400] [--reloc 8,32] [--hypotheses 2048]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from group_step_subset import CUTOFF, LEVELS, PERIOD_MS, POSES, RES, SIZE, session_scans  # noqa: E402

ARMS = ("last", "resent", "loop")


def pct(v, q):
    return float(np.percentile(np.asarray(v) * 1e3, q))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="16,128")
    ap.add_argument("--window-ms", type=float, default=5.0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--ticks", type=int, default=400)
    ap.add_argument("--reloc", default="8,32")
    ap.add_argument("--hypotheses", type=int, default=2048)
    ap.add_argument("--reloc-rounds", type=int, default=200)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("scripts/group_score.py measures on a GPU and found none")
    from hector_slam_b200 import capi, synth

    sizes = [int(x) for x in args.sizes.split(",") if x]
    reloc = [int(x) for x in args.reloc.split(",") if x]
    Mmax = max(sizes + reloc)
    lib = capi.load_library()
    fmt = synth.SCAN_FORMAT
    nb = fmt["n_beams"]

    def make(s):
        rep = capi.MapRepB200(RES, SIZE, levels=LEVELS, update_factor_free=0.4, update_factor_occupied=0.9)
        rep.setMapUpdateMinDistDiff(0.4)
        rep.setMapUpdateMinAngleDiff(0.13)
        rep.set_laser_projection(**fmt, range_cutoff=CUTOFF)
        mount = synth.laser_transform(xyz=(0.05 + 0.001 * s, -0.02 + 0.0005 * s, 0.3),
                                      rpy=(0.002 * (s % 5), -0.003 * (s % 7), 0.01 * (s % 11)))
        rep.set_cloud_format(mount, **synth.CLOUD_FORMAT)
        return rep

    fleets = {a: [make(s) for s in range(Mmax)] for a in ARMS}
    data = [session_scans(900 + s) for s in range(Mmax)]
    # the endpoints of every scan, as the step's conversion keeps them (for the arms that send the scan)
    endpoints = [[np.ascontiguousarray(fleets["loop"][j].projected_scan_to_points(data[j][k][1])[0], np.float32)
                  for k in range(POSES)] for j in range(Mmax)]
    phase = np.random.default_rng(40).uniform(0.0, PERIOD_MS, Mmax)
    pose = {a: np.zeros((Mmax, 3), np.float32) for a in ARMS}
    cov = np.zeros((Mmax, 9), np.float32)
    upd = np.zeros(Mmax, np.int32)
    kept = np.zeros(Mmax, np.int32)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()

    def check(st, rep):
        if st != 0:
            raise capi.HsbError(st, lib.hsb_last_error(rep.h).decode())

    for M in sizes:
        groups = {a: capi.SlamGroup(fleets[a][:M]) for a in ARMS}
        scan_no = np.zeros(M, np.int64)
        lh = {a: np.zeros(M, np.float32) for a in ARMS}
        cw = {a: np.zeros((M, 9), np.float32) for a in ARMS}
        cm = {a: np.zeros((M, 9), np.float32) for a in ARMS}

        def window(t):
            lo = (t * args.window_ms) % PERIOD_MS
            d = (phase[:M] - lo) % PERIOD_MS
            members = np.ascontiguousarray(np.nonzero(d < args.window_ms)[0][np.argsort(d[d < args.window_ms])], np.int32)
            ks = [int(scan_no[j] % POSES) for j in members]
            scan_no[members] += 1
            K = len(members)
            hints = np.ascontiguousarray(np.stack([data[j][k][0] for j, k in zip(members, ks)]) if K
                                         else np.zeros((0, 3), np.float32), np.float32)
            ranges = np.ascontiguousarray(np.concatenate([data[j][k][1] for j, k in zip(members, ks)]) if K
                                          else np.zeros(0, np.float32), np.float32)
            scans = [endpoints[j][k] for j, k in zip(members, ks)]
            so = np.zeros(K + 1, np.int32)
            so[1:] = np.cumsum([s.shape[0] for s in scans])
            pts = np.ascontiguousarray(np.concatenate(scans) if K else np.zeros((1, 2), np.float32), np.float32)
            return members, hints, ranges, np.arange(K + 1, dtype=np.int32) * nb, scans, so, pts, \
                np.arange(K + 1, dtype=np.int32)

        def step(a, w):
            members, hints, ranges, offs = w[:4]
            check(lib.hsb_group_slam_update_projected_subset(groups[a].g, len(members), members.ctypes.data,
                                                             hints.ctypes.data, ranges.ctypes.data, offs.ctypes.data,
                                                             None, None, 1, pose[a].ctypes.data, cov.ctypes.data,
                                                             upd.ctypes.data, kept.ctypes.data), fleets[a][0])

        def score(a, w, covariance):
            members, _, _, _, scans, so, pts, po = w
            K = len(members)
            p = pose[a]
            if a == "loop":
                for k, j in enumerate(members):
                    rep = fleets[a][j]
                    s = scans[k]
                    if covariance:
                        check(lib.hsb_covariance_batch(rep.h, 0, 1, p[k:].ctypes.data, s.ctypes.data, None, s.shape[0],
                                                       cm[a][k:].ctypes.data, cw[a][k:].ctypes.data), rep)
                    else:
                        check(lib.hsb_likelihood_batch(rep.h, 0, 1, p[k:].ctypes.data, s.ctypes.data, None, s.shape[0],
                                                       lh[a][k:].ctypes.data), rep)
                return
            pp, sp = (pts.ctypes.data, so.ctypes.data) if a == "resent" else (None, None)
            if covariance:
                check(lib.hsb_group_covariance_subset(groups[a].g, K, members.ctypes.data, 0, po.ctypes.data, p.ctypes.data,
                                                      pp, sp, cm[a].ctypes.data, cw[a].ctypes.data), fleets[a][0])
            else:
                check(lib.hsb_group_likelihood_subset(groups[a].g, K, members.ctypes.data, 0, po.ctypes.data, p.ctypes.data,
                                                      pp, sp, lh[a].ctypes.data), fleets[a][0])

        lh_s = {a: [] for a in ARMS}
        cov_s = {a: [] for a in ARMS}
        tick_s = {a: [] for a in ARMS}
        h2d = {a: [] for a in ARMS}
        t, n_q, plausible = 0, 0, 0
        for rnd in range(-1, args.rounds):   # round -1 warms up: modules, staging growth, the maps' first writes
            for i in range(args.ticks if rnd >= 0 else 100):
                w = window(t)
                t += 1
                K = len(w[0])
                if K == 0:
                    continue
                for a in (ARMS[n_q % 3:] + ARMS[:n_q % 3]):
                    t0 = time.perf_counter()
                    step(a, w)
                    t1 = time.perf_counter()
                    score(a, w, False)
                    t2 = time.perf_counter()
                    score(a, w, True)
                    t3 = time.perf_counter()
                    if rnd >= 0:
                        lh_s[a].append(t2 - t1)
                        cov_s[a].append(t3 - t2)
                        tick_s[a].append(t2 - t0)
                n_q += 1
                total = int(w[5][-1])
                if rnd >= 0:
                    h2d["last"].append(K * 16 + (K + 1) * 4 + K * 12)
                    h2d["resent"].append(K * 16 + (K + 1) * 4 + K * 12 + total * 8)
                    h2d["loop"].append(K * 12 + total * 8)
                for a in ARMS[1:]:
                    assert np.array_equal(pose[a][:K].view(np.uint32), pose["last"][:K].view(np.uint32)), (M, t, a)
                    assert np.array_equal(lh[a][:K].view(np.uint32), lh["last"][:K].view(np.uint32)), (M, t, a)
                    assert np.array_equal(cm[a][:K].view(np.uint32), cm["last"][:K].view(np.uint32)), (M, t, a)
                    assert np.array_equal(cw[a][:K].view(np.uint32), cw["last"][:K].view(np.uint32)), (M, t, a)
                plausible += int((lh["last"][:K] > 0.5).sum())
        for a in ARMS:
            groups[a].close()
            for r in fleets[a][:M]:
                r.onMapUpdated()
        res = {"M": M, "map": f"{SIZE}^2 x {LEVELS} levels, level 0 scored", "scored": "the poses each tick's step returned",
               "rounds_per_arm": len(lh_s["last"]), "likelihoods_above_0.5": plausible, "results_identical": True,
               "card": card}
        for a in ARMS:
            res[f"{a}_h2d_bytes_mean"] = round(float(np.mean(h2d[a])), 1)
            res[f"{a}_likelihood_ms_p50"] = round(pct(lh_s[a], 50), 3)
            res[f"{a}_likelihood_ms_p99"] = round(pct(lh_s[a], 99), 3)
            res[f"{a}_covariance_ms_p50"] = round(pct(cov_s[a], 50), 3)
            res[f"{a}_covariance_ms_p99"] = round(pct(cov_s[a], 99), 3)
            res[f"{a}_tick_ms_p50"] = round(pct(tick_s[a], 50), 3)
            res[f"{a}_tick_ms_p99"] = round(pct(tick_s[a], 99), 3)
        print(json.dumps(res), flush=True)

    # relocalisation: K lost robots, H hypotheses each, scored against each robot's current scan
    H = args.hypotheses
    rng = np.random.default_rng(42)
    for K in reloc:
        reps = fleets["last"][:K]
        g = capi.SlamGroup(reps)
        members = np.arange(K, dtype=np.int32)
        scans = [endpoints[j][0] for j in range(K)]
        so = np.zeros(K + 1, np.int32)
        so[1:] = np.cumsum([s.shape[0] for s in scans])
        pts = np.ascontiguousarray(np.concatenate(scans), np.float32)
        po = (np.arange(K + 1) * H).astype(np.int32)
        hyp = np.ascontiguousarray(np.concatenate([data[j][0][0][None] + rng.normal(0, 1, (H, 3)) * [0.5, 0.5, 0.3]
                                                   for j in range(K)]), np.float32)
        d_hyp = [torch.from_numpy(hyp[j * H:(j + 1) * H].reshape(-1)).cuda() for j in range(K)]
        d_pts = [torch.from_numpy(s.reshape(-1)).cuda() for s in scans]
        d_best = [torch.zeros(4, device="cuda") for _ in range(K)]
        best_g, idx_g = np.zeros((K, 4), np.float32), np.zeros(K, np.int32)
        best_l = np.zeros((K, 4), np.float32)

        def run_group():
            check(lib.hsb_group_best_hypothesis_subset(g.g, K, members.ctypes.data, 0, po.ctypes.data, hyp.ctypes.data,
                                                       pts.ctypes.data, so.ctypes.data, None, best_g.ctypes.data,
                                                       idx_g.ctypes.data), reps[0])

        def run_loop():
            for j in range(K):
                reps[j].best_hypothesis_device(0, H, d_hyp[j].data_ptr(), d_pts[j].data_ptr(), None, scans[j].shape[0],
                                               d_best[j].data_ptr(), None, 0)
                best_l[j] = d_best[j].cpu().numpy()

        runs = {"group": run_group, "loop": run_loop}
        times = {a: [] for a in runs}
        for r in range(-20, args.reloc_rounds):
            for a in (("group", "loop") if r % 2 == 0 else ("loop", "group")):
                t0 = time.perf_counter()
                runs[a]()
                if r >= 0:
                    times[a].append(time.perf_counter() - t0)
            assert np.array_equal(best_g.view(np.uint32), best_l.view(np.uint32)), (K, r)
        g.close()
        res = {"relocalisation_members": K, "hypotheses_each": H, "rounds_per_arm": args.reloc_rounds,
               "group_h2d_bytes": int(K * 16 + (K + 1) * 4 + K * H * 12 + so[-1] * 8),
               "loop_h2d_bytes": 0, "winners_identical": True, "best_likelihood_min": float(best_g[:, 0].min()),
               "card": card}
        for a in runs:
            res[f"{a}_ms_p50"] = round(pct(times[a], 50), 3)
            res[f"{a}_ms_p99"] = round(pct(times[a], 99), 3)
        print(json.dumps(res), flush=True)
    for a in ARMS:
        for r in fleets[a]:
            r.close()


if __name__ == "__main__":
    main()
