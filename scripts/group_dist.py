"""What answering a fleet's obstacle-distance queries in one pass buys a server of robots.

Workload: M robots (--sizes), each a handle with a 3-level 2048^2 map, stepped as in scripts/group_step_subset.py: 40 Hz
lidars with seeded random phases, a tick every --window-ms (5 ms) steps the robots whose scan falls into it with one
hsb_group_slam_update_projected_subset(nowait = 1).  Right after every step, a seeded share of the robots (--share,
at least one) asks hector_map_server's get_distance_to_obstacle question: --rays world-frame rays of 5 m
(hector_map_server.cpp:113-116) from the robot's pose, at level 0.

Two twin fleets get the same scans and the same rays, one per arm:
  group     one hsb_group_get_dist_subset over the queried robots
  loop      per queried robot one hsb_get_dist_batch (the per-member C-ABI path, driven from Python through ctypes)
Both fleets are stepped every tick and queried right after their step; the order of the two arms alternates from tick
to tick, in each of --rounds rounds of --ticks ticks.  Reported per arm: query-round time p50 / p99 (host clock around
the round, which ends in a synchronise) and the tick time, step included, p50 / p99.  Every round's distances, hit
points and found flags of the two arms are compared bit for bit.  Prints one JSON line per M, with the card and power
limit read in the same run.

    python scripts/group_dist.py [--sizes 16,128] [--rounds 3] [--ticks 400]
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

RAY_M = 5.0   # hector_map_server extends every query ray to 5 m


def pct(v, q):
    return float(np.percentile(np.asarray(v) * 1e3, q))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="16,128")
    ap.add_argument("--window-ms", type=float, default=5.0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--ticks", type=int, default=400)
    ap.add_argument("--share", type=float, default=0.25)
    ap.add_argument("--rays", type=int, default=8)
    args = ap.parse_args()
    from hector_slam_b200 import capi, synth

    sizes = [int(x) for x in args.sizes.split(",")]
    Mmax = max(sizes)
    lib = capi.load_library()
    fmt = synth.SCAN_FORMAT
    nb = fmt["n_beams"]
    arms = ("group", "loop")

    def make(s):
        rep = capi.MapRepB200(RES, SIZE, levels=LEVELS, update_factor_free=0.4, update_factor_occupied=0.9)
        rep.setMapUpdateMinDistDiff(0.4)
        rep.setMapUpdateMinAngleDiff(0.13)
        rep.set_laser_projection(**fmt, range_cutoff=CUTOFF)
        mount = synth.laser_transform(xyz=(0.05 + 0.001 * s, -0.02 + 0.0005 * s, 0.3),
                                      rpy=(0.002 * (s % 5), -0.003 * (s % 7), 0.01 * (s % 11)))
        rep.set_cloud_format(mount, **synth.CLOUD_FORMAT)
        return rep

    fleets = {a: [make(s) for s in range(Mmax)] for a in arms}
    data = [session_scans(900 + s) for s in range(Mmax)]
    phase = np.random.default_rng(40).uniform(0.0, PERIOD_MS, Mmax)
    pose = np.zeros((Mmax, 3), np.float32)
    cov = np.zeros((Mmax, 9), np.float32)
    upd = np.zeros(Mmax, np.int32)
    kept = np.zeros(Mmax, np.int32)
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip()
    except OSError:
        card = "unknown"

    def check(st, rep):
        if st != 0:
            raise capi.HsbError(st, lib.hsb_last_error(rep.h).decode())

    R = args.rays
    for M in sizes:
        groups = {a: capi.SlamGroup(fleets[a][:M]) for a in arms}
        scan_no = np.zeros(M, np.int64)
        qrng = np.random.default_rng(41)
        n_max = M * R
        out = {a: (np.zeros(n_max, np.float32), np.zeros((n_max, 2), np.float32), np.zeros(n_max, np.int32))
               for a in arms}

        def window(t):
            lo = (t * args.window_ms) % PERIOD_MS
            d = (phase[:M] - lo) % PERIOD_MS
            members = np.ascontiguousarray(np.nonzero(d < args.window_ms)[0][np.argsort(d[d < args.window_ms])], np.int32)
            ks = [int(scan_no[j] % POSES) for j in members]
            scan_no[members] += 1
            hints = np.ascontiguousarray(np.stack([data[j][k][0] for j, k in zip(members, ks)]) if len(members)
                                         else np.zeros((0, 3), np.float32), np.float32)
            ranges = np.ascontiguousarray(np.concatenate([data[j][k][1] for j, k in zip(members, ks)]) if len(members)
                                          else np.zeros(0, np.float32), np.float32)
            return members, hints, ranges, np.arange(len(members) + 1, dtype=np.int32) * nb

        def queries():
            """the robots that ask this tick (seeded), and R rays of RAY_M metres from each one's last hint pose"""
            K = max(1, int(round(args.share * M)))
            asked = np.ascontiguousarray(np.sort(qrng.choice(M, K, replace=False)), np.int32)
            origin = np.stack([data[j][int((scan_no[j] + POSES - 1) % POSES)][0][:2] for j in asked]).astype(np.float32)
            begin = np.repeat(origin, R, axis=0).astype(np.float32)
            ang = qrng.uniform(-np.pi, np.pi, K * R)
            end = (begin + RAY_M * np.stack([np.cos(ang), np.sin(ang)], axis=1)).astype(np.float32)
            offs = (np.arange(K + 1) * R).astype(np.int32)
            return asked, np.ascontiguousarray(begin), np.ascontiguousarray(end), offs

        def step(a, w):
            members, hints, ranges, offs = w
            check(lib.hsb_group_slam_update_projected_subset(groups[a].g, len(members), members.ctypes.data,
                                                             hints.ctypes.data, ranges.ctypes.data, offs.ctypes.data,
                                                             None, None, 1, pose.ctypes.data, cov.ctypes.data,
                                                             upd.ctypes.data, kept.ctypes.data), fleets[a][0])

        def query_group(q):
            asked, begin, end, offs = q
            d, h, f = out["group"]
            check(lib.hsb_group_get_dist_subset(groups["group"].g, len(asked), asked.ctypes.data, 0, offs.ctypes.data,
                                                begin.ctypes.data, end.ctypes.data, d.ctypes.data, h.ctypes.data,
                                                f.ctypes.data), fleets["group"][0])

        def query_loop(q):
            asked, begin, end, offs = q
            d, h, f = out["loop"]
            for k, j in enumerate(asked):
                rep = fleets["loop"][j]
                a = int(offs[k])
                check(lib.hsb_get_dist_batch(rep.h, 0, R, begin[a:].ctypes.data, end[a:].ctypes.data, d[a:].ctypes.data,
                                             h[a:].ctypes.data, f[a:].ctypes.data), rep)

        query = {"group": query_group, "loop": query_loop}
        round_s = {a: [] for a in arms}
        tick_s = {a: [] for a in arms}
        t, n_q, found = 0, 0, 0
        for rnd in range(args.rounds):
            for i in range(args.ticks):
                w = window(t)
                t += 1
                if len(w[0]) == 0:
                    continue
                q = queries()
                order = arms if n_q % 2 == 0 else arms[::-1]
                for a in order:
                    t0 = time.perf_counter()
                    step(a, w)
                    t1 = time.perf_counter()
                    query[a](q)
                    t2 = time.perf_counter()
                    round_s[a].append(t2 - t1)
                    tick_s[a].append(t2 - t0)
                n_q += 1
                Q = int(q[3][-1])
                for x, y in zip(out["group"], out["loop"]):
                    assert np.array_equal(x[:Q].view(np.uint32), y[:Q].view(np.uint32)), (M, t)
                found += int(out["group"][2][:Q].sum())
        for a in arms:
            groups[a].close()
            for r in fleets[a][:M]:
                r.onMapUpdated()
        res = {"M": M, "map": f"{SIZE}^2 x {LEVELS} levels, level 0 queried", "share": args.share, "rays_per_robot": R,
               "query_rounds_per_arm": n_q, "rays_found": found, "results_identical": True, "card": card}
        for a in arms:
            res[f"{a}_query_ms_p50"] = round(pct(round_s[a], 50), 3)
            res[f"{a}_query_ms_p99"] = round(pct(round_s[a], 99), 3)
            res[f"{a}_tick_ms_p50"] = round(pct(tick_s[a], 50), 3)
            res[f"{a}_tick_ms_p99"] = round(pct(tick_s[a], 99), 3)
        print(json.dumps(res), flush=True)
    for a in arms:
        for r in fleets[a]:
            r.close()


if __name__ == "__main__":
    main()
