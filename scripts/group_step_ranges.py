"""What the fused ranges steps buy a robot (or a server of robots) that runs without the laser tf and feeds raw LaserScan
ranges (HectorMappingRos.cpp:248-254).

Workload: M independent sessions, each its own handle with a 3-level 2048^2 map, driving synthetic 1081-beam scans along
its own closed trajectory through its own seeded world (the same scans as a Point32 cloud for the cloud arm).

Group part, per M in --sizes, arms alternated within each round on the same handles:
  group_ranges  one hsb_group_slam_update_ranges(nowait = 1): conversion, match, gate and map write for all M
  group_cloud   one hsb_group_slam_update_cloud(nowait = 1) on the same scans as projected clouds
  serial        hsb_slam_update_ranges(nowait = 1) on the M handles one after another from one thread
Per arm and round: 5 untimed ticks, then `--ticks` timed ones (host clock around the tick; every arm's last map writes
are waited for before the next arm starts).  p50 / p99 over all timed ticks of all rounds.

Single part, one session, arms alternated:
  fused     hsb_slam_update_ranges
  two_call  hsb_scan_to_points (a host round trip), then hsb_slam_update with the endpoints
  step time: the blocking form (map write included); pose latency: the nowait form, started after the previous step's
  map write has finished.

Host-to-device bytes per tick are computed, not timed: the scan payload is 4 B per beam for ranges and 12 B per point
for a cloud (the calls' small headers and per-session descriptors are left out).  Prints one JSON line per part, with
the card and power limit read in the same run.

    python scripts/group_step_ranges.py [--sizes 1,16,128] [--rounds 3] [--ticks 50]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZE, LEVELS, RES, POSES = 2048, 3, 0.05, 16


def session_scans(seed):
    """POSES points of a closed loop (radius 1.5-3 m) in the world of `seed`: hints, ranges and the same scans as clouds."""
    from hector_slam_b200 import synth

    rng = np.random.default_rng(seed)
    world = synth.World(1, seed=seed)
    cx, cy, r = rng.uniform(-2, 2), rng.uniform(-1.5, 1.5), rng.uniform(1.5, 3.0)
    ph = rng.uniform(0, 2 * np.pi)
    out = []
    for k in range(POSES):
        a = ph + 2 * np.pi * k / POSES
        p = np.array([cx + r * np.cos(a), cy + r * np.sin(a), a + np.pi / 2], np.float32)
        p[2] = np.float32((p[2] + np.pi) % (2 * np.pi) - np.pi)
        ranges = (world.cast(p) + rng.normal(0.0, 0.01, synth.N_BEAMS)).astype(np.float32)
        cloud = np.ascontiguousarray(synth.ranges_to_cloud(ranges), np.float32)
        hint = (p + rng.uniform(-1, 1, 3).astype(np.float32) * np.array([0.03, 0.03, 0.01], np.float32)).astype(np.float32)
        out.append((hint, ranges, cloud))
    return out


def pct(v, q):
    return float(np.percentile(np.asarray(v) * 1e3, q))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,16,128")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--ticks", type=int, default=50)
    args = ap.parse_args()
    from hector_slam_b200 import capi, synth

    sizes = [int(x) for x in args.sizes.split(",")]
    Mmax = max(sizes)
    lib = capi.load_library()
    reps = []
    for s in range(Mmax):
        rep = capi.MapRepB200(RES, SIZE, levels=LEVELS, update_factor_free=0.4, update_factor_occupied=0.9)
        rep.setMapUpdateMinDistDiff(0.4)
        rep.setMapUpdateMinAngleDiff(0.13)
        rep.set_scan_format(**synth.SCAN_FORMAT)
        rep.set_cloud_format(synth.laser_transform(xyz=(0.0, 0.0, 0.3), rpy=(0.0, 0.0, 0.0)), **synth.CLOUD_FORMAT)
        reps.append(rep)
    data = [session_scans(900 + s) for s in range(Mmax)]
    nb = synth.N_BEAMS
    pose = np.zeros((Mmax, 3), np.float32)
    cov = np.zeros((Mmax, 9), np.float32)
    upd = np.zeros(Mmax, np.int32)
    kept = np.zeros(Mmax, np.int32)
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip()
    except OSError:
        card = "unknown"

    def check(st, s=0):
        if st != 0:
            raise capi.HsbError(st, lib.hsb_last_error(reps[s].h).decode())

    for M in sizes:
        group = capi.SlamGroup(reps[:M])
        packed = []   # the group calls' host buffers, one set per trajectory point
        for k in range(POSES):
            hints = np.ascontiguousarray(np.stack([data[s][k][0] for s in range(M)]), np.float32)
            ranges = np.ascontiguousarray(np.concatenate([data[s][k][1] for s in range(M)]), np.float32)
            r_offs = np.arange(M + 1, dtype=np.int32) * nb
            clouds = [data[s][k][2] for s in range(M)]
            c_offs = np.zeros(M + 1, np.int32)
            c_offs[1:] = np.cumsum([x.shape[0] for x in clouds])
            packed.append((hints, ranges, r_offs, np.ascontiguousarray(np.concatenate(clouds), np.float32), c_offs))

        def group_ranges_tick(k):
            hints, ranges, r_offs, _, _ = packed[k % POSES]
            check(lib.hsb_group_slam_update_ranges(group.g, hints.ctypes.data, ranges.ctypes.data, r_offs.ctypes.data, None,
                                                   1, pose.ctypes.data, cov.ctypes.data, upd.ctypes.data,
                                                   kept.ctypes.data))

        def group_cloud_tick(k):
            hints, _, _, pts, c_offs = packed[k % POSES]
            check(lib.hsb_group_slam_update_cloud(group.g, hints.ctypes.data, pts.ctypes.data, c_offs.ctypes.data, None,
                                                  None, 1, pose.ctypes.data, cov.ctypes.data, upd.ctypes.data,
                                                  kept.ctypes.data))

        def serial_tick(k):
            for s in range(M):
                hint, ranges, _ = data[s][k % POSES]
                check(lib.hsb_slam_update_ranges(reps[s].h, hint.ctypes.data, ranges.ctypes.data, nb, 0, 1,
                                                 pose[s].ctypes.data, cov[s].ctypes.data, upd[s:].ctypes.data,
                                                 kept[s:].ctypes.data), s)

        arms = {"group_ranges": group_ranges_tick, "group_cloud": group_cloud_tick, "serial_ranges": serial_tick}
        times = {a: [] for a in arms}
        k = 0
        for _ in range(args.rounds):
            for name, fn in arms.items():
                for i in range(5 + args.ticks):
                    t0 = time.perf_counter()
                    fn(k)
                    t1 = time.perf_counter()
                    k += 1
                    if i >= 5:
                        times[name].append(t1 - t0)
                for r in reps[:M]:
                    r.onMapUpdated()   # the arm's last map writes are done before the next arm starts
        group.close()
        out = {"part": "group", "M": M, "map": f"{SIZE}^2 x {LEVELS} levels", "beams": nb,
               "ticks_per_arm": args.ticks * args.rounds,
               "h2d_scan_bytes_per_tick_ranges": int(sum(4 * nb for _ in range(M))),
               "h2d_scan_bytes_per_tick_cloud": int(np.mean([12 * int(packed[k][4][-1]) for k in range(POSES)])),
               "card": card}
        for name, v in times.items():
            out[f"{name}_ms_p50"] = round(pct(v, 50), 3)
            out[f"{name}_ms_p99"] = round(pct(v, 99), 3)
        print(json.dumps(out), flush=True)

    # single session: the fused step against the two calls it replaces
    rep = reps[0]
    pts = np.zeros((nb, 2), np.float32)
    n_out = C.c_int(0)
    zero2 = np.zeros(2, np.float32)

    def fused(k, nowait):
        hint, ranges, _ = data[0][k % POSES]
        check(lib.hsb_slam_update_ranges(rep.h, hint.ctypes.data, ranges.ctypes.data, nb, 0, int(nowait),
                                         pose.ctypes.data, cov.ctypes.data, upd.ctypes.data, kept.ctypes.data))

    def two_call(k, nowait):
        hint, ranges, _ = data[0][k % POSES]
        check(lib.hsb_scan_to_points(rep.h, ranges.ctypes.data, pts.ctypes.data, C.byref(n_out)))
        fn = lib.hsb_slam_update_nowait if nowait else lib.hsb_slam_update
        check(fn(rep.h, hint.ctypes.data, pts.ctypes.data, n_out.value, zero2.ctypes.data, 0, pose.ctypes.data,
                 cov.ctypes.data, upd.ctypes.data))

    arms = {"fused": fused, "two_call": two_call}
    step = {a: [] for a in arms}
    latency = {a: [] for a in arms}
    k = 0
    for _ in range(args.rounds):
        for name, fn in arms.items():
            for i in range(5 + args.ticks):
                t0 = time.perf_counter()
                fn(k, False)
                t1 = time.perf_counter()
                k += 1
                if i >= 5:
                    step[name].append(t1 - t0)
            for i in range(5 + args.ticks):
                rep.onMapUpdated()
                t0 = time.perf_counter()
                fn(k, True)
                t1 = time.perf_counter()
                k += 1
                if i >= 5:
                    latency[name].append(t1 - t0)
            rep.onMapUpdated()
    out = {"part": "single", "map": f"{SIZE}^2 x {LEVELS} levels", "beams": nb, "ticks_per_arm": args.ticks * args.rounds,
           "h2d_scan_bytes_fused": 4 * nb, "h2d_scan_bytes_two_call": 4 * nb + 8 * int(np.median(
               [rep.scan_to_points(data[0][j][1]).shape[0] for j in range(POSES)])), "card": card}
    for name in arms:
        out[f"{name}_step_ms_p50"] = round(pct(step[name], 50), 3)
        out[f"{name}_pose_latency_ms_p50"] = round(pct(latency[name], 50), 3)
    print(json.dumps(out), flush=True)
    for r in reps:
        r.close()


if __name__ == "__main__":
    main()
