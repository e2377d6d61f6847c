"""What stepping M SLAM sessions together buys when they are fed the node's default input (projected point clouds).

Workload: M independent sessions (M in {1, 8, 32, 128}), each its own handle with a 3-level 2048^2 map and its own
laser transform, each driving synthetic 1081-beam clouds (synth.ranges_to_cloud) along its own closed trajectory through
its own seeded world.  One tick steps every session once.  Arms, alternated within each round on the same handles:
  group_cloud  one hsb_group_slam_update_cloud(nowait = 1): conversion, match, gate and map write for all M
  serial       hsb_slam_update_cloud(nowait = 1) on the M handles one after another from one thread
  two_call     M x hsb_cloud_to_points (a host round trip each), then one hsb_group_slam_update(nowait = 1)
Per arm and round: 5 untimed ticks, then `--ticks` timed ones (host clock around the tick; every arm's last map writes
are waited for before the next arm starts).  Prints one JSON line per M with p50 / p99 over all timed ticks of all
rounds, and the card and power limit it ran on.

    python scripts/group_step_cloud.py [--sizes 1,8,32,128] [--rounds 3] [--ticks 50]
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


def session_clouds(seed):
    """POSES points of a closed loop (radius 1.5-3 m) in the world of `seed`, their clouds and hints."""
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
        cloud = np.ascontiguousarray(synth.ranges_to_cloud(world.cast(p) + rng.normal(0.0, 0.01, 1081)), np.float32)
        hint = (p + rng.uniform(-1, 1, 3).astype(np.float32) * np.array([0.03, 0.03, 0.01], np.float32)).astype(np.float32)
        out.append((hint, cloud))
    return out


def pct(v, q):
    return float(np.percentile(np.asarray(v) * 1e3, q))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,8,32,128")
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
        T = synth.laser_transform(xyz=(0.1 + 0.01 * (s % 5), -0.02 * (s % 3), 0.3), rpy=(0.0, -0.01 * (s % 4), 0.02 * (s % 7)))
        rep.set_cloud_format(T, **synth.CLOUD_FORMAT)
        reps.append(rep)
    data = [session_clouds(700 + s) for s in range(Mmax)]
    pose = np.zeros((Mmax, 3), np.float32)
    cov = np.zeros((Mmax, 9), np.float32)
    upd = np.zeros(Mmax, np.int32)
    kept = np.zeros(Mmax, np.int32)
    origo = np.zeros((Mmax, 2), np.float32)
    max_pts = max(c.shape[0] for d in data for _, c in d)
    endpoints = np.zeros((Mmax * max_pts, 2), np.float32)   # the two-call route's converted scans, packed
    ep_offs = np.zeros(Mmax + 1, np.int32)
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
        # the group calls' host buffers, one set per trajectory point
        packed = []
        for k in range(POSES):
            hints = np.ascontiguousarray(np.stack([data[s][k][0] for s in range(M)]), np.float32)
            clouds = [data[s][k][1] for s in range(M)]
            offs = np.zeros(M + 1, np.int32)
            offs[1:] = np.cumsum([x.shape[0] for x in clouds])
            packed.append((hints, np.ascontiguousarray(np.concatenate(clouds), np.float32), offs))

        def group_cloud_tick(k):
            hints, pts, offs = packed[k % POSES]
            check(lib.hsb_group_slam_update_cloud(group.g, hints.ctypes.data, pts.ctypes.data, offs.ctypes.data, None, None,
                                                  1, pose.ctypes.data, cov.ctypes.data, upd.ctypes.data, kept.ctypes.data))

        def serial_tick(k):
            for s in range(M):
                hint, cloud = data[s][k % POSES]
                check(lib.hsb_slam_update_cloud(reps[s].h, hint.ctypes.data, cloud.ctypes.data, cloud.shape[0], None, 0, 1,
                                                pose[s].ctypes.data, cov[s].ctypes.data, upd[s:].ctypes.data,
                                                kept[s:].ctypes.data), s)

        n_out = C.c_int(0)

        def two_call_tick(k):
            hints = packed[k % POSES][0]
            for s in range(M):
                cloud = data[s][k % POSES][1]
                check(lib.hsb_cloud_to_points(reps[s].h, cloud.ctypes.data, cloud.shape[0],
                                              endpoints.ctypes.data + 8 * int(ep_offs[s]), C.byref(n_out),
                                              origo[s].ctypes.data), s)
                ep_offs[s + 1] = ep_offs[s] + n_out.value
            check(lib.hsb_group_slam_update(group.g, hints.ctypes.data, endpoints.ctypes.data, ep_offs.ctypes.data,
                                            origo.ctypes.data, None, 1, pose.ctypes.data, cov.ctypes.data, upd.ctypes.data))

        arms = {"group_cloud": group_cloud_tick, "serial": serial_tick, "two_call": two_call_tick}
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
        out = {"M": M, "map": f"{SIZE}^2 x {LEVELS} levels", "cloud_points": int(data[0][0][1].shape[0]),
               "ticks_per_arm": args.ticks * args.rounds, "card": card}
        for name, v in times.items():
            out[f"{name}_ms_p50"] = round(pct(v, 50), 3)
            out[f"{name}_ms_p99"] = round(pct(v, 99), 3)
        print(json.dumps(out), flush=True)
    for r in reps:
        r.close()


if __name__ == "__main__":
    main()
