"""What stepping M SLAM sessions together buys: one hsb_group_slam_update per tick against M single steps.

Workload: M independent sessions (M in {1, 8, 32, 128}), each its own handle with a 3-level 2048^2 map (88 MB), each
driving synthetic 1081-point scans along its own closed trajectory through its own seeded world.  One tick steps every
session once.  Arms, alternated within each round on the same handles:
  group_wait    one hsb_group_slam_update(nowait = 0): returns when every map write is done
  group_nowait  one hsb_group_slam_update(nowait = 1): returns when every pose has arrived
  serial        hsb_slam_update_nowait on the M handles one after another from one thread
  threads       M host threads, each calling hsb_slam_update_nowait on its handle (a barrier starts and ends the tick)
Per arm and round: 5 untimed ticks, then `--ticks` timed ones (host clock around the tick; every nowait arm's last map
writes are waited for before the next arm starts).  Prints one JSON line per M with p50 / p99 over all timed ticks of
all rounds, and the card it ran on.

    python scripts/group_step.py [--sizes 1,8,32,128] [--rounds 3] [--ticks 50]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZE, LEVELS, RES, POSES = 2048, 3, 0.05, 16


def session_scans(seed):
    """POSES points of a closed loop (radius 1.5-3 m) in the world of `seed`, their scans and hints."""
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
        scan = np.ascontiguousarray(synth.make_scan(world, p, rng, scale_to_map=1.0 / RES), np.float32)
        hint = (p + rng.uniform(-1, 1, 3).astype(np.float32) * np.array([0.03, 0.03, 0.01], np.float32)).astype(np.float32)
        out.append((hint, scan))
    return out


def pct(v, q):
    return float(np.percentile(np.asarray(v) * 1e3, q))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,8,32,128")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--ticks", type=int, default=50)
    args = ap.parse_args()
    from hector_slam_b200 import capi

    sizes = [int(x) for x in args.sizes.split(",")]
    Mmax = max(sizes)
    lib = capi.load_library()
    reps = []
    for s in range(Mmax):
        rep = capi.MapRepB200(RES, SIZE, levels=LEVELS, update_factor_free=0.4, update_factor_occupied=0.9)
        rep.setMapUpdateMinDistDiff(0.4)
        rep.setMapUpdateMinAngleDiff(0.13)
        reps.append(rep)
    data = [session_scans(500 + s) for s in range(Mmax)]
    pose = np.zeros((Mmax, 3), np.float32)
    cov = np.zeros((Mmax, 9), np.float32)
    upd = np.zeros(Mmax, np.int32)
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip()
    except OSError:
        card = "unknown"

    def single(s, k):
        hint, scan = data[s][k % POSES]
        st = lib.hsb_slam_update_nowait(reps[s].h, hint.ctypes.data, scan.ctypes.data, scan.shape[0], None, 0,
                                        pose[s].ctypes.data, cov[s].ctypes.data, upd[s:].ctypes.data)
        if st != 0:
            raise capi.HsbError(st, lib.hsb_last_error(reps[s].h).decode())

    for M in sizes:
        group = capi.SlamGroup(reps[:M])
        # the group call's host buffers, one set per trajectory point
        packed = []
        for k in range(POSES):
            hints = np.ascontiguousarray(np.stack([data[s][k][0] for s in range(M)]), np.float32)
            scans = [data[s][k][1] for s in range(M)]
            offs = np.zeros(M + 1, np.int32)
            offs[1:] = np.cumsum([x.shape[0] for x in scans])
            packed.append((hints, np.ascontiguousarray(np.concatenate(scans), np.float32), offs))

        def group_tick(k, nowait):
            hints, pts, offs = packed[k % POSES]
            st = lib.hsb_group_slam_update(group.g, hints.ctypes.data, pts.ctypes.data, offs.ctypes.data, None, None,
                                           nowait, pose.ctypes.data, cov.ctypes.data, upd.ctypes.data)
            if st != 0:
                raise capi.HsbError(st, lib.hsb_last_error(reps[0].h).decode())

        def serial_tick(k):
            for s in range(M):
                single(s, k)

        # M host threads, released together at the start of a tick; the tick ends when the last one has its pose
        start, done = threading.Barrier(M + 1), threading.Barrier(M + 1)
        tick_no = [0]
        stop = [False]

        def worker(s):
            while True:
                start.wait()
                if stop[0]:
                    return
                single(s, tick_no[0])
                done.wait()

        threads = [threading.Thread(target=worker, args=(s,), daemon=True) for s in range(M)]
        for t in threads:
            t.start()

        def thread_tick(k):
            tick_no[0] = k
            start.wait()
            done.wait()

        arms = {"group_wait": lambda k: group_tick(k, 0), "group_nowait": lambda k: group_tick(k, 1),
                "serial": serial_tick, "threads": thread_tick}
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
        stop[0] = True
        start.wait()
        for t in threads:
            t.join()
        group.close()
        out = {"M": M, "map": f"{SIZE}^2 x {LEVELS} levels", "scan_points": int(data[0][0][1].shape[0]),
               "ticks_per_arm": args.ticks * args.rounds, "card": card}
        for name, v in times.items():
            out[f"{name}_ms_p50"] = round(pct(v, 50), 3)
            out[f"{name}_ms_p99"] = round(pct(v, 99), 3)
        print(json.dumps(out), flush=True)
    for r in reps:
        r.close()


if __name__ == "__main__":
    main()
