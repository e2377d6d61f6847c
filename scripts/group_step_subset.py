"""What the subset group steps buy a server of robots whose lidars do not scan in step.

Workload: M robots (--sizes), each a handle with a 3-level 2048^2 map and its own laser mount, sending synthetic
1081-beam LaserScans on the node's default projected path.  Every robot scans at 40 Hz with a seeded random phase; a
tick collects the robots whose scan falls into a --window-ms window (default 5 ms), i.e. about M * window / 25 ms robots
per tick, and steps them.

Per M, arms alternated within each round on the same handles:
  subset   one hsb_group_slam_update_projected_subset(nowait = 1) per tick on a group of all M handles made once
  rebuild  hsb_group_create over the tick's robots, hsb_group_slam_update_projected(nowait = 1), hsb_group_destroy:
           what a caller that keeps one group per set of stepped robots does on every tick of an unsynchronised fleet
  serial   hsb_slam_update_projected(nowait = 1) for each robot of the tick, one after another from one thread
Per arm and round: 5 untimed ticks, then `--ticks` timed ones (host clock around the tick; every arm's last map writes
are waited for before the next arm starts).  Reported per arm: ms per tick (p50, p99 over all timed ticks of all rounds)
and scans stepped per second (scans of the timed ticks over their summed time).  A tick with no robot costs every arm
nothing and is left out of the timing.  Prints one JSON line per M, with the card and power limit read in the same run.

    python scripts/group_step_subset.py [--sizes 16,128] [--window-ms 5] [--rounds 3] [--ticks 100]
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

SIZE, LEVELS, RES, POSES, CUTOFF, PERIOD_MS = 2048, 3, 0.05, 16, 30.0, 25.0


def session_scans(seed):
    """POSES points of a closed loop (radius 1.5-3 m) in the world of `seed`: hints and ranges."""
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
        hint = (p + rng.uniform(-1, 1, 3).astype(np.float32) * np.array([0.03, 0.03, 0.01], np.float32)).astype(np.float32)
        out.append((hint, ranges))
    return out


def pct(v, q):
    return float(np.percentile(np.asarray(v) * 1e3, q))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="16,128")
    ap.add_argument("--window-ms", type=float, default=5.0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--ticks", type=int, default=100)
    args = ap.parse_args()
    from hector_slam_b200 import capi, synth

    sizes = [int(x) for x in args.sizes.split(",")]
    Mmax = max(sizes)
    lib = capi.load_library()
    fmt = synth.SCAN_FORMAT
    nb = fmt["n_beams"]
    reps = []
    for s in range(Mmax):
        rep = capi.MapRepB200(RES, SIZE, levels=LEVELS, update_factor_free=0.4, update_factor_occupied=0.9)
        rep.setMapUpdateMinDistDiff(0.4)
        rep.setMapUpdateMinAngleDiff(0.13)
        rep.set_laser_projection(**fmt, range_cutoff=CUTOFF)
        mount = synth.laser_transform(xyz=(0.05 + 0.001 * s, -0.02 + 0.0005 * s, 0.3),
                                      rpy=(0.002 * (s % 5), -0.003 * (s % 7), 0.01 * (s % 11)))
        rep.set_cloud_format(mount, **synth.CLOUD_FORMAT)
        reps.append(rep)
    data = [session_scans(900 + s) for s in range(Mmax)]
    phase = np.random.default_rng(40).uniform(0.0, PERIOD_MS, Mmax)   # each lidar's 40 Hz phase
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
        scan_no = np.zeros(M, np.int64)   # each robot's next scan: its trajectory advances when it is stepped

        def window(t):
            """the robots (in phase order) whose scan falls into window t, and their packed inputs"""
            lo = (t * args.window_ms) % PERIOD_MS
            d = (phase[:M] - lo) % PERIOD_MS
            members = np.ascontiguousarray(np.nonzero(d < args.window_ms)[0][np.argsort(d[d < args.window_ms])], np.int32)
            ks = [int(scan_no[j] % POSES) for j in members]
            scan_no[members] += 1
            hints = np.ascontiguousarray(np.stack([data[j][k][0] for j, k in zip(members, ks)]) if len(members)
                                         else np.zeros((0, 3), np.float32), np.float32)
            ranges = np.ascontiguousarray(np.concatenate([data[j][k][1] for j, k in zip(members, ks)]) if len(members)
                                          else np.zeros(0, np.float32), np.float32)
            offs = np.arange(len(members) + 1, dtype=np.int32) * nb
            return members, hints, ranges, offs

        def subset_tick(w):
            members, hints, ranges, offs = w
            check(lib.hsb_group_slam_update_projected_subset(group.g, len(members), members.ctypes.data,
                                                             hints.ctypes.data, ranges.ctypes.data, offs.ctypes.data,
                                                             None, None, 1, pose.ctypes.data, cov.ctypes.data,
                                                             upd.ctypes.data, kept.ctypes.data))

        def rebuild_tick(w):
            members, hints, ranges, offs = w
            hs = (C.c_void_p * len(members))(*[reps[j].h for j in members])
            g = C.c_void_p()
            check(lib.hsb_group_create(C.cast(hs, C.c_void_p), len(members), C.byref(g)))
            try:
                check(lib.hsb_group_slam_update_projected(g, hints.ctypes.data, ranges.ctypes.data, offs.ctypes.data,
                                                          None, None, 1, pose.ctypes.data, cov.ctypes.data,
                                                          upd.ctypes.data, kept.ctypes.data))
            finally:
                lib.hsb_group_destroy(g)

        def serial_tick(w):
            members, hints, ranges, _ = w
            for i, j in enumerate(members):
                check(lib.hsb_slam_update_projected(reps[j].h, hints[i].ctypes.data, ranges[i * nb:].ctypes.data, nb,
                                                    None, 0, 1, pose[i].ctypes.data, cov[i].ctypes.data,
                                                    upd[i:].ctypes.data, kept[i:].ctypes.data), j)

        arms = {"subset": subset_tick, "rebuild": rebuild_tick, "serial": serial_tick}
        times = {a: [] for a in arms}
        scans = {a: 0 for a in arms}
        t = 0
        for _ in range(args.rounds):
            for name, fn in arms.items():
                i = 0
                while i < 5 + args.ticks:
                    w = window(t)
                    t += 1
                    if len(w[0]) == 0:
                        continue
                    t0 = time.perf_counter()
                    fn(w)
                    dt = time.perf_counter() - t0
                    if i >= 5:
                        times[name].append(dt)
                        scans[name] += len(w[0])
                    i += 1
                for r in reps[:M]:
                    r.onMapUpdated()
        group.close()
        out = {"M": M, "map": f"{SIZE}^2 x {LEVELS} levels", "beams": nb, "window_ms": args.window_ms,
               "ticks_per_arm": args.ticks * args.rounds,
               "scans_per_tick_mean": round(scans["subset"] / max(1, len(times["subset"])), 2), "card": card}
        for name, v in times.items():
            out[f"{name}_ms_p50"] = round(pct(v, 50), 3)
            out[f"{name}_ms_p99"] = round(pct(v, 99), 3)
            out[f"{name}_scans_per_s"] = round(scans[name] / sum(v), 1)
        print(json.dumps(out), flush=True)
    for r in reps:
        r.close()


if __name__ == "__main__":
    main()
