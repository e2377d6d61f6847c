"""What the projected steps buy a default-configured robot (or a server of such robots) that receives raw LaserScans and
has the node project them with laser_geometry before the cloud conversion (HectorMappingRos.cpp:258-297).

Workload: M independent sessions, each its own handle with a 3-level 2048^2 map and its own laser mount, driving
synthetic 1081-beam scans along its own closed trajectory through its own seeded world.

Per M in --sizes, arms alternated within each round on the same handles:
  group_projected  one hsb_group_slam_update_projected(nowait = 1): projection, conversion, match, gate and map write
                   for all M from the ranges
  group_cloud      the host projects every robot's scan (laser_geometry's arithmetic in numpy, the unit vectors
                   precomputed), then one hsb_group_slam_update_cloud(nowait = 1); the host projection is timed on its
                   own (host_projection_ms) and the step without it (group_cloud_ms)
  serial_projected hsb_slam_update_projected(nowait = 1) on the M handles one after another from one thread
Per arm and round: 5 untimed ticks, then `--ticks` timed ones (host clock around the tick; every arm's last map writes
are waited for before the next arm starts).  p50 / p99 over all timed ticks of all rounds.

Host-to-device scan bytes per tick are computed, not timed: 4 B per beam for ranges and 12 B per projected point for a
cloud (the calls' small headers and per-session descriptors are left out).  Prints one JSON line per M, with the card
and power limit read in the same run.

    python scripts/group_step_projected.py [--sizes 1,16,128] [--rounds 3] [--ticks 50]
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZE, LEVELS, RES, POSES, CUTOFF = 2048, 3, 0.05, 16, 30.0


def unit_vectors(fmt):
    a0, da = float(np.float32(fmt["angle_min"])), float(np.float32(fmt["angle_increment"]))
    a = [a0 + i * da for i in range(fmt["n_beams"])]
    return np.array([math.cos(x) for x in a]), np.array([math.sin(x) for x in a])


def host_project(ranges, unit, range_min):
    """laser_geometry's projectLaser_ (PointCloud output) with the precomputed unit vectors."""
    with np.errstate(invalid="ignore"):
        keep = (ranges.astype(np.float64) < CUTOFF) & (ranges >= np.float32(range_min))
    r = ranges[keep].astype(np.float64)
    pts = np.zeros((r.size, 3), np.float32)
    pts[:, 0] = (r * unit[0][keep]).astype(np.float32)
    pts[:, 1] = (r * unit[1][keep]).astype(np.float32)
    return pts


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
    ap.add_argument("--sizes", default="1,16,128")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--ticks", type=int, default=50)
    args = ap.parse_args()
    from hector_slam_b200 import capi, synth

    sizes = [int(x) for x in args.sizes.split(",")]
    Mmax = max(sizes)
    lib = capi.load_library()
    fmt = synth.SCAN_FORMAT
    unit = unit_vectors(fmt)
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
    nb = fmt["n_beams"]
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
        packed = []
        for k in range(POSES):
            hints = np.ascontiguousarray(np.stack([data[s][k][0] for s in range(M)]), np.float32)
            ranges = np.ascontiguousarray(np.concatenate([data[s][k][1] for s in range(M)]), np.float32)
            packed.append((hints, ranges))
        r_offs = np.arange(M + 1, dtype=np.int32) * nb
        c_offs = np.zeros(M + 1, np.int32)
        proj_s, cloud_bytes = [], []

        def group_projected_tick(k):
            hints, ranges = packed[k % POSES]
            check(lib.hsb_group_slam_update_projected(group.g, hints.ctypes.data, ranges.ctypes.data, r_offs.ctypes.data,
                                                      None, None, 1, pose.ctypes.data, cov.ctypes.data, upd.ctypes.data,
                                                      kept.ctypes.data))

        def group_cloud_tick(k):
            hints, _ = packed[k % POSES]
            t0 = time.perf_counter()
            clouds = [host_project(data[s][k % POSES][1], unit, fmt["range_min"]) for s in range(M)]
            c_offs[1:] = np.cumsum([c.shape[0] for c in clouds])
            pts = np.ascontiguousarray(np.concatenate(clouds), np.float32)
            proj_s.append(time.perf_counter() - t0)
            cloud_bytes.append(12 * int(c_offs[-1]))
            t1 = time.perf_counter()
            check(lib.hsb_group_slam_update_cloud(group.g, hints.ctypes.data, pts.ctypes.data, c_offs.ctypes.data, None,
                                                  None, 1, pose.ctypes.data, cov.ctypes.data, upd.ctypes.data,
                                                  kept.ctypes.data))
            return time.perf_counter() - t1

        def serial_tick(k):
            for s in range(M):
                hint, ranges = data[s][k % POSES]
                check(lib.hsb_slam_update_projected(reps[s].h, hint.ctypes.data, ranges.ctypes.data, nb, None, 0, 1,
                                                    pose[s].ctypes.data, cov[s].ctypes.data, upd[s:].ctypes.data,
                                                    kept[s:].ctypes.data), s)

        arms = {"group_projected": group_projected_tick, "group_cloud": group_cloud_tick,
                "serial_projected": serial_tick}
        times = {a: [] for a in arms}
        k = 0
        for _ in range(args.rounds):
            for name, fn in arms.items():
                n_proj = len(proj_s)
                for i in range(5 + args.ticks):
                    t0 = time.perf_counter()
                    dt = fn(k)
                    t1 = time.perf_counter()
                    k += 1
                    if i >= 5:
                        times[name].append(dt if dt is not None else t1 - t0)
                if name == "group_cloud":
                    del proj_s[n_proj:n_proj + 5]   # the untimed ticks
                for r in reps[:M]:
                    r.onMapUpdated()
        group.close()
        out = {"M": M, "map": f"{SIZE}^2 x {LEVELS} levels", "beams": nb, "ticks_per_arm": args.ticks * args.rounds,
               "h2d_scan_bytes_per_tick_ranges": 4 * nb * M,
               "h2d_scan_bytes_per_tick_cloud": int(np.mean(cloud_bytes)), "card": card}
        for name, v in times.items():
            out[f"{name}_ms_p50"] = round(pct(v, 50), 3)
            out[f"{name}_ms_p99"] = round(pct(v, 99), 3)
        out["host_projection_ms_p50"] = round(pct(proj_s, 50), 3)
        out["host_projection_ms_p99"] = round(pct(proj_s, 99), 3)
        print(json.dumps(out), flush=True)
    for r in reps:
        r.close()


if __name__ == "__main__":
    main()
