"""What publishing a fleet's occupancy grids in one pass buys a server of robots.

Workload: M robots (--sizes), each a handle with a 3-level 2048^2 map, stepped as in scripts/group_step_subset.py: 40 Hz
lidars with seeded random phases, a tick every --window-ms (5 ms) steps the robots whose scan falls into it with one
hsb_group_slam_update_projected_subset(nowait = 1).  Every 80 ticks (2 s of lidar time, the node's map_pub_period) one
publish round brings every robot's level-0 grid up to date, as publishMapLoop does (HectorMappingRos.cpp:577-595).

Three twin fleets get the same scans, one per arm:
  group     hsb_group_sync_occupancy over all M members (one pass)
  loop      per member hsb_get_mirror_dirty_rect(reset = 1) + hsb_download_occupancy_rect + the rows copied into the
            grid (the per-member C-ABI path, driven from Python through ctypes)
  full      per member the façade's getGridMap (hsb_download_level, the whole log-odds plane) + a numpy threshold
Each fleet is stepped every tick; the three arms publish in rotating order in each round (--rounds 3, --publishes per
round).  Reported per arm: publish-round time p50 / p99 (host clock around the round, which ends in a synchronise),
bytes copied to the host per round (hsb_get_d2h_bytes) and the time of the first tick after a round next to the median
tick of that fleet.  After every round the three arms' grids are compared byte for byte.  Prints one JSON line per M,
with the card and power limit read in the same run.

    python scripts/group_occupancy.py [--sizes 16,128] [--rounds 3] [--publishes 4]
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
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from group_step_subset import CUTOFF, LEVELS, PERIOD_MS, POSES, RES, SIZE, session_scans  # noqa: E402

TICKS_PER_PUBLISH = 80   # 2 s of 40 Hz lidar time at the default map_pub_period


def pct(v, q):
    return float(np.percentile(np.asarray(v) * 1e3, q))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="16,128")
    ap.add_argument("--window-ms", type=float, default=5.0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--publishes", type=int, default=4)
    args = ap.parse_args()
    from hector_slam_b200 import capi, synth

    sizes = [int(x) for x in args.sizes.split(",")]
    Mmax = max(sizes)
    lib = capi.load_library()
    fmt = synth.SCAN_FORMAT
    nb = fmt["n_beams"]
    arms = ("group", "loop", "full")

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

    for M in sizes:
        groups = {a: capi.SlamGroup(fleets[a][:M]) for a in arms}
        sx, sy, _ = fleets["group"][0].level_info(0)
        grids = {a: [np.full((sy, sx), -1, np.int8) for _ in range(M)] for a in arms}
        for a in arms:   # a grid that starts at -1 is a fresh map's: forget what earlier sizes wrote
            for rep, g in zip(fleets[a][:M], grids[a]):
                g[...] = rep.download_occupancy(0)
                rep.get_mirror_dirty_rect(0, reset=True)
        grid_ptrs = (C.c_void_p * M)(*[g.ctypes.data for g in grids["group"]])
        rects = np.zeros((M, 4), np.int32)
        rect1 = (C.c_int * 4)()
        packed = np.zeros(sx * sy, np.int8)
        plane = np.zeros((sy, sx), np.float32)
        scan_no = np.zeros(M, np.int64)

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

        def step(a, w):
            members, hints, ranges, offs = w
            check(lib.hsb_group_slam_update_projected_subset(groups[a].g, len(members), members.ctypes.data,
                                                             hints.ctypes.data, ranges.ctypes.data, offs.ctypes.data,
                                                             None, None, 1, pose.ctypes.data, cov.ctypes.data,
                                                             upd.ctypes.data, kept.ctypes.data), fleets[a][0])

        def publish_group():
            check(lib.hsb_group_sync_occupancy(groups["group"].g, 0, C.cast(grid_ptrs, C.c_void_p), rects.ctypes.data, 1),
                  fleets["group"][0])

        def publish_loop():
            for rep, g in zip(fleets["loop"][:M], grids["loop"]):
                check(lib.hsb_get_mirror_dirty_rect(rep.h, 0, rect1, 1), rep)
                x0, y0, x1, y1 = rect1
                if x1 < x0:
                    continue
                w, h = x1 - x0 + 1, y1 - y0 + 1
                check(lib.hsb_download_occupancy_rect(rep.h, 0, rect1, packed.ctypes.data), rep)
                g[y0:y1 + 1, x0:x1 + 1] = packed[:w * h].reshape(h, w)

        def publish_full():
            for rep, g in zip(fleets["full"][:M], grids["full"]):
                check(lib.hsb_download_level(rep.h, 0, plane.ctypes.data), rep)
                g[...] = -1
                g[plane < 0] = 0
                g[plane > 0] = 100

        publish = {"group": publish_group, "loop": publish_loop, "full": publish_full}
        round_s = {a: [] for a in arms}
        bytes_round = {a: [] for a in arms}
        first_tick = {a: [] for a in arms}
        ticks = {a: [] for a in arms}
        t, n_pub = 0, 0
        for rnd in range(args.rounds):
            for p in range(args.publishes):
                after = n_pub > 0
                for i in range(TICKS_PER_PUBLISH):
                    w = window(t)
                    t += 1
                    if len(w[0]) == 0:
                        continue
                    for a in arms:
                        t0 = time.perf_counter()
                        step(a, w)
                        dt = time.perf_counter() - t0
                        (first_tick[a] if after else ticks[a]).append(dt)
                    after = False
                order = arms[n_pub % 3:] + arms[:n_pub % 3]
                for a in order:
                    d2h = sum(r.d2h_bytes for r in fleets[a][:M])
                    t0 = time.perf_counter()
                    publish[a]()
                    round_s[a].append(time.perf_counter() - t0)
                    bytes_round[a].append(sum(r.d2h_bytes for r in fleets[a][:M]) - d2h)
                n_pub += 1
                for j in range(M):
                    g = grids["group"][j]
                    assert np.array_equal(g, grids["loop"][j]) and np.array_equal(g, grids["full"][j]), (M, n_pub, j)
        for a in arms:
            groups[a].close()
            for r in fleets[a][:M]:
                r.onMapUpdated()
        out = {"M": M, "map": f"{SIZE}^2 x {LEVELS} levels, level 0 published", "ticks_per_publish": TICKS_PER_PUBLISH,
               "publish_rounds_per_arm": n_pub, "grids_identical": True, "card": card}
        for a in arms:
            out[f"{a}_round_ms_p50"] = round(pct(round_s[a], 50), 3)
            out[f"{a}_round_ms_p99"] = round(pct(round_s[a], 99), 3)
            out[f"{a}_bytes_per_round"] = int(np.mean(bytes_round[a]))
            out[f"{a}_first_tick_ms_p50"] = round(pct(first_tick[a], 50), 3)
            out[f"{a}_tick_ms_p50"] = round(pct(ticks[a], 50), 3)
        print(json.dumps(out), flush=True)
    for a in arms:
        for r in fleets[a]:
            r.close()


if __name__ == "__main__":
    main()
