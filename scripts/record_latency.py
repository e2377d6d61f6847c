"""What the per-evaluation record costs one matchData call: hsb_match_data without and with the record
(hsb_match_data_record), in alternating rounds on the same map and scans.

Workload: BASELINE config 3's size — a 3-level 4096^2 map built by mapping with known poses, 64 seeded 1081-point
scans, hints perturbed by 5 cm / 0.02 rad.  Per round the median of 100 calls (after 20 untimed ones) through the ctypes
wrapper; prints one JSON line with the rounds of both arms and the card it ran on.

    python scripts/record_latency.py [--rounds 8] [--calls 120]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--calls", type=int, default=120)
    args = ap.parse_args()
    from hector_slam_b200 import capi, synth

    size, levels, res = 4096, 3, 0.05
    rep = capi.MapRepB200(res, size, levels=levels, update_factor_free=0.4, update_factor_occupied=0.9)
    world = synth.World.for_map_size(size)
    rng = np.random.default_rng(11)
    for p in world.mapping_poses():
        scan = synth.make_scan(world, p, rng)
        p32 = p.astype(np.float32)
        rep.matchData(p32, scan)
        rep.updateByScan(scan, p32)
        rep.onMapUpdated()
    rng = np.random.default_rng(31)
    poses = world.sample_free_poses(64, rng)
    scans = [np.ascontiguousarray(synth.make_scan(world, p, rng)) for p in poses]
    hints = synth.perturb_hints(poses, seed=32, dxy=0.05, dpsi=0.02)
    rounds = {False: [], True: []}
    for _ in range(args.rounds):
        for record in (False, True):
            lat = []
            for i in range(args.calls):
                k = i % len(scans)
                t0 = time.perf_counter()
                rep.matchData(hints[k], scans[k], record=record)
                t1 = time.perf_counter()
                if i >= 20:
                    lat.append(t1 - t0)
            rounds[record].append(float(np.median(lat) * 1e6))
    rep.close()
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip()
    except OSError:
        card = "unknown"
    print(json.dumps({"match_data_us_p50_rounds": rounds[False], "match_data_record_us_p50_rounds": rounds[True],
                      "card": card}))


if __name__ == "__main__":
    main()
