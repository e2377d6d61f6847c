"""What one mixed group buys a server whose robots' maps differ in size, resolution and start.

Workload: M robots (--sizes), spread round-robin over three 3-level map geometries
  wide     2048 x 2048 at 0.05 m, centred start
  offset   1024 x 1536 at 0.05 m, start (0.3, 0.4)
  fine     1536 x 1536 at 0.025 m, centred start
each stepping synthetic 1081-beam LaserScans from raw ranges (hsb_group_slam_update_ranges, nowait = 0) along its own
closed loop (scripts/group_step_subset.py's trajectories).  Three twin fleets get the same scans, one per arm:
  mixed    one hsb_group_create_mixed group of all M robots: one step call per tick
  uniform  one hsb_group_create group per geometry: one step call per geometry with a robot in the tick
  single   hsb_slam_update_ranges for each robot of the tick, one after another
Two phases per M: `full` steps every robot every tick (the full form; uniform: the three full-form calls), `subset` steps
a seeded random ~M/5 of the robots per tick (the _subset forms).  Per phase, 3 untimed ticks, then --ticks timed ticks;
within every tick the arms run one after another in a rotating order.  Reported per arm: ms per tick (host clock
around the arm's calls of the tick, which return after the map writes: p50 / p90), kernel launches per tick (summed
over the arm's handles: hsb_get_launch_count) and step calls per tick; each step call is one host-to-device copy (the
header's contract for every step form), so that is also the host-to-device copies per tick.  Every tick's poses are
compared bit for bit across the arms, and at the end every level's log-odds plane of every robot.

Prints one JSON line per (M, phase) and a final one with the plane comparison, with the card's name and power limit
read in the same run.  Needs a GPU; there is no fall-back.

    python scripts/group_mixed.py [--sizes 16,128] [--ticks 40]
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

from group_step_subset import POSES, session_scans  # noqa: E402

LEVELS = 3
GEOMS = {"wide": (2048, 2048, 0.05, (0.5, 0.5)), "offset": (1024, 1536, 0.05, (0.3, 0.4)),
         "fine": (1536, 1536, 0.025, (0.5, 0.5))}
NAMES = list(GEOMS)
ARMS = ("mixed", "uniform", "single")


def pct(v, q):
    return float(np.percentile(np.asarray(v) * 1e3, q))


def make_rep(s):
    from hector_slam_b200 import capi, synth

    sx, sy, res, start = GEOMS[NAMES[s % 3]]
    rep = capi.MapRepB200(res, sx, sy, levels=LEVELS, start=start, update_factor_free=0.4, update_factor_occupied=0.9)
    rep.setMapUpdateMinDistDiff(0.4)
    rep.setMapUpdateMinAngleDiff(0.13)
    rep.set_scan_format(**synth.SCAN_FORMAT)
    return rep


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="16,128")
    ap.add_argument("--ticks", type=int, default=40)
    args = ap.parse_args()
    from hector_slam_b200 import capi

    sizes = [int(x) for x in args.sizes.split(",")]
    Mmax = max(sizes)
    fleets = {a: [make_rep(s) for s in range(Mmax)] for a in ARMS}
    data = [session_scans(900 + s) for s in range(Mmax)]
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip()
    except OSError:
        card = "unknown"
    equal_poses = True

    for M in sizes:
        mixed = capi.SlamGroup(fleets["mixed"][:M], mixed=True)
        by_geom = [[j for j in range(M) if j % 3 == g] for g in range(3)]   # each geometry's robots, in order
        uniform = [capi.SlamGroup([fleets["uniform"][j] for j in js]) if js else None for js in by_geom]
        scan_no = np.zeros(M, np.int64)   # each robot's next scan: its loop advances when it is stepped

        def run(arm, members, hints, ranges):
            """one tick of `arm` over `members` (None: every robot) -> (poses in member order, step calls)"""
            sel = list(range(M)) if members is None else members
            if arm == "mixed":
                return mixed.slam_update_ranges(hints, ranges, members=members)[0], 1
            if arm == "single":
                reps = fleets["single"]
                return np.stack([reps[j].slam_update_ranges(hints[k], ranges[k])[0] for k, j in enumerate(sel)]), len(sel)
            out, calls = np.zeros((len(sel), 3), np.float32), 0
            for g, js in enumerate(by_geom):
                ks = [k for k, j in enumerate(sel) if j % 3 == g]
                if not ks:
                    continue
                local = None if members is None else [js.index(sel[k]) for k in ks]
                out[ks] = uniform[g].slam_update_ranges(hints[ks], [ranges[k] for k in ks], members=local)[0]
                calls += 1
            return out, calls

        for phase in ("full", "subset"):
            rng = np.random.default_rng(7 + M)
            times = {a: [] for a in ARMS}
            launches = {a: 0 for a in ARMS}
            calls = {a: 0 for a in ARMS}
            for t in range(3 + args.ticks):
                if phase == "full":
                    members, sel = None, list(range(M))
                else:
                    sel = [int(j) for j in rng.permutation(M)[:max(1, M // 5)]]
                    members = sel
                ks = [int(scan_no[j] % POSES) for j in sel]
                scan_no[sel] += 1
                hints = np.ascontiguousarray(np.stack([data[j][k][0] for j, k in zip(sel, ks)]), np.float32)
                ranges = [data[j][k][1] for j, k in zip(sel, ks)]
                poses = {}
                for i in range(len(ARMS)):
                    arm = ARMS[(t + i) % len(ARMS)]
                    before = sum(r.launch_count for r in fleets[arm][:M])
                    t0 = time.perf_counter()
                    poses[arm], n = run(arm, members, hints, ranges)
                    dt = time.perf_counter() - t0
                    if t >= 3:
                        times[arm].append(dt)
                        launches[arm] += sum(r.launch_count for r in fleets[arm][:M]) - before
                        calls[arm] += n
                ref = poses["single"].view(np.uint32)
                equal_poses &= all(np.array_equal(poses[a].view(np.uint32), ref) for a in ("mixed", "uniform"))
            rec = {"M": M, "phase": phase, "robots_per_tick": len(sel), "ticks": args.ticks,
                   "geometries": {n: GEOMS[n][:3] for n in NAMES}, "card": card}
            for a in ARMS:
                rec[a] = {"p50_ms": round(pct(times[a], 50), 3), "p90_ms": round(pct(times[a], 90), 3),
                          "launches_per_tick": launches[a] / args.ticks, "step_calls_per_tick": calls[a] / args.ticks,
                          "h2d_copies_per_tick": calls[a] / args.ticks}
            rec["poses_equal_across_arms"] = bool(equal_poses)
            print(json.dumps(rec), flush=True)
        for g in uniform:
            if g is not None:
                g.close()
        mixed.close()

    planes_equal = True
    for s in range(Mmax):
        for l in range(LEVELS):
            ref = fleets["single"][s].download_level(l).view(np.uint32)
            planes_equal &= all(np.array_equal(fleets[a][s].download_level(l).view(np.uint32), ref)
                                for a in ("mixed", "uniform"))
    print(json.dumps({"planes_equal_across_arms": bool(planes_equal), "poses_equal_across_arms": bool(equal_poses),
                      "robots": Mmax, "card": card}), flush=True)
    for a in ARMS:
        for r in fleets[a]:
            r.close()
    if not (planes_equal and equal_poses):
        sys.exit(1)


if __name__ == "__main__":
    main()
