"""What the step record (hsb_set_step_record) costs a group step and a single nowait step.

Workload: M robots (--sizes), each the node's default pyramid (3 levels, 1024 x 1024 at 0.05 m, texture gathers),
stepping synthetic 1081-beam LaserScans from raw ranges along its own closed loop (scripts/group_step_subset.py's
trajectories) in one heterogeneous group, one hsb_group_slam_update_ranges call per tick (nowait = 0: the call returns
after the map writes).  Three arms, alternated tick by tick on the same fleet so that they share the machine's state:
  none   no robot records
  one    robot 0 records
  all    every robot records
The switch is a host flag (every robot's record buffer is allocated before the first tick), so changing it between
ticks costs nothing.  Reported per arm: ms per tick (host clock around the step call: p50 / p99) and kernel launches
per tick.  Then a single robot's nowait step (hsb_slam_update_ranges, nowait = 1, which returns once the pose, and the
record, are in host memory) with the switch off and on, alternated step by step.

Prints one JSON line per M and one for the single step, with the card's name and power limit read in the same run.
Needs a GPU; there is no fall-back.

    python scripts/group_step_record.py [--sizes 16,128] [--ticks 300] [--single-steps 600]
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

ARMS = ("none", "one", "all")


def pct(v, q):
    return float(np.percentile(np.asarray(v) * 1e3, q))


def make_rep():
    from hector_slam_b200 import capi, synth

    rep = capi.MapRepB200(0.05, 1024, 1024, levels=3, update_factor_free=0.4, update_factor_occupied=0.9,
                          gather_mode=capi.GATHER_TEX)
    rep.setMapUpdateMinDistDiff(0.4)
    rep.setMapUpdateMinAngleDiff(0.13)
    rep.set_scan_format(**synth.SCAN_FORMAT)
    rep.set_step_record(True)    # allocates the record buffer; the arms set the switch per tick
    rep.set_step_record(False)
    return rep


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="16,128")
    ap.add_argument("--ticks", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=15)
    ap.add_argument("--single-steps", type=int, default=600)
    args = ap.parse_args()
    import torch

    from hector_slam_b200 import capi

    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    gpu = card()
    sizes = [int(x) for x in args.sizes.split(",")]
    for M in sizes:
        reps = [make_rep() for _ in range(M)]
        data = [session_scans(900 + s) for s in range(M)]
        g = capi.SlamGroup(reps, heterogeneous=True)
        times = {a: [] for a in ARMS}
        launches = {a: [] for a in ARMS}
        records = 0
        for t in range(args.warmup + 3 * args.ticks):
            arm = ARMS[t % 3]
            for j, r in enumerate(reps):
                r.set_step_record(arm == "all" or (arm == "one" and j == 0))
            k = t % POSES
            hints = np.ascontiguousarray(np.stack([data[j][k][0] for j in range(M)]), np.float32)
            ranges = [data[j][k][1] for j in range(M)]
            l0 = reps[0].launch_count
            t0 = time.perf_counter()
            g.slam_update_ranges(hints, ranges)
            dt = time.perf_counter() - t0
            if arm != "none":
                records += sum(r.step_record(raw=True) is not None for r in (reps if arm == "all" else reps[:1]))
            if t >= args.warmup:
                times[arm].append(dt)
                launches[arm].append(reps[0].launch_count - l0)
        print(json.dumps({"M": M, "ticks_per_arm": args.ticks, "card": gpu,
                          **{f"{a}_ms_p50": round(pct(times[a], 50), 4) for a in ARMS},
                          **{f"{a}_ms_p99": round(pct(times[a], 99), 4) for a in ARMS},
                          **{f"{a}_launches_per_tick": float(np.mean(launches[a])) for a in ARMS},
                          "records_read": records}), flush=True)
        g.close()
        for r in reps:
            r.close()

    rep = make_rep()
    d = session_scans(77)
    times = {False: [], True: []}
    for t in range(args.warmup + 2 * args.single_steps):
        on = t % 2 == 1
        rep.set_step_record(on)
        hint, ranges = d[t % POSES]
        t0 = time.perf_counter()
        rep.slam_update_ranges(hint, ranges, nowait=True)
        dt = time.perf_counter() - t0
        if t >= args.warmup:
            times[on].append(dt)
    print(json.dumps({"single_nowait_steps_per_arm": args.single_steps, "card": gpu,
                      "off_ms_p50": round(pct(times[False], 50), 4), "off_ms_p99": round(pct(times[False], 99), 4),
                      "on_ms_p50": round(pct(times[True], 50), 4), "on_ms_p99": round(pct(times[True], 99), 4)}),
          flush=True)
    rep.close()


if __name__ == "__main__":
    main()
