"""What one heterogeneous group buys a server whose robots' map pyramids differ in level count and gather path.

Workload: M robots (--sizes), spread round-robin over four robot classes:
  ugv       1 level  (hector_ugv.launch),           1024 x 1024 at 0.05 m, texture gathers
  mapping   2 levels (mapping_default.launch),      768 x 1024 at 0.05 m, start (0.3, 0.4), texture gathers
  default   3 levels (the node's default),          1024 x 1024 at 0.05 m, texture gathers
  outdoor   3 levels, LDG gathers (what HSB_GATHER_AUTO resolves to past the texture limit), 1536 x 1536 at 0.05 m
each stepping synthetic 1081-beam LaserScans from raw ranges (hsb_group_slam_update_ranges, nowait = 0) along its own
closed loop (scripts/group_step_subset.py's trajectories).  Three twin fleets get the same scans, one per arm:
  hetero    one hsb_group_create_heterogeneous group of all M robots: one step call per tick
  classes   one hsb_group_create_mixed group per class: one step call per class with a robot in the tick
  single    hsb_slam_update_ranges for each robot of the tick, one after another
Two phases per M, as scripts/group_mixed.py runs them: `full` steps every robot every tick, `subset` a seeded random
~M/5 of them.  Reported per arm: ms per tick (host clock around the arm's calls, which return after the map writes: p50 /
p90), kernel launches per tick (summed over the arm's handles) and step calls per tick.  Host-to-device copies per tick
are not counted: the field h2d_copies_per_tick_by_contract is the step calls per tick, each of which is one copy by the
header's contract for every step form (which the group step tests hold).
Every tick's poses are compared bit for bit across the arms, and at the end every level of every robot's plane.

Then the replication tick for the hetero and classes arms: after a full step, pack every robot's dirty tiles (reset) into
one buffer per group and unpack it on a replica group of twin handles listed in the same order — one buffer for the
heterogeneous group against one per class — timed with CUDA events around pack + unpack; the replicas are compared with
their owners at the end.

Prints one JSON line per (M, phase), one per M for the replication tick and a final one with the plane comparison, with
the card's name and power limit read in the same run.  Needs a GPU; there is no fall-back.

    python scripts/group_hetero.py [--sizes 16,128] [--ticks 40] [--rep-ticks 20]
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

TEX, LDG = 2, 1
# map_size_x, map_size_y, map_resolution, start, levels, gather mode
CLASSES = {"ugv": (1024, 1024, 0.05, (0.5, 0.5), 1, TEX), "mapping": (768, 1024, 0.05, (0.3, 0.4), 2, TEX),
           "default": (1024, 1024, 0.05, (0.5, 0.5), 3, TEX), "outdoor": (1536, 1536, 0.05, (0.5, 0.5), 3, LDG)}
NAMES = list(CLASSES)
NC = len(NAMES)
ARMS = ("hetero", "classes", "single")


def pct(v, q):
    return float(np.percentile(np.asarray(v) * 1e3, q))


def make_rep(s):
    from hector_slam_b200 import capi, synth

    sx, sy, res, start, levels, mode = CLASSES[NAMES[s % NC]]
    rep = capi.MapRepB200(res, sx, sy, levels=levels, start=start, update_factor_free=0.4, update_factor_occupied=0.9,
                          gather_mode=mode)
    rep.setMapUpdateMinDistDiff(0.4)
    rep.setMapUpdateMinAngleDiff(0.13)
    rep.set_scan_format(**synth.SCAN_FORMAT)
    return rep


def buffer_words(reps):
    cells = sum(r.level_info(l)[0] * r.level_info(l)[1] for r in reps for l in range(r.levels))
    return (5 + 2 * len(reps) + 3) // 4 * 4 + 64 * len(reps) + cells


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="16,128")
    ap.add_argument("--ticks", type=int, default=40)
    ap.add_argument("--rep-ticks", type=int, default=20)
    args = ap.parse_args()
    import torch

    from hector_slam_b200 import capi

    sizes = [int(x) for x in args.sizes.split(",")]
    Mmax = max(sizes)
    fleets = {a: [make_rep(s) for s in range(Mmax)] for a in ARMS}
    replicas = {a: [make_rep(s) for s in range(Mmax)] for a in ("hetero", "classes")}
    data = [session_scans(900 + s) for s in range(Mmax)]
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip()
    except OSError:
        card = "unknown"
    equal_poses = True
    replicas_equal = True

    for M in sizes:
        hetero = capi.SlamGroup(fleets["hetero"][:M], heterogeneous=True)
        by_class = [[j for j in range(M) if j % NC == c] for c in range(NC)]   # each class's robots, in order
        classes = [capi.SlamGroup([fleets["classes"][j] for j in js], mixed=True) if js else None for js in by_class]
        scan_no = np.zeros(M, np.int64)   # each robot's next scan: its loop advances when it is stepped

        def run(arm, members, hints, ranges):
            """one tick of `arm` over `members` (None: every robot) -> (poses in member order, step calls)"""
            sel = list(range(M)) if members is None else members
            if arm == "hetero":
                return hetero.slam_update_ranges(hints, ranges, members=members)[0], 1
            if arm == "single":
                reps = fleets["single"]
                return np.stack([reps[j].slam_update_ranges(hints[k], ranges[k])[0] for k, j in enumerate(sel)]), len(sel)
            out, calls = np.zeros((len(sel), 3), np.float32), 0
            for c, js in enumerate(by_class):
                ks = [k for k, j in enumerate(sel) if j % NC == c]
                if not ks:
                    continue
                local = None if members is None else [js.index(sel[k]) for k in ks]
                out[ks] = classes[c].slam_update_ranges(hints[ks], [ranges[k] for k in ks], members=local)[0]
                calls += 1
            return out, calls

        def tick_inputs(sel):
            ks = [int(scan_no[j] % POSES) for j in sel]
            scan_no[sel] += 1
            hints = np.ascontiguousarray(np.stack([data[j][k][0] for j, k in zip(sel, ks)]), np.float32)
            return hints, [data[j][k][1] for j, k in zip(sel, ks)]

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
                hints, ranges = tick_inputs(sel)
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
                equal_poses &= all(np.array_equal(poses[a].view(np.uint32), ref) for a in ("hetero", "classes"))
            rec = {"M": M, "phase": phase, "robots_per_tick": len(sel), "ticks": args.ticks,
                   "classes": {n: CLASSES[n] for n in NAMES}, "card": card}
            for a in ARMS:
                rec[a] = {"p50_ms": round(pct(times[a], 50), 3), "p90_ms": round(pct(times[a], 90), 3),
                          "launches_per_tick": launches[a] / args.ticks, "step_calls_per_tick": calls[a] / args.ticks,
                          "h2d_copies_per_tick_by_contract": calls[a] / args.ticks}
            rec["poses_equal_across_arms"] = bool(equal_poses)
            print(json.dumps(rec), flush=True)

        # the replication tick: a full step of both arms, then pack (reset) + unpack, one buffer per group
        rep_hetero = capi.SlamGroup(replicas["hetero"][:M], heterogeneous=True)
        rep_classes = [capi.SlamGroup([replicas["classes"][j] for j in js], mixed=True) if js else None
                       for js in by_class]
        pairs = {"hetero": [(hetero, rep_hetero, fleets["hetero"][:M])],
                 "classes": [(g, r, [fleets["classes"][j] for j in js])
                             for g, r, js in zip(classes, rep_classes, by_class) if g is not None]}
        bufs = {a: [torch.zeros(buffer_words(reps), dtype=torch.float32, device="cuda") for _, _, reps in pairs[a]]
                for a in pairs}
        st = torch.cuda.current_stream()
        rtimes = {a: [] for a in pairs}
        for t in range(2 + args.rep_ticks):
            hints, ranges = tick_inputs(list(range(M)))
            run("single", None, hints, ranges)   # (every arm takes every scan: the planes stay comparable)
            for a in ("hetero", "classes"):
                run(a, None, hints, ranges)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(st)
                for (g, r, _), b in zip(pairs[a], bufs[a]):
                    g.pack_dirty_device(b.data_ptr(), 4 * b.numel(), True, st.cuda_stream)
                    r.unpack_dirty_device(b.data_ptr(), 4 * b.numel(), st.cuda_stream)
                e1.record(st)
                torch.cuda.synchronize()
                if t >= 2:
                    rtimes[a].append(e0.elapsed_time(e1) / 1e3)
        rec = {"M": M, "phase": "replication", "ticks": args.rep_ticks, "card": card}
        for a in pairs:
            rec[a] = {"p50_ms": round(pct(rtimes[a], 50), 3), "p90_ms": round(pct(rtimes[a], 90), 3),
                      "buffers_per_tick": len(pairs[a])}
        for a in pairs:
            for j in range(M):
                for l in range(fleets[a][j].levels):
                    replicas_equal &= np.array_equal(replicas[a][j].download_level(l).view(np.uint32),
                                                     fleets[a][j].download_level(l).view(np.uint32))
        rec["replicas_equal_owners"] = bool(replicas_equal)
        print(json.dumps(rec), flush=True)
        for g in rep_classes + classes:
            if g is not None:
                g.close()
        rep_hetero.close()
        hetero.close()

    planes_equal = True
    for s in range(Mmax):
        for l in range(fleets["single"][s].levels):
            ref = fleets["single"][s].download_level(l).view(np.uint32)
            planes_equal &= all(np.array_equal(fleets[a][s].download_level(l).view(np.uint32), ref)
                                for a in ("hetero", "classes"))
    print(json.dumps({"planes_equal_across_arms": bool(planes_equal), "poses_equal_across_arms": bool(equal_poses),
                      "replicas_equal_owners": bool(replicas_equal), "robots": Mmax, "card": card}), flush=True)
    for fl in list(fleets.values()) + list(replicas.values()):
        for r in fl:
            r.close()
    if not (planes_equal and equal_poses and replicas_equal):
        sys.exit(1)


if __name__ == "__main__":
    main()
