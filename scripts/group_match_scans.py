"""What re-matching lost robots from their new LaserScans in one pass buys a fleet server.

Workload: M robots (--sizes), each a handle with a 3-level 2048^2 map and its own laser mount, mapped by --steps group
steps from synthetic 1081-beam LaserScans on the node's default projected path (hsb_group_slam_update_projected, the
workload of scripts/group_match.py).  Then every robot is "lost": its next scan (a fresh 1081-beam LaserScan, not yet
written into any map) is re-matched from H hints (--hints) spread 0.3 m / 0.2 rad around the pose it was taken at, and
each robot's most likely matched pose is picked.

Arms per (M, H), alternated in rotating order within each round, each timed by the host clock around the whole
relocalisation round (every arm ends in a synchronise):
  scans   one hsb_group_match_batch_projected_subset with the likelihoods and the pick asked for: conversion, match and
          scoring on the device, one copy each way
  points  today's path: per robot one hsb_projected_scan_to_points, then hsb_group_match_batch_subset with those
          endpoints, then hsb_group_best_hypothesis_subset on the returned poses with the same endpoints
Poses, Hessians, likelihoods, winners and their indices are compared bit for bit every round.

Reported: p50 / p99 ms per arm and the host-to-device bytes of one round, computed from its inputs (descriptor sizes
from csrc/hsb_internal.h: a session 24 bytes, a conversion table entry 104).  Prints one JSON line per case, with the
card and power limit read in the same run.  Needs a GPU; there is no fall-back.

    python scripts/group_match_scans.py [--sizes 8,32] [--hints 64,512,2048] [--rounds 40]
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from group_step_subset import CUTOFF, LEVELS, POSES, RES, SIZE, session_scans  # noqa: E402

SESSION_BYTES, CONV_ENTRY_BYTES, TRANSFORM_BYTES = 24, 104, 96


def pct(v, q):
    return float(np.percentile(np.asarray(v) * 1e3, q))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="8,32")
    ap.add_argument("--hints", default="64,512,2048")
    ap.add_argument("--steps", type=int, default=POSES)
    ap.add_argument("--rounds", type=int, default=40)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("scripts/group_match_scans.py measures on a GPU and found none")
    from hector_slam_b200 import capi, synth

    sizes = [int(x) for x in args.sizes.split(",") if x]
    hint_counts = [int(x) for x in args.hints.split(",") if x]
    Mmax = max(sizes)
    lib = capi.load_library()
    fmt = synth.SCAN_FORMAT
    nb = fmt["n_beams"]
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()

    def check(st, rep):
        if st != 0:
            raise capi.HsbError(st, lib.hsb_last_error(rep.h).decode())

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
    fleet = capi.SlamGroup(reps)
    for t in range(args.steps):
        k = t % POSES
        hints = np.stack([data[j][k][0] for j in range(Mmax)]).astype(np.float32)
        fleet.slam_update_projected(hints, [data[j][k][1] for j in range(Mmax)])
    fleet.close()
    rng = np.random.default_rng(45)
    k_next = args.steps % POSES   # the scan after the last step, with fresh noise: written into no map
    fresh = [(data[j][k_next][1] + rng.normal(0.0, 0.01, nb)).astype(np.float32) for j in range(Mmax)]
    centre = np.stack([data[j][k_next][0] for j in range(Mmax)])   # within 3 cm / 0.01 rad of where it was taken

    for M in sizes:
        g = capi.SlamGroup(reps[:M])
        members = np.arange(M, dtype=np.int32)
        ranges = np.ascontiguousarray(np.concatenate(fresh[:M]), np.float32)
        ro = (np.arange(M + 1) * nb).astype(np.int32)
        for H in hint_counts:
            Q = M * H
            ho = (np.arange(M + 1) * H).astype(np.int32)
            hints = np.ascontiguousarray(np.concatenate([centre[j][None] + rng.uniform(-1, 1, (H, 3)) * [0.3, 0.3, 0.2]
                                                         for j in range(M)]), np.float32)
            arrays = ("poses", "cov", "lh", "best4", "index")
            out = {a: dict(poses=np.zeros((Q, 3), np.float32), cov=np.zeros((Q, 9), np.float32),
                           lh=np.zeros(Q, np.float32), best4=np.zeros((M, 4), np.float32), index=np.zeros(M, np.int32))
                   for a in ("scans", "points")}
            kept = np.zeros(M, np.int32)
            conv_xy = np.zeros((M, nb, 2), np.float32)
            conv_n = np.zeros(M, np.int32)
            n_points = [0]

            def scans():
                o = out["scans"]
                check(lib.hsb_group_match_batch_projected_subset(
                    g.g, M, members.ctypes.data, ho.ctypes.data, hints.ctypes.data, ranges.ctypes.data, ro.ctypes.data,
                    None, o["poses"].ctypes.data, o["cov"].ctypes.data, o["lh"].ctypes.data, o["best4"].ctypes.data,
                    o["index"].ctypes.data, kept.ctypes.data), reps[0])

            def points():
                o = out["points"]
                origo = np.zeros(2, np.float32)
                n = ctypes.c_int(0)
                for j in range(M):
                    check(lib.hsb_projected_scan_to_points(reps[j].h, fresh[j].ctypes.data, nb, None,
                                                           conv_xy[j].ctypes.data, ctypes.byref(n), origo.ctypes.data),
                          reps[j])
                    conv_n[j] = n.value
                so = np.zeros(M + 1, np.int32)
                so[1:] = np.cumsum(conv_n)
                pts = np.ascontiguousarray(np.concatenate([conv_xy[j, :conv_n[j]] for j in range(M)]), np.float32)
                n_points[0] = int(so[-1])
                check(lib.hsb_group_match_batch_subset(g.g, M, members.ctypes.data, ho.ctypes.data, hints.ctypes.data,
                                                       pts.ctypes.data, so.ctypes.data, o["poses"].ctypes.data,
                                                       o["cov"].ctypes.data), reps[0])
                check(lib.hsb_group_best_hypothesis_subset(g.g, M, members.ctypes.data, 0, ho.ctypes.data,
                                                           o["poses"].ctypes.data, pts.ctypes.data, so.ctypes.data,
                                                           o["lh"].ctypes.data, o["best4"].ctypes.data,
                                                           o["index"].ctypes.data), reps[0])

            arms = {"scans": scans, "points": points}
            names = list(arms)
            times = {a: [] for a in names}
            for r in range(-3, args.rounds):   # the first rounds warm up: modules, staging growth
                order = names[r % len(names):] + names[:r % len(names)]
                for a in order:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    arms[a]()
                    if r >= 0:
                        times[a].append(time.perf_counter() - t0)
                for name in arrays:
                    x, y = out["scans"][name], out["points"][name]
                    assert np.array_equal(x.view(np.uint32), y.view(np.uint32)), (M, H, r, name)
                assert np.array_equal(kept, conv_n), (M, H, r, "kept")
            d = np.abs(out["scans"]["best4"][:, 1:3] - centre[:M, :2]).max(axis=1)
            n_pts = n_points[0]
            desc = M * SESSION_BYTES + (M + 1) * 4
            res = {"M": M, "hints_each": H, "Q": Q, "map": f"{SIZE}^2 x {LEVELS} levels", "beams": nb,
                   "kept_mean": n_pts / M, "rounds_per_arm": args.rounds,
                   "W": reps[0].last_launch_shape()["warps_per_scan"], "results_identical": True,
                   "winners_within_10cm_of_scan_pose": int((d < 0.1).sum()), "card": card,
                   "h2d_bytes": {"scans": desc + Q * 12 + M * (CONV_ENTRY_BYTES + TRANSFORM_BYTES) + M * nb * 4,
                                 "points": M * (nb * 4 + CONV_ENTRY_BYTES + TRANSFORM_BYTES)
                                 + 2 * (desc + Q * 12 + n_pts * 8)},
                   "d2h_bytes": {"scans": Q * (12 + 36 + 4) + M * (4 + 16 + 4),
                                 "points": M * 4 + n_pts * 8 + Q * (12 + 36) + Q * 4 + M * (16 + 4)}}
            for a in names:
                res[f"{a}_ms_p50"] = round(pct(times[a], 50), 3)
                res[f"{a}_ms_p99"] = round(pct(times[a], 99), 3)
            print(json.dumps(res), flush=True)
        g.close()
    for r in reps:
        r.close()


if __name__ == "__main__":
    main()
