"""What matching a fleet's pose hints in one pass buys a server that relocalises robots.

Workload: M robots (--sizes), each a handle with a 3-level 2048^2 map and its own laser mount, mapped by --steps group
steps from synthetic 1081-beam LaserScans on the node's default projected path (hsb_group_slam_update_projected, the
workload of scripts/group_step_subset.py with every robot stepped every tick).  Then every robot is "lost": its last
scan is re-matched from H hints (--hints) spread 0.3 m / 0.2 rad around the pose of its last step.

Arms per (M, H), alternated in rotating order within each round, each timed by the host clock around the call (every
arm ends in a synchronise or a read-back):
  group        one hsb_group_match_batch_subset over the M robots on their last-match containers (no scan sent)
  resent       the same call with the scans' endpoints sent
  loop         per robot one hsb_match_batch in shared-scan mode, warps per scan pinned to the group call's W
  group_w      the group call with handles[0]'s warps per scan set to what one robot's own call of H hints takes
  loop_auto    per robot one hsb_match_batch with its own default launch shape
group, resent and loop are compared bit for bit every round, and so are group_w and loop_auto: the reduction order
follows W, and the group call picks W by hsb_match_batch's rule for ONE batch of M x H hints, which may be narrower
than each robot's own call would take.  group_w / loop_auto show what that choice costs or saves.

Relocalisation round per (M, H): the group call, then hsb_group_best_hypothesis_subset on the returned poses with the
last matched scans (the winners read back) — against per robot hsb_match_batch_device + hsb_best_hypothesis_device on
device tensors (hints and scans already on the device, W pinned to the group call's) and the read-back of the winner.
Winners are compared bit for bit.

Reported: p50 / p99 ms per arm and the host-to-device bytes of one call / round, computed from its inputs.  Prints one
JSON line per case, with the card and power limit read in the same run.  Needs a GPU; there is no fall-back.

    python scripts/group_match.py [--sizes 8,32] [--hints 64,512,2048] [--rounds 40]
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

from group_step_subset import CUTOFF, LEVELS, POSES, RES, SIZE, session_scans  # noqa: E402


def pct(v, q):
    return float(np.percentile(np.asarray(v) * 1e3, q))


def auto_w(sm, B):
    """hsb_match_batch's warps per scan for one batch of B scans under the default tuning"""
    want, W = sm * 24 // max(B, 1), 1
    while W * 2 <= want and W < 8:
        W *= 2
    return W


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="8,32")
    ap.add_argument("--hints", default="64,512,2048")
    ap.add_argument("--steps", type=int, default=POSES)
    ap.add_argument("--rounds", type=int, default=40)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("scripts/group_match.py measures on a GPU and found none")
    from hector_slam_b200 import capi, synth

    sizes = [int(x) for x in args.sizes.split(",") if x]
    hint_counts = [int(x) for x in args.hints.split(",") if x]
    Mmax = max(sizes)
    lib = capi.load_library()
    fmt = synth.SCAN_FORMAT
    nb = fmt["n_beams"]
    sm = torch.cuda.get_device_properties(0).multi_processor_count
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
    # the maps: every robot stepped every tick by one group step of the projected input
    fleet = capi.SlamGroup(reps)
    last_pose = np.zeros((Mmax, 3), np.float32)
    for t in range(args.steps):
        k = t % POSES
        hints = np.stack([data[j][k][0] for j in range(Mmax)]).astype(np.float32)
        ranges = [data[j][k][1] for j in range(Mmax)]
        last_pose = fleet.slam_update_projected(hints, ranges)[0]
    fleet.close()
    k_last = (args.steps - 1) % POSES
    endpoints = [np.ascontiguousarray(reps[j].projected_scan_to_points(data[j][k_last][1])[0], np.float32)
                 for j in range(Mmax)]
    rng = np.random.default_rng(44)

    for M in sizes:
        g = capi.SlamGroup(reps[:M])
        members = np.arange(M, dtype=np.int32)
        scans = endpoints[:M]
        so = np.zeros(M + 1, np.int32)
        so[1:] = np.cumsum([s.shape[0] for s in scans])
        pts = np.ascontiguousarray(np.concatenate(scans), np.float32)
        d_pts = [torch.from_numpy(s.reshape(-1)).cuda() for s in scans]
        for H in hint_counts:
            Q = M * H
            ho = (np.arange(M + 1) * H).astype(np.int32)
            hints = np.ascontiguousarray(np.concatenate([last_pose[j][None] + rng.uniform(-1, 1, (H, 3)) * [0.3, 0.3, 0.2]
                                                         for j in range(M)]), np.float32)
            d_hints = [torch.from_numpy(hints[j * H:(j + 1) * H].reshape(-1)).cuda() for j in range(M)]
            d_out = [torch.zeros(H * 3, device="cuda") for _ in range(M)]
            d_best = [torch.zeros(4, device="cuda") for _ in range(M)]
            out = {a: (np.zeros((Q, 3), np.float32), np.zeros((Q, 9), np.float32))
                   for a in ("group", "resent", "loop", "group_w", "loop_auto")}
            best_g, idx_g = np.zeros((M, 4), np.float32), np.zeros(M, np.int32)
            best_l = np.zeros((M, 4), np.float32)
            w_own = auto_w(sm, H)

            def group(a, w=0):
                pp, sp = (pts.ctypes.data, so.ctypes.data) if a == "resent" else (None, None)
                reps[0].set_tuning(warps_per_scan=w)
                check(lib.hsb_group_match_batch_subset(g.g, M, members.ctypes.data, ho.ctypes.data, hints.ctypes.data,
                                                       pp, sp, out[a][0].ctypes.data, out[a][1].ctypes.data), reps[0])
                reps[0].set_tuning(warps_per_scan=0)

            W = None

            def loop(a, w):
                p, c = out[a]
                for j in range(M):
                    reps[j].set_tuning(warps_per_scan=w)
                    check(lib.hsb_match_batch(reps[j].h, H, hints[j * H:].ctypes.data, scans[j].ctypes.data, None,
                                              scans[j].shape[0], p[j * H:].ctypes.data, c[j * H:].ctypes.data), reps[j])
                    reps[j].set_tuning(warps_per_scan=0)

            def reloc_group():
                group("group")
                check(lib.hsb_group_best_hypothesis_subset(g.g, M, members.ctypes.data, 0, ho.ctypes.data,
                                                           out["group"][0].ctypes.data, None, None, None,
                                                           best_g.ctypes.data, idx_g.ctypes.data), reps[0])

            def reloc_loop():
                for j in range(M):
                    n = scans[j].shape[0]
                    reps[j].set_tuning(warps_per_scan=W)
                    reps[j].match_batch_device(H, d_hints[j].data_ptr(), d_pts[j].data_ptr(), None, n, n,
                                               d_out[j].data_ptr(), None, 0)
                    reps[j].set_tuning(warps_per_scan=0)
                    reps[j].best_hypothesis_device(0, H, d_out[j].data_ptr(), d_pts[j].data_ptr(), None, n,
                                                   d_best[j].data_ptr(), None, 0)
                    best_l[j] = d_best[j].cpu().numpy()

            group("group")
            W = reps[0].last_launch_shape()["warps_per_scan"]
            arms = {"group": lambda: group("group"), "resent": lambda: group("resent"), "loop": lambda: loop("loop", W),
                    "group_w": lambda: group("group_w", w_own), "loop_auto": lambda: loop("loop_auto", 0),
                    "reloc_group": reloc_group, "reloc_loop": reloc_loop}
            names = list(arms)
            times = {a: [] for a in names}
            for r in range(-3, args.rounds):   # the first rounds warm up: modules, staging growth, carve-outs
                order = names[r % len(names):] + names[:r % len(names)]
                for a in order:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    arms[a]()
                    if r >= 0:
                        times[a].append(time.perf_counter() - t0)
                for a in ("resent", "loop"):
                    for x, y in zip(out[a], out["group"]):
                        assert np.array_equal(x.view(np.uint32), y.view(np.uint32)), (M, H, r, a)
                for x, y in zip(out["loop_auto"], out["group_w"]):
                    assert np.array_equal(x.view(np.uint32), y.view(np.uint32)), (M, H, r, "group_w")
                assert np.array_equal(best_g.view(np.uint32), best_l.view(np.uint32)), (M, H, r, "reloc")
            d = np.abs(out["group"][0][:, :2].reshape(M, H, 2) - last_pose[:M, None, :2]).max(axis=2)
            n_scan = int(so[-1])
            res = {"M": M, "hints_each": H, "Q": Q, "map": f"{SIZE}^2 x {LEVELS} levels", "scan_points_mean": n_scan / M,
                   "rounds_per_arm": args.rounds, "W_group": W, "W_own": w_own, "results_identical": True,
                   "hints_matched_within_5cm_of_last_pose": int((d < 0.05).sum()), "best_likelihood_min":
                   round(float(best_g[:, 0].min()), 4), "card": card,
                   "h2d_bytes": {"group": M * 16 + (M + 1) * 4 + Q * 12,
                                 "resent": M * 16 + (M + 1) * 4 + Q * 12 + n_scan * 8,
                                 "loop": Q * 12 + n_scan * 8,
                                 "reloc_group": 2 * (M * 16 + (M + 1) * 4 + Q * 12), "reloc_loop": 0}}
            for a in names:
                res[f"{a}_ms_p50"] = round(pct(times[a], 50), 3)
                res[f"{a}_ms_p99"] = round(pct(times[a], 99), 3)
            print(json.dumps(res), flush=True)
        g.close()
    for r in reps:
        r.close()


if __name__ == "__main__":
    main()
