"""What hsb_group_reset buys a server that resets robots' maps (reset_map, restart_mapping_with_new_pose, a "reset"
system message) and replicates them.

Workload: M robots (--sizes), each a handle with a 3-level 2048^2 map at 0.05 m, stepped on the node's LaserScan path
(hsb_group_slam_update_ranges, scans of scripts/group_step_subset.py's closed loops).  Two twin owner fleets A and B
are stepped identically.
  (a) Resetting K of the M robots (K = 1, M/4, M; a seeded random member list):
        group       one hsb_group_reset_subset on A, then a device synchronise
        per-member  hsb_reset on each of B's K members (each synchronises), then a device synchronise
      p50 and p99 of a host clock around each arm over --reps repetitions, the arms alternating which runs first.  After
      every size, both fleets' listed members are compared in bits (log-odds, P, gate pose, both rectangles).
  (b) The replication tick after r resets (r = 1, 4, M), with a group buffer of 1 MiB per robot: each owner fleet has a
      replica fleet of fresh twins on the same GPU.  A tick resets r robots, steps every robot once and replicates:
        group       A: hsb_group_reset_subset, the step, one group pack (reset) and one group unpack into A's replicas:
                    the reset robots ship their clear record and the cells written since
        today       B: hsb_reset per robot, the step, one group pack and unpack (the reset robots' whole levels do not
                    fit: deferred), then the host-synchronous two-step protocol for the deferred robots
                    (hsb_get_dirty_rects + hsb_pack_rect_device / hsb_unpack_rect_device per level, what
                    parallel.broadcast_dirty_tiles does around its two collectives; no collective on one GPU)
      Per arm: bytes shipped (the group buffer's words used, plus the two-step rows), deferred blocks, and the time of
      the replication (pack + unpack, and the two-step protocol) from a host clock ending in a device synchronise.
      After every tick both replica fleets and both owner fleets are compared in bits on the reset robots and one other.
The NCCL form needs two GPUs and is not run here.  Prints one JSON line per measurement, with the card and power limit
read in the same run.

    python scripts/group_reset.py [--sizes 16,128] [--reps 30] [--ticks 5]
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

SIZE, LEVELS, RES = 2048, 3, 0.05
MB_PER_ROBOT = 1 << 20


def pct(v, q):
    return float(np.percentile(np.asarray(v) * 1e3, q))


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def same(a, b, members):
    """members of fleets a and b equal in bits: planes, probabilities, gate pose, both rectangles"""
    for m in members:
        for l in range(LEVELS):
            if not np.array_equal(bits(a[m].download_level(l)), bits(b[m].download_level(l))):
                return False
            if not np.array_equal(bits(a[m].download_prob(l)), bits(b[m].download_prob(l))):
                return False
            if a[m].get_mirror_dirty_rect(l) != b[m].get_mirror_dirty_rect(l):
                return False
        if a[m].get_dirty_rects() != b[m].get_dirty_rects():
            return False
        if not np.array_equal(bits(a[m].last_map_update_pose()), bits(b[m].last_map_update_pose())):
            return False
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="16,128")
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--ticks", type=int, default=5)
    args = ap.parse_args()
    import torch

    from group_step_subset import POSES, session_scans
    from hector_slam_b200 import capi, synth

    assert torch.cuda.is_available(), "group_reset.py measures on a GPU"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    stream = torch.cuda.current_stream().cuda_stream

    def fleet(M):
        reps = []
        for _ in range(M):
            r = capi.MapRepB200(RES, SIZE, levels=LEVELS)
            r.set_scan_format(**synth.SCAN_FORMAT)
            reps.append(r)
        return reps

    for M in [int(x) for x in args.sizes.split(",")]:
        A, B, RA, RB = fleet(M), fleet(M), fleet(M), fleet(M)
        gA, gB, gRA, gRB = (capi.SlamGroup(f) for f in (A, B, RA, RB))
        scans = [session_scans(1000 + s) for s in range(M)]
        at = [0]

        def step():
            k = at[0] % POSES
            at[0] += 1
            hints = np.stack([scans[s][k][0] for s in range(M)])
            ranges = [scans[s][k][1] for s in range(M)]
            outs = [g.slam_update_ranges(hints, ranges) for g in (gA, gB)]
            assert all(np.array_equal(bits(x), bits(y)) for x, y in zip(outs[0][:2], outs[1][:2])), "owners diverged"

        step()
        rng = np.random.default_rng(M)

        # (a) reset latency
        for K in sorted({1, max(1, M // 4), M}):
            members = [int(m) for m in rng.choice(M, K, replace=False)]
            t_group, t_single = [], []
            for rep in range(args.reps + 3):
                arms = ["group", "single"] if rep % 2 == 0 else ["single", "group"]
                for arm in arms:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    if arm == "group":
                        gA.reset(members=members)
                    else:
                        for m in members:
                            B[m].reset()
                    torch.cuda.synchronize()
                    dt = time.perf_counter() - t0
                    if rep >= 3:
                        (t_group if arm == "group" else t_single).append(dt)
            check = sorted({members[0], members[len(members) // 2], members[-1]})
            ok = same(A, B, check)
            # the group arm leaves the cleared flags set; consume both fleets' rectangles so (b) starts level
            for f in (A, B):
                for r in f:
                    r.get_dirty_rects(reset=True)
            print(json.dumps({"part": "a", "card": card, "M": M, "K": K, "reps": args.reps,
                              "group_ms_p50": pct(t_group, 50), "group_ms_p99": pct(t_group, 99),
                              "per_member_ms_p50": pct(t_single, 50), "per_member_ms_p99": pct(t_single, 99),
                              "bytes_written_per_member": SIZE * SIZE * 16 * (1 + 1 / 4 + 1 / 16),
                              "bitwise_equal": ok}), flush=True)
            assert ok, "group reset differs from hsb_reset"

        # (b) the replication tick after r resets
        cap = M * MB_PER_ROBOT
        buf = torch.zeros(cap // 4, dtype=torch.float32, device="cuda")
        rows = torch.zeros(SIZE * SIZE, dtype=torch.float32, device="cuda")
        # start level: every owner reset (equal to its fresh replica), every rectangle and cleared flag consumed
        gA.reset()
        for r in B:
            r.reset()
        for r in A + B:
            r.get_dirty_rects(reset=True)
        for r_count in sorted({1, 4, M}):
            res = {"group": [], "today": []}
            for tick in range(args.ticks):
                members = [int(m) for m in rng.choice(M, r_count, replace=False)]
                gA.reset(members=members)
                for m in members:
                    B[m].reset()
                step()
                arms = ["group", "today"] if tick % 2 == 0 else ["today", "group"]
                for arm in arms:
                    og, rg, owners, replicas = (gA, gRA, A, RA) if arm == "group" else (gB, gRB, B, RB)
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    og.pack_dirty_device(buf.data_ptr(), cap, True, stream)
                    rg.unpack_dirty_device(buf.data_ptr(), cap, stream)
                    head = buf[:5].view(torch.int32).cpu().tolist()   # synchronises: the deferred blocks
                    deferred, used = head[3], head[4]
                    two_step = 0
                    if deferred:
                        gh = buf[:5 + 2 * M].view(torch.int32).cpu().numpy()
                        for k in range(M):
                            start = int(gh[6 + 2 * k])
                            if int(buf[start + 2:start + 3].view(torch.int32).item()) == 0:
                                continue
                            m = int(gh[5 + 2 * k])
                            for l, rect in enumerate(owners[m].get_dirty_rects(reset=True)):
                                if rect is None:
                                    continue
                                owners[m].pack_rect_device(l, rect, rows.data_ptr(), stream)
                                replicas[m].unpack_rect_device(l, rect, rows.data_ptr(), stream)
                                two_step += (rect[2] - rect[0] + 1) * (rect[3] - rect[1] + 1)
                    torch.cuda.synchronize()
                    dt = time.perf_counter() - t0
                    res[arm].append((dt, 4 * used, 4 * two_step, deferred))
                check = sorted(set(members[:3]) | {(members[0] + 1) % M})
                ok = same(RA, RB, check) and same(A, B, check)
                for m in check:
                    for l in range(LEVELS):
                        ok = ok and np.array_equal(bits(RA[m].download_level(l)), bits(A[m].download_level(l)))
                assert ok, ("replicas differ", M, r_count, tick)
            out = {"part": "b", "card": card, "M": M, "resets": r_count, "ticks": args.ticks, "buffer_bytes": cap}
            for arm, v in res.items():
                out[arm] = {"ms_p50": pct([x[0] for x in v], 50), "ms_max": pct([x[0] for x in v], 100),
                            "buffer_bytes_used_p50": float(np.median([x[1] for x in v])),
                            "two_step_bytes_p50": float(np.median([x[2] for x in v])),
                            "deferred_blocks_p50": float(np.median([x[3] for x in v]))}
            out["bitwise_equal"] = True
            print(json.dumps(out), flush=True)
        for g in (gA, gB, gRA, gRB):
            g.close()
        for f in (A, B, RA, RB):
            for r in f:
                r.close()
        del buf, rows
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
