"""What the group replication calls buy a server that replicates a fleet's maps on every tick.

Workload: M robots (--sizes), each a handle with a 3-level 2048^2 map, stepped with the subset workload of
scripts/group_step_subset.py (40 Hz lidars with seeded random phases; a tick steps the robots whose scan falls into a
--window-ms window, on the node's default projected path).  Two twin owner fleets are stepped identically (one
hsb_group_slam_update_projected_subset each), each with a replica fleet of fresh twins on the same GPU.  After every
tick the stepped members are replicated, on one caller stream:
  group       one hsb_group_pack_dirty_device_subset (reset) into one buffer and one hsb_group_unpack_dirty_device
  per-member  for each stepped member, hsb_pack_dirty_device (reset) into its own 4 MB buffer slot and
              hsb_unpack_dirty_device from it
The arms alternate which runs first from tick to tick.  Per arm: replication time per tick from CUDA events on the
caller stream (p50, p99; a tick's enqueue gaps count), bytes the pack wrote (headers and rows), the bytes a fixed-size
broadcast of the buffers would move, and launches.  After every tick, outside the timed region, both replica fleets
are compared with their owners in bits on the device (every member, every level); a difference stops the run.  The NCCL form (one broadcast per tick against one per member) needs two GPUs; it is not
run here and reported as not measured.  Prints one JSON line per M, with the card and power limit read in the same run.

    python scripts/group_tiles.py [--sizes 16,128] [--window-ms 5] [--ticks 200]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

SIZE, LEVELS, RES, CUTOFF, PERIOD_MS = 2048, 3, 0.05, 30.0, 25.0
SLOT_BYTES = 4 << 20   # the documented one-shot buffer of the single protocol


def pct(v, q):
    return float(np.percentile(np.asarray(v), q))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="16,128")
    ap.add_argument("--window-ms", type=float, default=5.0)
    ap.add_argument("--ticks", type=int, default=200)
    ap.add_argument("--group-mb-per-robot", type=float, default=1.0,
                    help="group buffer capacity per robot of the fleet (MB)")
    args = ap.parse_args()
    import torch

    from group_step_subset import POSES, session_scans
    from hector_slam_b200 import capi, parallel, synth

    assert torch.cuda.is_available(), "group_tiles.py measures on a GPU"
    dev = torch.device("cuda", 0)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    fmt = synth.SCAN_FORMAT
    nb = fmt["n_beams"]
    lib = capi.load_library()

    def make(s):
        rep = capi.MapRepB200(RES, SIZE, levels=LEVELS, update_factor_free=0.4, update_factor_occupied=0.9)
        rep.setMapUpdateMinDistDiff(0.4)
        rep.setMapUpdateMinAngleDiff(0.13)
        rep.set_laser_projection(**fmt, range_cutoff=CUTOFF)
        mount = synth.laser_transform(xyz=(0.05 + 0.001 * s, -0.02 + 0.0005 * s, 0.3),
                                      rpy=(0.002 * (s % 5), -0.003 * (s % 7), 0.01 * (s % 11)))
        rep.set_cloud_format(mount, **synth.CLOUD_FORMAT)
        rep.get_dirty_rects(reset=True)
        return rep

    stream = torch.cuda.current_stream(dev)
    for M in [int(x) for x in args.sizes.split(",")]:
        fleets = {a: ([make(s) for s in range(M)], [make(s) for s in range(M)]) for a in ("group", "per_member")}
        groups = {a: (capi.SlamGroup(o), capi.SlamGroup(r)) for a, (o, r) in fleets.items()}
        data = [session_scans(900 + s) for s in range(M)]
        phase = np.random.default_rng(40).uniform(0.0, PERIOD_MS, M)
        scan_no = np.zeros(M, np.int64)
        gcap = int(args.group_mb_per_robot * M * (1 << 20)) & ~3
        gbuf = torch.zeros(gcap // 4, dtype=torch.float32, device=dev)
        slots = torch.zeros((M, SLOT_BYTES // 4), dtype=torch.float32, device=dev)
        pose, cov = np.zeros((M, 3), np.float32), np.zeros((M, 9), np.float32)
        upd, kept = np.zeros(M, np.int32), np.zeros(M, np.int32)
        stats = {a: dict(ms=[], bytes=0, fixed=0, launches=0, deferred=0) for a in fleets}
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

        def step(members, hints, ranges, offs):
            for og, _ in groups.values():
                st = lib.hsb_group_slam_update_projected_subset(og.g, len(members), members.ctypes.data, hints.ctypes.data,
                                                                ranges.ctypes.data, offs.ctypes.data, None, None, 0,
                                                                pose.ctypes.data, cov.ctypes.data, upd.ctypes.data,
                                                                kept.ctypes.data)
                og._check(st)

        def group_arm(members):
            owner, replica = fleets["group"]
            og, rg = groups["group"]
            l0 = owner[0].launch_count + replica[0].launch_count
            ev[0].record(stream)
            og.pack_dirty_device(gbuf.data_ptr(), gcap, True, stream.cuda_stream, members=members)
            rg.unpack_dirty_device(gbuf.data_ptr(), gcap, stream.cuda_stream)
            ev[1].record(stream)
            s = stats["group"]
            s["launches"] += owner[0].launch_count + replica[0].launch_count - l0
            hdr = gbuf[:5].view(torch.int32).cpu().numpy()
            s["bytes"] += 4 * int(hdr[4])
            s["deferred"] += int(hdr[3])
            s["fixed"] += gcap

        def per_member_arm(members):
            owner, replica = fleets["per_member"]
            l0 = sum(r.launch_count for r in owner + replica)
            ev[0].record(stream)
            for j in members:
                ptr = slots[j].data_ptr()
                owner[j].pack_dirty_device(ptr, SLOT_BYTES, True, stream.cuda_stream)
                replica[j].unpack_dirty_device(ptr, SLOT_BYTES, stream.cuda_stream)
            ev[1].record(stream)
            s = stats["per_member"]
            s["launches"] += sum(r.launch_count for r in owner + replica) - l0
            hdr = slots[torch.as_tensor(members.astype(np.int64), device=dev), :4].view(torch.int32).cpu().numpy()
            s["bytes"] += int(sum(4 * (64 + int(h[3])) for h in hdr))
            s["deferred"] += int(sum(int(h[2]) for h in hdr))
            s["fixed"] += SLOT_BYTES * len(members)

        planes = {arm: [(parallel.level_plane_tensor(o, l, dev).view(torch.int32),
                         parallel.level_plane_tensor(r, l, dev).view(torch.int32))
                        for o, r in zip(owner, replica) for l in range(LEVELS)]
                  for arm, (owner, replica) in fleets.items()}

        def check_equal(tag):
            """every member's every level of both fleets, bit for bit: one device-to-host read"""
            diff = torch.stack([(a != b).any() for pairs in planes.values() for a, b in pairs])
            if bool(diff.any()):
                bad = int(torch.nonzero(diff)[0])
                arm = list(planes)[bad // (M * LEVELS)]
                raise AssertionError((tag, arm, "member", bad % (M * LEVELS) // LEVELS, "level", bad % LEVELS))

        t = tick = 0
        while tick < args.ticks:
            lo = (t * args.window_ms) % PERIOD_MS
            t += 1
            d = (phase - lo) % PERIOD_MS
            sel = d < args.window_ms
            members = np.ascontiguousarray(np.nonzero(sel)[0][np.argsort(d[sel])], np.int32)
            if len(members) == 0:
                continue
            ks = [int(scan_no[j] % POSES) for j in members]
            scan_no[members] += 1
            hints = np.ascontiguousarray(np.stack([data[j][k][0] for j, k in zip(members, ks)]), np.float32)
            ranges = np.ascontiguousarray(np.concatenate([data[j][k][1] for j, k in zip(members, ks)]), np.float32)
            offs = np.arange(len(members) + 1, dtype=np.int32) * nb
            step(members, hints, ranges, offs)
            order = (group_arm, per_member_arm) if tick % 2 == 0 else (per_member_arm, group_arm)
            for fn in order:
                fn(members)
                torch.cuda.synchronize(dev)
                stats["group" if fn is group_arm else "per_member"]["ms"].append(ev[0].elapsed_time(ev[1]))
            tick += 1
            check_equal(f"M {M} tick {tick}")   # after both arms' timed regions
        out = {"M": M, "map": f"{SIZE}^2 x {LEVELS} levels", "window_ms": args.window_ms, "ticks": args.ticks,
               "group_capacity_bytes": gcap, "slot_bytes": SLOT_BYTES, "card": card, "replicas_equal_owners": True}
        warm = 5   # the first ticks load modules
        for arm, s in stats.items():
            v = s["ms"][warm:]
            out[f"{arm}_ms_p50"] = round(pct(v, 50), 4)
            out[f"{arm}_ms_p99"] = round(pct(v, 99), 4)
            out[f"{arm}_packed_bytes_per_tick"] = round(s["bytes"] / args.ticks)
            out[f"{arm}_fixed_broadcast_bytes_per_tick"] = round(s["fixed"] / args.ticks)
            out[f"{arm}_launches_per_tick"] = round(s["launches"] / args.ticks, 2)
            out[f"{arm}_deferred_blocks"] = s["deferred"]
        out["nccl"] = "not measured (needs two GPUs; not run by this script)"
        print(json.dumps(out), flush=True)
        for og, rg in groups.values():
            og.close()
            rg.close()
        for owner, replica in fleets.values():
            for r in owner + replica:
                r.close()
        del gbuf, slots
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
