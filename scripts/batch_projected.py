"""What hsb_match_batch_projected buys someone who replays or relocalises a default node's LaserScans against a map.

Workload: bench.py's (bench.make_workload / build_map_on_gpu): 4096 scans of 1081 beams, 3-level 2048^2 map, the
laser projection of synth.SCAN_FORMAT with the node's 30 m cutoff, one laser transform (synth.laser_transform()).

Arms, alternated within each of --rounds rounds on one handle, each `--steps` timed steps after `--warmup` untimed ones:
  projected_host  pinned host ranges -> hsb_match_batch_projected_submit / _wait, pipelined as bench.py's time_host
                  (step k+1 submitted before step k is waited for)
  cloud_host      the same scans projected on the host by the restatement in tests/laser_projection.py (not timed)
                  -> hsb_match_batch_cloud_submit / _wait, pipelined the same way
  ranges_host     hsb_match_batch_ranges_submit / _wait (the ranges conversion, not the node's default path)
  *_device        the three device-resident calls (_projected_device, _cloud_device, _ranges_device), the inputs
                  already in HBM: the in-kernel cost of each conversion
Host arms: wall clock around the steps, ending in a device synchronise.  Device arms: CUDA events around the steps.
Prints one JSON line: scans/s per arm (median and range over rounds), H2D input bytes per scan (computed), the max abs
difference of projected_host against cloud_host (poses, covariances, origo), and the card and power limit read in
the same run.

    python scripts/batch_projected.py [--rounds 3] [--steps 20] [--warmup 5]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

CUTOFF = 30.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()

    import torch

    import bench
    from hector_slam_b200 import capi, synth
    from laser_projection import project, unit_vectors

    if not torch.cuda.is_available():
        raise SystemExit("batch_projected.py: no CUDA device")
    dev = torch.device("cuda", 0)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    B = bench.BATCH
    world, _, _, _, hints = bench.make_workload(0, B)
    ranges = np.ascontiguousarray(bench.make_workload.ranges, dtype=np.float32)
    rep = capi.MapRepB200(bench.RES, bench.MAP_SIZE, levels=bench.LEVELS, update_factor_free=0.4,
                          update_factor_occupied=0.9)
    bench.build_map_on_gpu(rep, world)
    proj = dict(synth.SCAN_FORMAT, range_cutoff=CUTOFF)
    rep.set_laser_projection(**proj)
    rep.set_scan_format(**synth.SCAN_FORMAT)
    rep.set_cloud_format(synth.laser_transform(), **synth.CLOUD_FORMAT)
    u = unit_vectors(proj["n_beams"], proj["angle_min"], proj["angle_increment"])
    clouds = [project(ranges[b], proj, u) for b in range(B)]
    c_offs = np.concatenate([[0], np.cumsum([c.shape[0] for c in clouds])]).astype(np.int32)
    cloud_all = np.ascontiguousarray(np.concatenate(clouds), dtype=np.float32)

    NSET = 2
    h_hints = [capi.pinned_copy(hints) for _ in range(NSET)]
    h_ranges = [capi.pinned_copy(ranges) for _ in range(NSET)]
    h_cloud = [capi.pinned_copy(cloud_all) for _ in range(NSET)]
    h_poses = [capi.PinnedArray((B, 3)) for _ in range(NSET)]
    h_cov = [capi.PinnedArray((B, 9)) for _ in range(NSET)]
    h_origo = [capi.PinnedArray((B, 2)) for _ in range(NSET)]

    def submit_projected(i):
        k = i % NSET
        return rep.match_batch_projected_submit(h_hints[k].array, h_ranges[k].array, h_poses[k].array, h_cov[k].array,
                                                h_origo[k].array)

    def submit_cloud(i):
        k = i % NSET
        return rep.match_batch_cloud_submit(h_hints[k].array, h_cloud[k].array, c_offs, h_poses[k].array, h_cov[k].array,
                                            h_origo[k].array)

    def submit_ranges(i):
        k = i % NSET
        return rep.match_batch_ranges_submit(h_hints[k].array, h_ranges[k].array, h_poses[k].array, h_cov[k].array)

    def time_host(submit):
        for i in range(max(3, args.warmup)):
            rep.match_batch_wait(submit(i))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pending = submit(0)
        for i in range(1, args.steps):
            nxt = submit(i)
            rep.match_batch_wait(pending)
            pending = nxt
        rep.match_batch_wait(pending)
        torch.cuda.synchronize()
        return B * args.steps / (time.perf_counter() - t0)

    d_hints = torch.from_numpy(hints).to(dev)
    d_ranges = torch.from_numpy(ranges).to(dev)
    d_cloud = torch.from_numpy(cloud_all).to(dev)
    d_coffs = torch.from_numpy(c_offs).to(dev)
    d_poses = torch.empty((B, 3), dtype=torch.float32, device=dev)
    d_cov = torch.empty((B, 9), dtype=torch.float32, device=dev)
    d_origo = torch.empty((B, 2), dtype=torch.float32, device=dev)
    max_cloud = int(np.diff(c_offs).max())
    stream = torch.cuda.current_stream().cuda_stream

    def dev_projected():
        rep.match_batch_projected_device(B, d_hints.data_ptr(), d_ranges.data_ptr(), None, d_poses.data_ptr(),
                                         d_cov.data_ptr(), d_origo.data_ptr(), stream)

    def dev_cloud():
        rep.match_batch_cloud_device(B, d_hints.data_ptr(), d_cloud.data_ptr(), d_coffs.data_ptr(), max_cloud, None,
                                     d_poses.data_ptr(), d_cov.data_ptr(), d_origo.data_ptr(), stream)

    def dev_ranges():
        rep.match_batch_ranges_device(B, d_hints.data_ptr(), d_ranges.data_ptr(), d_poses.data_ptr(), d_cov.data_ptr(),
                                      stream)

    def time_device(fn):
        for _ in range(args.warmup):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            fn()
        e1.record()
        e1.synchronize()
        return B * args.steps / (e0.elapsed_time(e1) * 1e-3)

    arms = {"projected_host": lambda: time_host(submit_projected), "cloud_host": lambda: time_host(submit_cloud),
            "ranges_host": lambda: time_host(submit_ranges), "projected_device": lambda: time_device(dev_projected),
            "cloud_device": lambda: time_device(dev_cloud), "ranges_device": lambda: time_device(dev_ranges)}
    rates = {a: [] for a in arms}
    for _ in range(args.rounds):
        for name, fn in arms.items():
            rates[name].append(fn())

    # (a) against (b): the same scans, projected in the kernel or on the host
    a = rep.match_batch_projected(hints, ranges)
    b = rep.match_batch_cloud(hints, cloud_all, c_offs)
    diff = max(float(np.abs(x - y).max()) for x, y in zip(a, b))
    out = {"workload": f"{B} x {proj['n_beams']}-beam scans, {bench.MAP_SIZE}^2 x {bench.LEVELS} levels",
           "card": card, "rounds": args.rounds, "steps": args.steps, "unit": "scans/s",
           "h2d_input_bytes_per_scan": {"projected": 4 * proj["n_beams"], "ranges": 4 * proj["n_beams"],
                                        "cloud": round(12 * c_offs[-1] / B, 1)},
           "max_abs_diff_projected_vs_cloud": diff}
    for name, v in rates.items():
        out[name] = {"median": round(float(np.median(v))), "min": round(min(v)), "max": round(max(v))}
    print(json.dumps(out), flush=True)
    for x in h_hints + h_ranges + h_cloud + h_poses + h_cov + h_origo:
        x.free()
    rep.close()


if __name__ == "__main__":
    main()
