"""Where a host-buffer scoring call's time goes: hsb_likelihood_batch and hsb_covariance_batch on a 2048^2 level (the
arms of scripts/single_queries.py that move megabytes or launch many poses), split into the call's host-clock time and
the device time of its host-to-device copies, its kernels and its device-to-host copies, from torch.profiler's CUDA
activity records over --calls calls per arm after a warm-up.  The rest of a call is host work: staging, launch and
synchronise overheads (the copies and the kernel may overlap the host's staging, so the parts need not add up).

    python scripts/score_breakdown.py [--libs hector_slam_b200/lib/libhsb200.so,/path/to/other.so] [--calls 20]

Prints one JSON line per library and arm, in ms per call, with the card and power limit read in the same run.
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

from single_queries import RES, SCAN, plane  # noqa: E402

ARMS = [("likelihood", "shared", 65536, SCAN), ("likelihood", "per_pose", 1024, SCAN),
        ("likelihood", "per_pose", 65536, 16), ("covariance", "per_pose", 1024, SCAN)]


def worker(calls):
    import torch
    from torch.profiler import ProfilerActivity, profile

    from hector_slam_b200 import capi

    lib = capi.load_library()
    torch.cuda.init()
    for mode, mode_name in ((capi.GATHER_LDG, "ldg"), (capi.GATHER_TEX, "tex")):
        rep = capi.MapRepB200(RES, 2048, levels=1, gather_mode=mode)
        rep.upload_level(0, plane(2048, 1))
        origin = rep.map_origin(0)
        rng = np.random.default_rng(3)
        for call, layout, B, n in ARMS:
            poses = np.concatenate([origin + RES * rng.uniform(512, 1536, (B, 2)), rng.uniform(-np.pi, np.pi, (B, 1))],
                                   axis=1).astype(np.float32)
            pts = rng.uniform(-200, 200, ((B if layout == "per_pose" else 1) * n, 2)).astype(np.float32)
            offsets = np.arange(B + 1, dtype=np.int32) * n
            offp, n_shared = (offsets.ctypes.data, 0) if layout == "per_pose" else (None, n)
            out = [np.zeros((B, 9), np.float32) for _ in range(2)]
            if call == "likelihood":
                fn = lambda: lib.hsb_likelihood_batch(rep.h, 0, B, poses.ctypes.data, pts.ctypes.data, offp, n_shared,
                                                      out[0].ctypes.data)
            else:
                fn = lambda: lib.hsb_covariance_batch(rep.h, 0, B, poses.ctypes.data, pts.ctypes.data, offp, n_shared,
                                                      out[0].ctypes.data, out[1].ctypes.data)
            for _ in range(5):
                assert fn() == 0
            wall = []
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                for _ in range(calls):
                    t0 = time.perf_counter()
                    fn()
                    wall.append(time.perf_counter() - t0)
            parts = {"h2d": 0.0, "kernel": 0.0, "d2h": 0.0}
            copies = 0
            for e in prof.events():
                if e.device_type != torch.autograd.DeviceType.CUDA:
                    continue
                t = e.time_range.elapsed_us() / 1e3 / calls
                if "HtoD" in e.name:
                    parts["h2d"] += t
                    copies += 1
                elif "DtoH" in e.name:
                    parts["d2h"] += t
                elif "Memcpy" not in e.name and "Memset" not in e.name:
                    parts["kernel"] += t
            name = f"{call}_{layout}{'' if n == SCAN else f'{n}pt'}_{B}_{mode_name}"
            print(json.dumps({"arm": name, "wall_p50": round(float(np.median(wall)) * 1e3, 4),
                              **{k: round(v, 4) for k, v in parts.items()}, "h2d_copies": copies / calls}), flush=True)
        rep.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--libs", default=os.path.join(ROOT, "hector_slam_b200", "lib", "libhsb200.so"))
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--worker", action="store_true")
    args = ap.parse_args()
    if args.worker:
        worker(args.calls)
        return
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip()
    except OSError:
        card = "unknown"
    for p in [os.path.abspath(p) for p in args.libs.split(",")]:
        res = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", "--calls", str(args.calls)],
                             env=dict(os.environ, HSB_LIB_PATH=p), capture_output=True, text=True, check=True)
        for line in res.stdout.strip().splitlines():
            if line.startswith("{"):
                print(json.dumps({"lib": p, "card": card, **json.loads(line)}), flush=True)


if __name__ == "__main__":
    main()
