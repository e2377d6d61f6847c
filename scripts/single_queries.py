"""Per-call time of one handle's map queries: hsb_raycast_batch and hsb_get_dist_batch at B = 8, 1024 and 65536 rays on
a 2048^2 level, hsb_download_occupancy of a whole 2048^2 and 4096^2 level, and pose scoring on the 2048^2 level in both
gather modes (ldg / tex): hsb_likelihood_batch of B = 8, 1024 and 65536 poses against one shared 1081-point scan, of
B = 8, 1024 and 8192 poses with a 1081-point scan each, and of 65536 poses with a 16-point scan each (the most sessions
per scanned point); hsb_covariance_batch of B = 8, 1024 and 16384 poses against one shared scan and of 8 and 1024 poses
with a scan each.

Each call ends in a stream synchronise, so a host clock around the call is its time.  The map is a seeded log-odds
plane with about 3 % occupied cells; the rays are seeded cell rays and world rays of up to 20 m; the poses lie in the
map's middle, the scans' endpoints within 10 m of them.  Every arm is warmed up first and then called --calls times (a
tenth of that above 1024 poses or rays and at 4096^2).

Two libraries can be compared (--libs A,B: the first is the default build): each round runs one worker process per
library, their order alternating from round to round, and the per-call samples of all rounds are pooled per library.
Every call's results are hashed, and the hashes of the libraries must agree.  Prints one JSON line per library with the
p50 / p99 of each arm in ms, each round's p50 (the spread between rounds of one build), and the card and power limit
read in the same run.

    python scripts/single_queries.py [--libs hector_slam_b200/lib/libhsb200.so,/path/to/other.so] [--rounds 5]
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

RES = 0.05
RAYS = (8, 1024, 65536)
OCC = (2048, 4096)
SCAN = 1081
# (call, layout, poses B, points per scan)
SCORES = [("likelihood", "shared", 8, SCAN), ("likelihood", "shared", 1024, SCAN), ("likelihood", "shared", 65536, SCAN),
          ("likelihood", "per_pose", 8, SCAN), ("likelihood", "per_pose", 1024, SCAN),
          ("likelihood", "per_pose", 8192, SCAN), ("likelihood", "per_pose", 65536, 16),
          ("covariance", "shared", 8, SCAN), ("covariance", "shared", 1024, SCAN), ("covariance", "shared", 16384, SCAN),
          ("covariance", "per_pose", 8, SCAN), ("covariance", "per_pose", 1024, SCAN)]


def plane(n, seed):
    rng = np.random.default_rng(seed)
    p = rng.uniform(-2.0, -0.1, (n, n)).astype(np.float32)
    p[rng.random((n, n)) < 0.03] = np.float32(1.5)
    return p


def worker(calls):
    import ctypes as C

    from hector_slam_b200 import capi

    lib = capi.load_library()
    times, digest = {}, hashlib.sha256()

    def check(st, rep):
        if st != 0:
            raise capi.HsbError(st, lib.hsb_last_error(rep.h).decode())

    def timed(name, n, fn):
        for _ in range(10):
            fn()
        ts = []
        for _ in range(n):
            t0 = time.perf_counter()
            fn()
            ts.append(time.perf_counter() - t0)
        times[name] = ts

    rep = capi.MapRepB200(RES, 2048, levels=1)
    rep.upload_level(0, plane(2048, 1))
    origin = rep.map_origin(0)
    rng = np.random.default_rng(2)
    for B in RAYS:
        n = calls if B < 65536 else max(1, calls // 10)
        cb = rng.integers(0, 2048, (B, 2)).astype(np.int32)
        ce = np.clip(cb + rng.integers(-400, 401, (B, 2)), 0, 2047).astype(np.int32)
        wb = (origin + RES * rng.uniform(0, 2048, (B, 2))).astype(np.float32)
        ang = rng.uniform(-np.pi, np.pi, B)
        we = (wb + 20.0 * np.stack([np.cos(ang), np.sin(ang)], axis=1)).astype(np.float32)
        dist, hit = np.zeros(B, np.float32), np.zeros((B, 2), np.int32)
        gd, gh, gf = np.zeros(B, np.float32), np.zeros((B, 2), np.float32), np.zeros(B, np.int32)
        timed(f"raycast_{B}", n, lambda: check(lib.hsb_raycast_batch(rep.h, 0, B, cb.ctypes.data, ce.ctypes.data,
                                                                      dist.ctypes.data, hit.ctypes.data), rep))
        timed(f"get_dist_{B}", n, lambda: check(lib.hsb_get_dist_batch(rep.h, 0, B, wb.ctypes.data, we.ctypes.data,
                                                                        gd.ctypes.data, gh.ctypes.data,
                                                                        gf.ctypes.data), rep))
        for a in (dist, hit, gd, gh, gf):
            digest.update(a.tobytes())
    rep.close()
    for mode, mode_name in ((capi.GATHER_LDG, "ldg"), (capi.GATHER_TEX, "tex")):
        rep = capi.MapRepB200(RES, 2048, levels=1, gather_mode=mode)
        rep.upload_level(0, plane(2048, 1))
        rng = np.random.default_rng(3)
        for call, layout, B, n in SCORES:
            poses = np.concatenate([origin + RES * rng.uniform(512, 1536, (B, 2)), rng.uniform(-np.pi, np.pi, (B, 1))],
                                   axis=1).astype(np.float32)
            scans = B if layout == "per_pose" else 1
            pts = rng.uniform(-200, 200, (scans * n, 2)).astype(np.float32)   # level-0 cells: 10 m
            offsets = np.arange(B + 1, dtype=np.int32) * n if layout == "per_pose" else None
            offp, n_shared = (offsets.ctypes.data, 0) if layout == "per_pose" else (None, n)
            if call == "likelihood":
                outs = (np.zeros(B, np.float32),)
                fn = lambda: check(lib.hsb_likelihood_batch(rep.h, 0, B, poses.ctypes.data, pts.ctypes.data, offp,
                                                            n_shared, outs[0].ctypes.data), rep)
            else:
                outs = (np.zeros((B, 9), np.float32), np.zeros((B, 9), np.float32))
                fn = lambda: check(lib.hsb_covariance_batch(rep.h, 0, B, poses.ctypes.data, pts.ctypes.data, offp,
                                                            n_shared, outs[0].ctypes.data, outs[1].ctypes.data), rep)
            name = f"{call}_{layout}{'' if n == SCAN else f'{n}pt'}_{B}_{mode_name}"
            timed(name, calls if B <= 1024 else max(1, calls // 10), fn)
            for a in outs:
                digest.update(a.tobytes())
        rep.close()
    for n_cells in OCC:
        rep = capi.MapRepB200(RES, n_cells, levels=1)
        rep.upload_level(0, plane(n_cells, n_cells))
        out = np.zeros((n_cells, n_cells), np.int8)
        timed(f"occupancy_{n_cells}", calls if n_cells < 4096 else max(1, calls // 10),
              lambda: check(lib.hsb_download_occupancy(rep.h, 0, C.c_void_p(out.ctypes.data)), rep))
        digest.update(out.tobytes())
        rep.close()
    print(json.dumps({"times": times, "digest": digest.hexdigest()}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--libs", default=os.path.join(ROOT, "hector_slam_b200", "lib", "libhsb200.so"))
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=300)
    ap.add_argument("--worker", action="store_true")
    args = ap.parse_args()
    if args.worker:
        worker(args.calls)
        return
    libs = [os.path.abspath(p) for p in args.libs.split(",")]
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip()
    except OSError:
        card = "unknown"
    pooled = {p: {} for p in libs}
    per_round = {p: {} for p in libs}
    digests = set()
    for r in range(args.rounds):
        for p in (libs if r % 2 == 0 else libs[::-1]):
            env = dict(os.environ, HSB_LIB_PATH=p)
            res = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", "--calls", str(args.calls)],
                                 env=env, capture_output=True, text=True, check=True)
            w = json.loads(res.stdout.strip().splitlines()[-1])
            digests.add(w["digest"])
            for k, v in w["times"].items():
                pooled[p].setdefault(k, []).extend(v)
                per_round[p].setdefault(k, []).append(round(float(np.percentile(np.asarray(v) * 1e3, 50)), 4))
    for p in libs:
        line = {"lib": p, "rounds": args.rounds, "card": card, "results_identical": len(digests) == 1}
        for k, v in pooled[p].items():
            line[f"{k}_ms_p50"] = round(float(np.percentile(np.asarray(v) * 1e3, 50)), 4)
            line[f"{k}_ms_p99"] = round(float(np.percentile(np.asarray(v) * 1e3, 99)), 4)
            line[f"{k}_ms_p50_rounds"] = per_round[p][k]
        print(json.dumps(line), flush=True)
    if len(digests) != 1:
        sys.exit("the libraries' results differ")


if __name__ == "__main__":
    main()
