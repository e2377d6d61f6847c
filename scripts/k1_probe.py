"""K1 diagnostics on the BASELINE batch (4096 scans, 2048^2 3-level map): launch-shape / staging variants timed
with CUDA events (8 input batches cycled, like bench.py's `value`), bit-equality of their results, and the
per-scan timeline (%globaltimer at start / after each level / end, %smid) of the default launch.

  python scripts/k1_probe.py [B] > gpurun_out/k1_probe.log
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from hector_slam_b200 import capi  # noqa: E402

B = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
dev = torch.device("cuda", 0)
rep = capi.MapRepB200(bench.RES, bench.MAP_SIZE, levels=3, update_factor_free=0.4, update_factor_occupied=0.9)
world, poses, pts, offs, hints = bench.make_workload(0, B)
bench.build_map_on_gpu(rep, world)
nbuf = 8 if B <= 8192 else 2
d_pts = [torch.from_numpy(pts).to(dev).clone() for _ in range(nbuf)]
d_hints = [torch.from_numpy(hints).to(dev).clone() for _ in range(nbuf)]
d_offs = torch.from_numpy(offs).to(dev)
d_poses = torch.empty((B, 3), dtype=torch.float32, device=dev)
d_cov = torch.empty((B, 9), dtype=torch.float32, device=dev)
stream = torch.cuda.current_stream().cuda_stream


def run(k=0):
    rep.match_batch_device(B, d_hints[k % nbuf].data_ptr(), d_pts[k % nbuf].data_ptr(), d_offs.data_ptr(), 0, bench.N_PTS,
                           d_poses.data_ptr(), d_cov.data_ptr(), stream)


def timed(iters=20):
    for i in range(5):
        run(i)
    torch.cuda.synchronize()
    best = []
    for rep_i in range(3):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(iters):
            run(i)
        e1.record()
        torch.cuda.synchronize()
        best.append(e0.elapsed_time(e1) / iters)
    return min(best), float(np.median(best))


base = dict(warps_per_scan=0, scans_per_block=0, stage_smem=1, unroll=0, partial=0, prefetch=0, trace=0, seq=0, pace=0, auto_group=0)
variants = [
    ("G=1 unstaged (round-1 shape)", {}),
    ("G=1 partial staging", dict(partial=1)),
    ("auto (grouped, staged prefix)", dict(auto_group=1, partial=1)),
]
for G in (28, 14):
    for pace in (0, 1):
        for stage, part in ((0, 0), (1, 1)):
            variants.append((f"G={G} pace={pace} " + ("staged prefix" if stage else "unstaged"),
                             dict(warps_per_scan=1, scans_per_block=G, pace=pace, stage_smem=stage, partial=part)))
if B > 8192:   # many waves: only the staging question matters
    variants = [("default", {}), ("always fully staged", dict(stage_smem=2)), ("never staged", dict(stage_smem=0))]
ref = None
for name, kw in variants:
    t = dict(base)
    t.update(kw)
    try:
        rep.set_tuning(**t)
        run(0)
        torch.cuda.synchronize()
        got = d_poses.cpu().numpy().copy()
        if ref is None:
            ref = got
        same = np.array_equal(got, ref)
        dmax = float(np.abs(got - ref).max())
        mn, med = timed()
        print(f"{name:34s} {mn * 1e3:8.1f} us (median {med * 1e3:8.1f})  {B / mn / 1e3:6.2f} M matches/s   "
              f"bit-identical to default: {same} (max diff {dmax:.1e})", flush=True)
    except Exception as e:  # noqa: BLE001
        print(f"{name:34s} failed: {e}", flush=True)


def timeline(label, kw):
    t = dict(base)
    t.update(kw)
    t["trace"] = 1
    rep.set_tuning(**t)
    for i in range(3):
        run(i)
    torch.cuda.synchronize()
    run(3)
    torch.cuda.synchronize()
    tr = rep.read_trace(B).astype(np.int64)
    t0 = tr[:, 0].min()
    start, end = (tr[:, 0] - t0) / 1e3, (tr[:, 4] - t0) / 1e3
    dur = end - start
    lv = np.diff(tr[:, 0:5], axis=1) / 1e3
    sm = tr[:, 7]
    print(f"--- timeline: {label} (us, %globaltimer resolution ~1 us)")
    print(f"span first start -> last end {end.max():.1f}; starts: p50 {np.median(start):.1f} max {start.max():.1f}; "
          f"ends: min {end.min():.1f} p10 {np.percentile(end, 10):.1f} p50 {np.median(end):.1f} p90 {np.percentile(end, 90):.1f} max {end.max():.1f}")
    print(f"per-scan duration: min {dur.min():.1f} p10 {np.percentile(dur, 10):.1f} p50 {np.median(dur):.1f} "
          f"p90 {np.percentile(dur, 90):.1f} max {dur.max():.1f}")
    print("per-level duration p50 (coarse -> fine, + tail):", " ".join(f"{np.median(lv[:, k]):.1f}" for k in range(4)))
    full = sum(rep.level_evals())
    ran = tr[:, 5]   # evaluations each scan ran (a level ends at its first evaluation that leaves the pose unchanged)
    hist = np.bincount(ran, minlength=full + 1)
    print(f"evaluations run per scan (of {full}), count: " + " ".join(f"{k}:{c}" for k, c in enumerate(hist) if c) +
          f"; {1 - ran.sum() / (full * ran.size):.1%} of all evaluations skipped")
    cnt = np.bincount(sm, minlength=torch.cuda.get_device_properties(0).multi_processor_count)
    per_sm_end = np.array([end[sm == s].max() if (sm == s).any() else 0 for s in range(cnt.size)])
    print(f"scans per SM: min {cnt[cnt > 0].min()} max {cnt.max()} (SMs used {(cnt > 0).sum()}); "
          f"last end per SM: min {per_sm_end[cnt > 0].min():.1f} p50 {np.median(per_sm_end[cnt > 0]):.1f} max {per_sm_end.max():.1f}")
    for c in sorted(set(cnt[cnt > 0])):
        sel = np.isin(sm, np.flatnonzero(cnt == c))
        print(f"  SMs with {c} scans: {int((cnt == c).sum())} SMs, scan duration p50 {np.median(dur[sel]):.1f}, last end p50 "
              f"{np.median(per_sm_end[cnt == c]):.1f} max {per_sm_end[cnt == c].max():.1f}")
    edges = np.arange(0, end.max() + 10, 10.0)
    alive = [(int(((start <= e) & (end > e)).sum())) for e in edges]
    print("scans alive at t = 0,10,20.. us:", alive)


def slot_study():
    """Which scans are slow: the same ones in two runs (data) or the same warp slots (scheduling)?"""
    t = dict(base)
    t["trace"] = 1
    rep.set_tuning(**t)
    durs, slots = [], []
    for k in range(3):
        run(0)
        torch.cuda.synchronize()
        tr = rep.read_trace(B).astype(np.int64)
        durs.append((tr[:, 4] - tr[:, 0]) / 1e3)
        slots.append(tr[:, 6])
    c01 = np.corrcoef(durs[0], durs[1])[0, 1]
    print(f"--- slot study: correlation of per-scan durations between two runs on identical inputs: {c01:.3f}")
    d, w = durs[2], slots[2]
    print("duration p50 by hardware warp slot (%warpid):")
    for slot in sorted(set(w.tolist())):
        sel = w == slot
        print(f"  warpid {slot:2d} (scheduler {slot % 4}): n={int(sel.sum()):4d} p50 {np.median(d[sel]):6.1f} us")


if B > 8192:
    rep.set_tuning(**base)
    rep.close()
    sys.exit(0)
timeline("G=1 unstaged (round-1 shape)", {})
slot_study()
timeline("auto (grouped, staged prefix)", dict(auto_group=1, partial=1))
rep.set_tuning(**base)
rep.close()
