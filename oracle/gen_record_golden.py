"""Generate tests/golden/record.npz from the COMPILED REFERENCE (oracle/_ref/libhsref_record.so).

TEST INFRASTRUCTURE.  Run in the build container, where the reference headers exist:

    make -C oracle && make -C oracle -f record.mk && python oracle/gen_record_golden.py

record.npz holds what ScanMatcher::matchData (matcher/ScanMatcher.h:54-190) reports to its DrawInterface /
HectorDebugInfoInterface — the start arrow of every level, then per reported evaluation the Hessian and the arrow — on the
match3 / match1 golden maps: ordinary scans, an empty scan, a scan entirely out of the map, a scan whose first step hits
the +-0.2 rad clamp, a single evaluation per level (maxIterations = -1) and uneven iteration counts.
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.record_oracle import RecordOracle, port_hooks  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")

RECORD_CASES = (
    # (name, golden map, scan source, hint offset (x, y, psi), maxIterations per level or None for the defaults)
    ("match3_s0", "match3", 0, (0, 0, 0), None),
    ("match3_s1", "match3", 1, (0, 0, 0), None),
    ("match3_s2", "match3", 2, (0, 0, 0), None),
    ("match3_s3", "match3", 3, (0, 0, 0), None),
    ("match1_s0", "match1", 0, (0, 0, 0), None),
    ("match1_s1", "match1", 1, (0, 0, 0), None),
    ("empty", "match3", "empty", (0, 0, 0), None),
    ("far", "match3", "far", (0, 0, 0), None),
    ("clamp", "match1", "near6", (0.0, 0.0, 0.3), None),
    ("one_eval", "match3", 4, (0, 0, 0), [-1, -1, -1]),
    ("iters_214", "match3", 6, (0.05, -0.05, 0.02), [2, 1, 4]),
)


def record_inputs(g, src, offset):
    """the scan and hint of one RECORD_CASES entry on golden `g`"""
    if src == "empty":
        scan = np.zeros((0, 2), np.float32)
        k = 0
    elif src == "near6":
        # the six endpoints of scan 0 closest to the sensor: rotation is barely constrained, the first step in psi
        # is beyond the +-0.2 rad clamp (ScanMatcher.h:209-215)
        sc = g["scans"][0]
        scan = np.ascontiguousarray(sc[np.argsort(np.hypot(sc[:, 0], sc[:, 1]), kind="stable")[:6]], np.float32)
        k = 0
    elif src == "far":
        scan = (g["scans"][0] + np.float32(1e5)).astype(np.float32)   # every endpoint out of the map: H = 0
        k = 0
    else:
        k = int(src)
        scan = g["scans"][k]
    hint = (g["hints"][k] + np.float32(offset)).astype(np.float32)
    return scan, hint


def load_map(kind, name):
    g = np.load(os.path.join(OUT, name + ".npz"))
    size, levels = int(g["size"]), int(g["levels"])
    orc = RecordOracle(kind, float(g["res"]), size, levels)
    for l in range(levels):
        p = np.zeros((size >> l) ** 2, np.float32)
        p[g[f"map_idx{l}"]] = g[f"map_val{l}"]
        orc.set_logodds(l, p.reshape(size >> l, size >> l))
    return g, orc


def record_arrays(kind="reference"):
    """The arrays of record.npz, from the compiled reference's hooks or (kind="port") the C port's record reduced to the
    hooks' view (drawn points are counted by the reference only: zeros)."""
    maps = {name: load_map(kind, name) for name in ("match3", "match1")}
    out = {}
    for name, mp, src, offset, iters in RECORD_CASES:
        g, orc = maps[mp]
        scan, hint = record_inputs(g, src, offset)
        if kind == "reference":
            pose, cov, hooks, npts = orc.match_record(hint, scan, iters)
        else:
            pose, cov, rec = orc.match_record(hint, scan, iters)
            hooks, npts = port_hooks(orc, rec, scan.shape[0], iters), np.zeros(orc.levels, np.int32)
        out[f"{name}_hint"] = hint
        out[f"{name}_iters"] = np.int32(iters if iters is not None else [0] * orc.levels)
        out[f"{name}_pose"] = pose
        out[f"{name}_cov"] = cov.reshape(9)
        out[f"{name}_hooks"] = hooks
        out[f"{name}_points"] = npts
    out["cases"] = np.array([c[0] for c in RECORD_CASES])
    for g, orc in maps.values():
        orc.close()
    return out


if __name__ == "__main__":
    np.savez_compressed(os.path.join(OUT, "record.npz"), **record_arrays())
