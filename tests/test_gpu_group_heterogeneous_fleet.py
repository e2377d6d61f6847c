"""Heterogeneous groups (hsb_group_create_heterogeneous) at fleet size, and in each way the members of one may differ.

GPU.  Every member has a twin handle driven by single calls and a replica handle in a heterogeneous replica group that
lists the handles in the owner's order; every comparison is bit for bit.
  - test_fleet_300: 300 members round-robin over the 1-, 2- and 3-level classes (the 3-level class in both gather modes)
    and three small geometries.  Full steps and permuted subsets of K = 121 and K = 129 in all four input kinds, with
    nowait and map_without_matching; subset packs of K = 129 and 121 and a full pack, each block equal to the member's
    single pack and each unpacked on the replica group; subset resets of K = 129 and 121 followed by steps, the next
    full pack shipping the clear records.  K = 129 goes past 128 sessions: the subset kernels that list up to 4096
    members, the second 128-session pass of the pack and unpack layout, and the first-fit loop over more than 32
    blocks, all with per-member level counts.
  - test_group_kinds: a small group for each way its members may differ on their own — gather mode at one level count
    (the group kernels in MODE_ANY), level count at one gather mode (TEX and LDG: the group kernels in that mode, each
    session, block and reset on its member's own level count), and per-level iteration counts only (each member's own
    evaluation counts): steps, the match at W = 1 and 8, scoring, tile replication and a subset reset."""
import numpy as np
import pytest

from test_gpu_group_match import assert_match
from test_gpu_group_score import assert_sessions, hypotheses, thinned
from test_gpu_group_subset import (KINDS, assert_same_session, assert_same_state, beam_angles, bits, close_all,
                                   geometry, group_step, member_cloud, member_transform, scan_of, session_data,
                                   single_step)
from test_gpu_group_tiles import HEADER_WORDS, group_header_words

pytestmark = pytest.mark.gpu

F32 = np.float32
TEX, LDG = 2, 1   # capi.GATHER_TEX, capi.GATHER_LDG
CLEARED_WORD = 4 + 4 * 8   # HSB_TILE_CLEARED_WORD (hsb_internal.h)
# map_size_x, map_size_y, map_resolution, start
GEOMS = [(128, 128, 0.1, (0.5, 0.5)), (136, 104, 0.1, (0.3, 0.6)), (96, 160, 0.05, (0.5, 0.5))]


def fleet_spec(s):
    """member s of the 300-member fleet: (geometry, levels, gather mode, max_iterations)"""
    levels = 1 + s % 3
    mode = LDG if levels == 3 and (s // 3) % 2 else TEX
    return GEOMS[(s // 3) % 3] + (levels, mode, None)


def make_rep(spec, s):
    from hector_slam_b200 import capi

    sx, sy, res, start, levels, mode, iters = spec
    rep = capi.MapRepB200(res, sx, sy, levels=levels, start=start, max_iterations=iters,
                          update_factor_free=0.4 + 0.02 * (s % 5), update_factor_occupied=0.6 + 0.1 * (s % 4),
                          gather_mode=mode)
    dist, ang = ((0.0, 0.0), (0.15, 0.1), (0.3, 0.5))[(s // 2) % 3]
    rep.setMapUpdateMinDistDiff(dist)
    rep.setMapUpdateMinAngleDiff(ang)
    g = geometry(s // 2)
    rep.set_scan_format(**g)
    rep.set_laser_projection(**g, range_cutoff=30.0)
    rep.set_cloud_format(member_transform(s), **member_cloud(s))
    assert rep.gather_mode == mode and rep.levels == levels
    return rep


class HetFleet:
    """A heterogeneous group of members `specs`, their twins and replicas, and every member's trajectory position."""

    def __init__(self, specs, ticks):
        from hector_slam_b200 import capi, synth

        self.specs, self.M = specs, len(specs)
        self.grp = [make_rep(sp, s) for s, sp in enumerate(specs)]
        self.one = [make_rep(sp, s) for s, sp in enumerate(specs)]
        self.replica = [make_rep(sp, s) for s, sp in enumerate(specs)]
        self.g = capi.SlamGroup(self.grp, heterogeneous=True)
        self.rg = capi.SlamGroup(self.replica, heterogeneous=True)
        self.data = []
        for s, sp in enumerate(specs):
            g = geometry(s // 2)
            d = session_data(1300 + s, ticks, g)
            d["scans"] = [np.ascontiguousarray(synth.ranges_to_points(r, 1.0 / sp[2], beam_angles(g)), F32)
                          for r in d["ranges"]]
            self.data.append(d)
        self.at = [0] * self.M
        self.covs = [np.full((3, 3), 5.0, F32) for _ in range(self.M)]

    def levels(self, j):
        return self.specs[j][4]

    def tick(self, kind, members, nowait, rng, without_share=0.2):
        sel = list(range(self.M)) if members is None else members
        without = [bool(rng.random() < without_share) and self.at[j] > 0 for j in sel]
        hints = np.asarray([self.data[j]["truth" if w else "hints"][self.at[j]] for j, w in zip(sel, without)],
                           F32).reshape(len(sel), 3)
        scans = [thinned(kind, scan_of(kind, self.data[j], self.at[j])) for j in sel]
        cov = np.stack([self.covs[j] for j in sel])
        launches = self.grp[0].launch_count
        out = group_step(self.g, kind, hints, scans, without, members=members, nowait=nowait, cov=cov)
        assert self.grp[0].launch_count - launches == 3, kind
        for i, j in enumerate(sel):
            ref = single_step(self.one[j], kind, hints[i], scans[i], without[i], cov=self.covs[j].copy())
            assert_same_session(out, i, ref, (kind, i, j))
            self.covs[j] = out[1][i].copy()
            self.at[j] += 1

    def assert_states(self, tag, members=None, probe=False):
        for j in range(self.M) if members is None else members:
            assert_same_state(self.grp[j], self.one[j], (tag, j), probe=probe, levels=self.levels(j))

    def replicate(self, members, tag, check=None, cleared=()):
        """Pack the members' dirty tiles (reset) on the group and on the twins one by one: every block (or those of the
        sessions in `check`) equals the twin's single pack, except that of a member in `cleared` (reset by the group
        since its last pack, where hsb_reset leaves its twin shipping whole levels): that block carries the clear record
        of all its own levels.  Then unpack on the replica group.  -> the group header"""
        import torch

        K = self.M if members is None else len(members)
        sel = list(range(self.M)) if members is None else members
        cells = sum(r.level_info(l)[0] * r.level_info(l)[1] for r in self.grp for l in range(r.levels))
        words = group_header_words(K) + K * HEADER_WORDS + cells
        buf = torch.zeros(words, dtype=torch.float32, device="cuda")
        single = torch.zeros(HEADER_WORDS + cells, dtype=torch.float32, device="cuda")
        st = torch.cuda.current_stream().cuda_stream
        self.g.pack_dirty_device(buf.data_ptr(), 4 * words, True, st, members=members)
        torch.cuda.synchronize()
        hdr = buf[:group_header_words(K)].view(torch.int32).cpu().numpy()
        assert hdr[1] == K and hdr[2] == max(sp[4] for sp in self.specs) and hdr[3] == 0, (tag, hdr[:5])
        for k, j in enumerate(sel):
            single.zero_()
            self.one[j].pack_dirty_device(single.data_ptr(), 4 * single.numel(), True, st)
            torch.cuda.synchronize()
            if check is not None and k not in check:
                continue
            assert int(hdr[5 + 2 * k]) == j, (tag, k)
            start = int(hdr[6 + 2 * k])
            if j in cleared:
                blk = buf[start:start + HEADER_WORDS].view(torch.int32).cpu().numpy()
                assert blk[1] == self.levels(j) and blk[2] == 0, (tag, k, j, blk[:4])
                assert blk[CLEARED_WORD] == (1 << self.levels(j)) - 1, (tag, k, j, blk[CLEARED_WORD])
                continue
            head = single[:HEADER_WORDS].view(torch.int32)
            assert int(head[1]) == self.levels(j), (tag, k, j)
            n = HEADER_WORDS + int(head[3])
            assert torch.equal(buf[start:start + n].view(torch.int32), single[:n].view(torch.int32)), (tag, k, j)
        self.rg.unpack_dirty_device(buf.data_ptr(), 4 * words, st)
        torch.cuda.synchronize()
        assert self.replica[0].replication_overflows(reset=True) == 0, tag
        return hdr

    def assert_replicas(self, tag):
        for j in range(self.M):
            for l in range(self.levels(j)):
                assert np.array_equal(bits(self.replica[j].download_level(l)), bits(self.grp[j].download_level(l))), \
                    (tag, j, l)

    def close(self):
        self.rg.close()
        self.g.close()
        close_all(self.grp, self.one, self.replica)


def test_fleet_300(hsb_lib):
    M = 300
    f = HetFleet([fleet_spec(s) for s in range(M)], 12)
    try:
        assert sorted({sp[4] for sp in f.specs}) == [1, 2, 3] and {sp[5] for sp in f.specs} == {TEX, LDG}
        rng = np.random.default_rng(41)
        samples = [0, 31, 32, 120, 121, 127, 128, 129, 255, 256, M - 1]
        plan = [(None, False), (129, False), (121, True), (None, True), (129, True), (121, False)]
        for t, (K, nowait) in enumerate(plan):
            members = None if K is None else [int(j) for j in rng.permutation(M)[:K]]
            f.tick(KINDS[t % 4], members, nowait, rng)
        f.assert_states("steps")
        f.assert_states("steps, probed", members=samples, probe=True)
        # tiles: subset packs of 129 (the 4096-member subset kernel) and 121 sessions, then the rest in a full pack
        sub129 = [int(j) for j in rng.permutation(M)[:129]]
        f.replicate(sub129, "pack 129")
        f.replicate([int(j) for j in rng.permutation(M)[:121]], "pack 121")
        f.replicate(None, "pack all")
        f.assert_replicas("replicas")
        f.assert_states("after packs")
        # resets of 129 and 121 members, steps, and the clear records shipped by the next full pack
        was_reset = set()
        for K in (129, 121):
            members = [int(j) for j in rng.permutation(M)[:K]]
            was_reset.update(members)
            f.g.reset(members=members)
            for j in members:
                f.one[j].reset()
            f.assert_states(("reset", K))
        f.tick("ranges", None, True, rng, without_share=0.0)
        f.tick("endpoints", sub129, False, rng)
        f.assert_states("after reset and steps")
        f.replicate(None, "pack after reset", check=set(samples) | set(range(0, M, 7)), cleared=was_reset)
        f.assert_replicas("replicas after reset")
    finally:
        f.close()


# each way the members of a heterogeneous group may differ on their own
KIND_SPECS = {
    "modes": [GEOMS[0] + (3, TEX, None), GEOMS[1] + (3, LDG, None), GEOMS[2] + (3, TEX, None), GEOMS[0] + (3, LDG, None)],
    "levels_tex": [GEOMS[0] + (1, TEX, None), GEOMS[1] + (2, TEX, None), GEOMS[2] + (3, TEX, None),
                   GEOMS[0] + (4, TEX, None)],
    "levels_ldg": [GEOMS[1] + (3, LDG, None), GEOMS[0] + (1, LDG, None), GEOMS[2] + (2, LDG, None),
                   GEOMS[0] + (4, LDG, None)],
    "iterations": [GEOMS[0] + (3, TEX, None), GEOMS[1] + (3, TEX, [6, 0, -1]), GEOMS[2] + (3, TEX, [2, 4, 1]),
                   GEOMS[0] + (3, TEX, [0, -1, 7])],
}


@pytest.mark.parametrize("kind", list(KIND_SPECS))
def test_group_kinds(hsb_lib, kind):
    f = HetFleet(KIND_SPECS[kind], 12)
    try:
        rng = np.random.default_rng(7)
        for t in range(8):
            members = None if t % 2 == 0 else [int(j) for j in rng.permutation(f.M)[:int(rng.integers(1, f.M + 1))]]
            f.tick(KINDS[t % 4], members, t % 3 == 1, rng)
        f.assert_states("steps", probe=True)
        # the match at W = 1 and 8, and scoring at level 0 and at the coarsest level every member has
        hints = [hypotheses(rng, f.data[j]["truth"][f.at[j] - 1], 3 + j, specials=False) for j in range(f.M)]
        scans = [f.data[j]["scans"][f.at[j] - 1] for j in range(f.M)]
        try:
            for W in (1, 8):
                f.grp[0].set_tuning(warps_per_scan=W)
                assert assert_match(f.g, f.grp, None, hints, scans, scans, (kind, "match"))[2] == W
        finally:
            f.grp[0].set_tuning(warps_per_scan=0)
        for level in sorted({0, min(f.levels(j) for j in range(f.M)) - 1}):
            poses = [hypotheses(rng, f.data[j]["truth"][f.at[j] - 1], 5 + j) for j in range(f.M)]
            assert_sessions(f.g, f.one, level, None, poses, scans, scans, (kind, "score", level))
        f.replicate(None, (kind, "pack"))
        f.assert_replicas((kind, "replicas"))
        members = [f.M - 1, 0]
        f.g.reset(members=members)
        for j in members:
            f.one[j].reset()
        f.tick("endpoints", None, False, rng)
        f.assert_states("after reset", probe=True)
        f.replicate(None, (kind, "pack after reset"), cleared=set(members))
        f.assert_replicas((kind, "replicas after reset"))
    finally:
        f.close()
