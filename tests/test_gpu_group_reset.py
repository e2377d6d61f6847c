"""Map reset for a group's members in one launch (hsb_group_reset, hsb_group_reset_subset), and the clear record that
replicates it (block-header word 36 of the tile transport) instead of whole levels.

GPU, in both gather modes, on the tile tests' square-ish three-level geometry, a two-level one whose width is not a
multiple of 4, and a mixed group of three map sizes; before each reset the members are written by full, subset, nowait
and map_without_matching group steps, single SLAM steps and hsb_update_level_by_scan calls:
  - against hsb_reset: a twin fleet reset member by member with hsb_reset holds the same planes, probabilities, texture
    twin, occupancy grids, rectangles, gate pose and last-match container, and stepping both fleets afterwards gives the
    same poses, covariances, gate decisions and planes; members left out of a subset reset are untouched;
  - ordering without a synchronise: a reset straight after a nowait step of the same group, of another group holding
    the member and of the member alone, then a nowait step and queries straight after the reset;
  - replication between an owner and a replica fleet: the clear record in every block, cleared blocks of a few cells
    under a buffer smaller than one level-0 plane, a 0-cell block after a reset with no write, the replica equal to the
    owner, a deferred cleared block shipped as a union, a single pack equal to its group block, the two-step protocol
    after a group reset, hsb_reset still shipping whole levels, and a mask bit >= levels rejected;
  - a 300-member fleet with subsets across the 32- and 128-session boundaries; launches and rejections; the C++ façade.
"""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import ROOT
from oracle import mapwrite as mw
from test_gpu_group_dist import make_rep, step
from test_gpu_group_subset import geometry, session_data
from test_gpu_group_tiles import HEADER_WORDS, MAGIC, cells_of, group_header_words
from twin_probe import probe_twin

pytestmark = pytest.mark.gpu

MODES = pytest.mark.parametrize("mode", [2, 1], ids=["tex", "ldg"])   # capi.GATHER_TEX, capi.GATHER_LDG
FLT_MAX = np.float32(3.4028234663852886e38)
CLEARED_WORD = 4 + 4 * 8   # HSB_TILE_CLEARED_WORD (hsb_internal.h)
HSB_ERR_INVALID_ARG = -1
# per member (map_size_x, map_size_y, levels, start); the mixed set differs in size and start, one width is 243
SETS = {
    "404x300x3": [(404, 300, 3, (0.5, 0.5))] * 4,
    "243x200x2": [(243, 200, 2, (0.5, 0.5))] * 4,
    "mixed": [(404, 300, 3, (0.5, 0.5)), (243, 200, 3, (0.5, 0.5)), (300, 404, 3, (0.3, 0.6))],
}
SET_IDS = list(SETS)


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


class Twins:
    """An owner fleet and a twin fleet written identically (each in a group of its own, mixed for the mixed set), and
    optionally a replica fleet in a third group, all preloaded identically with clean rectangles."""

    def __init__(self, set_id, mode, seed, replica=False):
        from hector_slam_b200 import capi

        self.geoms = SETS[set_id]
        self.M = M = len(self.geoms)
        self.levels = self.geoms[0][2]
        self.lv = [mw.geometry(0.05, g[0], g[1], g[2], g[3]) for g in self.geoms]
        mixed = set_id == "mixed"
        fleets = 3 if replica else 2
        self.fleets = [[make_rep(g, s, mode) for s, g in enumerate(self.geoms)] for _ in range(fleets)]
        self.owner, self.twin = self.fleets[0], self.fleets[1]
        self.replica = self.fleets[2] if replica else None
        self.rng = np.random.default_rng(seed)
        for s in range(M):
            for l, L in enumerate(self.lv[s]):
                p = mw.preload((L.sy, L.sx), self.rng)
                for fl in self.fleets:
                    fl[s].upload_level(l, p)
            for fl in self.fleets:
                fl[s].get_dirty_rects(reset=True)
                for l in range(self.levels):
                    fl[s].get_mirror_dirty_rect(l, reset=True)
        self.groups = [capi.SlamGroup(fl, mixed=mixed) for fl in self.fleets]
        self.og, self.tg = self.groups[0], self.groups[1]
        self.rg = self.groups[2] if replica else None
        self.data = [session_data(seed + s, 40, geometry(s)) for s in range(M)]
        self.at = [0] * M
        self.t = self.w = 0   # group steps taken, writes() ticks taken

    def group_step(self, members=None, nowait=False):
        out = step([self.og, self.tg], self.data, self.at, self.t, members, np.random.default_rng(100 + self.t), nowait)
        self.t += 1
        for a, b in zip(*out):
            assert np.array_equal(bits(a), bits(b)) if a.dtype == np.float32 else np.array_equal(a, b), self.t
        return out

    def single_step(self, s, nowait=False):
        d, k = self.data[s], self.at[s]
        res = [rep.slam_update(d["hints"][k], d["scans"][k], nowait=nowait) for rep in (self.owner[s], self.twin[s])]
        self.at[s] += 1
        assert all(np.array_equal(bits(a), bits(b)) for a, b in zip(res[0][:2], res[1][:2])) and res[0][2] == res[1][2]

    def level_writes(self, s, levels, k):
        """hsb_update_level_by_scan on `levels` of member s, the same on owner and twin"""
        rng_state = self.rng.bit_generator.state
        for rep in (self.owner[s], self.twin[s]):
            self.rng.bit_generator.state = rng_state
            for l in levels:
                L = self.lv[s][l]
                c = (L.sx // 3 + 7 * k + 11 * s) % L.sx, (L.sy // 2 + 5 * k + 3 * s) % L.sy
                pose = mw.pose_for_cell(L, c[0], c[1], 0.3 * k)
                pts = mw.points_for_targets(L, pose, mw.family_targets(L, c, self.rng, 16))
                rep.update_level_by_scan(l, pts, pose)

    def writes(self, ticks, members=None):
        """every kind of write, on `members` (None: all)"""
        sel = list(range(self.M)) if members is None else list(members)
        for i in range(ticks):
            kind = self.w % 4
            self.w += 1
            if kind == 0:
                self.group_step(members=members)
            elif kind == 1:
                self.group_step(members=sel[::-1], nowait=True)
            elif kind == 2:
                self.single_step(sel[i % len(sel)])
            else:
                self.level_writes(sel[-1], [0, self.levels - 1], self.w)

    def close(self):
        for g in self.groups:
            g.close()
        for fl in self.fleets:
            for r in fl:
                r.close()


def state(rep, levels):
    """everything hsb_reset defines, read without consuming a rectangle"""
    return ([bits(rep.download_level(l)).copy() for l in range(levels)],
            [bits(rep.download_prob(l)).copy() for l in range(levels)],
            rep.get_dirty_rects(), [rep.get_dirty_rect(l) for l in range(levels)],
            [rep.get_mirror_dirty_rect(l) for l in range(levels)], bits(rep.last_map_update_pose()).copy())


def assert_same(a, b, tag):
    for i, (x, y) in enumerate(zip(a, b)):
        if isinstance(x, list) and x and isinstance(x[0], np.ndarray):
            for l, (p, q) in enumerate(zip(x, y)):
                assert np.array_equal(p, q), (tag, i, l)
        elif isinstance(x, np.ndarray):
            assert np.array_equal(x, y), (tag, i)
        else:
            assert x == y, (tag, i, x, y)


def assert_reset_state(f, m, tag):
    """member m of the owner fleet is in hsb_reset's end state (the twin holds it too: compared bit for bit)"""
    rep = f.owner[m]
    for l, L in enumerate(f.lv[m]):
        zero = np.zeros((L.sy, L.sx), np.float32)
        assert np.array_equal(bits(rep.download_level(l)), bits(zero)), (tag, m, l)
        assert np.array_equal(bits(rep.download_prob(l)), bits(mw.prob(zero))), (tag, m, l)
        probe_twin(rep, l, L, zero, (0, 0, L.sx - 1, L.sy - 1), (tag, m), max_cells=3000)
        whole = (0, 0, L.sx - 1, L.sy - 1)
        assert rep.get_mirror_dirty_rect(l) == whole and rep.get_dirty_rect(l) == whole, (tag, m, l)
    assert np.array_equal(rep.last_map_update_pose(), np.full(3, FLT_MAX, np.float32)), (tag, m)
    assert_same(state(rep, f.levels), state(f.twin[m], f.levels), (tag, m))


@MODES
@pytest.mark.parametrize("set_id", SET_IDS)
def test_against_hsb_reset(hsb_lib, set_id, mode):
    """A group reset (full, then a permuted subset) against hsb_reset on a twin fleet: every state hsb_reset defines in
    bits, the synced occupancy grids, the last-match container; the members left out untouched; then several ticks of
    steps on both fleets stay identical."""
    f = Twins(set_id, mode, seed=31 + mode)
    M, L = f.M, f.levels
    for rnd, members in enumerate((None, [M - 1, 0])):
        f.writes(6)
        sel = list(range(M)) if members is None else members
        before = {m: state(f.owner[m], L) for m in range(M) if m not in sel}
        f.og.reset(members=members)
        for m in sel:
            f.twin[m].reset()
        for m in range(M):
            if m in sel:
                assert_reset_state(f, m, f"round {rnd}")
            else:
                assert_same(state(f.owner[m], L), before[m], ("unlisted", rnd, m))
                assert_same(state(f.owner[m], L), state(f.twin[m], L), ("unlisted twin", rnd, m))
        # the last-match container survives the reset: likelihood against it on both fleets
        poses = [f.data[m]["truth"][max(0, f.at[m] - 1)][None, :] for m in range(M)]
        for level in range(L):
            assert np.array_equal(bits(f.og.likelihood(level, poses)), bits(f.tg.likelihood(level, poses))), level
        # publishMap's grids: all -1 over the whole level (the twin's equal), the mirror rectangles consumed
        for level in range(L):
            grids = [[np.full((f.lv[m][level].sy, f.lv[m][level].sx), 5, np.int8) for m in sel] for _ in range(2)]
            rects = [g.sync_occupancy(level, gr, members=sel) for g, gr in zip((f.og, f.tg), grids)]
            assert rects[0] == rects[1] == [(0, 0, f.lv[m][level].sx - 1, f.lv[m][level].sy - 1) for m in sel]
            for k, m in enumerate(sel):
                assert (grids[0][k] == -1).all() and np.array_equal(grids[0][k], grids[1][k]), (level, m)
        f.writes(6)   # stamps, gate and container pinned by the steps after the reset
        for m in range(M):
            assert_same(state(f.owner[m], L), state(f.twin[m], L), ("after steps", rnd, m))
    f.close()


@MODES
def test_ordering_without_synchronise(hsb_lib, mode):
    """A reset queued straight after a nowait step of the same group, of another group holding the member and of the
    member alone runs after it; a nowait step and queries straight after the reset run after the reset."""
    from hector_slam_b200 import capi

    f = Twins("404x300x3", mode, seed=41 + mode)
    M, L = f.M, f.levels
    og2, tg2 = capi.SlamGroup(f.owner[2:]), capi.SlamGroup(f.twin[2:])
    f.writes(4)
    # the same group
    f.group_step(nowait=True)
    f.og.reset(members=[1, 0])
    for m in (1, 0):
        f.twin[m].reset()
    # another group holding member 2 (its index 0 there)
    d = f.data[2]
    for g in (og2, tg2):
        g.slam_update([d["hints"][f.at[2]], f.data[3]["hints"][f.at[3]]], [d["scans"][f.at[2]], f.data[3]["scans"][f.at[3]]],
                      nowait=True)
    f.at[2] += 1
    f.at[3] += 1
    f.og.reset(members=[2])
    f.twin[2].reset()
    # member 3 alone
    f.single_step(3, nowait=True)
    f.og.reset(members=[3])
    f.twin[3].reset()
    # a nowait step straight after the reset, then queries
    f.group_step(nowait=True)
    for level in range(L):
        poses = [f.data[m]["truth"][f.at[m] - 1][None, :] for m in range(M)]
        assert np.array_equal(bits(f.og.likelihood(level, poses)), bits(f.tg.likelihood(level, poses))), level
    f.og.reset()
    for r in f.twin:
        r.reset()
    scans = [f.data[m]["scans"][f.at[m] - 1] for m in range(M)]
    poses = [f.data[m]["truth"][f.at[m] - 1][None, :] for m in range(M)]
    assert np.array_equal(bits(f.og.likelihood(0, poses, points=scans)), bits(f.tg.likelihood(0, poses, points=scans)))
    f.group_step()
    for m in range(M):
        assert_same(state(f.owner[m], L), state(f.twin[m], L), ("ordering", m))
    og2.close()
    tg2.close()
    f.close()


class Buffers:
    def __init__(self, f):
        import torch

        self.G = group_header_words(f.M)
        big = self.G + f.M * HEADER_WORDS + f.M * sum(L.sx * L.sy for L in f.lv[0])
        self.big = 4 * big
        self.buf = torch.zeros(big + 64, dtype=torch.float32, device="cuda")
        self.single = torch.zeros(HEADER_WORDS + sum(L.sx * L.sy for L in f.lv[0]) + 64, dtype=torch.float32,
                                  device="cuda")
        self.stream = torch.cuda.current_stream().cuda_stream

    def words(self, t, lo, n):
        import torch

        torch.cuda.synchronize()
        return t[lo:lo + n].view(torch.int32).cpu().numpy()

    def blocks(self, f):
        """(member, start) per session of the group buffer, and each block's header words"""
        K = int(self.words(self.buf, 1, 1)[0])
        gh = self.words(self.buf, 0, 5 + 2 * K)
        out = []
        for k in range(K):
            m, start = int(gh[5 + 2 * k]), int(gh[6 + 2 * k])
            out.append((m, start, self.words(self.buf, start, HEADER_WORDS)))
        return out


def assert_replica(f, m, tag, mirror_whole=True):
    """the replica of member m equals its owner in bits, P = mapwrite.prob, the texture probe; its replication state
    clean (rectangles and cleared flags: get_dirty_rects reports a set flag as the whole level)"""
    rep, own = f.replica[m], f.owner[m]
    for l, L in enumerate(f.lv[m]):
        got, want = rep.download_level(l), own.download_level(l)
        assert np.array_equal(bits(got), bits(want)), (tag, m, l, int((bits(got) != bits(want)).sum()))
        assert np.array_equal(bits(rep.download_prob(l)), bits(mw.prob(got))), (tag, m, l)
        probe_twin(rep, l, L, got, (0, 0, L.sx - 1, L.sy - 1), (tag, m), max_cells=3000)
        if mirror_whole:
            assert rep.get_mirror_dirty_rect(l, reset=True) == (0, 0, L.sx - 1, L.sy - 1), (tag, m, l)
    assert rep.get_dirty_rects() == [None] * f.levels, (tag, m)


@MODES
@pytest.mark.parametrize("set_id", SET_IDS)
def test_replication_clear_record(hsb_lib, set_id, mode):
    import torch

    f = Twins(set_id, mode, seed=53 + mode, replica=True)
    M, L = f.M, f.levels
    B = Buffers(f)
    full = (1 << L) - 1
    f.writes(4)
    f.og.pack_dirty_device(B.buf.data_ptr(), B.big, True, B.stream)   # replicas in step with their owners
    f.rg.unpack_dirty_device(B.buf.data_ptr(), B.big, B.stream)
    for m in range(M):
        f.replica[m].get_dirty_rects(reset=True)
        for l in range(L):
            f.replica[m].get_mirror_dirty_rect(l, reset=True)

    # (1) a reset with no write after it: a 0-cell block with the whole mask, the others mask 0
    R = [M - 1, 0]
    f.og.reset(members=R)
    f.tg.reset(members=R)
    small = 4 * (B.G + M * HEADER_WORDS + 64)
    assert small // 4 < min(lv[0].sx * lv[0].sy for lv in f.lv)   # smaller than one level-0 plane
    B.buf.fill_(0)
    f.og.pack_dirty_device(B.buf.data_ptr(), small, True, B.stream)
    f.rg.unpack_dirty_device(B.buf.data_ptr(), small, B.stream)
    for m, start, hdr in B.blocks(f):
        assert hdr[0] == MAGIC and hdr[2] == 0 and hdr[3] == 0, (m, hdr[:8])
        assert hdr[CLEARED_WORD] == (full if m in R else 0), (m, hdr[CLEARED_WORD])
    for m in R:
        assert f.owner[m].get_dirty_rects() == [None] * L   # shipped: flags and rectangles consumed
        assert_replica(f, m, "reset, no write")
    assert all(r.replication_overflows() == 0 for r in f.replica)

    # (2) reset, then writes: only the cells written since ship.  The twin group, reset and written the same way, packs
    # each member alone first (the exact capacity, and the blocks the group pack must equal byte for byte); one block
    # applies with the single unpack.  First with a few level writes under a buffer smaller than one level-0 plane, then
    # with every kind of write.
    def ship(tag, write, narrow):
        f.og.reset(members=R)
        f.tg.reset(members=R)
        write()
        singles = []
        for m in R:
            B.single.fill_(0)
            f.twin[m].pack_dirty_device(B.single.data_ptr(), 4 * B.single.numel(), True, B.stream)
            n = int(B.words(B.single, 3, 1)[0])
            singles.append(B.words(B.single, 0, HEADER_WORDS + n))
        cap = 4 * (group_header_words(len(R)) + len(R) * HEADER_WORDS + sum(w.size - HEADER_WORDS for w in singles))
        if narrow:
            assert cap // 4 < min(lv[0].sx * lv[0].sy for lv in f.lv), cap
        else:
            cap = B.big
        B.buf.fill_(0)
        f.og.pack_dirty_device(B.buf.data_ptr(), cap, True, B.stream, members=R)
        f.rg.unpack_dirty_device(B.buf.data_ptr(), cap, B.stream)
        for k, (m, start, hdr) in enumerate(B.blocks(f)):
            assert m == R[k] and hdr[2] == 0 and hdr[CLEARED_WORD] == full, (tag, m, hdr[:8])
            rects = [None if hdr[6 + 4 * l] < hdr[4 + 4 * l] else tuple(int(v) for v in hdr[4 + 4 * l:8 + 4 * l])
                     for l in range(L)]
            n = cells_of(rects)
            assert hdr[3] == n and 0 < n, (tag, m, n)
            for l, r in enumerate(rects):   # nothing was written outside the shipped rectangle since the reset
                plane = f.owner[m].download_level(l)
                if r is not None:
                    plane[r[1]:r[3] + 1, r[0]:r[2] + 1] = 0
                assert not plane.any(), (tag, m, l)
            assert np.array_equal(B.words(B.buf, start, HEADER_WORDS + n), singles[k]), (tag, m)
            assert_replica(f, m, tag)
        solo = make_rep(f.geoms[R[0]], R[0], mode)
        for l in range(L):
            solo.upload_level(l, f.replica[R[0]].download_level(l) + 1.0)   # anything: the clear record overwrites it
        B.single.fill_(0)
        B.single[:singles[0].size] = torch.from_numpy(singles[0].view(np.float32).copy()).cuda()
        solo.unpack_dirty_device(B.single.data_ptr(), 4 * singles[0].size, B.stream)
        for l in range(L):
            assert np.array_equal(bits(solo.download_level(l)), bits(f.owner[R[0]].download_level(l))), (tag, l)
        assert solo.replication_overflows() == 0
        solo.close()

    def short_beams():   # one beam of a few cells on level 0 of each member
        for m in R:
            L0 = f.lv[m][0]
            c = (L0.sx // 3, L0.sy // 2)
            pose = mw.pose_for_cell(L0, c[0], c[1], 0.0)
            pts = mw.points_for_targets(L0, pose, np.float64([[c[0] + 3, c[1] + 2]]))
            for rep in (f.owner[m], f.twin[m]):
                rep.update_level_by_scan(0, pts, pose)

    ship("a short beam, small buffer", short_beams, True)
    ship("every kind of write", lambda: f.writes(4, members=R), False)

    # (3) a deferred cleared block keeps its flags; the next pack ships the union of its writes
    a, b = R[0], 1
    f.og.reset(members=[a])
    f.level_writes(a, [0], 1)
    f.owner[b].upload_level(0, mw.preload((f.lv[b][0].sy, f.lv[b][0].sx), f.rng))   # b: its whole level 0
    sub = [b, a]
    G2 = group_header_words(2)
    cap = 4 * (G2 + 2 * HEADER_WORDS + f.lv[b][0].sx * f.lv[b][0].sy)
    f.og.pack_dirty_device(B.buf.data_ptr(), cap, True, B.stream, members=sub)
    f.rg.unpack_dirty_device(B.buf.data_ptr(), cap, B.stream)
    blk = B.blocks(f)
    assert [(m, int(h[2]), int(h[CLEARED_WORD])) for m, _, h in blk] == [(b, 0, 0), (a, 1, full)], blk
    assert f.replica[a].replication_overflows(reset=True) == 1
    assert f.owner[a].get_dirty_rects()[0] == (0, 0, f.lv[a][0].sx - 1, f.lv[a][0].sy - 1)   # the flag is kept
    f.level_writes(a, [0, L - 1], 2)
    f.og.pack_dirty_device(B.buf.data_ptr(), B.big, True, B.stream, members=sub)
    f.rg.unpack_dirty_device(B.buf.data_ptr(), B.big, B.stream)
    blk = B.blocks(f)
    assert int(blk[1][2][2]) == 0 and int(blk[1][2][CLEARED_WORD]) == full
    assert_replica(f, a, "deferred, shipped next")
    assert_replica(f, b, "the other member", mirror_whole=False)

    # (4) the two-step protocol after a group reset ships the whole levels, and consumes the flags
    c = 1
    f.og.reset(members=[c])
    f.level_writes(c, [0], 3)
    rects = f.owner[c].get_dirty_rects(reset=True)
    assert rects == [(0, 0, lv.sx - 1, lv.sy - 1) for lv in f.lv[c]]
    tmp = torch.zeros(max(lv.sx * lv.sy for lv in f.lv[c]), dtype=torch.float32, device="cuda")
    for l, r in enumerate(rects):
        f.owner[c].pack_rect_device(l, r, tmp.data_ptr(), B.stream)
        f.replica[c].unpack_rect_device(l, r, tmp.data_ptr(), B.stream)
    assert f.owner[c].get_dirty_rects() == [None] * L
    assert_replica(f, c, "two-step")
    f.og.pack_dirty_device(B.buf.data_ptr(), B.big, False, B.stream, members=[c])
    h = B.blocks(f)[0][2]
    assert h[3] == 0 and h[CLEARED_WORD] == 0

    # (5) hsb_reset: mask 0, whole-level rectangles, as before
    f.owner[0].reset()
    f.og.pack_dirty_device(B.buf.data_ptr(), B.big, True, B.stream, members=[0])
    h = B.blocks(f)[0][2]
    assert h[CLEARED_WORD] == 0 and h[3] == sum(lv.sx * lv.sy for lv in f.lv[0])
    assert [tuple(int(v) for v in h[4 + 4 * l:8 + 4 * l]) for l in range(L)] == \
        [(0, 0, lv.sx - 1, lv.sy - 1) for lv in f.lv[0]]
    f.rg.unpack_dirty_device(B.buf.data_ptr(), B.big, B.stream)
    assert_replica(f, 0, "hsb_reset")

    # (6) a mask bit >= levels: the buffer does not fit, counted once on handles[0], nothing applied
    f.og.reset(members=[0])
    f.og.pack_dirty_device(B.buf.data_ptr(), B.big, False, B.stream, members=[0])
    start = B.blocks(f)[0][1]
    torch.cuda.synchronize()
    B.buf[start + CLEARED_WORD:start + CLEARED_WORD + 1].view(torch.int32).fill_(1 << L)
    snap = [f.replica[0].download_level(l) for l in range(L)]
    f.rg.unpack_dirty_device(B.buf.data_ptr(), B.big, B.stream)
    B.single.fill_(0)
    f.owner[0].pack_dirty_device(B.single.data_ptr(), 4 * B.single.numel(), False, B.stream)
    torch.cuda.synchronize()
    B.single[CLEARED_WORD:CLEARED_WORD + 1].view(torch.int32).fill_(full | (1 << L))
    f.replica[0].unpack_dirty_device(B.single.data_ptr(), 4 * B.single.numel(), B.stream)
    assert f.replica[0].replication_overflows(reset=True) == 2   # once per buffer, both on handles[0]
    assert all(r.replication_overflows() == 0 for r in f.replica[1:])
    for l in range(L):
        assert np.array_equal(bits(f.replica[0].download_level(l)), bits(snap[l])), l
    f.close()


@MODES
def test_fleet_300(hsb_lib, mode):
    """About 300 members of the fleet test's mixed group: subset resets of K = 121 and K = 129 across the 32- and
    128-session boundaries (both member-list forms of the launch) and a full one; the listed members in hsb_reset's
    state, sampled unlisted ones untouched, and a full pack ships every listed member's clear record."""
    import torch

    from hector_slam_b200 import capi
    from test_gpu_group_fleet import LEVELS, fleet_size, make_rep as fleet_rep, member_data, state_of, same_state
    from test_gpu_group_match import sm_count

    M = fleet_size(sm_count())
    owner = [fleet_rep(s, mode) for s in range(M)]
    replica = [fleet_rep(s, mode) for s in range(M)]
    og, rg = capi.SlamGroup(owner, mixed=True), capi.SlamGroup(replica, mixed=True)
    data = [member_data(s) for s in range(M)]
    og.slam_update([d["hints"][0] for d in data], [d["scans"][0] for d in data])
    G = group_header_words(M)
    cap = 4 * (G + M * HEADER_WORDS + sum(r.level_info(l)[0] * r.level_info(l)[1] for r in owner for l in range(LEVELS)))
    buf = torch.zeros(cap // 4 + 64, dtype=torch.float32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    og.pack_dirty_device(buf.data_ptr(), cap, True, st)
    rg.unpack_dirty_device(buf.data_ptr(), cap, st)
    rng = np.random.default_rng(7)
    for rnd, sel in enumerate((list(rng.permutation(np.arange(20, 141))), list(rng.permutation(np.arange(M - 129, M))),
                               None)):
        og.slam_update([d["hints"][rnd + 1] for d in data], [d["scans"][rnd + 1] for d in data])
        listed = set(range(M)) if sel is None else {int(m) for m in sel}
        probe = [m for m in (0, 19, 31, 32, 127, 128, 129, 141, 255, 256, M - 130, M - 1) if m not in listed]
        before = {m: state_of(owner[m]) for m in probe}
        og.reset(members=sel)
        for m in probe:
            assert same_state(state_of(owner[m]), before[m]), (rnd, m)
        for m in sorted(listed)[::17] + [max(listed)]:
            rep = owner[m]
            for l in range(LEVELS):
                sx, sy, _ = rep.level_info(l)
                assert not rep.download_level(l).any() and (rep.download_prob(l) == 0.5).all(), (rnd, m, l)
                assert rep.get_mirror_dirty_rect(l) == rep.get_dirty_rect(l) == (0, 0, sx - 1, sy - 1), (rnd, m, l)
            assert np.array_equal(rep.last_map_update_pose(), np.full(3, FLT_MAX, np.float32)), (rnd, m)
        buf.fill_(0)
        og.pack_dirty_device(buf.data_ptr(), cap, True, st)
        rg.unpack_dirty_device(buf.data_ptr(), cap, st)
        torch.cuda.synchronize()
        w = buf.view(torch.int32).cpu().numpy()
        assert w[3] == 0
        for k in range(M):
            start = int(w[6 + 2 * k])
            assert w[5 + 2 * k] == k and w[start + CLEARED_WORD] == ((1 << LEVELS) - 1 if k in listed else 0), (rnd, k)
        for m in probe[:3] + sorted(listed)[:3] + [max(listed)]:
            for l in range(LEVELS):
                assert np.array_equal(bits(replica[m].download_level(l)), bits(owner[m].download_level(l))), (rnd, m, l)
    og.close()
    rg.close()
    for r in owner + replica:
        r.close()


@MODES
def test_launches_and_rejections(hsb_lib, mode):
    from hector_slam_b200 import capi

    f = Twins("243x200x2", mode, seed=61 + mode)
    M = f.M
    lib = capi.load_library()
    h0 = f.owner[0]
    for members in (None, [2, 1], list(range(M))):
        a = h0.launch_count
        f.og.reset(members=members)
        assert h0.launch_count - a == 1, members
    snap = [state(r, f.levels) for r in f.owner]
    mem = lambda *v: (C.c_int * max(1, len(v)))(*v)   # noqa: E731
    bad = [
        ((f.og.g, -1, mem(0)), "K is -1"),
        ((f.og.g, M + 1, mem(*range(M + 1))), "K is"),
        ((f.og.g, 2, None), "members is NULL"),
        ((f.og.g, 2, mem(0, M)), "session 1"),
        ((f.og.g, 2, mem(0, -1)), "session 1"),
        ((f.og.g, 3, mem(1, 2, 1)), "session 2"),
    ]
    la = h0.launch_count
    for args, msg in bad:
        assert lib.hsb_group_reset_subset(*args) == HSB_ERR_INVALID_ARG, msg
        err = (lib.hsb_last_error(h0.h) or b"").decode()
        assert msg in err and "hsb_group_reset_subset" in err, (msg, err)
    assert lib.hsb_group_reset_subset(f.og.g, 0, None) == 0   # K = 0
    assert lib.hsb_group_reset(None) == HSB_ERR_INVALID_ARG
    assert h0.launch_count == la
    for r, s in zip(f.owner, snap):
        assert_same(state(r, f.levels), s, "rejections change nothing")
    f.close()


def test_facade(hsb_lib):
    """hsb200::SlamProcessor::resetMany (all, and a member list) against reset() per processor on a twin set: the same
    poses, covariances and maps from the following updates (which read the processors' lastMapUpdatePose)."""
    L = C.CDLL(os.path.join(ROOT, "hector_slam_b200", "lib", "libhsb200_host.so"))
    vp, i, fl = C.c_void_p, C.c_int, C.c_float
    L.hsbp_create.restype = vp
    L.hsbp_create.argtypes = [fl, i, i, fl, fl, i, i]
    L.hsbp_destroy.argtypes = [vp]
    L.hsbp_update.argtypes = [vp, vp, i, vp, vp, i, vp, vp]
    L.hsbp_reset.argtypes = [vp]
    L.hsbp_reset_many.argtypes = [vp, i, vp, i]
    L.hsbp_get_grid_map.argtypes = [vp, i, vp]
    sx, sy, levels, start = SETS["404x300x3"][0]
    M, ticks = 4, 12
    data = [session_data(8100 + s, ticks, geometry(s)) for s in range(M)]
    sets = [[L.hsbp_create(0.05, sx, sy, start[0], start[1], levels, 0) for _ in range(M)] for _ in range(2)]
    assert all(q for s in sets for q in s)
    many, single = sets
    arr = C.cast((C.c_void_p * M)(*many), vp)
    for t in range(ticks):
        if t in (4, 8):
            members = None if t == 4 else np.ascontiguousarray([3, 1], np.int32)
            assert L.hsbp_reset_many(arr, M, None if members is None else members.ctypes.data,
                                     0 if members is None else 2) == 0
            for s in (range(M) if members is None else members):
                assert L.hsbp_reset(single[int(s)]) == 0
        for s in range(M):
            x = data[s]["scans"][t]
            out = []
            for st in sets:
                pose, cov = np.zeros(3, np.float32), np.zeros(9, np.float32)
                assert L.hsbp_update(st[s], x.ctypes.data, x.shape[0], None, data[s]["hints"][t].ctypes.data, 0,
                                     pose.ctypes.data, cov.ctypes.data) == 0
                out.append((pose, cov))
            assert np.array_equal(bits(out[0][0]), bits(out[1][0])) and np.array_equal(bits(out[0][1]), bits(out[1][1]))
    for s in range(M):
        for l in range(levels):
            n = (sx >> l) * (sy >> l)
            a, b = np.zeros(n, np.float32), np.zeros(n, np.float32)
            assert L.hsbp_get_grid_map(many[s], l, a.ctypes.data) == 0 and L.hsbp_get_grid_map(single[s], l, b.ctypes.data) == 0
            assert np.array_equal(bits(a), bits(b)), (s, l)
    for st in sets:
        for q in st:
            L.hsbp_destroy(q)
