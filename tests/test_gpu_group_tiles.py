"""Map replication for a group's members in one pass (hsb_group_pack_dirty_device, its _subset form and
hsb_group_unpack_dirty_device): every session's dirty tiles packed into one self-describing buffer with one launch and
applied on a replica group with one launch.

GPU, in both gather modes, on a square-ish three-level geometry and a two-level one whose width is not a multiple of 4,
the owners written by full, subset, nowait and map_without_matching group steps, single SLAM steps and
hsb_update_level_by_scan calls that leave a level clean between two dirty ones:
  - round trip: replica log-odds equal the owner's in bits, P equals mapwrite.prob, the texture twin follows, the
    replica's mirror rectangle is the union of what it received and its replication rectangles are clean, the owner's
    rectangles are cleared for shipped members only;
  - format: each block is byte for byte the buffer hsb_pack_dirty_device writes on a twin owner with the same writes,
    the group header is what the host computes, and one block copied out applies with hsb_unpack_dirty_device;
  - subsets in permuted order, first-fit placement at its exact boundaries, foreign buffers, ordering without a
    synchronise (after a nowait step; group queries right after an unpack), launch accounting and rejections.
CPU: the multi-process plumbing (parallel.broadcast_group_dirty_tiles_async) on gloo with a host stand-in for the
group; with two GPUs, one NCCL round trip."""
import os
import socket

import numpy as np
import pytest

from oracle import mapwrite as mw

HEADER_WORDS, MAGIC, GROUP_MAGIC = 64, 0x48534254, 0x48534247   # hsb_internal.h
INT_MAX = 2 ** 31 - 1
CLEAN = (INT_MAX, INT_MAX, -1, -1)
HSB_ERR_INVALID_ARG = -1
M = 5


def group_header_words(K):
    return (5 + 2 * K + 3) & ~3


def cells_of(rects):
    return sum(0 if r is None else (r[2] - r[0] + 1) * (r[3] - r[1] + 1) for r in rects)


def layout(rects, members, cap_bytes, levels):
    """The host's view of a group pack: (group header words, [(block start, shipped)] per session).  rects: per session
    the member's replication rectangles before the pack."""
    K = len(members)
    G = group_header_words(K)
    room = min(cap_bytes // 4, 2 ** 32 - 1) - G - HEADER_WORDS * K
    used, blocks = 0, []
    for k in range(K):
        c = cells_of(rects[k])
        start = G + HEADER_WORDS * k + used
        ship = used + c <= room
        blocks.append((start, ship))
        used += c if ship else 0
    hdr = [GROUP_MAGIC, K, levels, sum(not s for _, s in blocks), G + HEADER_WORDS * K + used]
    for m, (start, _) in zip(members, blocks):
        hdr += [m, start]
    hdr += [0] * (G - len(hdr))
    return hdr, blocks


# ---- CPU: multi-process plumbing ------------------------------------------------------------------------------------

def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


class HostGroup:
    """A host stand-in for capi.SlamGroup (same method names): M members of one level each, the group buffer format
    written and read with numpy over the memory of a CPU tensor."""

    def __init__(self, M, n):
        self.planes = [np.zeros((n, n), np.float32) for _ in range(M)]
        self.dirty = [None] * M
        self.overflows = [0] * M
        self.foreign = 0

    def write(self, m, x0, y0, x1, y1, v):
        self.planes[m][y0:y1 + 1, x0:x1 + 1] += v
        self.dirty[m] = mw.union(self.dirty[m], (x0, y0, x1, y1))

    @staticmethod
    def _view(ptr, n):
        import ctypes

        return np.ctypeslib.as_array((ctypes.c_float * n).from_address(ptr))

    def pack_dirty_device(self, ptr, nbytes, reset, stream=0, members=None):
        members = list(range(len(self.planes))) if members is None else list(members)
        words = self._view(ptr, nbytes // 4)
        iw = words.view(np.int32)
        hdr, blocks = layout([[self.dirty[m]] for m in members], members, nbytes, 1)
        iw[:len(hdr)] = hdr
        for m, (start, ship) in zip(members, blocks):
            r = self.dirty[m] or CLEAN
            iw[start:start + 8] = [MAGIC, 1, 0 if ship else 1, cells_of([self.dirty[m]])] + list(r)
            if ship and self.dirty[m] is not None:
                x0, y0, x1, y1 = r
                n = (x1 - x0 + 1) * (y1 - y0 + 1)
                words[start + HEADER_WORDS:start + HEADER_WORDS + n] = self.planes[m][y0:y1 + 1, x0:x1 + 1].reshape(-1)
            if ship and reset:
                self.dirty[m] = None

    def unpack_dirty_device(self, ptr, nbytes, stream=0):
        words = self._view(ptr, nbytes // 4)
        iw = words.view(np.int32)
        if iw[0] != GROUP_MAGIC or iw[2] != 1 or not 0 <= iw[1] <= len(self.planes):
            self.foreign += 1
            return
        for k in range(int(iw[1])):
            m, start = int(iw[5 + 2 * k]), int(iw[6 + 2 * k])
            if iw[start + 2] != 0:
                self.overflows[m] += 1
                continue
            x0, y0, x1, y1 = (int(v) for v in iw[start + 4:start + 8])
            if x1 >= x0:
                n = (x1 - x0 + 1) * (y1 - y0 + 1)
                o = start + HEADER_WORDS
                self.planes[m][y0:y1 + 1, x0:x1 + 1] = words[o:o + n].reshape(y1 - y0 + 1, x1 - x0 + 1)


def _gloo_worker(rank, world, port, q):
    import sys

    import torch
    import torch.distributed as dist

    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    ok = True
    try:
        from hector_slam_b200 import parallel

        g = HostGroup(4, 16)
        G = group_header_words(4)
        buf = torch.zeros(G + 4 * HEADER_WORDS + 40, dtype=torch.float32)   # 40 words of rows
        if rank == 0:
            g.write(0, 1, 1, 4, 2, 1.0)     # 8 cells
            g.write(2, 0, 0, 1, 1, -2.0)    # 4 cells
        parallel.broadcast_group_dirty_tiles_async(g, buf, src=0)
        ok = ok and float(g.planes[0].sum()) == 8.0 and float(g.planes[2].sum()) == -8.0
        ok = ok and g.dirty == [None] * 4
        # member 1 larger than what is left behind member 0's rows: deferred, member 3 still ships
        before = g.planes[1].copy()
        if rank == 0:
            g.write(0, 0, 0, 4, 3, 1.0)     # 20 cells
            g.write(1, 0, 0, 9, 2, 5.0)     # 30 cells: 20 + 30 > 40
            g.write(3, 0, 0, 2, 2, 3.0)     # 9 cells
        parallel.broadcast_group_dirty_tiles_async(g, buf, src=0)
        if rank == 0:
            ok = ok and g.dirty[1] == (0, 0, 9, 2) and g.dirty[0] is None and g.dirty[3] is None
        else:
            ok = ok and g.overflows == [0, 1, 0, 0] and bool(np.array_equal(g.planes[1], before))
            ok = ok and float(g.planes[3].sum()) == 27.0
        # the next call ships the deferred member; a subset leaves the others alone
        parallel.broadcast_group_dirty_tiles_async(g, buf, src=0, members=[1])
        ok = ok and float(g.planes[1].sum()) == 150.0 and (rank != 0 or g.dirty == [None] * 4)
        q.put((rank, ok))
    except Exception as e:   # reported through the queue: the parent asserts on it
        q.put((rank, repr(e)))
    finally:
        dist.destroy_process_group()


def test_group_broadcast_two_ranks_gloo():
    import torch.multiprocessing as mp

    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_gloo_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=180) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert sorted(r[0] for r in results) == [0, 1]
    assert all(r[1] is True for r in results), results


def test_layout_first_fit():
    """The host model the GPU tests compare against: first fit in session order, deferred blocks keep their place."""
    rects = [[(0, 0, 9, 9)], [(0, 0, 19, 19)], [(0, 0, 4, 4)], [None]]
    G = group_header_words(4)
    cap = 4 * (G + 4 * HEADER_WORDS + 100 + 25)
    hdr, blocks = layout(rects, [3, 0, 1, 2], cap, 1)
    assert [s for _, s in blocks] == [True, False, True, True]
    assert [b for b, _ in blocks] == [G, G + 64 + 100, G + 128 + 100, G + 192 + 125]
    assert hdr[:5] == [GROUP_MAGIC, 4, 1, 1, G + 256 + 125] and hdr[5:13] == [3, G, 0, G + 164, 1, G + 228, 2, G + 317]
    assert len(hdr) == G == 16 and hdr[13:] == [0, 0, 0]


# ---- GPU ------------------------------------------------------------------------------------------------------------

MODES = pytest.mark.parametrize("mode", [2, 1], ids=["tex", "ldg"])   # capi.GATHER_TEX, capi.GATHER_LDG
GEOMS = [(404, 300, 3, (0.5, 0.5)), (243, 200, 2, (0.5, 0.5))]     # test_gpu_map_io / maptools_cases geometries
GEOM_IDS = ["404x300x3", "243x200x2"]


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def make_rep(geom, s, mode):
    from test_gpu_group_dist import make_rep as dist_rep

    return dist_rep(geom, s, mode)


class Fleets:
    """An owner group, a twin owner group written identically (packed member by member with the single call), and a
    replica group of fresh twins, all preloaded identically; the planes each replica member must hold and the
    rectangles it received since its last mirror reset."""

    def __init__(self, geom, mode, seed):
        import torch

        from hector_slam_b200 import capi
        from test_gpu_group_subset import geometry, session_data

        self.geom, self.levels = geom, geom[2]
        self.lv = mw.geometry(0.05, geom[0], geom[1], geom[2], geom[3])
        self.owner = [make_rep(geom, s, mode) for s in range(M)]
        self.twin = [make_rep(geom, s, mode) for s in range(M)]
        self.replica = [make_rep(geom, s, mode) for s in range(M)]
        self.rng = np.random.default_rng(seed)
        for s in range(M):
            for l, L in enumerate(self.lv):
                p = mw.preload((L.sy, L.sx), self.rng)
                for rep in (self.owner[s], self.twin[s], self.replica[s]):
                    rep.upload_level(l, p)
            for rep in (self.owner[s], self.twin[s], self.replica[s]):
                rep.get_dirty_rects(reset=True)
                for l in range(self.levels):
                    rep.get_mirror_dirty_rect(l, reset=True)
        self.og, self.tg, self.rg = (capi.SlamGroup(r) for r in (self.owner, self.twin, self.replica))
        self.data = [session_data(seed + s, 16, geometry(s)) for s in range(M)]
        self.at = [0] * M
        self.shipped = [[[] for _ in range(self.levels)] for _ in range(M)]
        words = group_header_words(M) + M * HEADER_WORDS + M * sum(L.sx * L.sy for L in self.lv)
        self.cap = 4 * words
        self.buf = torch.zeros(words + 64, dtype=torch.float32, device="cuda")
        self.single = torch.zeros(HEADER_WORDS + sum(L.sx * L.sy for L in self.lv) + 64, dtype=torch.float32,
                                  device="cuda")
        self.stream = torch.cuda.current_stream().cuda_stream

    # writes, applied identically to owner and twin
    def group_step(self, t, members=None, nowait=False):
        from test_gpu_group_dist import step

        step([self.og, self.tg], self.data, self.at, t, members, np.random.default_rng(100 + t), nowait)

    def single_step(self, s):
        d, k = self.data[s], self.at[s]
        for rep in (self.owner[s], self.twin[s]):
            rep.slam_update(d["hints"][k], d["scans"][k])
        self.at[s] += 1

    def level_writes(self, s, levels, k):
        """hsb_update_level_by_scan on `levels` of member s (test_gpu_map_io.Replication.write's scan family)."""
        rng_state = self.rng.bit_generator.state
        for rep in (self.owner[s], self.twin[s]):
            self.rng.bit_generator.state = rng_state
            for l in levels:
                L = self.lv[l]
                c = (L.sx // 3 + 7 * k + 11 * s) % L.sx, (L.sy // 2 + 5 * k + 3 * s) % L.sy
                pose = mw.pose_for_cell(L, c[0], c[1], 0.3 * k)
                pts = mw.points_for_targets(L, pose, mw.family_targets(L, c, self.rng, 16))
                rep.update_level_by_scan(l, pts, pose)

    def rects(self, members=None):
        return [self.owner[m].get_dirty_rects() for m in (range(M) if members is None else members)]

    def words(self, lo, n):
        import torch

        torch.cuda.synchronize()
        return self.buf[lo:lo + n].view(torch.int32).cpu().numpy()

    def note_shipped(self, m, rects):
        for l, r in enumerate(rects):
            if r is not None:
                self.shipped[m][l].append(r)

    def check_member(self, m, what):
        from test_gpu_map_io import union
        from twin_probe import probe_twin

        rep = self.replica[m]
        for l, L in enumerate(self.lv):
            got, want = rep.download_level(l), self.owner[m].download_level(l)
            bad = bits(got) != bits(want)
            assert not bad.any(), (what, m, l, int(bad.sum()), np.argwhere(bad)[:5].tolist())
            assert np.array_equal(bits(rep.download_prob(l)), bits(mw.prob(got))), (what, m, l)
            probe_twin(rep, l, L, got, union(self.shipped[m][l]), what, max_cells=8000)
            assert rep.get_mirror_dirty_rect(l) == union(self.shipped[m][l]), (what, m, l)
        assert rep.get_dirty_rects() == [None] * self.levels, (what, m)

    def close(self):
        for g in (self.og, self.tg, self.rg):
            g.close()
        for r in self.owner + self.twin + self.replica:
            r.close()


@pytest.mark.gpu
@MODES
@pytest.mark.parametrize("geom", GEOMS, ids=GEOM_IDS)
def test_round_trip_and_format(hsb_lib, geom, mode):
    """After every tick of mixed writes: a full group pack with reset and a group unpack; the replica equals the owner;
    each block is the single pack of the twin member; the group header is the host's; block 0 applies alone on a
    fourth handle with hsb_unpack_dirty_device."""
    import torch

    f = Fleets(geom, mode, seed=geom[0] + mode)
    L = f.levels
    solo = make_rep(geom, 0, mode)   # receives member 0's block through the single unpack
    for l, Lv in enumerate(f.lv):
        solo.upload_level(l, f.owner[0].download_level(l))
    solo.get_dirty_rects(reset=True)
    for tick in range(6):
        if tick % 3 == 0:
            f.group_step(tick)
        elif tick % 3 == 1:
            f.group_step(tick, members=[3, 0, 2], nowait=True)
        else:
            f.single_step(1)
            f.level_writes(4, [0, L - 1], tick)   # a clean level between two dirty ones when L = 3
        if tick == 2 and L == 3:
            r4 = f.owner[4].get_dirty_rects()
            assert r4[1] is None and r4[0] is not None and r4[2] is not None
        rects = f.rects()
        f.buf.fill_(0)
        f.og.pack_dirty_device(f.buf.data_ptr(), f.cap, True, f.stream)
        f.rg.unpack_dirty_device(f.buf.data_ptr(), f.cap, f.stream)
        hdr, blocks = layout(rects, list(range(M)), f.cap, L)
        assert list(f.words(0, len(hdr))) == hdr, (tick, list(f.words(0, len(hdr))), hdr)
        assert all(ship for _, ship in blocks)
        for m in range(M):
            start = blocks[m][0]
            n = cells_of(rects[m])
            f.single.fill_(0)
            f.twin[m].pack_dirty_device(f.single.data_ptr(), 4 * f.single.numel(), True, f.stream)
            torch.cuda.synchronize()
            want = f.single[:HEADER_WORDS + n].view(torch.int32).cpu().numpy()
            got = f.buf[start:start + HEADER_WORDS + n].view(torch.int32).cpu().numpy()
            assert np.array_equal(got, want), (tick, m, np.argwhere(got != want)[:5].tolist())
            assert list(got[:4]) == [MAGIC, L, 0, n]
            f.note_shipped(m, rects[m])
            assert f.owner[m].get_dirty_rects() == [None] * L, (tick, m)
            f.check_member(m, f"tick {tick} {geom} mode {mode}")
        # one block copied out applies with the single unpack
        n0 = cells_of(rects[0])
        f.single.fill_(0)
        f.single[:HEADER_WORDS + n0] = f.buf[blocks[0][0]:blocks[0][0] + HEADER_WORDS + n0]
        solo.unpack_dirty_device(f.single.data_ptr(), 4 * (HEADER_WORDS + n0), f.stream)
        for l in range(L):
            assert np.array_equal(bits(solo.download_level(l)), bits(f.owner[0].download_level(l))), (tick, l)
        assert all(r.replication_overflows() == 0 for r in f.replica + [solo])
    solo.close()
    f.close()


@pytest.mark.gpu
@MODES
def test_subsets_permuted_and_untouched(hsb_lib, mode):
    """A member left out of a pack keeps its rectangles and its replica is not changed; permuted sessions land on
    the right replica members; a later full pack ships the union."""
    geom = GEOMS[0]
    f = Fleets(geom, mode, seed=7 + mode)
    L = f.levels
    for s in range(M):
        f.level_writes(s, list(range(L)), 1)
    rects_all = f.rects()
    before = [[f.replica[m].download_level(l) for l in range(L)] for m in range(M)]
    sub = [4, 1, 3]
    f.og.pack_dirty_device(f.buf.data_ptr(), f.cap, True, f.stream, members=sub)
    f.rg.unpack_dirty_device(f.buf.data_ptr(), f.cap, f.stream)
    hdr, _ = layout([rects_all[m] for m in sub], sub, f.cap, L)
    assert list(f.words(0, len(hdr))) == hdr
    for m in range(M):
        if m in sub:
            f.note_shipped(m, rects_all[m])
            assert f.owner[m].get_dirty_rects() == [None] * L
            f.check_member(m, f"subset, member {m}")
        else:
            assert f.owner[m].get_dirty_rects() == rects_all[m]
            for l in range(L):
                assert np.array_equal(bits(f.replica[m].download_level(l)), bits(before[m][l])), (m, l)
                assert f.replica[m].get_mirror_dirty_rect(l) is None
    # more writes on a left-out member: the full pack ships the union of both
    f.level_writes(0, [0], 2)
    rects2 = f.rects()
    assert all(mw.union(a, b) == b for a, b in zip(rects_all[0], rects2[0]) if a is not None)
    f.og.pack_dirty_device(f.buf.data_ptr(), f.cap, True, f.stream)
    f.rg.unpack_dirty_device(f.buf.data_ptr(), f.cap, f.stream)
    for m in range(M):
        f.note_shipped(m, rects2[m])
        f.check_member(m, f"full after subset, member {m}")
    f.close()


@pytest.mark.gpu
@MODES
def test_first_fit_boundaries(hsb_lib, mode):
    """Members {0, 1, 2} dirty with cells1 > cells2: the exact capacity that ships 0 and 2 and defers 1, the one that
    ships all three, one word less (and capacities that are not a multiple of 4 bytes), the deferral counted once on
    the replica member, the rectangles kept on the owner and shipped by the next call; below the minimum rejected."""
    from hector_slam_b200 import capi

    geom = GEOMS[0]
    f = Fleets(geom, mode, seed=11 + mode)
    L = f.levels
    sub = [0, 1, 2]
    G = group_header_words(3)

    def dirty():
        f.level_writes(0, [0], 3)
        f.owner[1].upload_level(0, mw.preload((f.lv[0].sy, f.lv[0].sx), f.rng))   # the whole level
        f.level_writes(2, [L - 1], 4)
        r = f.rects(sub)
        c = [cells_of(x) for x in r]
        assert c[1] > c[2] > 0 and c[0] > 0, c
        return r, c

    def run(cap, reset):
        f.og.pack_dirty_device(f.buf.data_ptr(), cap, reset, f.stream, members=sub)
        f.rg.unpack_dirty_device(f.buf.data_ptr(), cap, f.stream)

    def deferred_of(r, cap):
        hdr, blocks = layout(r, sub, cap, L)
        assert list(f.words(0, len(hdr))) == hdr, (cap, list(f.words(0, len(hdr))), hdr)
        for (start, ship), m in zip(blocks, sub):
            assert f.words(start + 2, 1)[0] == (0 if ship else 1)
        return [m for (_, ship), m in zip(blocks, sub) if not ship]

    r, c = dirty()
    before1 = [f.replica[1].download_level(l) for l in range(L)]
    cap = 4 * (G + 3 * HEADER_WORDS + c[0] + c[2])
    run(cap, True)
    assert deferred_of(r, cap) == [1]
    assert [f.replica[m].replication_overflows(reset=True) for m in range(M)] == [0, 1, 0, 0, 0]
    assert f.rects(sub) == [[None] * L, r[1], [None] * L]
    for l in range(L):
        assert np.array_equal(bits(f.replica[1].download_level(l)), bits(before1[l]))
    for m in (0, 2):
        f.note_shipped(m, r[m])
        f.check_member(m, "first fit: shipped")
    run(cap + 4 * c[1], True)   # the next call ships the deferred member
    f.note_shipped(1, r[1])
    f.check_member(1, "first fit: deferred member shipped next")
    assert f.replica[1].replication_overflows() == 0

    r, c = dirty()
    W = G + 3 * HEADER_WORDS + sum(c)
    for cap, want in ((4 * W, []), (4 * W + 3, []), (4 * W - 1, [2]), (4 * (W - 1), [2])):
        run(cap, False)
        assert deferred_of(r, cap) == want, (cap, want)
        assert f.rects(sub) == r
        assert [f.replica[m].replication_overflows(reset=True) for m in range(M)] == [int(m in want) for m in range(M)]
    for m in sub:
        f.note_shipped(m, r[m])
        f.check_member(m, "first fit: all shipped")
    # below the minimum: rejected, nothing written
    f.buf.fill_(7.0)
    with pytest.raises(capi.HsbError) as e:
        f.og.pack_dirty_device(f.buf.data_ptr(), 4 * (G + 3 * HEADER_WORDS) - 1, True, f.stream, members=sub)
    assert e.value.status == HSB_ERR_INVALID_ARG and "minimum" in str(e.value)
    f.og.pack_dirty_device(f.buf.data_ptr(), 4 * (G + 3 * HEADER_WORDS), False, f.stream, members=sub)
    assert deferred_of(r, 4 * (G + 3 * HEADER_WORDS)) == [0, 1, 2]
    f.close()


@pytest.mark.gpu
@MODES
def test_deferred_block_wider_than_the_buffer(hsb_lib, mode):
    """A deferred member whose rectangle is wider (and larger) than the whole buffer does not make the buffer foreign:
    the member that fits ships and lands on its replica, the deferred one is counted once on its own replica and
    keeps its rectangles, and the next, larger pack ships it."""
    geom = GEOMS[0]
    f = Fleets(geom, mode, seed=23 + mode)
    L = f.levels
    sub = [0, 1]
    G = group_header_words(2)
    # member 0: one short beam on level 0 (a rectangle of a few cells); member 1: its whole level 0 (404 x 300)
    L0 = f.lv[0]
    c = (L0.sx // 3, L0.sy // 2)
    pose = mw.pose_for_cell(L0, c[0], c[1], 0.0)
    pts = mw.points_for_targets(L0, pose, np.float64([[c[0] + 3, c[1] + 2]]))
    for rep in (f.owner[0], f.twin[0]):
        rep.update_level_by_scan(0, pts, pose)
    f.owner[1].upload_level(0, mw.preload((L0.sy, L0.sx), f.rng))
    r = f.rects(sub)
    c0, c1 = cells_of(r[0]), cells_of(r[1])
    cap = 4 * (G + 2 * HEADER_WORDS + c0)
    assert 0 < c0 and r[1][0] == (0, 0, L0.sx - 1, L0.sy - 1) and L0.sx > cap // 4, (r, cap)
    before1 = [f.replica[1].download_level(l) for l in range(L)]
    f.og.pack_dirty_device(f.buf.data_ptr(), cap, True, f.stream, members=sub)
    f.rg.unpack_dirty_device(f.buf.data_ptr(), cap, f.stream)
    hdr, blocks = layout(r, sub, cap, L)
    assert list(f.words(0, len(hdr))) == hdr and [s for _, s in blocks] == [True, False]
    assert [f.replica[m].replication_overflows(reset=True) for m in range(M)] == [0, 1, 0, 0, 0]
    assert f.rects(sub) == [[None] * L, r[1]]
    for l in range(L):
        assert np.array_equal(bits(f.replica[1].download_level(l)), bits(before1[l])), l
    f.note_shipped(0, r[0])
    f.check_member(0, "deferred block wider than the buffer: the other member")
    cap2 = 4 * (G + 2 * HEADER_WORDS + c1)
    f.og.pack_dirty_device(f.buf.data_ptr(), cap2, True, f.stream, members=sub)
    f.rg.unpack_dirty_device(f.buf.data_ptr(), cap2, f.stream)
    assert [f.replica[m].replication_overflows() for m in range(M)] == [0] * M
    f.note_shipped(1, r[1])
    for m in sub:
        f.check_member(m, "deferred block wider than the buffer: shipped next")
    f.close()


@pytest.mark.gpu
@MODES
def test_foreign_buffers(hsb_lib, mode):
    """Counted once on the replica group's handles[0] and nothing applied: a member index >= M, another level count,
    a single-handle buffer."""
    import torch

    from hector_slam_b200 import capi

    geom = GEOMS[0]
    f = Fleets(geom, mode, seed=13 + mode)
    L = f.levels
    small = capi.SlamGroup(f.replica[:3])
    for s in range(M):
        f.level_writes(s, [0], 5)
    snap = [[r.download_level(l) for l in range(L)] for r in f.replica]

    def unchanged(tag):
        for m in range(M):
            for l in range(L):
                assert np.array_equal(bits(f.replica[m].download_level(l)), bits(snap[m][l])), (tag, m, l)
        assert f.replica[0].replication_overflows(reset=True) == 1, tag
        assert all(r.replication_overflows() == 0 for r in f.replica[1:]), tag

    f.og.pack_dirty_device(f.buf.data_ptr(), f.cap, False, f.stream, members=[1, 4])
    small.unpack_dirty_device(f.buf.data_ptr(), f.cap, f.stream)
    unchanged("member index >= M")
    other = [make_rep((geom[0], geom[1], L - 1, geom[3]), s, mode) for s in range(2)]
    og2 = capi.SlamGroup(other)
    other[0].upload_level(0, mw.preload((f.lv[0].sy, f.lv[0].sx), f.rng))
    og2.pack_dirty_device(f.buf.data_ptr(), f.cap, True, f.stream)
    f.rg.unpack_dirty_device(f.buf.data_ptr(), f.cap, f.stream)
    unchanged("another level count")
    f.owner[0].pack_dirty_device(f.buf.data_ptr(), f.cap, False, f.stream)
    f.rg.unpack_dirty_device(f.buf.data_ptr(), f.cap, f.stream)
    unchanged("single-handle buffer")
    torch.cuda.synchronize()
    og2.close()
    small.close()
    for r in other:
        r.close()
    f.close()


@pytest.mark.gpu
@MODES
def test_ordering_without_synchronise(hsb_lib, mode):
    """A pack straight after a nowait group step ships that step's write; getDist, likelihood and group matches on the
    replica group straight after an unpack return the owner's results bit for bit."""
    import maptools_cases as mc

    geom = GEOMS[0]
    f = Fleets(geom, mode, seed=17 + mode)
    L = f.levels
    for t in range(3):
        f.group_step(2 * t, nowait=True)   # endpoints: every member matched, its last-match container set
        f.og.pack_dirty_device(f.buf.data_ptr(), f.cap, True, f.stream)
        f.rg.unpack_dirty_device(f.buf.data_ptr(), f.cap, f.stream)
        # the replica's containers are not replicated: queries pass their scans explicitly
        scans = [f.data[m]["scans"][f.at[m] - 1] for m in range(M)]
        level = t % L
        wb, we = [], []
        for m in range(M):
            sx, sy, cell = f.owner[m].level_info(level)
            b, e, _ = mc.world_rays(sx, sy, f.owner[m].map_origin(level), cell, 31 * t + m)
            pick = np.random.default_rng(t + m).choice(b.shape[0], 40)
            wb.append(np.ascontiguousarray(b[pick]))
            we.append(np.ascontiguousarray(e[pick]))
        got = f.rg.get_dist(level, wb, we)
        want = f.og.get_dist(level, wb, we)
        assert all(np.array_equal(bits(a), bits(b)) for a, b in zip(got[:2], want[:2])) and np.array_equal(got[2], want[2])
        poses = [f.data[m]["truth"][f.at[m] - 1][None, :] + np.float32([[0.0, 0.0, 0.0], [0.02, -0.01, 0.01]])
                 for m in range(M)]
        got = f.rg.likelihood(level, poses, points=scans)
        want = f.og.likelihood(level, poses, points=scans)
        assert np.array_equal(bits(got), bits(want)), t
        hints = [f.data[m]["hints"][f.at[m] - 1][None, :] for m in range(M)]
        got = f.rg.match_batch(hints, points=scans)
        want = f.og.match_batch(hints, points=scans)
        assert np.array_equal(bits(got[0]), bits(want[0])) and np.array_equal(bits(got[1]), bits(want[1])), t
    for m in range(M):
        for l in range(L):
            assert np.array_equal(bits(f.replica[m].download_level(l)), bits(f.owner[m].download_level(l))), (m, l)
    f.close()


@pytest.mark.gpu
@MODES
def test_launches_and_rejections(hsb_lib, mode):
    import ctypes as C

    import torch

    from hector_slam_b200 import capi

    geom = GEOMS[1]
    f = Fleets(geom, mode, seed=19 + mode)
    lib = capi.load_library()
    h0o, h0r = f.owner[0], f.replica[0]
    for reset, n in ((True, 2), (False, 1)):
        a = h0o.launch_count
        f.og.pack_dirty_device(f.buf.data_ptr(), f.cap, reset, f.stream, members=[2, 4])
        assert h0o.launch_count - a == n
        a = h0o.launch_count
        f.og.pack_dirty_device(f.buf.data_ptr(), f.cap, reset, f.stream)
        assert h0o.launch_count - a == n
    a = h0r.launch_count
    f.rg.unpack_dirty_device(f.buf.data_ptr(), f.cap, f.stream)
    assert h0r.launch_count - a == 1

    torch.cuda.synchronize()
    f.buf.fill_(3.0)
    ptr = f.buf.data_ptr()
    mem = lambda *v: (C.c_int * max(1, len(v)))(*v)   # noqa: E731
    cap = f.cap
    bad = [
        (lib.hsb_group_pack_dirty_device_subset, (f.og.g, -1, mem(0), ptr, cap, 1, f.stream), "K is -1"),
        (lib.hsb_group_pack_dirty_device_subset, (f.og.g, M + 1, mem(*range(M + 1)), ptr, cap, 1, f.stream), "K is"),
        (lib.hsb_group_pack_dirty_device_subset, (f.og.g, 2, None, ptr, cap, 1, f.stream), "members is NULL"),
        (lib.hsb_group_pack_dirty_device_subset, (f.og.g, 2, mem(0, M), ptr, cap, 1, f.stream), "session 1"),
        (lib.hsb_group_pack_dirty_device_subset, (f.og.g, 3, mem(1, 2, 1), ptr, cap, 1, f.stream), "session 2"),
        (lib.hsb_group_pack_dirty_device_subset, (f.og.g, 2, mem(0, 1), None, cap, 1, f.stream), "d_buf is NULL"),
        (lib.hsb_group_pack_dirty_device, (f.og.g, None, cap, 1, f.stream), "d_buf is NULL"),
        (lib.hsb_group_pack_dirty_device, (f.og.g, ptr, 4 * (group_header_words(M) + 64 * M) - 1, 1, f.stream),
         f"minimum of {4 * (group_header_words(M) + 64 * M)}"),
        (lib.hsb_group_pack_dirty_device_subset, (f.og.g, 2, mem(0, 1), ptr, 4 * (group_header_words(2) + 128) - 1, 1,
                                                     f.stream), f"minimum of {4 * (group_header_words(2) + 128)}"),
        (lib.hsb_group_unpack_dirty_device, (f.rg.g, None, cap, f.stream), "d_buf is NULL"),
        (lib.hsb_group_unpack_dirty_device, (f.rg.g, ptr, 4 * (8 + 64) - 1, f.stream), "minimum"),
    ]
    la, lb = h0o.launch_count, h0r.launch_count
    for fn, args, msg in bad:
        st = fn(*args)
        assert st == HSB_ERR_INVALID_ARG, (fn, msg)
        h = h0r.h if fn is lib.hsb_group_unpack_dirty_device else h0o.h
        err = (lib.hsb_last_error(h) or b"").decode()
        assert msg in err, (msg, err)
    assert lib.hsb_group_pack_dirty_device_subset(f.og.g, 0, None, ptr, 0, 1, f.stream) == 0   # K = 0
    assert (h0o.launch_count, h0r.launch_count) == (la, lb)
    torch.cuda.synchronize()
    assert bool((f.buf == 3.0).all())
    f.close()


@pytest.mark.gpu
def test_nccl_round_trip_two_gpus():
    """With two GPUs: one NCCL broadcast per tick replicates an owner group on rank 0 into a replica group on rank 1."""
    import torch

    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_nccl_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    results = [q.get(timeout=300) for _ in range(2)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    by_rank = {rank: (tag, value) for rank, tag, value in results}
    assert sorted(by_rank) == [0, 1] and all(tag == "ok" for tag, _ in by_rank.values()), by_rank
    assert by_rank[0][1] == by_rank[1][1], by_rank


def _nccl_worker(rank, world, port, q):
    import hashlib
    import sys

    import torch
    import torch.distributed as dist

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    sys.path.insert(0, os.path.join(root, "tests"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    try:
        from hector_slam_b200 import capi, parallel
        from test_gpu_group_subset import geometry, session_data

        geom = GEOMS[0]
        reps = []
        for s in range(3):
            rep = capi.MapRepB200(0.05, geom[0], geom[1], levels=geom[2], start=geom[3], device=rank)
            rep.set_scan_format(**geometry(s))
            reps.append(rep)
        g = capi.SlamGroup(reps)
        data = [session_data(s, 4, geometry(s)) for s in range(3)]
        buf = parallel.tile_buffer(torch.device("cuda", rank), 8 << 20)
        for t in range(4):
            if rank == 0:
                g.slam_update([d["hints"][t] for d in data], [d["scans"][t] for d in data])
            parallel.broadcast_group_dirty_tiles_async(g, buf, src=0)
        torch.cuda.synchronize()
        h = hashlib.sha256()
        for rep in reps:
            for l in range(geom[2]):
                h.update(rep.download_level(l).tobytes())
        g.close()
        for rep in reps:
            rep.close()
        q.put((rank, "ok", h.hexdigest()))
    except Exception as e:   # reported through the queue, tagged: the parent accepts only "ok" from both ranks
        q.put((rank, "error", repr(e)))
    finally:
        dist.destroy_process_group()
