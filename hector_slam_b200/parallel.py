"""Multi-GPU plumbing: one process per GPU, `torch.distributed` (NCCL on the GPUs, gloo in the CPU
tests).  The match path shards by scan / hypothesis and needs NO collective on the data path:
every rank holds a replica of the map and matches its contiguous share.  Collectives appear only
where the path has a real exchange: replicating the map (broadcast of the log-odds planes from the
rank that owns / writes the map) and, optionally, assembling the result poses (all_gather).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.distributed as dist


def _parse_cpulist(text: str) -> set[int]:
    cpus: set[int] = set()
    for part in text.strip().split(","):
        if not part:
            continue
        if "-" in part:
            lo, hi = part.split("-")
            cpus.update(range(int(lo), int(hi) + 1))
        else:
            cpus.add(int(part))
    return cpus


def bind_process_to_gpu_numa_node(device_index: int):
    """Pin this process to the CPUs of the NUMA node the GPU hangs off, so that pinned host buffers
    allocated afterwards are local to the GPU's PCIe root (a far-socket buffer copies at a fraction of the
    near one's rate).  Returns the previous
    affinity (to restore with os.sched_setaffinity) or None if nothing could be done."""
    import os

    try:
        prop = torch.cuda.get_device_properties(device_index)
        bdf = f"{prop.pci_domain_id:04x}:{prop.pci_bus_id:02x}:{prop.pci_device_id:02x}.0"
        with open(f"/sys/bus/pci/devices/{bdf}/numa_node") as f:
            node = int(f.read().strip())
        if node < 0:
            return None
        with open(f"/sys/devices/system/node/node{node}/cpulist") as f:
            cpus = _parse_cpulist(f.read())
        prev = os.sched_getaffinity(0)
        cpus &= prev
        if not cpus:
            return None
        os.sched_setaffinity(0, cpus)
        return prev
    except Exception:
        return None


def pinned_copy(array) -> "torch.Tensor":
    """Pinned host tensor holding a copy of `array` (numpy or tensor): the pinned block is allocated first, by the
    calling thread (so on the NUMA node the process is bound to), then filled.  (freshly allocated pinned blocks
    copy to the device at a steady rate, `tensor.pin_memory()` results at widely varying ones.)"""
    src = array if isinstance(array, torch.Tensor) else torch.from_numpy(array)
    out = torch.empty(src.shape, dtype=src.dtype, pin_memory=True)
    out.copy_(src)
    return out


def pinned_empty(shape, dtype=torch.float32) -> "torch.Tensor":
    return torch.empty(shape, dtype=dtype, pin_memory=True)


def shard_range(n: int, rank: int, world: int) -> tuple[int, int]:
    """Contiguous balanced partition of range(n): shard sizes differ by at most one."""
    lo = (n * rank) // world
    hi = (n * (rank + 1)) // world
    return lo, hi


def shard_scans(hints, pts, offsets, rank: int, world: int):
    """This rank's contiguous share of a ragged scan batch, offsets rebased to zero."""
    B = hints.shape[0]
    lo, hi = shard_range(B, rank, world)
    offsets = np.asarray(offsets)
    p0, p1 = int(offsets[lo]), int(offsets[hi])
    return hints[lo:hi], pts[p0:p1], (offsets[lo:hi + 1] - p0).astype(np.int32), (lo, hi)


class _DevicePlane:
    """Zero-copy torch view of a raw device plane (the handle owns the memory)."""

    def __init__(self, ptr: int, shape):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": "<f4", "data": (int(ptr), False), "version": 2}


def level_plane_tensor(rep, level: int, device) -> torch.Tensor:
    """The handle's log-odds plane of `level` as a torch CUDA tensor (no copy)."""
    sx, sy, _ = rep.level_info(level)
    return torch.as_tensor(_DevicePlane(rep.level_logodds_device_ptr(level), (sy, sx)), device=device)


def broadcast_planes(planes: list[torch.Tensor], src: int = 0, group=None) -> None:
    """Replicate the map: one broadcast per level plane from the owner rank."""
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return
    for p in planes:
        dist.broadcast(p, src=src, group=group)


def replicate_map(rep, device, src: int = 0, group=None) -> list[torch.Tensor]:
    """Broadcast every level's log-odds plane from `src` into this rank's handle and refresh the
    probability planes of the receivers. Returns the plane views."""
    planes = [level_plane_tensor(rep, l, device) for l in range(rep.getMapLevels())]
    if dist.is_initialized() and dist.get_world_size(group) > 1:
        broadcast_planes(planes, src, group)
        torch.cuda.synchronize(device)
        if dist.get_rank(group) != src:
            for l in range(rep.getMapLevels()):
                rep.refresh_level(l, 0)
            torch.cuda.synchronize(device)
    return planes


def gather_rows(local: torch.Tensor, n_total: int, group=None) -> torch.Tensor:
    """all_gather of per-rank row blocks produced by shard_range (uneven blocks are padded)."""
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return local
    world = dist.get_world_size(group)
    sizes = [shard_range(n_total, r, world) for r in range(world)]
    mx = max(hi - lo for lo, hi in sizes)
    pad = torch.zeros((mx,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    pad[: local.shape[0]] = local
    out = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(out, pad, group=group)
    return torch.cat([o[: hi - lo] for o, (lo, hi) in zip(out, sizes)], dim=0)


def match_sharded(match_fn, hints, pts, offsets, group=None, device="cpu"):
    """Match a ragged batch sharded over the ranks of `group`: every rank runs `match_fn(hints,
    pts, offsets) -> (poses (b,3), cov (b,3,3))` on its contiguous share (no collective on the data
    path) and the poses / covariances are assembled on every rank."""
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    h, p, o, (lo, hi) = shard_scans(hints, pts, offsets, rank, world)
    poses, cov = match_fn(h, p, o)
    poses_t = torch.as_tensor(np.ascontiguousarray(poses, dtype=np.float32), device=device).reshape(hi - lo, 3)
    cov_t = torch.as_tensor(np.ascontiguousarray(cov, dtype=np.float32), device=device).reshape(hi - lo, 9)
    B = hints.shape[0]
    return gather_rows(poses_t, B, group), gather_rows(cov_t, B, group).reshape(B, 3, 3)


def broadcast_dirty_tiles(rep, device, src: int = 0, group=None, stats: dict | None = None) -> int:
    """After the owner rank (`src`) has written its map (hsb_update_by_scan / hsb_slam_update), ship what changed to
    the replicas.  Two collectives per call, whatever the number of levels: the dirty rectangles of ALL levels (levels x 4
    int32, read from the owner's device with one copy) and ONE packed buffer holding the log-odds rows of every
    level's rectangle back to back; replicas write the rows into their planes and refresh the probabilities (and the
    texture twin) there.  pack / unpack are ordered against the handle's own streams inside the C-ABI (see
    hsb_pack_rect_device), so the caller needs no synchronisation before the next match or map write.
    Returns the number of cells shipped.  `stats` (optional dict) receives "cells", "bytes".  No-op without a
    process group (the rectangles are still reset)."""
    levels = rep.getMapLevels()
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        rep.get_dirty_rects(reset=True)
        return 0
    rank = dist.get_rank(group)
    on_gpu = torch.device(device).type == "cuda"
    stream = torch.cuda.current_stream(device).cuda_stream if on_gpu else 0
    rects_t = torch.empty(levels * 4, dtype=torch.int32, device=device)
    if rank == src:
        flat = []
        for r in rep.get_dirty_rects(reset=True):
            flat.extend(r if r is not None else (0, 0, -1, -1))       # clean: x1 < x0
        rects_t.copy_(torch.tensor(flat, dtype=torch.int32))
    dist.broadcast(rects_t, src=src, group=group)
    rects = rects_t.cpu().view(levels, 4).tolist()
    sizes = [max(0, r[2] - r[0] + 1) * max(0, r[3] - r[1] + 1) for r in rects]
    total = int(sum(sizes))
    if stats is not None:
        stats["cells"], stats["bytes"] = total, 4 * total + 16 * levels
    if total == 0:
        return 0
    buf = torch.empty(total, dtype=torch.float32, device=device)
    off = 0
    if rank == src:
        for l, (r, n) in enumerate(zip(rects, sizes)):
            if n:
                rep.pack_rect_device(l, r, buf.data_ptr() + 4 * off, stream)
            off += n
    dist.broadcast(buf, src=src, group=group)
    if rank != src:
        off = 0
        for l, (r, n) in enumerate(zip(rects, sizes)):
            if n:
                rep.unpack_rect_device(l, r, buf.data_ptr() + 4 * off, stream)
            off += n
        # `buf` may be recycled by torch's allocator as soon as this function returns: the unpack kernels were
        # queued on torch's current stream, which is the stream the allocator tracks the block on — safe.
    return total


def tile_buffer(device, capacity_bytes: int = 4 << 20) -> torch.Tensor:
    """A device buffer for broadcast_dirty_tiles_async (allocate once, reuse every step)."""
    return torch.empty(capacity_bytes // 4, dtype=torch.float32, device=device)


def broadcast_dirty_tiles_async(rep, buf: torch.Tensor, src: int = 0, group=None) -> None:
    """The same replication step with no host in the loop: the owner packs the dirty rectangles of all levels AND their
    descriptions into `buf` on the device (hsb_pack_dirty_device), ONE fixed-size broadcast moves it, the replicas
    unpack from the buffer's own header (hsb_unpack_dirty_device).  Nothing is read back, nothing synchronises: the
    three operations are queued on torch's current stream and ordered against the handle's streams inside the C-ABI, so
    the call costs the host three launches (the two-step protocol needs the rectangle sizes on every host first).  If the dirty area exceeds the buffer the owner ships nothing and keeps its rectangles; replicas
    count that (rep.replication_overflows()) — call broadcast_dirty_tiles() then."""
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return
    nbytes = buf.numel() * 4
    stream = torch.cuda.current_stream(buf.device).cuda_stream if buf.is_cuda else 0   # (CPU tensors: the gloo tests)
    if dist.get_rank(group) == src:
        rep.pack_dirty_device(buf.data_ptr(), nbytes, True, stream)
    dist.broadcast(buf, src=src, group=group)
    if dist.get_rank(group) != src:
        rep.unpack_dirty_device(buf.data_ptr(), nbytes, stream)


def broadcast_group_dirty_tiles_async(group, buf: torch.Tensor, src: int = 0, members=None, pg=None) -> None:
    """The group form of broadcast_dirty_tiles_async: the owner rank packs every listed member's dirty tiles into `buf`
    with one launch (SlamGroup.pack_dirty_device: a group header, then one block per session, rows placed first-fit),
    ONE fixed-size broadcast moves it, and the replica ranks apply it to their group with one launch
    (SlamGroup.unpack_dirty_device), which must list its handles in the owner group's order.  One collective per tick
    whatever the number of robots, nothing read back, nothing synchronised.  A member whose rows did not fit is deferred:
    it keeps its rectangles on the owner and ships with the next call; its replica counts it
    (reps[k].replication_overflows()).  `members` (owner side): pack only these members, in session order."""
    if not dist.is_initialized() or dist.get_world_size(pg) == 1:
        return
    nbytes = buf.numel() * 4
    stream = torch.cuda.current_stream(buf.device).cuda_stream if buf.is_cuda else 0   # (CPU tensors: the gloo tests)
    if dist.get_rank(pg) == src:
        group.pack_dirty_device(buf.data_ptr(), nbytes, True, stream, members=members)
    dist.broadcast(buf, src=src, group=pg)
    if dist.get_rank(pg) != src:
        group.unpack_dirty_device(buf.data_ptr(), nbytes, stream)
