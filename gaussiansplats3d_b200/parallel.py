"""Multi-GPU plumbing for the hot path: one process per GPU (torch.distributed), the rasteriser sharded by screen tile, the frame
assembled with ONE collective (the only one on the data path).

Ownership: coarse tile (cx, cy) (8 x 4 fine tiles: 128x64 px at 16-px tiles, 256x128 px at 32-px tiles, see tile_px) belongs to rank
(cx + cy) % world -- a diagonal interleave that spreads the dense centre and the empty border over all ranks.  Every rank holds the
whole scene (0.7 GB for 16M SH0 splats: replicas only) and sorts the full depth list, or from GS_SUBSET_MIN splats only the splats
that reach its own tiles (the order restricted to a rank's tiles is the global order, SURVEY.md 8e), so no splat data ever crosses
NVLink.  Each
rank writes its tiles into a full-size frame that is zero elsewhere; the frames are summed with one NCCL all-reduce on the ENGINE's
stream ("the final tile gather").
"""
from __future__ import annotations

import numpy as np

TILE = 16
COARSE_W, COARSE_H = 128, 64   # pixels (8 x 4 fine tiles of 16 px), csrc/raster_kernels.cuh kCoarseW/kCoarseH


def tile_px(width: int, height: int) -> int:
    """Fine-tile edge the engine uses for a frame (csrc/raster_kernels.cuh frame_tile_shift): 16 px while that gives at most 256 coarse
    tiles, else 32 px (a coarse tile is always 8 x 4 fine tiles)."""
    cx, cy = -(-width // COARSE_W), -(-height // COARSE_H)
    return TILE if cx * cy <= 256 else 2 * TILE


def owner_of_coarse(cx: int, cy: int, world: int) -> int:
    return (cx + cy) % world if world > 1 else 0


def ownership_map(width: int, height: int, world: int) -> np.ndarray:
    """[height, width] array of the rank that rasterises each pixel (GL row order)."""
    t = tile_px(width, height)
    ys, xs = np.mgrid[0:height, 0:width]
    return ((xs // (8 * t) + ys // (4 * t)) % max(world, 1)).astype(np.int32)


def combine_frames(frames: list):
    """Sum of the per-rank frames (what the all-reduce computes); numpy arrays or torch tensors."""
    out = frames[0].copy() if isinstance(frames[0], np.ndarray) else frames[0].clone()
    for f in frames[1:]:
        out += f
    return out


class _DevicePointer:
    """Expose a raw device pointer to torch through __cuda_array_interface__ (no copy)."""

    def __init__(self, ptr: int, nbytes: int):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 2}


class TileGather:
    """The final tile gather: every rank's finished tiles -> the whole frame on every rank, one NCCL all-reduce (SUM of frames that
    are zero outside their own tiles) enqueued on the ENGINE's stream (torch.cuda.ExternalStream), so it is ordered after the blend
    kernel without a host sync."""

    def __init__(self, engine, width: int, height: int, rank: int, world: int, fmt: int):
        import torch
        import torch.distributed as dist
        from . import _native as N
        self.torch, self.dist = torch, dist
        self.engine, self.width, self.height, self.rank, self.world = engine, width, height, rank, world
        self.rgba8 = fmt == N.GS_FRAME_RGBA8
        ptr, _ = engine.buffer_dev(N.GS_BUF_FRAME)
        nbytes = width * height * (4 if self.rgba8 else 16)
        dev = torch.device("cuda", torch.cuda.current_device())
        raw = torch.as_tensor(_DevicePointer(ptr, nbytes), device=dev)
        self.frame = raw if self.rgba8 else raw.view(torch.float32)      # summed in place: afterwards every rank holds the picture
        self.stream = torch.cuda.ExternalStream(engine.stream(), device=dev)

    def all_reduce(self) -> None:
        with self.torch.cuda.stream(self.stream):
            self.dist.all_reduce(self.frame, op=self.dist.ReduceOp.SUM)

    all_gather = all_reduce   # historical name used by bench.py

    def sync_to_torch(self) -> None:
        self.torch.cuda.current_stream().wait_stream(self.stream)

    def image(self):
        """[height, width, 4] view of the assembled frame (uint8 or float32) on the device."""
        return self.frame.view(self.height, self.width, -1) if self.rgba8 else self.frame.view(self.height, self.width, 4)


class PeerGather:
    """The final tile gather fused into the blend kernel: ranks > 0 store their finished pixels directly into rank 0's frame buffer
    over NVLink (CUDA IPC mapping, device-side release/arrive handshake); no collective call at all on the data path.  The IPC
    handles travel once through torch.distributed at set-up.  After a frame, only rank 0 holds the picture."""

    def __init__(self, engine, rank: int, world: int):
        import torch.distributed as dist
        self.engine, self.rank, self.world = engine, rank, world
        payload = [None]
        if rank == 0:
            payload = [engine.peer_export()]
        dist.broadcast_object_list(payload, src=0)
        if rank != 0:
            engine.peer_attach(*payload[0])
        dist.barrier()

    def all_gather(self) -> None:   # nothing to do: the gather happened inside the blend kernel
        pass

    all_reduce = all_gather


# ---- sort-only on N GPUs: one sortIndexes call split by input position (SURVEY.md 8(e), "depth + sort") -------------------------
def shard_bounds(sort_start: int, sort_count: int, world: int) -> list[tuple[int, int]]:
    """Input-position slice [lo, hi) of every rank (the C side uses the same integer formula)."""
    return [(sort_start + (sort_count * g) // world, sort_start + (sort_count * (g + 1)) // world) for g in range(world)]


def merge_sharded_order(sort_start: int, range_: int, per_rank: list[tuple[np.ndarray, np.ndarray]]) -> np.ndarray:
    """Host restatement of the exchange the kernels perform, for tests and documentation.

    per_rank[g] = (buckets, values) of rank g's slice in ORIGINAL input order (buckets computed with the GLOBAL min/max).
    Each rank orders its slice like the reference orders the whole window (bucket descending, later input position first,
    sorter.cpp:151-167); rank g's run of bucket b then starts after every run of a larger bucket and after the runs of bucket b
    held by ranks > g (their input positions are higher).  Returns the sorted part of indexesOut (without the head)."""
    world = len(per_rank)
    counts = np.zeros((world, range_), np.int64)
    local = []
    for g, (b, v) in enumerate(per_rank):
        b = np.asarray(b, np.int64)
        key = (range_ - 1) - b[::-1]                      # ascending key over the reversed slice == the reference's order
        order = np.argsort(key, kind="stable")
        local.append((key[order], np.asarray(v)[::-1][order]))
        counts[g] = np.bincount(key, minlength=range_)
    total = counts.sum(axis=0)
    before_key = np.concatenate([[0], np.cumsum(total)[:-1]])
    out = np.empty(int(total.sum()), np.uint32)
    for g in range(world):
        ahead = counts[g + 1:].sum(axis=0)                # same key, ranks with higher input positions
        start_local = np.concatenate([[0], np.cumsum(counts[g])[:-1]])
        keys, vals = local[g]
        j = np.arange(keys.size)
        out[j + (before_key + ahead - start_local)[keys]] = vals
    return out


class ShardedSort:
    """N processes, one GPU each: every rank sorts its slice of input positions and stores its part of the global order into
    rank 0's sortedIndexes over NVLink (CUDA IPC); the IPC handles travel once through torch.distributed at set-up."""

    def __init__(self, engine, rank: int, world: int):
        import torch.distributed as dist
        self.engine, self.rank, self.world = engine, rank, world
        mine = engine.shard_export()
        gathered = [None] * world
        dist.all_gather_object(gathered, mine)
        engine.shard_attach([h[0] for h in gathered], gathered[0][1])
        dist.barrier()

    def sort(self, mvp, sort_count: int, render_count: int, indexes=None, *, out=None, transforms=None, precomputed=None):
        """Collective: every rank calls it with the same arguments.  Rank 0 gets (sortedIndexes, ms); others (None, ms)."""
        if self.rank == 0 and out is None:
            out = np.empty(render_count, np.uint32)
        res, ms = self.engine.sort_sharded(mvp, sort_count, render_count, indexes, transforms=transforms, precomputed=precomputed,
                                           out=out if self.rank == 0 else None)
        return (res if self.rank == 0 else None), ms
