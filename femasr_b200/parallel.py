"""Data-parallel sharding of the hot path across the GPUs of one node (one process per GPU).

Images (and test_tile tiles) are independent - GroupNorm is per-sample, LayerNorm per-token, attention
per-window, the VQ per-pixel against a replicated codebook (SURVEY.md 8e) - so the batch is split
contiguously, every rank runs the whole path on its shard with replicated weights, and the only
collective is ONE all-gather of the output shards (NCCL over NVLink on the GPU box; gloo in the CPU tests).
The reference has no multi-GPU inference path (basicsr/models/femasr_model.py:229-232).
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Tuple

import torch
import torch.distributed as dist


def shard_range(n: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous [start, stop) of rank's images; the first n % world ranks get one extra."""
    base, rem = divmod(n, world)
    start = rank * base + min(rank, rem)
    return start, start + base + (1 if rank < rem else 0)


def shard_counts(n: int, world: int) -> List[int]:
    return [shard_range(n, r, world)[1] - shard_range(n, r, world)[0] for r in range(world)]


def all_gather_outputs(local: torch.Tensor, counts: List[int], group: Optional[dist.ProcessGroup] = None) -> torch.Tensor:
    """Concatenate the per-rank output shards (rank order) on every rank with a single all-gather.
    Equal shards use all_gather_into_tensor directly into the result; ragged shards are padded to the
    largest shard for the collective and trimmed afterwards."""
    world = len(counts)
    if world == 1:
        return local
    tail = tuple(local.shape[1:])
    mx = max(counts)
    if mx == 0:
        return local.new_zeros((0,) + tail)
    if all(c == mx for c in counts):
        out = local.new_empty((world * mx,) + tail)
        dist.all_gather_into_tensor(out, local.contiguous(), group=group)
        return out
    padded = local.new_zeros((mx,) + tail)
    padded[: local.shape[0]] = local
    buf = local.new_empty((world * mx,) + tail)
    dist.all_gather_into_tensor(buf, padded, group=group)
    return torch.cat([buf[r * mx: r * mx + c] for r, c in enumerate(counts)], 0)


class PeerGather:
    """All-gather of EQUAL output shards by copy-engine peer writes instead of an NCCL kernel (one node, one process per GPU).

    Why: the tensor-core kernels of this path are persistent - 132 CTAs, one per SM, each with a STATIC share of the tiles
    and the whole 227 KB of shared memory.  An NCCL all-gather kernel that overlaps them (side stream) takes a few SMs for
    its own CTAs; the tc_igemm CTAs that find no SM start only when another CTA of the same launch has finished its share,
    so every launch in that window runs for up to two shares.  Peer-to-peer `cudaMemcpyAsync` over NVLink runs on the DMA
    engines and takes no SM.  Every rank owns `nbuf` gather buffers [world * B, ...]; their CUDA IPC handles are exchanged
    once (the mechanism torch.multiprocessing uses), and `push(k, shard)` writes the rank's shard into slot `rank` of buffer
    k on EVERY rank.  A buffer is complete on all ranks once every rank's pushes have finished (stream sync + barrier, or -
    as in bench.py - a timed region that ends with the max over ranks of each rank's own completion).

    Raises at construction when a peer cannot be mapped / accessed or the self-check against `all_gather_into_tensor`
    fails; callers fall back to the NCCL collective.
    """

    def __init__(self, shard_shape, dtype, device: torch.device, rank: int, world: int, nbuf: int = 2,
                 group: Optional[dist.ProcessGroup] = None):
        from torch.multiprocessing.reductions import reduce_tensor
        self.rank, self.world, self.B = rank, world, int(shard_shape[0])
        self.device = device
        self.full, self.peer = [], []
        # every step that can fail locally is followed by a collective vote, so that ALL ranks raise (and fall back) together
        mine, why = None, ""
        try:
            for r in range(world):
                if r != rank and not torch.cuda.can_device_access_peer(device.index, r):
                    raise RuntimeError(f"no peer access {device.index} -> {r}")
            tail = tuple(shard_shape[1:])
            self.full = [torch.empty((world * self.B,) + tail, dtype=dtype, device=device) for _ in range(nbuf)]
            mine = [reduce_tensor(t) for t in self.full]                # (rebuild function, picklable arguments)
        except Exception as ex:                                         # noqa: BLE001 - reported through the vote
            why = f"{type(ex).__name__}: {ex}"
        everyone: list = [None] * world
        dist.all_gather_object(everyone, mine, group=group)
        if mine is not None and all(e is not None for e in everyone):
            try:                                                        # peer[r][k]: rank r's buffer k, mapped into this process
                self.peer = [self.full if r == rank else [fn(*args) for fn, args in everyone[r]] for r in range(world)]
            except Exception as ex:                                     # noqa: BLE001
                why = f"{type(ex).__name__}: {ex}"
                self.peer = []
        elif not why:
            why = "another rank could not export its buffers"
        self._vote(bool(self.peer), group, why or "another rank could not map its peers")
        self.stream = torch.cuda.Stream(device=device)
        self._self_check(group)

    def _vote(self, ok: bool, group, why: str):
        flag = torch.tensor([1 if ok else 0], device=self.device)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=group)
        if int(flag.item()) != 1:
            self.close()
            raise RuntimeError(f"peer-copy all-gather unavailable ({why})")

    def close(self):
        """Drop the mapped peer buffers (before the process group goes away: the exporting process must outlive the maps)."""
        self.peer = []

    def push(self, k: int, shard: torch.Tensor, after: Optional[torch.cuda.Event] = None) -> torch.cuda.Event:
        """Enqueue (on the gather's own stream, after `after`) the copies of `shard` into slot `rank` of buffer k on every
        rank; returns the event that marks their completion on this rank."""
        lo, hi = self.rank * self.B, (self.rank + 1) * self.B
        with torch.cuda.stream(self.stream):
            if after is not None:
                self.stream.wait_event(after)
            for d in range(self.world):                                 # start with the next rank: no common first target
                r = (self.rank + 1 + d) % self.world
                self.peer[r][k][lo:hi].copy_(shard, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.stream)
        return ev

    def _self_check(self, group):
        g = torch.Generator(device="cpu").manual_seed(1234 + self.rank)
        probe = torch.rand((self.B,) + tuple(self.full[0].shape[1:]), generator=g).to(self.full[0].dtype).to(self.device)
        want = torch.empty_like(self.full[0])
        dist.all_gather_into_tensor(want, probe, group=group)
        ok, why = True, "self-check against all_gather_into_tensor failed"
        try:
            for k in range(len(self.full)):
                self.full[k].zero_()
            torch.cuda.synchronize(self.device)
        except Exception as ex:                                         # noqa: BLE001 - a local failure must not desynchronise the ranks
            ok, why = False, f"{type(ex).__name__}: {ex}"
        dist.barrier(group=group)
        try:
            if ok:
                for k in range(len(self.full)):
                    self.push(k, probe)
                self.stream.synchronize()
        except Exception as ex:                                         # noqa: BLE001
            ok, why = False, f"{type(ex).__name__}: {ex}"
        dist.barrier(group=group)                                       # every rank's pushes have landed
        ok = ok and all(torch.equal(self.full[k], want) for k in range(len(self.full)))
        self._vote(ok, group, why)


def sharded_forward(run: Callable[[torch.Tensor], torch.Tensor], x_global: torch.Tensor, rank: int, world: int,
                    group: Optional[dist.ProcessGroup] = None, out_shape_fn: Optional[Callable] = None) -> torch.Tensor:
    """Run `run` (e.g. FeMaSRNet.test) on this rank's contiguous slice of x_global [N,3,H,W] and return
    the gathered [N,3,sH,sW] result on every rank."""
    n = x_global.shape[0]
    a, b = shard_range(n, rank, world)
    counts = shard_counts(n, world)
    if b > a:
        local = run(x_global[a:b])
    else:
        if out_shape_fn is None:
            raise ValueError("an empty shard needs out_shape_fn to size its (empty) output")
        local = x_global.new_zeros((0,) + tuple(out_shape_fn(x_global.shape)[1:]))
    return all_gather_outputs(local, counts, group)


def tile_classes(height: int, width: int, tile_size: int, tile_pad: int) -> Dict[Tuple[int, int], List[dict]]:
    """The tiles of FeMaSRNet.test_tile (femasr_arch.py:387-447) grouped by the shape of their padded input window:
    tiles of one class can be stacked into one batch.  Deterministic order (row-major inside a class)."""
    from .net import tile_plan                      # pure Python (no CUDA needed to plan)
    classes: Dict[Tuple[int, int], List[dict]] = {}
    for t in tile_plan(height, width, tile_size, tile_pad):
        py0, py1, px0, px1 = t["in"]
        classes.setdefault((py1 - py0, px1 - px0), []).append(t)
    return classes


def sharded_test_tile(run: Callable[[torch.Tensor], torch.Tensor], x: torch.Tensor, scale: int, tile_size: int,
                      tile_pad: int, rank: int, world: int, group: Optional[dist.ProcessGroup] = None,
                      max_batch: int = 64) -> torch.Tensor:
    """test_tile with the TILE LIST sharded over the ranks (SURVEY.md 8e): inside every same-shape class the tiles are
    dealt round-robin, each rank runs `run` (e.g. FeMaSRNet.test) on stacks of its tiles, one all-gather per class
    brings the SR tiles to every rank, and every rank pastes the full [B,3,sH,sW] result.  `run` maps
    [n,3,th,tw] -> [n,3,s*th,s*tw]; tiles are independent on this path, so stacking does not change their values."""
    B, C, H, W = x.shape
    s = scale
    out = x.new_zeros((B, C, H * s, W * s))
    for (th, tw), tiles in tile_classes(H, W, tile_size, tile_pad).items():
        mine = tiles[rank::world]
        counts = [len(tiles[r::world]) * B for r in range(world)]
        parts = []
        per = max(1, max_batch // B)
        for i in range(0, len(mine), per):
            chunk = mine[i:i + per]
            stack = torch.cat([x[:, :, t["in"][0]:t["in"][1], t["in"][2]:t["in"][3]] for t in chunk], 0)
            parts.append(run(stack.contiguous()))
        local = torch.cat(parts, 0) if parts else x.new_zeros((0, C, th * s, tw * s))
        full = all_gather_outputs(local, counts, group)          # rank-major: rank 0's tiles, rank 1's tiles, ...
        order = [t for r in range(world) for t in tiles[r::world]]
        for k, t in enumerate(order):
            y0, y1, x0, x1 = t["out"]
            cy, cx = t["crop"]
            sr = full[k * B:(k + 1) * B]
            out[:, :, y0 * s:y1 * s, x0 * s:x1 * s] = sr[:, :, cy * s:(cy + y1 - y0) * s, cx * s:(cx + x1 - x0) * s]
    return out
