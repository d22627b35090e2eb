"""Single-node multi-GPU sharding of the hot path (SURVEY.md 8e): one process per GPU, ``torch.distributed``
(NCCL on GPUs; the host logic below is backend-agnostic and is tested with ``gloo`` on CPU).

* video-parallel (configs 2/3): videos dealt to ranks by longest-processing-time-first on ``video_cost`` =
  N_q * T * (T + 1) * c_map + T * c_frame; no data-path collective.
* frame-sharded long video (config 4): rank r owns a contiguous block of frames, runs ViT + delta-DINO for them
  writing straight into its slice of the full ``[T][P][C]`` buffer, then ONE in-place all-gather of the refined
  features (each (query, frame) correlation map needs only that frame + one descriptor, so any frame sharding is
  exact); query points are then sharded across ranks and the results gathered.
* best-buddies (config 5): features replicated, unordered frame pairs dealt round-robin
  (``best_buddies.best_buddies(rank=, world=)``), results gathered as objects.
"""
from typing import Callable, List, Sequence

import torch
import torch.distributed as dist


def frame_shard(T: int, world: int, rank: int):
    """Contiguous block of frames of ``rank``: sizes differ by at most one, earlier ranks get the extras."""
    base, extra = divmod(T, world)
    start = rank * base + min(rank, extra)
    return start, start + base + (1 if rank < extra else 0)


def query_shard(N: int, world: int, rank: int):
    return frame_shard(N, world, rank)


def video_cost(T: int, n_query_points: int, c_map: float = 2.5e-8, c_frame: float = 1.55e-2) -> float:
    """Seconds one video costs on one GPU: every query point is tracked into every frame (T maps) and, from each of its T
    track points, re-tracked into every anchor frame (<= T * T maps) -> N_q * T * (T + 1) correlation maps; the feature
    stage (ViT + delta-DINO) is per frame.  Defaults: relative weights of the two terms for the exact-window pipeline with ViT-L/14@15
    features; only their ratio matters to the assignment."""
    return n_query_points * T * (T + 1) * c_map + T * c_frame


def lpt_assign(costs: Sequence[float], world: int) -> List[List[int]]:
    """Longest-processing-time-first assignment of videos to ranks (costs: ``video_cost`` per video)."""
    order = sorted(range(len(costs)), key=lambda i: -costs[i])
    loads = [0.0] * world
    out = [[] for _ in range(world)]
    for i in order:
        r = min(range(world), key=lambda k: loads[k])
        out[r].append(i)
        loads[r] += costs[i]
    return out


def allgather_frames(full: torch.Tensor, T: int, world: int, rank: int, group=None) -> torch.Tensor:
    """In-place all-gather of a frame-sharded ``[T][...]`` buffer: every rank has filled its own block
    ``frame_shard(T, world, rank)`` of ``full``; afterwards all blocks are valid everywhere.
    Equal blocks go through one ``all_gather_into_tensor`` directly on ``full`` (NCCL: NVLink/NVSwitch ring or
    NVLS); ragged blocks (T % world != 0) are padded to the largest block in a staging buffer."""
    if world == 1:
        return full
    base, extra = divmod(T, world)
    if extra == 0:
        s, e = frame_shard(T, world, rank)
        dist.all_gather_into_tensor(full, full[s:e].contiguous() if not full[s:e].is_contiguous() else full[s:e], group=group)
        return full
    blk = base + 1
    stage = torch.zeros((world * blk,) + tuple(full.shape[1:]), dtype=full.dtype, device=full.device)
    s, e = frame_shard(T, world, rank)
    mine = torch.zeros((blk,) + tuple(full.shape[1:]), dtype=full.dtype, device=full.device)
    mine[: e - s] = full[s:e]
    dist.all_gather_into_tensor(stage, mine, group=group)
    for r in range(world):
        rs, re = frame_shard(T, world, r)
        if r != rank:
            full[rs:re] = stage[r * blk: r * blk + (re - rs)]
    return full


def gather_rows(local: torch.Tensor, N: int, world: int, rank: int, group=None) -> torch.Tensor:
    """All ranks end up with the ``[N][...]`` concatenation of their row shards (``query_shard``)."""
    if world == 1:
        return local
    blk = -(-N // world)
    mine = torch.zeros((blk,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    mine[: local.shape[0]] = local
    stage = torch.zeros((world * blk,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(stage, mine, group=group)
    parts = []
    for r in range(world):
        rs, re = query_shard(N, world, r)
        parts.append(stage[r * blk: r * blk + (re - rs)])
    return torch.cat(parts, dim=0)


def sharded_long_video_infer(T: int, N: int, world: int, rank: int, refine_block: Callable, infer_rows: Callable,
                             full_features: torch.Tensor, group=None):
    """Config-4 driver, generic over the compute callables so that it runs under gloo/CPU in tests:
      refine_block(s, e)      -> fills full_features[s:e] (ViT + delta-DINO of this rank's frames)
      infer_rows(qs, qe)      -> (traj [qe-qs][T][2], occ [qe-qs][T]) for this rank's query rows, using full_features
    Returns (traj [N][T][2], occ [N][T]) on every rank."""
    s, e = frame_shard(T, world, rank)
    refine_block(s, e)
    allgather_frames(full_features, T, world, rank, group)
    qs, qe = query_shard(N, world, rank)
    traj, occ = infer_rows(qs, qe)
    traj = gather_rows(traj, N, world, rank, group)
    occ = gather_rows(occ.to(torch.uint8), N, world, rank, group).bool()
    return traj, occ


class _DevPtr:
    """Minimal __cuda_array_interface__ carrier so that torch can view a raw device allocation."""

    def __init__(self, ptr, shape):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": "<f4", "data": (int(ptr), False), "version": 3}


class PeerFeatureBuffer:
    """A full ``[T][P][C]`` fp32 feature video on every rank of one node whose allocation is mapped into all peers
    (cudaMalloc + CUDA IPC), so that a producing kernel can store rows straight into every GPU's copy over NVLink.
    ``tensor`` views this rank's copy; ``peer_ptrs`` are the peers' mapped base pointers (own rank excluded)."""

    def __init__(self, T, P, C, rank, world, group=None):
        import ctypes
        from . import _lib
        self._lib = _lib.load()
        self.rank, self.world = rank, world
        nbytes = T * P * C * 4
        ptr = ctypes.c_void_p()
        handle = ctypes.create_string_buffer(64)
        _lib.check(self._lib.dinotrk_peer_alloc(nbytes, ctypes.byref(ptr), handle), "peer_alloc")
        self._own = ptr
        self.tensor = torch.as_tensor(_DevPtr(ptr.value, (T, P, C)), device=f"cuda:{torch.cuda.current_device()}")
        self.peer_ptrs, self._opened = [], []
        if world > 1:
            handles = [None] * world
            dist.all_gather_object(handles, handle.raw, group=group)
            for r, hraw in enumerate(handles):
                if r == rank:
                    continue
                p = ctypes.c_void_p()
                _lib.check(self._lib.dinotrk_peer_open(hraw, ctypes.byref(p)), "peer_open")
                self.peer_ptrs.append(p.value)
                self._opened.append(p)

    def sync(self, group=None):
        """Make every rank's peer stores visible: drain the local stream, then a rank barrier."""
        torch.cuda.synchronize()
        if self.world > 1:
            dist.barrier(group=group)

    def close(self):
        for p in self._opened:
            self._lib.dinotrk_peer_close(p)
        self._opened = []
        if self._own is not None:
            self.tensor = None
            self._lib.dinotrk_peer_free(self._own)
            self._own = None
