"""Multi-GPU host logic (SURVEY.md section 8e): one process per GPU.

* classify / embed: prompts are independent -> every rank takes a contiguous slice of the request batch, weights
  are replicated, NO data-path collective.
* partitioned semantic cache: rank r owns rows [r*N/G, (r+1)*N/G); every rank scans its shard for the whole query
  batch (queries are replicated at enqueue), the per-shard [B,k] (score, GLOBAL id) lists are exchanged with ONE
  all-gather (B*k*8 bytes per rank: {fp32 score, int32 global id} entries; NCCL over NVLink on GPUs, gloo in the CPU tests) and merged with the reference
  tie rule (descending score, lower global index first).  Exact caches take the same exchange with fp32 queries: each
  shard's list holds the exact scores of its own rows, so the merge is the unsharded exact result.
"""
from __future__ import annotations

from typing import Tuple

import numpy as np


def shard_range(n: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous, balanced partition of n items: first (n % world) ranks get one extra."""
    base, rem = divmod(n, world)
    start = rank * base + min(rank, rem)
    return start, start + base + (1 if rank < rem else 0)


def _gather_pairs(payload, group=None):
    """payload int32 [B,k,2] = 8-byte entries {score bits, global id} -> [world, B, k, 2] (ONE collective)."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(group)
    out = torch.empty((world,) + tuple(payload.shape), dtype=payload.dtype, device=payload.device)
    try:
        dist.all_gather_into_tensor(out, payload, group=group)
    except (RuntimeError, NotImplementedError):      # a backend without the flat form
        parts = [torch.empty_like(payload) for _ in range(world)]
        dist.all_gather(parts, payload, group=group)
        out = torch.stack(parts)
    return out


def allgather_topk(idx, score, group=None):
    """idx int32 [B,k], score float32 [B,k] (torch tensors on this rank's device, GLOBAL ids) ->
    merged (idx, score) numpy arrays, identical on every rank.  The exchange is B*k*8 bytes per rank: one int32 pair
    {score bits, id} per entry.  CUDA tensors are merged on the device (merge_packed_kernel), CPU tensors (the gloo
    tests) on the host with the same tie rule."""
    import torch
    payload = torch.stack([score.contiguous().view(torch.int32), idx.to(torch.int32)], dim=-1).contiguous()
    gathered = _gather_pairs(payload, group)
    world, b, k = gathered.shape[0], gathered.shape[1], gathered.shape[2]
    if gathered.is_cuda:
        from .binding import lib
        import ctypes as C
        oi = torch.empty((b, k), dtype=torch.int32, device=gathered.device)
        os_ = torch.empty((b, k), dtype=torch.float32, device=gathered.device)
        rc = lib().sr_cache_merge_packed_dev(gathered.device.index, C.c_void_p(gathered.data_ptr()), world, b, k,
                                             C.c_void_p(oi.data_ptr()), C.c_void_p(os_.data_ptr()),
                                             C.c_void_p(torch.cuda.current_stream().cuda_stream))
        if rc != 0:
            raise RuntimeError("sr_cache_merge_packed_dev failed")
        return oi.cpu().numpy(), os_.cpu().numpy()
    from .binding import merge_topk
    gs = gathered[..., 0].contiguous().view(torch.float32)
    gi = gathered[..., 1].contiguous()
    return merge_topk([gi[r].numpy() for r in range(world)], [gs[r].numpy() for r in range(world)])


def sharded_topk_dev(cache, d_queries, k: int, group=None):
    """The whole sharded lookup on the device (cfg 4): scan this rank's shard for the (replicated) query batch, pack,
    all-gather 8-byte entries over NCCL, merge.  `cache`: binding.Cache holding this rank's rows with id_offset = first
    global row; d_queries: torch CUDA tensor [B, D], fp16 (sr_cache_topk_packed_dev) or fp32
    (sr_cache_topk_packed_f32_dev: the route of exact caches, whose merged lists are the unsharded exact result).
    Returns (idx int32 [B,k], score fp32 [B,k]) CUDA tensors, identical on every rank.  Everything is queued on torch's
    current stream."""
    import ctypes as C
    import torch
    from .binding import lib
    b = d_queries.shape[0]
    dev = d_queries.device
    # torch's default stream is the legacy stream, handle 0, which the C ABI reads as "the cache's own stream": name it
    # cudaStreamLegacy (1) so that the scan is ordered before the all-gather
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream or 1)
    pairs = torch.empty((b, k, 2), dtype=torch.int32, device=dev)
    scan = lib().sr_cache_topk_packed_f32_dev if d_queries.dtype == torch.float32 else lib().sr_cache_topk_packed_dev
    if scan(cache.handle, C.c_void_p(d_queries.data_ptr()), b, k, C.c_void_p(pairs.data_ptr()), stream) != 0:
        raise RuntimeError(f"{scan.__name__} failed")
    gathered = _gather_pairs(pairs, group)
    oi = torch.empty((b, k), dtype=torch.int32, device=dev)
    os_ = torch.empty((b, k), dtype=torch.float32, device=dev)
    if lib().sr_cache_merge_packed_dev(dev.index, C.c_void_p(gathered.data_ptr()), gathered.shape[0], b, k,
                                       C.c_void_p(oi.data_ptr()), C.c_void_p(os_.data_ptr()), stream) != 0:
        raise RuntimeError("sr_cache_merge_packed_dev failed")
    return oi, os_
