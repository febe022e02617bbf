"""Multi-GPU plumbing (one process per GPU, torch.distributed).

The sampler path shards embarrassingly: every (audio, prompt, noise) sample is independent through the whole
DDIM loop and the decode (no cross-sample op exists in the U-Net; SURVEY §8e).  So the only collective is
the one-time broadcast of the packed weight blob from rank 0 over NCCL/NVLink; after that each rank runs
its contiguous slice of the batch with zero per-step traffic.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist

from .config import ModelConfig
from .packer import WeightBlob, pack_model


def shard_range(total: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous, balanced slice [lo, hi) of ``total`` samples for ``rank`` (first ranks get the remainder)."""
    base, rem = divmod(total, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_batch(tensors: Sequence[torch.Tensor], rank: int, world: int) -> List[torch.Tensor]:
    lo, hi = shard_range(tensors[0].shape[0], rank, world)
    return [t[lo:hi] for t in tensors]


def broadcast_blob(state_dict: Optional[Dict[str, torch.Tensor]], cfg: ModelConfig, device: torch.device, src: int = 0) -> WeightBlob:
    """Rank ``src`` packs the state_dict; everybody receives the flat fp32 blob (one broadcast of 0.56 GB: plain weights only) plus the
    small layout table (broadcast_object_list).  Works with NCCL (device tensors) and gloo (CPU)."""
    rank = dist.get_rank()
    blob = pack_model(state_dict, cfg.unet, cfg.decoder) if rank == src else None
    meta = [(blob.entries, blob.meta, blob.numel, blob.tc, blob.tc_lo_numel) if rank == src else None]
    dist.broadcast_object_list(meta, src=src)
    entries, bmeta, numel, tc, tc_lo_numel = meta[0]
    use_cuda = dist.get_backend() == "nccl"
    if rank == src:
        flat = blob.data.to(device) if use_cuda else blob.data
    else:
        flat = torch.empty(numel, dtype=torch.float32, device=device if use_cuda else "cpu")
    dist.broadcast(flat, src=src)
    if rank != src:
        blob = WeightBlob()
        blob.entries, blob.meta, blob._size = entries, bmeta, numel
        blob.tc, blob.tc_lo_numel = tc, tc_lo_numel
    blob.data = flat      # plain fp32, every weight once: each rank derives the TF32 hi / lo operands on its own device (MugEngine)
    return blob


def gather_batch(local: torch.Tensor, sizes: Sequence[int], dst: int = 0) -> Optional[torch.Tensor]:
    """Optional final gather of per-rank results (e.g. logits [b_r,16,8L]) onto ``dst``.  Shards may differ by one
    sample, collectives want equal shapes: pad to the largest shard, gather, trim."""
    world = dist.get_world_size()
    rank = dist.get_rank()
    mx = max(sizes)
    padded = local.contiguous()
    if padded.shape[0] < mx:
        pad = torch.zeros((mx - padded.shape[0],) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
        padded = torch.cat([padded, pad], dim=0)
    if rank == dst:
        bufs = [torch.empty_like(padded) for _ in range(world)]
        dist.gather(padded, bufs, dst=dst)
        return torch.cat([bufs[r][:sizes[r]] for r in range(world)], dim=0)
    dist.gather(padded, None, dst=dst)
    return None


def scatter_batch(tensors: Optional[Sequence[torch.Tensor]], shapes: Sequence[Sequence[int]], device: torch.device, src: int = 0) -> List[torch.Tensor]:
    """Rank ``src`` holds whole-batch tensors (``shapes[i]`` = their shapes, known on every rank); every rank receives its contiguous
    shard (shard_range).  Shards may differ by one sample, collectives want equal shapes: pad to the largest shard, scatter, trim."""
    world, rank = dist.get_world_size(), dist.get_rank()
    use_cuda = dist.get_backend() == "nccl"
    dev = device if use_cuda else torch.device("cpu")
    out = []
    for i, shape in enumerate(shapes):
        total = int(shape[0])
        spans = [shard_range(total, r, world) for r in range(world)]
        mx = max(b - a for a, b in spans)
        recv = torch.empty((mx,) + tuple(shape[1:]), dtype=torch.float32, device=dev)
        if rank == src:
            full = tensors[i].to(dev, torch.float32)
            chunks = []
            for a, b in spans:
                c = full[a:b]
                if b - a < mx:
                    c = torch.cat([c, torch.zeros((mx - (b - a),) + tuple(shape[1:]), dtype=torch.float32, device=dev)])
                chunks.append(c.contiguous())
            dist.scatter(recv, chunks, src=src)
        else:
            dist.scatter(recv, None, src=src)
        a, b = spans[rank]
        out.append(recv[:b - a].to(device))
    return out


def sample_sharded(sample_fn, request: Optional[Dict[str, object]], shapes: Dict[str, Sequence[int]], device: torch.device, src: int = 0,
                   z_lengths=None):
    """One sampling request over all ranks (BASELINE config 4: 256 charts on 8 GPUs): rank ``src`` holds the request
    (x_T [B,16,L], c / uc [B,128,T], w = the four audio feature maps), every rank receives its contiguous slice of the batch, runs
    ``sample_fn(x_T, c, uc, w) -> result [b, ...]`` on it -- the samples are independent through the whole DDIM loop and the decode, so
    there is no collective per step -- and the results are gathered on ``src`` in batch order (None elsewhere).
    ``shapes``: the whole-batch shapes of ``x_T``, ``c``, ``uc`` and ``w0..w3`` (known to every rank, e.g. from the request header)."""
    if z_lengths is not None:
        from .lib import MugdError
        raise MugdError("z_lengths: sharding a request of charts of different lengths is not supported; run it on one GPU")
    keys = ["x_T", "c", "uc", "w0", "w1", "w2", "w3"]
    rank, world = dist.get_rank(), dist.get_world_size()
    tensors = None
    if rank == src:
        tensors = [request["x_T"], request["c"], request["uc"]] + list(request["w"])[-4:]
    parts = scatter_batch(tensors, [shapes[k] for k in keys], device, src)
    local = sample_fn(parts[0], parts[1], parts[2], parts[3:])
    total = int(shapes["x_T"][0])
    sizes = [shard_range(total, r, world)[1] - shard_range(total, r, world)[0] for r in range(world)]
    if dist.get_backend() != "nccl":
        local = local.cpu()
    return gather_batch(local, sizes, dst=src)
