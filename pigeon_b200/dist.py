"""Multi-GPU plumbing: one process per GPU, batch sharded by sample, ONE all-gather per batch.

The reference's only inference-time collective is `accelerator.gather(output)` / `gather(index)` in
preprocessing/embed.py:36-37 (torch.distributed all_gather via accelerate).  Here the per-rank head outputs
(pooled embedding, top-k candidates, initial guess) are packed into one byte buffer and exchanged with a single
`all_gather_into_tensor` (NCCL over NVLink between the GPUs; gloo in the CPU tests), issued on the compute stream.
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import torch
import torch.distributed as dist


def is_distributed() -> bool:
    return dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1


def world_size() -> int:
    return dist.get_world_size() if (dist.is_available() and dist.is_initialized()) else 1


def shard_range(total: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous shard [lo, hi) of `total` samples for `rank` (remainder spread over the first ranks)."""
    base, rem = divmod(total, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def _pack(tensors: List[torch.Tensor]) -> Tuple[torch.Tensor, List[Tuple[torch.dtype, Tuple[int, ...], int]]]:
    metas, parts = [], []
    for t in tensors:
        t = t.contiguous()
        b = t.view(torch.uint8).reshape(-1)
        pad = (-b.numel()) % 16
        if pad:
            b = torch.cat([b, torch.zeros(pad, dtype=torch.uint8, device=b.device)])
        metas.append((t.dtype, tuple(t.shape), b.numel()))
        parts.append(b)
    return torch.cat(parts), metas


def all_gather_rows(tensors: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """Every tensor has the per-rank batch as dim 0 (same size on every rank). Returns the rank-ordered
    concatenation of each, using one collective for all of them."""
    if not is_distributed():
        return tensors
    world = dist.get_world_size()
    names = list(tensors)
    buf, metas = _pack([tensors[n] for n in names])
    out = torch.empty((world, buf.numel()), dtype=torch.uint8, device=buf.device)
    if dist.get_backend() == "nccl":
        dist.all_gather_into_tensor(out, buf)
    else:  # gloo (CPU tests)
        chunks = [torch.empty_like(buf) for _ in range(world)]
        dist.all_gather(chunks, buf)
        out = torch.stack(chunks)
    res, off = {}, 0
    for n, (dt, shape, nbytes) in zip(names, metas):
        real = 1
        for s in shape:
            real *= s
        real *= torch.empty((), dtype=dt).element_size()
        piece = out[:, off: off + real].contiguous().view(dt).reshape((world * shape[0],) + shape[1:])
        res[n] = piece
        off += nbytes
    return res


def merge_partials_by_owner(gathered: Dict[str, torch.Tensor], cand_cells: torch.Tensor, world: int) -> Dict[str, torch.Tensor]:
    """Cell-sharded retrieval: `gathered[name]` is the rank-ordered concatenation [world * B, topk, ...] of every rank's
    per-(query, candidate) partials; the partial of pair (b, j) that counts is the one of the rank holding geocell
    cand_cells[b, j], i.e. rank cand_cells[b, j] % world (bank.shard_bank).  Returns [B, topk, ...] tensors."""
    B, k = cand_cells.shape
    owner = torch.remainder(cand_cells, world).to(torch.int64)            # [B, k]
    out = {}
    for name, t in gathered.items():
        t = t.reshape((world, B) + tuple(t.shape[1:]))
        idx = owner.reshape((1, B, k) + (1,) * (t.dim() - 3)).expand((1,) + tuple(t.shape[1:]))
        out[name] = torch.gather(t, 0, idx)[0]
    return out
