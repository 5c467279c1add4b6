"""Multi-GPU partition of the DfM hot path (SURVEY.md section 8e).

The path shards over *pairs* (independent frames): the reference cannot batch
(dfm_backbone.py:160 supports B=1 only), so N GPUs run N frames with zero
data-path communication -- exact, and weak scaling.  The only collective is the
MAX-reduction of the per-rank step time for reporting.

Depth-slab sharding of ONE frame (what BASELINE.json's north_star sketches) is not a
single-exchange partition: every GroupNorm needs a global per-channel sum (18
all-reduces per frame) and every 3x3x3 conv a one-plane halo at its own resolution
(22 exchanges); with a single-GPU frame of ~10 ms (H100) made of sub-millisecond kernels those
~40 latency-bound exchanges cannot pay off.  It is documented in DESIGN.md and left out.
"""
import torch
import torch.distributed as dist


def shard_pairs(pairs, rank, world):
    """Round-robin ownership of frame pairs."""
    return [p for i, p in enumerate(pairs) if i % world == rank]


def reduce_step_time(ms, device):
    """max over ranks of a per-rank elapsed time (ms)."""
    t = torch.tensor([float(ms)], device=device)
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())
