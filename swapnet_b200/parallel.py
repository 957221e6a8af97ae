"""Data-parallel plumbing (one process per GPU, torch.distributed; NCCL on the GPUs, gloo in CPU tests).

The hot path shards over the batch with no data-path collective: convs, InstanceNorm (per sample),
ROIAlign and the batch-mean losses are all per-sample, so equal shards + gradient averaging
reproduce the single-process gradient (SURVEY §8e).  The only exchange step is one all-reduce of
the flat fp32 gradient buffer per optimizer step; the smooth-label scalars (one draw per loss call
for the whole batch, loss.py:65-77) come from an identically seeded generator on every rank.  Batch norm couples the
samples of a call: with `--b200_sync_bn 1` its statistics are exchanged per call (BNStatsExchange).  The texture
stage's style loss couples every pair of samples: with `--b200_sync_style 1` the fakes and targets are gathered over the
same exchange each step (engine.PerceptualEngine.style).
"""
from __future__ import annotations

from typing import Iterable, Optional

import torch
import torch.distributed as dist


def launched_distributed() -> bool:
    """True under torchrun / torch.distributed.run with more than one rank (WORLD_SIZE in the environment)."""
    import os

    return int(os.environ.get("WORLD_SIZE", "1")) > 1


def init_from_env() -> int:
    """Create the NCCL process group from torchrun's environment (idempotent) and return this rank's GPU index
    (LOCAL_RANK).  Called by BaseModel.__init__, so the reference's train.py needs no distributed code."""
    import os

    local = int(os.environ.get("LOCAL_RANK", "0"))
    # the gradient all-reduces overlap G-backward: cap the SMs NCCL may take from the persistent GEMM kernels (the
    # transfers are hidden behind ~25 ms of backward either way; measured at 2 GPUs: 65.3 vs 65.8 ms/step)
    os.environ.setdefault("NCCL_MAX_CTAS", "16")
    if dist.is_available() and not dist.is_initialized():
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device(f"cuda:{local}"))
    return local


def world_size() -> int:
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


def rank() -> int:
    return dist.get_rank() if dist.is_available() and dist.is_initialized() else 0


def sum_gradients(flat_grad: torch.Tensor) -> None:
    """In-place SUM over ranks (the consumer applies 1/world: the fused AdamW kernel's gscale)."""
    if world_size() > 1:
        dist.all_reduce(flat_grad, op=dist.ReduceOp.SUM)


def average_gradients(flat_grad: torch.Tensor) -> None:
    """In-place mean over ranks of a flat gradient buffer (sum all-reduce + scale)."""
    w = world_size()
    if w > 1:
        dist.all_reduce(flat_grad, op=dist.ReduceOp.SUM)
        flat_grad.mul_(1.0 / w)


class BucketedAverager:
    """Overlaps the gradient all-reduce with the rest of the backward pass.

    The flat gradient buffer is cut into contiguous buckets in the order the backward pass finishes them
    (WarpEngine: decoder+head, resblocks, cloth branch, body branch).  `ready(i)` is called right after
    the last weight-gradient launch of bucket i has been enqueued: the all-reduce of that slice starts on
    NCCL's stream as soon as those kernels finish, while the remaining backward keeps the SMs busy.
    `finish()` waits for all of them and applies the 1/world scale."""

    def __init__(self, flat_grad: torch.Tensor, bounds, scale: bool = True):
        """scale=False: leave the SUM in the buffer (the AdamW kernel multiplies by 1/world as it reads it)."""
        self.flat, self.bounds, self.work, self.scale = flat_grad, list(bounds), [], scale

    def ready(self, i: int) -> None:
        if world_size() > 1:
            lo, hi = self.bounds[i]
            self.work.append(dist.all_reduce(self.flat[lo:hi], op=dist.ReduceOp.SUM, async_op=True))

    def finish(self) -> None:
        w = world_size()
        if w > 1:
            for wk in self.work:
                wk.wait()
            self.work.clear()
            if self.scale:
                self.flat.mul_(1.0 / w)


class BNStatsExchange:
    """Cross-rank batch-norm statistics (`--b200_sync_bn 1`): each BatchNorm2d call of a training step contributes its
    per-group partials ([groups, C, 3] fp64: element count, sum, sum of squares; ops.bn_group_sums) and receives every
    rank's, stacked in rank order ([world, groups, C, 3]).  The kernels sum the slices in that order, so every rank
    computes the same bits whatever the transport's reduction algorithm, and unequal shards are weighted by their counts.

    The exchange has a process group of its own: the gradient all-reduces that overlap the backward pass
    (BucketedAverager) queue on the default group's communicator, and a gather behind a large bucket there would stall
    the backward chain.  Every rank issues the gathers in the same order (the launch sequence is fixed), so they need no
    further synchronisation.  `group`: an existing process group (tests pass a gloo group)."""

    def __init__(self, group=None):
        self.group = group if group is not None else dist.new_group()
        self.world = dist.get_world_size(self.group)
        self.rank = dist.get_rank(self.group)
        self.gathers = 0            # gathers issued so far (the cost of the exchange is one latency-bound gather each)

    def buffers(self, groups: int, c: int, device) -> tuple:
        """(part [groups, c, 3], gathered [world, groups, c, 3]): fp64 buffers of one BatchNorm2d call site."""
        part = torch.zeros(groups, c, 3, dtype=torch.float64, device=device)
        return part, torch.zeros(self.world, groups, c, 3, dtype=torch.float64, device=device)

    def gather(self, part: torch.Tensor, gathered: torch.Tensor) -> torch.Tensor:
        """gathered[r] <- rank r's part, on the current stream."""
        assert part.is_contiguous() and gathered.is_contiguous() and gathered.numel() == self.world * part.numel()
        dist.all_gather_into_tensor(gathered.view(-1), part.view(-1), group=self.group)
        self.gathers += 1
        return gathered


def broadcast_parameters(params: Iterable[torch.Tensor], src: int = 0) -> None:
    if world_size() > 1:
        for p in params:
            dist.broadcast(p.data if hasattr(p, "data") else p, src)


class LabelDraws:
    """Smooth GAN labels exactly as GANLoss.get_target_tensor computes them (loss.py:65-107):
    fp32 `rand(1) * (1.1 - 0.7) + 0.7` for real AND fake targets.  Single process: the CPU default
    generator, like the reference.  Under DP: a dedicated generator with the same seed on all ranks."""

    def __init__(self, shared_seed: Optional[int] = None):
        self.gen = torch.Generator().manual_seed(shared_seed) if shared_seed is not None else None

    def draw(self) -> float:
        low, high = torch.tensor((0.7, 1.1))
        r = torch.rand(1, generator=self.gen) if self.gen is not None else torch.rand(1)
        return float(r * (high - low) + low)


def shard_batch(batch: dict, r: int, w: int) -> dict:
    """Rank r's contiguous slice [r*B/w, (r+1)*B/w) of every batched entry (tensors and lists).
    ROI rows need no re-indexing: rois stay [b, 12, 4] and the batch index is implicit."""
    out = {}
    for k, v in batch.items():
        n = len(v)
        assert n % w == 0, f"batch entry {k} of length {n} does not split over {w} ranks"
        out[k] = v[r * n // w:(r + 1) * n // w]
    return out
