"""`--b200_sync_bn` without a GPU: the option, the statistics exchange over a gloo group of two ranks, and an fp64
restatement of what the kernels compute from the gathered partials (csrc/elementwise.cu bn_group_sums_kernel,
bn_finalize_gathered_kernel) against F.batch_norm on the concatenated batch."""
import os
from argparse import ArgumentParser, Namespace

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F

from swapnet_b200 import parallel
from swapnet_b200.models.base_gan import BaseGAN, batch_norm_exchange


def test_flag_is_registered_with_default_off():
    for is_train in (True, False):
        p = BaseGAN.modify_commandline_options(ArgumentParser(), is_train)
        assert p.parse_args([]).b200_sync_bn == 0
        assert p.parse_args(["--b200_sync_bn", "1"]).b200_sync_bn == 1
        with pytest.raises(SystemExit):
            p.parse_args(["--b200_sync_bn", "2"])


def test_refusal_names_the_flag():
    opt = Namespace(norm="batch")
    with pytest.raises(NotImplementedError, match="cross-rank batch statistics.*--b200_sync_bn 1"):
        batch_norm_exchange(opt, 2)
    with pytest.raises(NotImplementedError, match="--b200_sync_bn 1"):
        batch_norm_exchange(Namespace(norm="batch", b200_sync_bn=0), 4)
    # local statistics: one rank, or no batch norm, whatever the flag says
    for o, world in ((Namespace(norm="batch", b200_sync_bn=1), 1), (Namespace(norm="instance", b200_sync_bn=1), 2),
                     (Namespace(norm="none", b200_sync_bn=0), 2)):
        assert batch_norm_exchange(o, world) is None


def _partials(shard: torch.Tensor, groups: int) -> torch.Tensor:
    """[groups, C, 3] = (element count, sum, sum of squares) of the shard's samples of each group (NCHW fp64)."""
    n, c, h, w = shard.shape
    per = n // groups
    out = torch.zeros(groups, c, 3, dtype=torch.float64)
    for g in range(groups):
        x = shard[g * per:(g + 1) * per]
        out[g, :, 0] = per * h * w
        out[g, :, 1] = x.sum((0, 2, 3))
        out[g, :, 2] = (x * x).sum((0, 2, 3))
    return out


def _finalize(gathered: torch.Tensor, rm: torch.Tensor, rv: torch.Tensor, eps=1e-5, momentum=0.1):
    """The kernels' arithmetic on the gathered partials, group after group: (mean, biased variance) per group, the
    running buffers updated with the unbiased variance over the global count."""
    means, vars_ = [], []
    for g in range(gathered.shape[1]):
        cnt, s1, s2 = gathered[:, g].sum(0).unbind(-1)
        mean = s1 / cnt
        var = (s2 / cnt - mean * mean).clamp_min(0)
        rm.mul_(1 - momentum).add_(momentum * mean)
        rv.mul_(1 - momentum).add_(momentum * var * cnt / (cnt - 1))
        means.append(mean)
        vars_.append(var)
    return means, vars_


@pytest.mark.parametrize("shards,groups", [((3,), 1), ((2, 2), 2), ((1, 3), 1), ((2, 4, 1), 1), ((3, 1, 2), 2)])
def test_gathered_partials_restate_batch_norm_on_the_concatenated_batch(shards, groups):
    g = torch.Generator().manual_seed(len(shards) * 10 + groups)
    c, h = 5, 7
    ys = [torch.randn(n * groups, c, h, h, generator=g, dtype=torch.float64) * 1.7 + 0.3 for n in shards]
    gathered = torch.stack([_partials(y, groups) for y in ys])
    rm, rv = torch.zeros(c, dtype=torch.float64), torch.ones(c, dtype=torch.float64)
    means, vars_ = _finalize(gathered, rm, rv)
    rm_ref, rv_ref = torch.zeros(c, dtype=torch.float64), torch.ones(c, dtype=torch.float64)
    for gi in range(groups):
        full = torch.cat([y[gi * n:(gi + 1) * n] for y, n in zip(ys, shards)])
        z = F.batch_norm(full, rm_ref, rv_ref, None, None, True, 0.1, 1e-5)
        zr = (full - means[gi][None, :, None, None]) / torch.sqrt(vars_[gi][None, :, None, None] + 1e-5)
        torch.testing.assert_close(zr, z, rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(rm, rm_ref, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(rv, rv_ref, rtol=1e-12, atol=1e-12)


def _exchange_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        ex = parallel.BNStatsExchange(dist.group.WORLD)
        assert (ex.world, ex.rank) == (world, rank)
        part, gathered = ex.buffers(2, 4, "cpu")
        assert part.shape == (2, 4, 3) and gathered.shape == (world, 2, 4, 3)
        part.copy_(torch.arange(24, dtype=torch.float64).view(2, 4, 3) + 100 * rank)
        ex.gather(part, gathered)
        part.fill_(-1)        # a later gather into another buffer leaves this one as it is
        ex.gather(part, ex.buffers(2, 4, "cpu")[1])
        q.put((rank, gathered.tolist(), ex.gathers))     # plain lists: the worker exits before the parent reads
    finally:
        dist.destroy_process_group()


def test_exchange_gathers_in_rank_order_on_every_rank():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 27500 + os.getpid() % 2000
    procs = [ctx.Process(target=_exchange_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    outs = dict((r, (t, n)) for r, t, n in (q.get(timeout=300) for _ in procs))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    want = torch.stack([torch.arange(24, dtype=torch.float64).view(2, 4, 3) + 100 * r for r in range(2)])
    for r in range(2):
        assert torch.equal(torch.tensor(outs[r][0], dtype=torch.float64), want) and outs[r][1] == 2
