"""`--b200_sync_style` without a GPU: the option, an fp64 restatement of the row-block decomposition the kernels and
PerceptualEngine.style compute (gram_rows, gram_rows_mse with the `world` gradient factor, gram_rows_bwd, the rank-order
loss sum, the optimizer's 1/world) against the reference's gram_matrix + MSELoss autograd on the whole batch, and the
gather over a gloo group of two ranks."""
import os
from argparse import ArgumentParser

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F

from oracle import nets as ON
from swapnet_b200 import parallel
from swapnet_b200.models.texture_model import TextureModel


def test_flag_is_registered_with_default_off():
    p = TextureModel.modify_commandline_options(ArgumentParser(), True)
    assert p.parse_args([]).b200_sync_style == 0
    assert p.parse_args(["--b200_sync_style", "1"]).b200_sync_style == 1
    for bad in ("2", "-1", "yes"):
        with pytest.raises(SystemExit):
            p.parse_args(["--b200_sync_style", bad])


def _row_block_step(fakes, targets, world, lam):
    """What every emulated rank computes from the gathered batch: its [R_l, R] row blocks of both Gram matrices, its
    loss partial and m (scaled by world), and m @ X_all as its gradient rows.  Returns (the loss as the rank-order sum
    of the partials, the gradient w.r.t. all fakes after the SUM over ranks and the optimizer's 1/world)."""
    n, c, h, w = fakes.shape
    per = n // world
    xo, xt = fakes.reshape(n * c, h * w), targets.reshape(n * c, h * w)
    r, rl = n * c, per * c
    parts, grads = [], []
    for rank in range(world):
        rows = slice(rank * rl, (rank + 1) * rl)
        go, gt = xo[rows] @ xo.T, xt[rows] @ xt.T                 # gram_rows: this rank's rows x every rank's rows
        d = go - gt
        parts.append(5.0 * lam * (d * d).sum() / r ** 2)           # gram_rows_mse: loss partial
        m = world * 4.0 * 5.0 * lam * d / r ** 2                    # gram_rows_mse: m with the world factor
        grads.append(m @ xo)                                        # gram_rows_bwd: this rank's gradient rows
    loss = torch.zeros((), dtype=torch.float64)
    for p in parts:                                                 # rank order
        loss = loss + p
    # each rank's gradient reaches only its own samples; the G gradient all-reduce sums them, the optimizer takes 1/w
    g = torch.cat(grads) * (1.0 / world)
    return loss, g.view(n, c, h, w)


@pytest.mark.parametrize("world", [1, 2, 4])
@pytest.mark.parametrize("per,c,s", [(2, 3, 5), (3, 3, 8)])
def test_row_blocks_restate_the_full_batch_style_loss(world, per, c, s):
    g = torch.Generator().manual_seed(world * 100 + per * 10 + s)
    n = per * world
    fakes = (torch.rand(n, c, s, s, generator=g, dtype=torch.float64) * 2 - 1).requires_grad_()
    targets = torch.rand(n, c, s, s, generator=g, dtype=torch.float64) * 4.5 - 2
    lam = 1e-3
    ref = 5 * F.mse_loss(ON.gram_matrix(fakes), ON.gram_matrix(targets)) * lam
    (gref,) = torch.autograd.grad(ref, fakes)
    loss, grad = _row_block_step(fakes.detach(), targets, world, lam)
    torch.testing.assert_close(loss, ref.detach(), rtol=1e-12, atol=0)
    torch.testing.assert_close(grad, gref, rtol=1e-11, atol=1e-15)


def test_shard_local_term_is_not_the_full_batch_term():
    """Without the exchange each rank's Gram matrices cover its shard only: a different objective (the flag's reason)."""
    g = torch.Generator().manual_seed(5)
    fakes = torch.rand(4, 3, 6, 6, generator=g, dtype=torch.float64)
    targets = torch.rand(4, 3, 6, 6, generator=g, dtype=torch.float64) * 2
    full = 5 * F.mse_loss(ON.gram_matrix(fakes), ON.gram_matrix(targets))
    shards = [5 * F.mse_loss(ON.gram_matrix(fakes[i:i + 2]), ON.gram_matrix(targets[i:i + 2])) for i in (0, 2)]
    assert abs(float(sum(shards) / 2 - full)) > 1e-3 * float(full)
    assert abs(float(_row_block_step(fakes, targets, 2, 1.0)[0] - full)) <= 1e-12 * float(full)


def _gather_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        ex = parallel.BNStatsExchange(dist.group.WORLD)
        B, S = 2, 4
        full = torch.arange(world * B * S * S * 3, dtype=torch.float32).view(world * B, S, S, 3)
        fakes = full[rank * B:(rank + 1) * B].contiguous()           # NHWC, as the engine holds them
        tfull = -torch.arange(world * B * 3 * S * S, dtype=torch.float32).view(world * B, 3, S, S)
        targets = tfull[rank * B:(rank + 1) * B].contiguous()        # NCHW
        fa, ta = torch.zeros_like(full), torch.zeros_like(tfull)
        ex.gather(fakes, fa)
        ex.gather(targets, ta)
        part = torch.tensor([10.0 + rank], dtype=torch.float64)
        parts = ex.gather(part, torch.zeros(world, dtype=torch.float64))
        q.put((rank, torch.equal(fa, full), torch.equal(ta, tfull), parts.tolist(), ex.gathers))
    finally:
        dist.destroy_process_group()


def test_gather_puts_rows_in_global_sample_order():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 28500 + os.getpid() % 2000
    procs = [ctx.Process(target=_gather_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    outs = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, fakes_ok, targets_ok, parts, gathers in outs:
        assert fakes_ok and targets_ok, rank
        assert parts == [10.0, 11.0] and gathers == 3
