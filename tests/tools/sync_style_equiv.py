"""2-rank equivalence of `--b200_sync_style 1` (run under torchrun; tests/test_sync_style_gpu.py launches it).

Texture stage with the style term on (the reference's default lambda_style 1e-8; content off: it is per-sample and
shards exactly) and --norm instance, so the style term's exchange is one of its own.  Each rank runs the D and G phases
of one training step on ITS half of a batch through the plugin, and a single-process model (world forced to 1) runs
them on the whole batch with the same weights, label draws and dropout masks.  Checked on every rank:
  * flag 1: the summed flat D and G gradients (x 1/world) against the single process: < 5e-4 (the bar of dp_equiv.py);
    the losses (mean over ranks) against the single process: < 1e-5; loss_G_style bit-equal on every rank and within
    1e-5 of the single process's full-batch value; one whole optimize_parameters() on the shards, after which the
    parameters are bit-equal across ranks;
  * flag 0: each rank's loss_G_style is the style loss of its own shard (fp64 torch of the reference's formula on the
    rank's fakes and targets, < 1e-5), and not the full-batch value.
SN_SSTYLE_BACKEND=nccl: one rank per GPU, the process group from torchrun's environment (BaseModel.__init__).  gloo:
both ranks drive cuda:0 over a gloo group this script creates before the models (parallel.init_from_env leaves it be).
Prints one `SYNC_STYLE_EQUIV OK|FAIL flag=<0|1> ...` line per flag on rank 0.
"""
import gc
import os
import sys

import torch
import torch.distributed as dist
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

BACKEND = os.environ.get("SN_SSTYLE_BACKEND", "nccl")
if BACKEND == "gloo":
    os.environ["LOCAL_RANK"] = "0"
    dist.init_process_group("gloo")

from sync_bn_equiv import batch_of, equal_across_ranks, phases, relmax, state  # noqa: E402
from test_engine_gpu import _opt  # noqa: E402

from swapnet_b200 import parallel  # noqa: E402
from swapnet_b200.models import create_model  # noqa: E402

LAM_STYLE = 1e-8


def comm_device(model):
    """Where the script's own collectives run: the GPU with NCCL, host memory with gloo."""
    return model.device if BACKEND == "nccl" else torch.device("cpu")


def texture_opt(B, S, **over):
    return _opt(B, S, model="texture", netG="swapnet", lambda_l1=10, lambda_content=0, lambda_style=LAM_STYLE, **over)


def shard_style_loss(model):
    """5 lam MSE(gram(fakes), gram(targets)) of this rank's samples in fp64 (perceptual.py:6-10,58-63)."""
    fakes = model._eng_G.fakes.permute(0, 3, 1, 2).double()
    tgt = model.targets.double()
    b, c, h, w = fakes.shape
    go = fakes.reshape(b * c, h * w) @ fakes.reshape(b * c, h * w).T
    gt = tgt.reshape(b * c, h * w) @ tgt.reshape(b * c, h * w).T
    return (5 * F.mse_loss(go, gt) * LAM_STYLE).item()


def run(flag, S, per):
    world, rank = dist.get_world_size(), dist.get_rank()
    torch.manual_seed(0)
    dp = create_model(texture_opt(per, S, name=f"texture_dp{rank}_{flag}", b200_sync_style=flag))
    dp.setup(dp.opt)
    assert (dp._style_sync is not None) == bool(flag)
    B = per * world
    full = batch_of("texture", B, S)
    cdev = comm_device(dp)

    # single process on the same weights: world and rank forced to 1 / 0 while it is built, no all-reduce
    real_world, real_rank = parallel.world_size, parallel.rank
    parallel.world_size, parallel.rank = (lambda: 1), (lambda: 0)
    try:
        torch.manual_seed(0)
        ref = create_model(texture_opt(B, S, name=f"texture_ref{rank}_{flag}"))
        ref.setup(ref.opt)
        ref._labels = parallel.LabelDraws(1234)     # the draws of the data-parallel run
        ref.allreduce_grads = lambda eng: None
        ref.ensure_engines(B, S)
    finally:
        parallel.world_size, parallel.rank = real_world, real_rank
    for k, v in state(ref).items():
        assert torch.equal(v, state(dp)[k]), f"replicas diverged from the single-process initialisation: {k}"
    gD, gG, losses = phases(dp, parallel.shard_batch(full, rank, world))
    gD, gG = gD * dp.grad_scale(), gG * dp.grad_scale()
    rD, rG, rlosses = phases(ref, full)
    style = torch.tensor([losses["G_style"]], dtype=torch.float64, device=cdev)
    styles = [torch.zeros_like(style) for _ in range(world)]
    dist.all_gather(styles, style)
    styles = [float(s) for s in styles]
    full_style = rlosses["G_style"]
    if flag:
        eD, eG = relmax(gD, rD), relmax(gG, rG)
        lt = torch.tensor([losses[k] for k in sorted(losses)], dtype=torch.float64, device=cdev)
        dist.all_reduce(lt)
        el = max(abs(v / world - rlosses[k]) / abs(rlosses[k]) for v, k in zip(lt.tolist(), sorted(losses)))
        es = abs(losses["G_style"] - full_style) / abs(full_style)
        same_style = all(s == styles[0] for s in styles)
        dp.set_input(parallel.shard_batch(full, rank, world))
        dp.optimize_parameters()
        torch.cuda.synchronize()
        same_step = equal_across_ranks(state(dp), cdev)
        worst = torch.tensor([eD, eG, el, es, float(not same_style), float(not same_step)], dtype=torch.float64,
                             device=cdev)
        dist.all_reduce(worst, op=dist.ReduceOp.MAX)
        w = worst.tolist()
        ok = w[0] < 5e-4 and w[1] < 5e-4 and w[2] < 1e-5 and w[3] < 1e-5 and not any(w[4:])
        detail = (f"flat_grad_D={w[0]:.3e} flat_grad_G={w[1]:.3e} losses={w[2]:.3e} style_vs_full_batch={w[3]:.3e} "
                  f"style_bit_equal_across_ranks={not w[4]} step_bit_equal_across_ranks={not w[5]} "
                  f"loss_G_style={styles} full_batch={full_style:.9g}")
    else:
        own = shard_style_loss(dp)
        eo = abs(losses["G_style"] - own) / abs(own)
        off_full = abs(losses["G_style"] - full_style) / abs(full_style)
        worst = torch.tensor([eo, -off_full], dtype=torch.float64, device=cdev)
        dist.all_reduce(worst, op=dist.ReduceOp.MAX)
        w = worst.tolist()
        ok = w[0] < 1e-5 and -w[1] > 1e-3
        detail = (f"style_vs_own_shard={w[0]:.3e} min_style_off_full_batch={-w[1]:.3e} loss_G_style={styles} "
                  f"full_batch={full_style:.9g}")
    if rank == 0:
        print(f"SYNC_STYLE_EQUIV {'OK' if ok else 'FAIL'} flag={flag} backend={BACKEND} world={world} size={S} "
              f"per_rank={per} {detail}", flush=True)
    return ok


def main():
    ok = run(1, 128, 2)
    gc.collect()              # the models are reference cycles: free their device memory before the next pair
    ok &= run(0, 128, 2)
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
