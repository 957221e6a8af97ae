"""2-rank equivalence of `--norm batch --b200_sync_bn 1` (run under torchrun; tests/test_sync_bn_gpu.py launches it).

For the warp stage (batch norm in the PatchGAN only) and the texture stage (U-Net and PatchGAN), each rank runs the
D and G phases of one training step on ITS half of a batch through the plugin, and a single-process model (world
forced to 1) runs them on the whole batch with the same weights, label draws and dropout masks.  The perceptual terms
are off: the style Gram couples a shard's samples by design.  Checked on every rank:
  * the summed flat D and G gradients (x 1/world) against the single process: < 5e-4 (the bar of dp_equiv.py);
  * the losses (mean over ranks) against the single process: < 1e-5;
  * every running buffer against the single process: < 1e-5, and num_batches_tracked equal;
  * every BatchNorm buffer bit-equal across ranks; then one whole optimize_parameters() on the shards, after which the
    parameters and buffers are bit-equal across ranks.
SN_SBN_BACKEND=nccl: one rank per GPU, the process group from torchrun's environment (BaseModel.__init__).  gloo: both
ranks drive cuda:0 over a gloo group this script creates before the models (parallel.init_from_env leaves it be).
Prints one `SYNC_BN_EQUIV OK|FAIL <stage> ...` line per stage on rank 0.
"""
import gc
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

BACKEND = os.environ.get("SN_SBN_BACKEND", "nccl")
if BACKEND == "gloo":
    os.environ["LOCAL_RANK"] = "0"
    dist.init_process_group("gloo")

from test_engine_gpu import _opt, synth_texture_batch, synth_warp_batch  # noqa: E402

from swapnet_b200 import parallel  # noqa: E402
from swapnet_b200.models import create_model  # noqa: E402


def relmax(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


def randomise_bn(nets):
    """The same non-trivial affine parameters and running buffers on every rank and in the single process."""
    g = torch.Generator().manual_seed(9)
    for net in nets:
        for m in net.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                c = m.num_features
                with torch.no_grad():
                    m.weight.copy_(1.0 + 0.3 * torch.randn(c, generator=g))
                    m.bias.copy_(0.1 * torch.randn(c, generator=g))
                    m.running_mean.copy_(0.1 * torch.randn(c, generator=g))
                    m.running_var.copy_(1.0 + 0.5 * torch.rand(c, generator=g))


def phases(model, batch):
    model.set_input(batch)
    model._acc.zero_()
    model.forward()
    model._eng_Dd.zero_grad()
    model.backward_D()
    gD = model._eng_Dd.flat_grad.detach().clone()
    model._eng_G.zero_grad()
    model.backward_G()
    torch.cuda.synchronize()
    return gD, model._eng_G.flat_grad.detach().clone(), dict(model.get_current_losses())


def state(model, buffers_only=False):
    out = {}
    for pre, net in (("G.", model.net_generator), ("D.", model.net_discriminator)):
        items = net.named_buffers() if buffers_only else net.state_dict().items()
        out.update({pre + k: v.detach() for k, v in items})
    return out


def comm_device(model):
    """Where the script's own collectives run: the GPU with NCCL, host memory with gloo."""
    return model.device if BACKEND == "nccl" else torch.device("cpu")


def equal_across_ranks(tensors: dict, device) -> bool:
    """Every tensor bit-equal on all ranks (compared as raw bytes gathered from every rank)."""
    flat = torch.cat([v.reshape(-1).contiguous().view(torch.uint8) for _, v in sorted(tensors.items())]).to(device)
    got = [torch.empty_like(flat) for _ in range(dist.get_world_size())]
    dist.all_gather(got, flat)
    return all(torch.equal(got[0], x) for x in got[1:])


def stage_opt(stage, B, S, **over):
    if stage == "texture":
        return _opt(B, S, model="texture", netG="swapnet", lambda_l1=10, lambda_content=0, lambda_style=0,
                    norm="batch", **over)
    return _opt(B, S, norm="batch", **over)


def batch_of(stage, B, S):
    if stage == "texture":
        tex, rois, cloth, tgt = synth_texture_batch(B, S)
        return dict(input_textures=tex, rois=rois, cloths=cloth, target_textures=tgt, cloth_paths=["c"] * B,
                    texture_paths=["t"] * B)
    body, inp, tgt = synth_warp_batch(B, S)
    return dict(bodys=body, input_cloths=inp, target_cloths=tgt, cloth_paths=["c"] * B, body_paths=["b"] * B)


def run(stage, S, per):
    world, rank = dist.get_world_size(), dist.get_rank()
    torch.manual_seed(0)
    dp = create_model(stage_opt(stage, per, S, name=f"{stage}_dp{rank}", b200_sync_bn=1))
    dp.setup(dp.opt)
    assert dp._bn_sync is not None and dp._bn_sync.world == world
    randomise_bn((dp.net_generator, dp.net_discriminator))
    B = per * world
    full = batch_of(stage, B, S)
    cdev = comm_device(dp)

    # single process on the same weights: world and rank forced to 1 / 0 while it is built, no all-reduce
    real_world, real_rank = parallel.world_size, parallel.rank
    parallel.world_size, parallel.rank = (lambda: 1), (lambda: 0)
    try:
        torch.manual_seed(0)
        ref = create_model(stage_opt(stage, B, S, name=f"{stage}_ref{rank}"))
        ref.setup(ref.opt)
        randomise_bn((ref.net_generator, ref.net_discriminator))
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
    eD, eG = relmax(gD, rD), relmax(gG, rG)
    lt = torch.tensor([losses[k] for k in sorted(losses)], dtype=torch.float64, device=cdev)
    dist.all_reduce(lt)
    el = max(abs(v / world - rlosses[k]) / abs(rlosses[k]) for v, k in zip(lt.tolist(), sorted(losses)))
    bufs, rbufs = state(dp, buffers_only=True), state(ref, buffers_only=True)
    eb, counts_ok = 0.0, True
    for k, v in bufs.items():
        if k.endswith("num_batches_tracked"):
            counts_ok &= int(v) == int(rbufs[k])
        else:
            eb = max(eb, relmax(v, rbufs[k]))
    same_bufs = equal_across_ranks(bufs, cdev)

    # one whole training step on the shards: the updated parameters and buffers stay bit-equal across ranks
    dp.set_input(parallel.shard_batch(full, rank, world))
    dp.optimize_parameters()
    torch.cuda.synchronize()
    same_step = equal_across_ranks(state(dp), cdev)

    worst = torch.tensor([eD, eG, el, eb, float(not counts_ok), float(not same_bufs), float(not same_step)],
                         dtype=torch.float64, device=cdev)
    dist.all_reduce(worst, op=dist.ReduceOp.MAX)
    w = worst.tolist()
    ok = w[0] < 5e-4 and w[1] < 5e-4 and w[2] < 1e-5 and w[3] < 1e-5 and not any(w[4:])
    if rank == 0:
        print(f"SYNC_BN_EQUIV {'OK' if ok else 'FAIL'} {stage} backend={BACKEND} world={world} size={S} "
              f"per_rank={per} gathers/step={dp._bn_sync.gathers // 2} flat_grad_D={w[0]:.3e} flat_grad_G={w[1]:.3e} "
              f"losses={w[2]:.3e} running_buffers={w[3]:.3e} counters_equal={not w[4]} "
              f"buffers_bit_equal_across_ranks={not w[5]} step_bit_equal_across_ranks={not w[6]}", flush=True)
    return ok


def main():
    ok = run("warp", 128, 2)
    gc.collect()              # the warp models are reference cycles: free their device memory before the texture stage
    ok &= run("texture", 128, 2)
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
