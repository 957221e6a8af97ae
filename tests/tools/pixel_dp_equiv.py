"""2-rank equivalence of `--discriminator pixel` (run under torchrun; tests/test_pixel_disc_gpu.py launches it).

For the warp and the texture stage, each rank runs the D and G phases of one training step on ITS half of a batch
through the plugin, and a single-process model (world forced to 1) runs them on the whole batch with the same weights,
label draws and dropout masks.  Checked on every rank, as tests/tools/sync_bn_equiv.py checks batch norm:
  * the summed flat D and G gradients (x 1/world) against the single process: < 5e-4;
  * the losses (mean over ranks) against the single process: < 1e-5;
  * one whole optimize_parameters() on the shards leaves the parameters bit-equal across ranks.
SN_PIX_BACKEND=nccl: one rank per GPU.  gloo (default): both ranks drive cuda:0 over a gloo group this script creates
before the models.  Prints one `PIXEL_DP_EQUIV OK|FAIL <stage> ...` line per stage on rank 0.
"""
import gc
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

BACKEND = os.environ.get("SN_PIX_BACKEND", "gloo")
if BACKEND == "gloo":
    os.environ["LOCAL_RANK"] = "0"
    dist.init_process_group("gloo")

from test_engine_gpu import _opt, synth_texture_batch, synth_warp_batch  # noqa: E402

from swapnet_b200 import parallel  # noqa: E402
from swapnet_b200.models import create_model  # noqa: E402


def relmax(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


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


def stage_opt(stage, B, S, **over):
    if stage == "texture":
        return _opt(B, S, model="texture", netG="swapnet", lambda_l1=10, lambda_content=0, lambda_style=0,
                    discriminator="pixel", **over)
    return _opt(B, S, discriminator="pixel", **over)


def batch_of(stage, B, S):
    if stage == "texture":
        tex, rois, cloth, tgt = synth_texture_batch(B, S)
        return dict(input_textures=tex, rois=rois, cloths=cloth, target_textures=tgt, cloth_paths=["c"] * B,
                    texture_paths=["t"] * B)
    body, inp, tgt = synth_warp_batch(B, S)
    return dict(bodys=body, input_cloths=inp, target_cloths=tgt, cloth_paths=["c"] * B, body_paths=["b"] * B)


def equal_across_ranks(tensors: dict, device) -> bool:
    flat = torch.cat([v.reshape(-1).contiguous().view(torch.uint8) for _, v in sorted(tensors.items())]).to(device)
    got = [torch.empty_like(flat) for _ in range(dist.get_world_size())]
    dist.all_gather(got, flat)
    return all(torch.equal(got[0], x) for x in got[1:])


def run(stage, S, per):
    world, rank = dist.get_world_size(), dist.get_rank()
    torch.manual_seed(0)
    dp = create_model(stage_opt(stage, per, S, name=f"{stage}_dp{rank}"))
    dp.setup(dp.opt)
    B = per * world
    full = batch_of(stage, B, S)
    cdev = dp.device if BACKEND == "nccl" else torch.device("cpu")
    real_world, real_rank = parallel.world_size, parallel.rank
    parallel.world_size, parallel.rank = (lambda: 1), (lambda: 0)
    try:
        torch.manual_seed(0)
        ref = create_model(stage_opt(stage, B, S, name=f"{stage}_ref{rank}"))
        ref.setup(ref.opt)
        ref._labels = parallel.LabelDraws(1234)     # the draws of the data-parallel run
        ref.allreduce_grads = lambda eng: None
        ref.ensure_engines(B, S)
    finally:
        parallel.world_size, parallel.rank = real_world, real_rank
    gD, gG, losses = phases(dp, parallel.shard_batch(full, rank, world))
    gD, gG = gD * dp.grad_scale(), gG * dp.grad_scale()
    rD, rG, rlosses = phases(ref, full)
    eD, eG = relmax(gD, rD), relmax(gG, rG)
    lt = torch.tensor([losses[k] for k in sorted(losses)], dtype=torch.float64, device=cdev)
    dist.all_reduce(lt)
    el = max(abs(v / world - rlosses[k]) / abs(rlosses[k]) for v, k in zip(lt.tolist(), sorted(losses)))
    dp.set_input(parallel.shard_batch(full, rank, world))
    dp.optimize_parameters()
    torch.cuda.synchronize()
    params = {f"{p}.{k}": v.detach() for p, net in (("G", dp.net_generator), ("D", dp.net_discriminator))
              for k, v in net.state_dict().items()}
    same_step = equal_across_ranks(params, cdev)
    worst = torch.tensor([eD, eG, el, float(not same_step)], dtype=torch.float64, device=cdev)
    dist.all_reduce(worst, op=dist.ReduceOp.MAX)
    w = worst.tolist()
    ok = w[0] < 5e-4 and w[1] < 5e-4 and w[2] < 1e-5 and not w[3]
    if rank == 0:
        print(f"PIXEL_DP_EQUIV {'OK' if ok else 'FAIL'} {stage} backend={BACKEND} world={world} size={S} "
              f"per_rank={per} flat_grad_D={w[0]:.3e} flat_grad_G={w[1]:.3e} losses={w[2]:.3e} "
              f"step_bit_equal_across_ranks={not w[3]}", flush=True)
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
