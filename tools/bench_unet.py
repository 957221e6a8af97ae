"""Training-step cost of the two models on a bare U-Net next to the SwapNet texture stage: 512 x 512, batch 16, one
GPU, graph replay (the default), timed with CUDA events.  Three legs, alternated over `--rounds` rounds so that the
card's state drifts over all of them alike:
  * pix2pix:      --model pix2pix (--norm batch, unet_128 on the 36-zero + cloth operand, the 64-channel D operand);
  * texture_unet: --model texture --netG unet_128 (--norm instance);
  * texture:      --model texture --netG swapnet (--norm instance).
The texture legs run without the perceptual terms (--lambda_content 0 --lambda_style 0) so that the three legs differ
in their networks only.  Per leg: ms per step (median over rounds), and the device memory the leg's model added to the
peak while it was built and warmed up.  Prints the card's name and power limit, read in the same run, and one JSON line.

    python tools/bench_unet.py [--steps 10] [--warmup 3] [--rounds 3]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

LEGS = ("pix2pix", "texture_unet", "texture")


def build(leg: str, B: int, S: int):
    from swapnet_b200.models import create_model

    o = bench.warp_opt(B, S, "fp32x3")
    if leg == "pix2pix":
        o.model, o.name, o.norm, o.netG, o.lambda_l1, o.beta1, o.lr = "pix2pix", "pix2pix", "batch", "unet_128", 10.0, \
            0.5, 0.01
    else:
        o.model, o.name, o.lambda_l1, o.lambda_content, o.lambda_style = "texture", "texture", 10, 0, 0
        o.netG = "unet_128" if leg == "texture_unet" else "swapnet"
    batch = bench.synth_texture_batch(B, S, 1234, labels=True)
    if leg == "pix2pix":
        batch = {"cloths": batch["cloths"], "target_textures": batch["target_textures"]}
    torch.manual_seed(0)
    m = create_model(o)
    m.setup(m.opt)
    for k in ("input_textures", "rois", "cloths", "target_textures"):
        if k in batch:
            batch[k] = batch[k].cuda()
    return m, batch


def time_steps(m, batch, steps: int) -> float:
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        m.set_input(batch)
        m.optimize_parameters()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "tools/bench_unet.py measures on a GPU"
    B, S = args.batch, args.size
    models, peak = {}, {}
    for leg in LEGS:
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        m, batch = build(leg, B, S)
        time_steps(m, batch, args.warmup)          # eager warm-up steps, then the graph capture
        peak[leg] = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
        models[leg] = (m, batch)
    ms = {leg: [] for leg in LEGS}
    for _ in range(args.rounds):
        for leg in LEGS:
            m, batch = models[leg]
            ms[leg].append(time_steps(m, batch, args.steps))
    gpu = bench.gpu_info(torch.cuda.current_device())
    res = {"size": S, "batch": B, "steps": args.steps, "rounds": args.rounds, "gpu": gpu,
           "graph_replay": all(len(models[leg][0]._graphs) == 1 for leg in LEGS)}
    for leg in LEGS:
        res[leg] = {"ms_per_step": statistics.median(ms[leg]), "ms_rounds": ms[leg], "peak_added_gib": peak[leg]}
        print(f"{leg:13s} {statistics.median(ms[leg]):8.2f} ms/step  rounds {['%.2f' % x for x in ms[leg]]}  "
              f"peak +{peak[leg]:.2f} GiB")
    print(f"card: {gpu['name']}, power limit {gpu['power_limit_w']} W")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
