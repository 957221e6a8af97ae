"""Cost of the style term's kernels and of a one-GPU texture step with a large Gram matrix.

1. Kernels (CUDA events over `--launches` launches, 512 x 512, 16 images per rank): the style term as
   PerceptualEngine.style launches it, forward Gram matrices of fakes (NHWC) and targets (NCHW), the MSE and the
   gradient, in the default mode.
     * rows_w<w>:   `gram_rows` x 2, `gram_rows_mse`, `gram_rows_bwd` of ONE rank of w, its 48 rows against
                    R = 48 w rows of emulated ranks (the gathered batch is already on the device: the all-gather is
                    not in the number), for w = 1, 2, 4, 8.
2. Texture step (`--step-size` x `--step-size`, batch `--step-batch` on one GPU, content and style on with a
   seeded-random VGG16, graph replay): ms per optimize_parameters().  Batch 48 is 144 Gram rows.
Prints one JSON line with the card's name and power limit.

    python tools/bench_style.py [--launches 50] [--steps 10] [--warmup 3]
"""
from __future__ import annotations

import argparse
import contextlib
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from swapnet_b200 import ops  # noqa: E402


def time_launches(fn, launches: int) -> float:
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / launches


def kernel_legs(S: int, per: int, worlds, launches: int) -> dict:
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    out = {}
    rl = 3 * per
    acc = torch.zeros(1, dtype=torch.float64, device=dev)
    dx = torch.zeros(per, S, S, 3, device=dev)
    for w in worlds:
        fa = torch.rand(w * per, S, S, 3, generator=g, device=dev) * 2 - 1
        ta = torch.rand(w * per, 3, S, S, generator=g, device=dev) * 4.5 - 2
        mine = slice((w // 2) * per, (w // 2 + 1) * per)
        fl, tl = fa[mine].contiguous(), ta[mine].contiguous()
        gor = torch.zeros(rl, rl * w, dtype=torch.float64, device=dev)
        gtr, mr = torch.zeros_like(gor), torch.zeros(rl, rl * w, device=dev)

        def rows_path():
            ops.gram_rows(fl, fa, True, gor)
            ops.gram_rows(tl, ta, False, gtr)
            ops.gram_rows_mse(gor, gtr, 5e-8, acc, mr, gscale=float(w))
            ops.gram_rows_bwd(mr, fa, True, dx, accumulate=True)
        out[f"rows_w{w}"] = time_launches(rows_path, launches)
        del fa, ta
    return {k: round(v, 4) for k, v in out.items()}


def texture_step(B: int, S: int, warmup: int, steps: int) -> dict:
    from swapnet_b200.models import create_model

    o = bench.warp_opt(B, S, "fp32x3")
    o.model, o.name, o.netG, o.lambda_l1 = "texture", "texture", "swapnet", 10
    o.lambda_content, o.lambda_style, o.b200_vgg = 20.0, 1e-8, "random"
    batch = bench.synth_texture_batch(B, S, 1234, labels=True)
    with contextlib.redirect_stdout(sys.stderr):
        torch.manual_seed(0)
        m = create_model(o)
        m.setup(m.opt)
        for k in ("input_textures", "rois", "cloths", "target_textures"):
            batch[k] = batch[k].cuda()
        for _ in range(max(warmup, 3)):
            m.set_input(batch)
            m.optimize_parameters()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        m.set_input(batch)
        m.optimize_parameters()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    res = {"batch": B, "size": S, "ms_per_step": round(ms, 3), "images_per_s": round(1000.0 * B / ms, 2),
           "style_rows": m._eng_P.rows, "graph_replay": len(m._graphs) > 0,
           "peak_gb": round(torch.cuda.max_memory_allocated() / 1e9, 2), "G_style": m.get_current_losses()["G_style"]}
    del m, batch
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--per-rank", type=int, default=16)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--step-size", type=int, default=256)
    ap.add_argument("--step-batch", type=int, default=48)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_style.py needs a CUDA device")
    kernels = kernel_legs(args.size, args.per_rank, (1, 2, 4, 8), args.launches)
    step = texture_step(args.step_batch, args.step_size, args.warmup, args.steps)
    print(json.dumps({"gpu": bench.gpu_info(0), "kernels": {"size": args.size, "images_per_rank": args.per_rank,
                                                            "launches": args.launches, "unit": "ms per style term",
                                                            "ms": kernels, "all_gather": "not measured"},
                      "texture_step": step}))


if __name__ == "__main__":
    main()
