"""Cost of `--norm` (instance / batch / none): one plugin training step at the bench's shapes, timed with CUDA events.

Legs: texture at 512 x 512, batch 16, without and with the perceptual losses; warp at 512 x 512, batch 16 (the
generator always uses InstanceNorm there, so only the discriminator changes).  Each leg runs the same step as
bench.py (graph replay after the eager warm-up steps, device-resident inputs) for every norm, alternating the norms
over `--rounds` rounds so that clock drift affects all of them alike.  Prints the card's name and power limit with
the per-step milliseconds (median over the rounds) as one JSON line.

    python tools/bench_norm.py [--steps 10] [--warmup 3] [--rounds 3] [--size 512] [--batch 16]
"""
from __future__ import annotations

import argparse
import contextlib
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

NORMS = ("instance", "batch", "none")


def build(kind: str, norm: str, B: int, S: int, perceptual: bool):
    from swapnet_b200.models import create_model

    o = bench.warp_opt(B, S, "fp32x3")
    o.norm = norm
    if kind == "texture":
        o.model, o.name, o.netG, o.lambda_l1, o.lambda_content, o.lambda_style = "texture", "texture", "swapnet", 10, 0, 0
        if perceptual:
            o.lambda_content, o.lambda_style, o.b200_vgg = 20.0, 1e-8, "random"
        batch = bench.synth_texture_batch(B, S, 1234, labels=True)
        keys = ("input_textures", "rois", "cloths", "target_textures")
    else:
        batch = bench.synth_batch(B, S, 1234, labels=True)
        keys = ("bodys", "input_cloths", "target_cloths")
    torch.manual_seed(0)
    m = create_model(o)
    m.setup(m.opt)
    for k in keys:
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
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--batch", type=int, default=16)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_norm.py needs a CUDA device")
    B, S = args.batch, args.size
    legs = [("texture", False), ("texture", True), ("warp", False)]
    result = {"gpu": bench.gpu_info(0), "size": S, "batch": B, "steps": args.steps, "rounds": args.rounds,
              "unit": "ms/step (median over rounds)", "legs": {}}
    for kind, perceptual in legs:
        leg = f"{kind}{'+perceptual' if perceptual else ''}"
        ms = {n: [] for n in NORMS}
        for r in range(args.rounds):
            for norm in NORMS:
                with contextlib.redirect_stdout(sys.stderr):
                    m, batch = build(kind, norm, B, S, perceptual)
                    for _ in range(max(args.warmup, 3)):      # two eager steps, then the graph capture
                        m.set_input(batch)
                        m.optimize_parameters()
                ms[norm].append(time_steps(m, batch, args.steps))
                del m, batch
        med = {n: statistics.median(v) for n, v in ms.items()}
        result["legs"][leg] = {n: {"ms": round(med[n], 3), "all": [round(x, 3) for x in ms[n]],
                                   "vs_instance": round(med[n] / med["instance"], 4)} for n in NORMS}
        print(f"{leg}: " + ", ".join(f"{n} {med[n]:.2f} ms" for n in NORMS), file=sys.stderr)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
