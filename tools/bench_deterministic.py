"""Cost of `--b200_deterministic`: one plugin training step at the bench's shapes with the mode off and on, timed with
CUDA events.

Legs: warp at 512 x 512, batch 16, and texture at 512 x 512, batch 16, without and with the perceptual losses
(seeded-random VGG16 weights).  Each leg runs the same step as bench.py (graph replay after the eager
warm-up steps, device-resident inputs) in both modes, alternating the modes over `--rounds` rounds so that clock drift
affects both alike.  Prints the card's name and power limit, the per-step milliseconds (median over the rounds) and
the deterministic mode's workspace bytes per engine as one JSON line.

    python tools/bench_deterministic.py [--steps 10] [--warmup 3] [--rounds 3] [--size 512] [--batch 16]
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

MODES = (0, 1)


def build(kind: str, det: int, B: int, S: int, perceptual: bool = False):
    from swapnet_b200.models import create_model

    o = bench.warp_opt(B, S, "fp32x3")
    o.b200_deterministic = det
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
        raise SystemExit("tools/bench_deterministic.py needs a CUDA device")
    B, S = args.batch, args.size
    result = {"gpu": bench.gpu_info(0), "size": S, "batch": B, "steps": args.steps, "rounds": args.rounds,
              "unit": "ms/step (median over rounds)", "legs": {}, "workspace_bytes": {}}
    for kind, perceptual in (("warp", False), ("texture", False), ("texture", True)):
        leg = f"{kind}{'+perceptual' if perceptual else ''}"
        ms = {d: [] for d in MODES}
        for r in range(args.rounds):
            for det in MODES:
                with contextlib.redirect_stdout(sys.stderr):
                    m, batch = build(kind, det, B, S, perceptual)
                    for _ in range(max(args.warmup, 3)):      # two eager steps, then the graph capture
                        m.set_input(batch)
                        m.optimize_parameters()
                ms[det].append(time_steps(m, batch, args.steps))
                if det and r == 0:
                    result["workspace_bytes"][leg] = {k: m._eng_extra[k].workspace_bytes()
                                                      for k in ("G", "Dd", "Dg", "P") if k in m._eng_extra}
                del m, batch
        med = {d: statistics.median(v) for d, v in ms.items()}
        result["legs"][leg] = {("deterministic" if d else "default"): {"ms": round(med[d], 3),
                                                                       "all": [round(x, 3) for x in ms[d]]}
                                for d in MODES}
        result["legs"][leg]["ratio"] = round(med[1] / med[0], 4)
        print(f"{leg}: default {med[0]:.2f} ms, deterministic {med[1]:.2f} ms", file=sys.stderr)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
