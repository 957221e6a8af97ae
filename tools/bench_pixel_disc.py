"""Cost of `--discriminator pixel` against `basic` on one H100: ms per warp and per texture training step at 512^2,
batch 16, with CUDA-graph replay (the two discriminators alternated in one run), per-pass kernel times of the PixelGAN
from CUDA events, and the peak device memory of each step.  Prints one JSON line; the card's name and power limit are
read in the same run.

    python tools/bench_pixel_disc.py [--size 512] [--batch 16] [--steps 10] [--rounds 3]
"""
import argparse
import gc
import json
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip()


def build(model, disc, B, S):
    from test_engine_gpu import _opt, synth_texture_batch, synth_warp_batch
    from swapnet_b200.models import create_model

    extra = {} if model == "warp" else dict(name="texture", netG="swapnet", lambda_l1=10, lambda_content=0,
                                            lambda_style=0)
    opt = _opt(B, S, model=model, discriminator=disc, b200_graph=1, checkpoints_dir=tempfile.mkdtemp(), **extra)
    torch.manual_seed(0)
    m = create_model(opt)
    m.setup(opt)
    if model == "warp":
        body, inp, tgt = synth_warp_batch(B, S)
        batch = dict(bodys=body, input_cloths=inp, target_cloths=tgt, cloth_paths=["c"] * B, body_paths=["b"] * B)
    else:
        tex, rois, cloth, tgt = synth_texture_batch(B, S)
        batch = dict(input_textures=tex, rois=rois, cloths=cloth, target_textures=tgt, cloth_paths=["c"] * B,
                     texture_paths=["t"] * B)
    return m, batch


def step_ms(m, batch, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        m.set_input(batch)
        m.optimize_parameters()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def pass_ms(m, reps=20):
    """CUDA-event times of the D-step engine's passes (2B images)."""
    d = m._eng_Dd
    out = {}
    dpred = torch.randn_like(d.pred) * 1e-4
    for name, fn in (("forward", d.forward), ("backward", lambda: d.backward(dpred))):
        fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out[name] = e0.elapsed_time(e1) / reps
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs an H100"
    res = {"card": card(), "size": a.size, "batch": a.batch}
    for model in ("warp", "texture"):
        times = {"basic": [], "pixel": []}
        peak = {}
        for r in range(a.rounds):
            for disc in ("basic", "pixel"):
                gc.collect()             # a model is a reference cycle: free the previous one's buffers first
                torch.cuda.empty_cache()
                torch.cuda.reset_peak_memory_stats()
                m, batch = build(model, disc, a.batch, a.size)
                step_ms(m, batch, 3)                          # two eager steps, capture, one replay
                times[disc].append(step_ms(m, batch, a.steps))
                peak[disc] = torch.cuda.max_memory_allocated()
                if disc == "pixel" and r == 0:
                    res[f"{model}_pixel_D_step_passes_ms"] = pass_ms(m)
                del m
        res[f"{model}_step_ms"] = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
        res[f"{model}_step_ms_all"] = times
        res[f"{model}_peak_bytes"] = peak
    print(json.dumps(res))


if __name__ == "__main__":
    main()
