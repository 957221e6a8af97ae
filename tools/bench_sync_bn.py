"""Cost of `--norm batch --b200_sync_bn 1`: one texture training step per rank at 512 x 512, batch 16 per rank, timed
with CUDA events, in three configurations alternated over `--rounds` rounds:
  * sync_bn:    --norm batch --b200_sync_bn 1 over all ranks (with one rank the exchange is not built: the flag has no
                effect there, and this leg is the next one);
  * instance:   --norm instance over all ranks;
  * batch_1gpu: --norm batch on rank 0 alone (the other ranks wait).
Also prints, computed from the engines' shapes, the gathers one training step issues (a forward and a backward
gather per train-mode BatchNorm2d call: the D step's 2B call, the G step's D call, the texture U-Net) and the bytes
each one moves, plus the card's name and power limit.  Data-parallel steps run eagerly (graph replay needs world 1).

    torchrun --nproc-per-node <gpus> tools/bench_sync_bn.py [--steps 10] [--warmup 3] [--rounds 3]
    python tools/bench_sync_bn.py ...      (one GPU: the cross-rank cost is then not measured)
"""
from __future__ import annotations

import argparse
import contextlib
import json
import os
import statistics
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from swapnet_b200 import parallel  # noqa: E402

LEGS = ("sync_bn", "instance", "batch_1gpu")


def build(leg: str, B: int, S: int):
    from swapnet_b200.models import create_model

    o = bench.warp_opt(B, S, "fp32x3")
    o.model, o.name, o.netG, o.lambda_l1, o.lambda_content, o.lambda_style = "texture", "texture", "swapnet", 10, 0, 0
    o.norm = "instance" if leg == "instance" else "batch"
    o.b200_sync_bn = int(leg == "sync_bn")
    batch = bench.synth_texture_batch(B, S, 1234 + parallel.rank(), labels=True)
    torch.manual_seed(0)
    m = create_model(o)
    m.setup(m.opt)
    for k in ("input_textures", "rois", "cloths", "target_textures"):
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


def gathers_per_step(m, world: int) -> list:
    """(engine, stage, groups, channels, bytes each rank sends, bytes each rank receives) of every gather of a step:
    two per train-mode BatchNorm2d stage (forward statistics, backward gradient sums), [groups][C][3] fp64 each."""
    out = []
    for key in ("Dd", "Dg", "G"):
        for st in m._eng_extra[key].stages:
            if st.bn is not None:
                sent = st.groups * st.cout * 3 * 8
                out += [(key, st.name, st.groups, st.cout, sent, world * sent)] * 2
    return out


def run_leg(leg: str, B: int, S: int, warmup: int, steps: int, world: int):
    if leg == "batch_1gpu" and world > 1:
        # rank 0 alone: a single-process model (world and rank read as 1 / 0 while it is built)
        if parallel.rank() != 0:
            dist.barrier()
            return None, None
        real = parallel.world_size, parallel.rank
        parallel.world_size, parallel.rank = (lambda: 1), (lambda: 0)
        try:
            ms, gathers = run_leg(leg, B, S, warmup, steps, 1)
        finally:
            parallel.world_size, parallel.rank = real
        dist.barrier()
        return ms, gathers
    with contextlib.redirect_stdout(sys.stderr):
        m, batch = build(leg, B, S)
        for _ in range(max(warmup, 3)):
            m.set_input(batch)
            m.optimize_parameters()
    ms = time_steps(m, batch, steps)
    gathers = gathers_per_step(m, max(world, 2)) if leg != "instance" else None
    del m, batch
    return ms, gathers


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--batch", type=int, default=16, help="samples per rank")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_sync_bn.py needs a CUDA device")
    if parallel.launched_distributed():
        parallel.init_from_env()
    world, rank = parallel.world_size(), parallel.rank()
    B, S = args.batch, args.size
    ms = {leg: [] for leg in LEGS}
    gathers = None
    for _ in range(args.rounds):
        for leg in LEGS:
            t, g = run_leg(leg, B, S, args.warmup, args.steps, world)
            if t is not None:
                ms[leg].append(t)
            if leg == "sync_bn" and g is not None:
                gathers = g
    if rank == 0:
        med = {leg: statistics.median(v) for leg, v in ms.items()}
        result = {"gpu": bench.gpu_info(torch.cuda.current_device()), "world": world, "size": S, "batch_per_rank": B,
                  "steps": args.steps, "rounds": args.rounds, "unit": "ms/step (median over rounds)",
                  "legs": {leg: {"ms": round(med[leg], 3), "all": [round(x, 3) for x in ms[leg]]} for leg in LEGS},
                  "gathers_per_step": len(gathers),
                  "bytes_per_gather_received_at_world": max(world, 2),
                  "gathers": [dict(zip(("engine", "stage", "groups", "channels", "bytes_sent", "bytes_received"), g))
                              for g in gathers[::2]],
                  "cross_rank_cost_measured": world > 1}
        print(json.dumps(result))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
