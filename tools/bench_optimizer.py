"""Cost of the fused optimizer kernels: milliseconds per `launch()` of FusedAdamW and FusedAdaBound over a flat buffer
of the warp generator's size (137.6 M fp32 parameters by default), timed with CUDA events.

Both kernels read p, g, m, v and write p, m, v once: 28 bytes per parameter.  The two optimizers alternate over
`--rounds` rounds of `--launches` back-to-back launches each (after a warm-up), so that clock drift affects both alike.
Prints the card's name and power limit with the per-launch milliseconds (median over the rounds), the bytes moved over
that time, and its share of the H100 SXM data sheet's 3.35 TB/s of HBM3 bandwidth, as one JSON line.

    python tools/bench_optimizer.py [--params 137600000] [--launches 50] [--warmup 10] [--rounds 5]
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

BYTES_PER_PARAM = 28            # p, g, m, v read; p, m, v written; fp32
HBM_PEAK = 3.35e12              # bytes/s, H100 SXM data sheet


def build(kind: str, n: int):
    from swapnet_b200 import optim

    p = torch.nn.Parameter(torch.randn(n, device="cuda"))
    flat = optim.flatten_parameters([p])
    if kind == "AdaBound":
        o = optim.FusedAdaBound([p], flat, lr=1e-4, weight_decay=0.01, final_lr=0.1)
    else:
        o = optim.FusedAdamW([p], flat, lr=1e-4, weight_decay=0.01)
    o.flat_grad = torch.randn(n, device="cuda")
    hyper = torch.tensor(o.advance(1.0), dtype=torch.float32, device="cuda")
    return o, hyper


def time_launches(o, hyper, launches: int) -> float:
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        o.launch(hyper)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--params", type=int, default=137_600_000)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_optimizer.py needs a CUDA device")
    kinds = ("AdamW", "AdaBound")
    opts = {k: build(k, args.params) for k in kinds}
    for o, hyper in opts.values():
        for _ in range(args.warmup):
            o.launch(hyper)
    ms = {k: [] for k in kinds}
    for _ in range(args.rounds):
        for k in kinds:
            ms[k].append(time_launches(*opts[k], args.launches))
    nbytes = BYTES_PER_PARAM * args.params
    result = {"gpu": bench.gpu_info(0), "params": args.params, "bytes_per_launch": nbytes, "launches": args.launches,
              "rounds": args.rounds, "unit": "ms/launch (median over rounds)", "kernels": {}}
    for k in kinds:
        med = statistics.median(ms[k])
        rate = nbytes / (med * 1e-3)
        result["kernels"][k] = {"ms": round(med, 4), "all": [round(x, 4) for x in ms[k]],
                                "tb_per_s": round(rate / 1e12, 3), "share_of_hbm_peak": round(rate / HBM_PEAK, 3)}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
