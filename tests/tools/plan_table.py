"""Per-plan timing table of one warp-stage training step (the model and batch bench.py times), on the GPU.

    python tests/tools/plan_table.py [--size 512] [--batch 16] [--steps 3] [--json OUT]

Builds the warp model the way bench.py does, runs warm-up steps, then `--steps` eager steps with ops.Plan.trace
installed (every GEMM plan launch bracketed by CUDA events).  Prints one line per plan: layer, kind (fwd / dgrad /
wgrad), launches per step, median ms per step, algorithmic TFLOP/s, and the plan's launch geometry (M tiles x N tiles
x phases, block_n, A row chunk; for weight gradients the grid and the Y row chunk).  The totals line of the fwd +
dgrad plans is the figure bench.py reports as roofline.achieved.
"""
from __future__ import annotations

import argparse
import contextlib
import ctypes
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def plan_geometry(plan):
    from swapnet_b200 import _lib

    g = (ctypes.c_int * 6)()
    _lib.load().sn_plan_geometry(plan.handle, g)
    return list(g)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--json", default=None, help="also write the rows as JSON to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("plan_table.py needs a CUDA device")
    import bench
    from swapnet_b200 import ops
    from swapnet_b200.models import create_model

    torch.manual_seed(0)
    B, S = args.batch, args.size
    with contextlib.redirect_stdout(sys.stderr):
        m = create_model(bench.warp_opt(B, S, "fp32x3"))
        m.setup(m.opt)
    host = bench.synth_batch(B, S, 1234, labels=True)
    devb = dict(host)
    for k in ("bodys", "input_cloths", "target_cloths"):
        devb[k] = host[k].cuda()
    m.graph_enabled = False
    for _ in range(3):
        m.set_input(devb)
        m.optimize_parameters()
    torch.cuda.synchronize()

    info = {}
    engs = [m._eng_G, m._eng_Dd, m._eng_Dg]
    for eng in engs:
        for st in eng.stages:
            fl, ly = 2.0 * st.nominal_macs(), st.layer
            for p in ly.fwd_plans:
                info[id(p)] = (p, "fwd", fl / len(ly.fwd_plans), st.name)
            for p in ly.dgrad_plans:
                info[id(p)] = (p, "dgrad", fl / len(ly.dgrad_plans), st.name)
            if ly.wgrad_plan is not None:
                info[id(ly.wgrad_plan)] = (ly.wgrad_plan, "wgrad", fl, st.name)

    per_step = []          # one {plan id: [ms, launches]} per traced step
    for _ in range(args.steps):
        ops.Plan.trace = []
        m.set_input(devb)
        m.optimize_parameters()
        torch.cuda.synchronize()
        trace, ops.Plan.trace = ops.Plan.trace, None
        acc = {}
        for plan, a, b in trace:
            e = acc.setdefault(id(plan), [0.0, 0])
            e[0] += a.elapsed_time(b)
            e[1] += 1
        per_step.append(acc)

    rows = []
    for pid, (plan, kind, fl, name) in info.items():
        if pid not in per_step[0]:
            continue
        ms = statistics.median(s[pid][0] for s in per_step)
        n = per_step[0][pid][1]
        geo = plan_geometry(plan)
        rows.append({"layer": name, "kind": kind, "launches": n, "ms": ms,
                     "tflops": n * fl / (ms * 1e-3) / 1e12 if ms > 0 else 0.0,
                     "grid": geo[1:4], "block_n": geo[4], "chunk": geo[5]})
    gpu = bench.gpu_info(torch.cuda.current_device())
    print(f"# {gpu['name']}, power limit {gpu['power_limit_w']} W; warp step {S}x{S}, batch {B}; "
          f"median of {args.steps} traced eager steps")
    print(f"{'layer':<28} {'kind':<6} {'n':>2} {'ms':>8} {'TFLOP/s':>8}  {'tiles (m x n x z)':<18} {'block_n':>7} {'chunk':>5}")
    for r in rows:
        g = "x".join(str(v) for v in r["grid"])
        print(f"{r['layer']:<28} {r['kind']:<6} {r['launches']:>2} {r['ms']:>8.3f} {r['tflops']:>8.1f}  {g:<18} "
              f"{r['block_n']:>7} {r['chunk']:>5}")
    for kinds in (("fwd", "dgrad"), ("wgrad",)):
        sel = [r for r in rows if r["kind"] in kinds]
        ms = sum(r["ms"] for r in sel)
        fl = sum(r["tflops"] * r["ms"] for r in sel)
        print(f"# {'+'.join(kinds)}: {ms:.2f} ms per step, {fl / ms if ms else 0.0:.1f} TFLOP/s")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"gpu": gpu, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
