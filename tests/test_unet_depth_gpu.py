"""The conv GEMMs of the U-Net's deepest levels, 8x8 down to 1x1 planes, layer by layer against fp64.

The texture stage builds its U-Net with num_downs = log2(img_size) (9 levels at 512) and `--netG unet_128` / pix2pix
use 7 levels at 128: both reach a 1x1 innermost plane.  There the tap GEMM's M tile holds many whole images (or is
mostly padding), almost every tap reads outside the plane, the weight-gradient reduction over B * oh * ow pixels is a
single partial 64-pixel tile at small batches, and the fused InstanceNorm statistics must give way to plane_stats
because a tile spans images.  The cases are derived from the generators themselves, every conv whose input plane is
at most 8x8, with its real channels and bias, at the batches the texture stage runs (1, 2, 3, 16, and 40 for the 1x1
and 2x2 planes: the per-GPU batch `--b200_sync_style` allows).

Bounds as in test_kernels_gpu: forward (fp16-split x3) 1.5e-5, backward (bf16-split x3) 1e-4, as max|err| / max|ref|;
single-pass plans (nsplit = 1) 1.5e-5 of the fp64 product of the 16-bit operands they read.  References are fp64
torch on the GPU.
"""
import os
import sys

import pytest
import torch

from swapnet_b200 import lowering as L
from test_gemm_edges_gpu import BWD_TOL, FWD_TOL, SPLIT_SPREAD, geometry, grad_planes, sm_count
from test_kernels_gpu import (SP_SEP_BF16, SP_SEP_FP16, at_both_nsplits, check_single_pass, dev, make_layer,
                              model_dgrad, model_forward, model_wgrad, nhwc, record, ref_forward, relmax)

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "tools"))

pytestmark = pytest.mark.gpu

SENTINEL = 7.0
MAX_PLANE = 8          # input planes up to 8x8
# A conv4s2 of 512 channels on a 4x4 or 8x8 plane sums 512 x 9..16 in-bounds products per output (K = 8192) in one
# tensor-core accumulator, 3 truncating wgmma adds per 16 products at nsplit = 3.  Its fp16-split x3 forward measured
# 1.0e-5 .. 3.1e-5 against fp64 on an H100 80GB HBM3 (700 W limit), above the 1.5e-5 of test_conv_forward (K <= 2048
# there); the single-pass plans of the same shapes sit at up to 1.1e-5 of their operand model, the same floor with a
# third of the adds.  The 1024-channel convT4s2 skip joins (4 taps x 1024 channels per output phase) measured up to
# 1.7e-5.  The 512-channel convT4s2 and the conv4s2 of a 2x2 plane hold 1.5e-5.
LONG_K_FWD_TOL = 4e-5


def fwd_tol(kind, cin, h):
    return LONG_K_FWD_TOL if (kind == "conv4s2" and h >= 4) or cin >= 1024 else FWD_TOL


BATCHES = (1, 2, 3, 16)
WIDE_BATCH = 40        # the 1x1 and 2x2 planes also run at the largest per-GPU batch


def unet_generators():
    """(label, generator, image size) of the two U-Nets that reach a 1x1 plane, built as their models build them: the
    texture stage's at 512 (num_downs = log2(512) = 9, InstanceNorm: a bias on every conv) and the 7-level one of
    pix2pix / `--netG unet_128` at 128 (BatchNorm: a bias on the outermost up conv only)."""
    from swapnet_b200 import modules as M

    with torch.device("meta"):
        texture = M.TextureModule(3, 19, 12, "instance", 0.5, 512).unet
        unet_128 = M.UnetGenerator(3, 3, 7, 64, use_dropout=True, norm="batch")
    return [("texture_512", texture, 512), ("unet_128", unet_128, 128)]


def deep_convs(net, size):
    """(kind, cin, cout, input plane, bias) of every conv of `net` whose input plane is at most MAX_PLANE: block j's
    down conv reads the size >> j plane, its up conv the size >> (j + 1) plane."""
    rows = []
    for j, blk in enumerate(net.blocks()):
        for kind, conv, h in (("conv4s2", blk.down, size >> j), ("convT4s2", blk.up, size >> (j + 1))):
            if h <= MAX_PLANE:
                row = (kind, conv.in_channels, conv.out_channels, h, conv.bias is not None)
                if row not in rows:
                    rows.append(row)
    return rows


SHAPES = {label: deep_convs(net, size) for label, net, size in unet_generators()}
CASES = []
for _rows in SHAPES.values():
    for _row in _rows:
        for _n in BATCHES + ((WIDE_BATCH,) if _row[3] <= 2 else ()):
            if _row + (_n,) not in CASES:
                CASES.append(_row + (_n,))


def test_cases_cover_the_innermost_levels():
    """The table of the six deepest convs (both depths, without the bias flag): a change to the generator that moved
    them would otherwise empty these tests silently."""
    table = [("conv4s2", 512, 512, 8), ("conv4s2", 512, 512, 4), ("conv4s2", 512, 512, 2),
             ("convT4s2", 512, 512, 1), ("convT4s2", 1024, 512, 2), ("convT4s2", 1024, 512, 4)]
    for label, rows in SHAPES.items():
        assert set(table) <= {r[:4] for r in rows}, (label, rows)
    assert {r[4] for r in SHAPES["texture_512"]} == {True} and {r[4] for r in SHAPES["unet_128"]} == {False}
    batches = {(r[:5]): set() for r in CASES}
    for r in CASES:
        batches[r[:5]].add(r[5])
    for row, ns in batches.items():
        assert ns == set(BATCHES) | ({WIDE_BATCH} if row[3] <= 2 else set()), (row, ns)
    record("unet_depth_cases", f"{len(CASES)} cases: " + "; ".join(f"{k}: {v}" for k, v in SHAPES.items()))


def wgrad_pixels(kind, h):
    """Pixels per image of the weight-gradient reduction: the dy grid of a conv4s2, the input grid of a convT4s2."""
    return (h // 2) ** 2 if kind == "conv4s2" else h * h


def ref_grads(kind, x, wt, bias, gy):
    """fp64 output and gradients (input, weight, bias or None) of ref_forward for the output gradient gy, on the GPU."""
    d = dev()
    xr = x.to(d).double().requires_grad_()
    wr = wt.to(d).double().requires_grad_()
    br = None if bias is None else bias.to(d).double().requires_grad_()
    y = ref_forward(kind, xr, wr, br)
    g = torch.autograd.grad(y, [t for t in (xr, wr, br) if t is not None], gy.to(d).double())
    return y.detach(), g[0], g[1], (g[2] if br is not None else None)


def output_gradient(n, cout, oh, ow):
    return torch.randn((n, cout, oh, ow), generator=torch.Generator().manual_seed(99))


# ---------------------------------------------------------------------------------------------
# forward
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,cin,cout,h,bias,n,nsplit", at_both_nsplits(CASES))
def test_unet_depth_forward(kind, cin, cout, h, bias, n, nsplit):
    """The output bound as the first n images of an (n+1)-image buffer, inside a channel slice: the image after the
    batch and the channels on both sides must keep their sentinel (at 1x1 the valid rows end inside an M tile)."""
    layer, x, wt, b = make_layer(kind, n, cin, cout, h, h, nsplit, with_bias=bias)
    oh, ow = L.out_hw(kind, h, h)
    buf = torch.full((n + 1, oh, ow, cout + 5), SENTINEL, device=dev())
    y = buf[:n]
    layer.bind_forward(y, y_c_off=2)
    layer.pack()
    layer.forward()
    torch.cuda.synchronize()
    exact = nhwc(ref_forward(kind, x.to(dev()).double(), wt.to(dev()).double(),
                             None if b is None else b.to(dev()).double()))
    got = y[..., 2:2 + cout]
    geo = [geometry(p) for p in layer.fwd_plans]
    tag = f"unet_depth_fwd[{kind},{cin},{cout},{h}x{h},bias={bias},n={n}" + ("]" if nsplit == 3 else ",nsplit=1]")
    if nsplit == 3:
        err = relmax(got, exact)
        record(tag, f"{err:.3e} geometry {geo}")
        assert err < fwd_tol(kind, cin, h), err
    else:
        err, sep = check_single_pass(tag, got, model_forward(layer), exact, FWD_TOL, SP_SEP_FP16)
        record(tag, f"{err:.3e} (model vs exact {sep:.3e}) geometry {geo}")
    assert torch.all(buf[n] == SENTINEL), "wrote past the batch"
    assert torch.all(y[..., :2] == SENTINEL) and torch.all(y[..., 2 + cout:] == SENTINEL), "wrote outside its channels"


# ---------------------------------------------------------------------------------------------
# backward: input, weight and bias gradients
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,cin,cout,h,bias,n,nsplit", at_both_nsplits(CASES))
def test_unet_depth_backward(kind, cin, cout, h, bias, n, nsplit):
    layer, x, wt, b = make_layer(kind, n, cin, cout, h, h, nsplit, with_bias=bias)
    oh, ow = L.out_hw(kind, h, h)
    gy = output_gradient(n, cout, oh, ow)
    _, gx, gw, gb = ref_grads(kind, x, wt, b, gy)
    dy = grad_planes(gy.to(dev()), L.padc(cout))
    buf = torch.full((n + 1, h, h, cin + 3), 5.0, device=dev())
    dx = buf[:n]
    wg = torch.zeros_like(layer.weight)
    bg = torch.zeros(cout, device=dev()) if bias else None
    layer.bind_backward(dy, dx, wg, bg, dx_c_off=1)
    layer.pack()
    layer.backward()
    torch.cuda.synchronize()
    got_dx = dx[..., 1:1 + cin]
    e_b = relmax(bg, gb) if bias else 0.0   # no GEMM: bias_grad_kernel reads hi + lo whatever nsplit is
    tag = f"unet_depth_bwd[{kind},{cin},{cout},{h}x{h},bias={bias},n={n}" + ("]" if nsplit == 3 else ",nsplit=1]")
    if nsplit == 3:
        e_dx, e_w = relmax(got_dx, nhwc(gx)), relmax(wg, gw)
        record(tag, f"dx {e_dx:.3e} w {e_w:.3e} b {e_b:.3e}")
        assert e_dx < BWD_TOL and e_w < BWD_TOL, (e_dx, e_w)
    else:
        e_dx, s_dx = check_single_pass(f"{tag} dgrad", got_dx, model_dgrad(layer), nhwc(gx), FWD_TOL, SP_SEP_BF16)
        e_w, s_w = check_single_pass(f"{tag} wgrad", wg, model_wgrad(layer), gw, FWD_TOL, SP_SEP_BF16)
        record(tag, f"dx {e_dx:.3e} w {e_w:.3e} b {e_b:.3e} (model vs exact: dx {s_dx:.3e} w {s_w:.3e})")
    assert e_b < BWD_TOL, e_b
    assert torch.all(buf[n] == 5.0), "input gradient written past the batch"
    assert torch.all(dx[..., 0] == 5.0) and torch.all(dx[..., 1 + cin:] == 5.0), "input gradient outside its channels"


@pytest.mark.parametrize("kind,cin,cout,h,bias,n,nsplit", at_both_nsplits(CASES))
def test_unet_depth_wgrad_splits(kind, cin, cout, h, bias, n, nsplit):
    """The weight-gradient plans over B * oh * ow pixels (1 to 40 at the 1x1 planes): the split count the layer's plan
    got is the one sn_wgrad_ksplit gives; a split count above the number of 64-pixel tiles is clamped to it with the
    same result; deterministic plans, with the split count of their own rule and with one split per tile, give the same
    bits on three launches.  Every result within the bound of the layer's backward."""
    from swapnet_b200 import ops

    layer, x, wt, b = make_layer(kind, n, cin, cout, h, h, nsplit, with_bias=bias)
    oh, ow = L.out_hw(kind, h, h)
    gy = output_gradient(n, cout, oh, ow)
    _, _, gw, _ = ref_grads(kind, x, wt, b, gy)
    dy = grad_planes(gy.to(dev()), L.padc(cout))
    layer.bind_backward(dy, None, torch.zeros_like(layer.weight))
    (ws,) = L.wgrad_specs(kind, h, h)
    x_is_dy = ws.x_is == "dy"
    xs, ys = (dy, layer.x.twin) if x_is_dy else (layer.x.twin, dy)
    cx, cy = (cout, cin) if x_is_dy else (cin, cout)
    assert min(xs.c, ys.c) >= 64
    s_row, s_col = L.wgrad_out_strides(kind, cin, cout, x_is_dy)

    def plan_for(out, ksplit, det):   # the descriptor ConvLayer.bind_backward builds (both operands >= 64 channels)
        desc = ops.wgrad_desc(xs, ys, ws, out, s_row, s_col, list(ws.tap_ids), cx, cy, swap=cy > cx, nsplit=nsplit,
                              ksplit=ksplit, deterministic=det)
        return ops.wgrad_plan(desc, keep=(xs.hi, xs.lo, ys.hi, ys.lo, out)), desc

    pixels = n * wgrad_pixels(kind, h)
    per_image = wgrad_pixels(kind, h)
    tiles = -(-n // (64 // per_image))        # 64-pixel tiles of whole images (the planes divide 64)
    assert (ws.m_h * ws.m_w, layer.n) == (per_image, n)
    ks_rule = ops.wgrad_ksplit(plan_for(torch.zeros_like(layer.weight), 0, False)[1], sm_count())
    geo = geometry(layer.wgrad_plan)
    assert geo[0] == 1 and geo[3] == ks_rule, (geo, ks_rule)

    ref, tol = (gw, BWD_TOL) if nsplit == 3 else (model_wgrad(layer, dy), FWD_TOL)
    results, errs, splits = {}, {}, {}
    for label, ksplit, det in (("rule", 0, False), ("over", tiles + 3, False), ("det", 0, True),
                               ("det_over", tiles + 3, True)):
        out = torch.zeros_like(layer.weight)
        plan, _ = plan_for(out, ksplit, det)
        splits[label] = geometry(plan)[3]
        if ksplit:
            assert splits[label] == tiles, f"{label}: split count {splits[label]} not clamped to {tiles} tiles"
        runs = []
        for _ in range(3 if det else 1):
            out.zero_()
            plan.run()
            torch.cuda.synchronize()
            runs.append(out.clone())
        for i, r in enumerate(runs[1:]):
            assert torch.equal(r, runs[0]), f"{label}: launch {i + 2} differs from the first"
        results[label], errs[label] = runs[0], relmax(runs[0], ref)
    scale = gw.abs().max().item()
    spread = max((r.double() - results["rule"].double()).abs().max().item() / scale for r in results.values())
    tag = f"unet_depth_wgrad[{kind},{cin},{cout},{h}x{h},n={n}" + ("]" if nsplit == 3 else ",nsplit=1]")
    record(tag, f"K={pixels} px, {tiles} tiles, geometry {geo}, splits {splits}, "
           + " ".join(f"{k} {e:.3e}" for k, e in errs.items()) + f" spread {spread:.3e}")
    assert max(errs.values()) < tol, errs
    assert spread < SPLIT_SPREAD, spread


# ---------------------------------------------------------------------------------------------
# InstanceNorm statistics
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,cin,cout,h,bias,n,nsplit", at_both_nsplits(CASES))
def test_unet_depth_instance_norm_statistics(kind, cin, cout, h, bias, n, nsplit):
    """Statistics bound as test_fused_instance_norm_statistics binds them: a plan whose M tile spans images must refuse
    to fuse them (the layer then runs plane_stats); the mean and rstd of either path within 1e-5 of the fp64 statistics
    of the output the plan wrote."""
    from swapnet_b200 import ops

    layer, x, wt, b = make_layer(kind, n, cin, cout, h, h, nsplit, with_bias=bias)
    oh, ow = L.out_hw(kind, h, h)
    y = torch.zeros(n, oh, ow, cout, device=dev())
    stats = torch.zeros(n, cout, 2, dtype=torch.float64, device=dev())
    layer.bind_forward(y, stats=stats)
    # GEMM rows of one image: the output plane of a conv4s2, one output-parity phase (the input plane) of a convT4s2
    rows_per_image = oh * ow if kind == "conv4s2" else h * h
    spans = rows_per_image < 128 and n > 1
    assert layer.fused_stats == (not spans), (layer.fused_stats, spans)
    layer.pack()
    layer.forward()
    layer.forward()
    if layer.fused_stats:
        ops.stats_finalize(stats, n * cout, oh * ow)
    else:
        ops.plane_stats(y, cout, stats)
    torch.cuda.synchronize()
    exact = ref_forward(kind, x.to(dev()).double(), wt.to(dev()).double(), None if b is None else b.to(dev()).double())
    e_y = relmax(y.permute(0, 3, 1, 2), exact)
    assert nsplit == 1 or e_y < fwd_tol(kind, cin, h), e_y
    # the statistics of the output the plan wrote, in fp64: its distance from the exact output is the forward test's
    # (on a 2x2 plane of a channel with little spread, rstd = 1/std magnifies it past any fixed bound)
    ref = y.permute(0, 3, 1, 2).double()
    mean = ref.mean((2, 3))
    e_m = ((stats[..., 0] - mean).abs().max() / ref.abs().max()).item()
    # rstd per plane, relative to its fp64 value: both paths square the fp32 values in fp32 and sum a few of them in
    # fp32, an error of a few 2^-24 E[y^2] in the variance, which 1/sqrt(var + eps) turns into 2^-23 E[y^2] / (var + eps)
    # of rstd.  On planes of 1 to 4 pixels with little spread (var ~ 0: the 1x1 outputs of the innermost down conv,
    # which the U-Net does not normalise) that term, bounded here with 4x margin, is far above 1e-5.
    var = ref.var((2, 3), unbiased=False)
    rstd_ref = (var + 1e-5).rsqrt()
    cond = 2.0 ** -21 * (ref * ref).mean((2, 3)) / (var + 1e-5)
    e_r = ((stats[..., 1] - rstd_ref).abs() / rstd_ref / (1e-5 + cond)).max().item() * 1e-5
    tag = f"unet_depth_in_stats[{kind},{cin},{cout},{h}x{h},n={n}" + ("]" if nsplit == 3 else ",nsplit=1]")
    record(tag, f"fused={layer.fused_stats} mean {e_m:.3e} rstd {e_r:.3e} (output vs exact {e_y:.3e})")
    assert e_m < 1e-5 and e_r < 1e-5, (e_m, e_r)


# ---------------------------------------------------------------------------------------------
# an engine whose levels are all small
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("num_downs,B,norm", [(nd, B, norm) for nd in (5, 6) for B in (2, 16)
                                              for norm in ("instance", "batch", "none")])
def test_small_unet_engine_matches_oracle(num_downs, B, norm):
    """UnetEngine at S = 2**num_downs (32 and 64: the innermost level is 1x1, every level at most 32x32), train mode
    with dropout, on a random 55-channel input: fakes and every parameter gradient against the fp64 oracle, with the
    device's activation gates imposed on it as test_unet_engine_matches_oracle does."""
    import unet_oracle as UO
    from oracle import dropout as OD
    from oracle import nets as ON
    from swapnet_b200 import engine as E
    from swapnet_b200 import modules as M
    from swapnet_b200 import ops
    from test_batchnorm_gpu import _param_sd, _randomise_affine, bn_stage_gates

    S = 1 << num_downs
    torch.manual_seed(0)
    net = M.UnetGenerator(55, 3, num_downs, 64, use_dropout=True, norm=norm).to(dev())
    M.init_weights(net, "kaiming", 0.02)
    _randomise_affine((net,))
    sd, names = _param_sd(net)
    eng = E.UnetEngine(net, B, S, dev())
    eng.alloc_grads()
    eng.bind_backward()
    eng.pack()
    g = torch.Generator().manual_seed(5)
    x = torch.randn(B, 55, S, S, generator=g)
    up = torch.randn(B, S, S, 3, generator=g)
    eng.zero_grad()
    ops.pack_planes(x.to(dev()), eng.x_in)
    eng.forward(training=True, seed=77)
    eng.backward([ops.GradSrc(up.to(dev()))])
    torch.cuda.synchronize()
    got = {k: p.grad.detach().cpu().clone() for k, p in net.named_parameters()}
    gates = bn_stage_gates(eng)
    ON.gate_with(lambda name, _: gates[name])
    drop = OD.make_drop({s.name: E._mix_seed(eng.seed, s.id) for s in eng.stages}, 0.5)
    try:
        out, _ = UO.unet_forward(sd, x.double(), norm, True, drop, num_downs=num_downs)
        stats = dict(ON.GATE_STATS)
    finally:
        ON.gate_with(None)
    flips = sum(v for k, v in stats.items() if k != "__total__")
    assert flips <= 2e-5 * stats.get("__total__", 1), stats
    e_f = relmax(eng.fakes.cpu().permute(0, 3, 1, 2), out.detach())
    keys = [k for k in sd if k in names]
    refs = torch.autograd.grad((out * up.double().permute(0, 3, 1, 2)).sum(), [sd[k] for k in keys])
    mx = max(r.abs().max().item() for r in refs)
    worst = {}
    for k, r in zip(keys, refs):
        if r.abs().max().item() < 1e-6 * mx:     # a conv bias followed by InstanceNorm: its gradient is zero
            assert got[k].abs().max().item() < 1e-4 * mx, k
            continue
        worst[k] = relmax(got[k], r)
    record(f"small_unet_engine[nd={num_downs},S={S},B={B},{norm}]",
           f"fakes {e_f:.3e} flips {flips} worst grads {sorted(worst.items(), key=lambda kv: -kv[1])[:3]}")
    # Measured on an H100 80GB HBM3 (700 W limit): parameter gradients up to 9e-5 with batch norm and without a norm,
    # fakes up to 2.7e-4.  With InstanceNorm the weight gradients of the convs whose output is normalised over a 2x2
    # plane (D_{nd-2}, U_{nd-1}) reach 3.6e-4: rstd over 4 values magnifies the forward floor of the 512-channel
    # levels (LONG_K_FWD_TOL).  The gates are the device's, so no flip enters these numbers.
    assert e_f < 1e-3, e_f
    assert max(worst.values()) < (1e-3 if norm == "instance" else 1e-4), worst
