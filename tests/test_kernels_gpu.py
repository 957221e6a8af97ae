"""GPU parity of every CUDA kernel behind the C ABI, one op at a time, against fp64 torch
restatements of the reference ops (and the numpy ROI oracle).

Tolerances (max|err| / max|ref|; the north-star bar is 1e-3 relative fp32): forward GEMMs run
fp16-split x3 -> < 1.5e-5; backward GEMMs run bf16-split x3 -> < 1e-4.  Single-pass GEMMs (nsplit = 1,
`--b200_precision bf16`) are held to 1.5e-5 (3e-5 at the baseline shapes) against the fp64 product of the
16-bit operands they read (the operand model below).
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import roi_align as R  # noqa: E402
from swapnet_b200 import lowering as L  # noqa: E402


def dev():
    return torch.device("cuda:0")


def relmax(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


def record(name, value):
    from conftest import record as _r

    _r(name, value)


def ref_forward(kind, x, w, b=None):
    if kind == "conv4s2":
        return F.conv2d(x, w, b, 2, 1)
    if kind == "convT4s2":
        return F.conv_transpose2d(x, w, b, 2, 1)
    if kind == "conv3r":
        return F.conv2d(F.pad(x, (1, 1, 1, 1), mode="reflect"), w, b)
    if kind in ("conv4s1", "conv3z"):
        return F.conv2d(x, w, b, 1, 1)
    if kind == "head":
        return F.conv2d(F.pad(F.interpolate(x, scale_factor=2), (1, 0, 1, 0)), w, b, 1, 1)
    raise ValueError(kind)


def nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


# (kind, n, cin, cout, h, w) — shapes chosen to hit: multi M-tile, multi N-tile, partial tiles
# (63/62 PatchGAN planes), tiny planes (nb > 1), padded channels (3/19/22 -> 64), block_n 16/32/64/128
CONV_CASES = [
    ("conv4s2", 2, 3, 64, 32, 32),
    ("conv4s2", 2, 64, 128, 32, 64),
    ("conv4s2", 3, 128, 192, 16, 16),
    ("conv4s2", 5, 64, 64, 4, 4),
    ("conv4s2", 2, 22, 64, 64, 64),
    ("convT4s2", 2, 128, 64, 8, 8),
    ("convT4s2", 2, 192, 128, 16, 32),
    ("convT4s2", 3, 64, 3, 16, 16),
    ("conv3r", 2, 128, 128, 32, 32),
    ("conv3r", 1, 64, 192, 16, 16),
    ("conv4s1", 2, 128, 256, 64, 64),
    ("conv4s1", 2, 64, 1, 63, 63),
    ("conv4s1", 1, 64, 64, 8, 8),
    ("head", 2, 192, 19, 32, 32),
    ("head", 1, 64, 19, 16, 48),
    ("head", 2, 192, 27, 16, 16),        # more outputs than HEAD_SLOT: the unstacked 4-phase forward
    ("conv4s2", 2, 19, 64, 32, 32),      # 19 -> 32-channel rows (SWIZZLE_64B)
    ("conv4s1", 2, 16, 32, 16, 16),      # exactly 16 channels (SWIZZLE_32B), narrow dy too
    ("convT4s2", 2, 32, 16, 8, 8),
    ("conv3z", 2, 3, 64, 32, 32),        # vgg16.features.0 (3 -> 16-channel rows, 9 taps padded to 12)
    ("conv3z", 2, 64, 64, 32, 48),
    ("conv3z", 1, 128, 256, 16, 16),
    ("conv3z", 3, 256, 256, 4, 4),
    # the warp engine at S = 192: planes 96/48/24/12/6/3 wide, PatchGAN 23x23 (conv: 27-row tiles of 3 whole 3x3
    # images, a_rows % 8 != 0 -> unmerged A; weight gradient: 4x4 patches of 4 images over a 3x3 plane, masked)
    ("conv4s2", 2, 64, 128, 24, 24),
    ("conv4s2", 3, 128, 256, 6, 6),
    ("convT4s2", 3, 256, 128, 3, 3),
    ("conv3r", 2, 128, 128, 12, 12),
    ("conv4s1", 2, 256, 512, 24, 24),
    ("head", 2, 64, 19, 48, 48),
    # texture-stage widths: encode 36 -> 36, the U-Net's first conv 36 + 19 = 55 -> 64, the decoder's 36-channel output
    ("conv4s2", 2, 36, 36, 64, 64),
    ("conv4s2", 2, 55, 64, 64, 64),
    ("convT4s2", 2, 128, 36, 16, 16),
]


def make_layer(kind, n, cin, cout, h, w, nsplit, with_bias=True):
    from swapnet_b200 import ops
    from swapnet_b200.layers import ConvLayer

    g = torch.Generator().manual_seed(1234 + n * 7 + cin + cout + h)
    x = torch.randn(n, cin, h, w, generator=g)
    k = 3 if kind in ("conv3r", "conv3z") else 4
    wshape = (cin, cout, k, k) if kind == "convT4s2" else (cout, cin, k, k)
    wt = torch.randn(*wshape, generator=g) * (1.0 / (cin * k * k) ** 0.5)
    bias = torch.randn(cout, generator=g) if with_bias else None
    cp = L.padc(cin)   # 3 -> 16, 22 -> 32 (narrow TMA rows), else multiples of 64
    wide = cin * 33 * 4 > 48 * 1024      # the NCHW packer stages [c][33] floats in shared memory: wide inputs go NHWC
    put = (lambda t, pl: ops.pack_planes(nhwc(t).to(dev()), pl, nhwc=True)) if wide else \
        (lambda t, pl: ops.pack_planes(t.to(dev()), pl))
    if kind == "conv3r":
        xp = F.pad(x, (1, 1, 1, 1), mode="reflect")
        planes = ops.Planes(n, h + 2, w + 2, cp + 64, dev(), c=cp, c_off=64, dual=True)  # inside a wider buffer
        put(xp, planes)
    else:
        planes = ops.Planes(n, h, w, cp + 64, dev(), c=cp, c_off=0, dual=True)
        put(x, planes)
    wd = wt.to(dev()).contiguous()
    bd = None if bias is None else bias.to(dev())
    layer = ConvLayer(kind, wd, bd, planes, nsplit=nsplit, name=f"{kind}-{cin}-{cout}")
    return layer, x, wt, bias


# ---------------------------------------------------------------------------------------------
# the single-pass (nsplit = 1) operand model
# ---------------------------------------------------------------------------------------------
# A product of two 16-bit values is exact in fp32 (fp16 x fp16: 22 significant bits, bf16 x bf16: 16), so the only
# error a correct single-pass GEMM may have is its fp32 accumulation.  Its reference is therefore the fp64 contraction
# of the hi planes the plan reads, not of the fp32 tensors: decoded over the valid channels only (a pad channel counts
# as zero, so garbage read from one shows up as an error) and contracted by oracle/emulate.py over the lowering's specs,
# in fp64 on the device.
#
# Sensitivity: the distance of that model from the exact fp64 result is what the bound has to tell apart from the
# single-pass result.  bf16 operands (backward GEMMs, unit roundoff 2^-8) put it at more than 20x the bound.  fp16
# operands (forward, 2^-11) put it at 1.2e-4 .. 2.9e-4 whatever the shape: 8x .. 19x the 1.5e-5 bound of CONV_CASES
# and 5x .. 9x the 3e-5 of the baseline shapes, so the forward asserts >= 4x the bound.  Every case also asserts that
# the model is >= 20x farther from the exact result than the kernel is from the model.
SP_SEP_BF16, SP_SEP_FP16 = 20.0, 4.0


def hi_values(t, fmt):
    """fp64 values of the hi words of a split 16-bit buffer (fp16 or bf16 bit patterns stored as bfloat16)."""
    from swapnet_b200 import ops

    return (t.view(torch.float16) if fmt == ops.FMT_F16 else t).double()


def plane_hi(p, c):
    """fp64 [n, h, w, p.c]: the hi plane of operand planes p, channels >= c zero."""
    a = hi_values(p.hi[..., p.c_off:p.c_off + p.c], p.fmt).clone()
    a[..., c:] = 0
    return a


def model_forward(layer):
    """fp64 NHWC [n, out_h, out_w, cout]: the contraction of x.hi with the decoded packed weights wp.hi / wscale[0]
    (the head's effective taps as the packer summed them), plus the bias."""
    from oracle import emulate as E

    kind, k, cout = layer.kind, layer.k_pad, layer.cout
    a = plane_hi(layer.x, layer.cin)
    wm = hi_values(layer.wp.hi, layer.wp.fmt) / layer.wscale[0].double()
    b = None if layer.bias is None else layer.bias.double()
    out = a.new_zeros(layer.n, layer.out_h, layer.out_w, cout)
    if layer.stacked:   # one 9-shift contraction, the 4 output phases side by side along N
        slot, spec = L.HEAD_SLOT, L.head_stacked_spec(layer.in_h, layer.in_w)
        plain = L.GemmSpec(False, spec.m_h, spec.m_w, spec.taps, (1, 1), (0, 0), a_hw=spec.a_hw)
        acc = a.new_zeros(layer.n, spec.m_h, spec.m_w, 4 * slot)
        E.emul_tap_gemm(a, plain, wm, k, 4 * slot, acc)
        for p in range(4):
            out[:, p >> 1::2, p & 1::2] = acc[..., p * slot:p * slot + cout]
        return out if b is None else out + b
    for spec in L.forward_specs(kind, layer.in_h, layer.in_w):
        w = wm
        if kind == "head":   # per-phase matrices [rows_pad][ntaps_p * k] at HEAD_PHASE_OFF
            p = spec.w_phase
            nt = L.head_neff(p >> 1) * L.head_neff(p & 1)
            off = layer.rows_pad * k * L.HEAD_PHASE_OFF[p]
            w = wm.reshape(-1)[off:off + layer.rows_pad * nt * k].reshape(layer.rows_pad, nt * k)
        E.emul_tap_gemm(a, spec, w, k, cout, out, bias=b)
    return out


def model_dgrad(layer):
    """fp64 NHWC input gradient (over the padded grid for conv3r): dy.hi contracted with the bf16 pack wd.hi."""
    from oracle import emulate as E

    a = plane_hi(layer.dy, layer.cout)
    wm = hi_values(layer.wd.hi, layer.wd.fmt)
    ih, iw = (layer.in_h + 2, layer.in_w + 2) if layer.kind == "conv3r" else (layer.in_h, layer.in_w)
    dx = a.new_zeros(layer.n, ih, iw, layer.cin)
    for spec in L.dgrad_specs(layer.kind, layer.in_h, layer.in_w):
        E.emul_tap_gemm(a, spec, wm, layer.dy.c, layer.cin, dx)
    return dx


def model_wgrad(layer, dy=None):
    """fp64 weight gradient in torch layout: the hi planes of dy (default: the one bound to the layer) and of the bf16
    twin of the input, contracted over the pixels (emul_wgrad), scattered through the plan's output strides and, for
    the head, folded from effective taps."""
    from oracle import emulate as E

    kind, cin, cout = layer.kind, layer.cin, layer.cout
    dy = layer.dy if dy is None else dy
    (ws,) = L.wgrad_specs(kind, layer.in_h, layer.in_w)
    x_is_dy = ws.x_is == "dy"
    xin = layer.x if layer.x.fmt == dy.fmt else layer.x.twin
    a, d = plane_hi(xin, cin), plane_hi(dy, cout)
    xd, yd = (d, a) if x_is_dy else (a, d)
    cx, cy = (cout, cin) if x_is_dy else (cin, cout)
    g = E.emul_wgrad(xd, yd, ws, cx, cy)
    s_row, s_col = L.wgrad_out_strides(kind, cin, cout, x_is_dy)
    n_out = cout * 25 * cin if kind == "head" else layer.weight.numel()
    tap_off = [t * cin for t in ws.tap_ids] if kind == "head" else list(ws.tap_ids)
    flat = g.new_zeros(n_out)
    rc = (torch.arange(cx, device=g.device)[:, None] * s_row + torch.arange(cy, device=g.device)[None, :] * s_col)
    for t, off in enumerate(tap_off):
        flat.index_add_(0, (rc + off).reshape(-1), g[t].reshape(-1))
    if kind == "head":
        return E.fold_head_wgrad_ref(flat.reshape(cout, 25, cin))
    return flat.reshape(layer.weight.shape)


def at_both_nsplits(cases):
    """Parameter rows of a test over nsplit: every case at nsplit = 3 under the id it had before the nsplit = 1 rows
    came, then every case at nsplit = 1 with '-nsplit1' appended; the last argument of the test is nsplit."""
    rows = []
    for ns in (3, 1):
        for c in cases:
            c = c if isinstance(c, tuple) else (c,)
            cid = "-".join(str(v) for v in c)
            rows.append(pytest.param(*c, ns, id=cid if ns == 3 else f"{cid}-nsplit1"))
    return rows


def check_single_pass(what, got, model, exact, tol, sep_factor):
    """got within tol of the operand model, and the model far enough from the exact result that the bound tells the
    single-pass result apart from it.  Returns (err, sep) for record()."""
    model = model.to(got.device)
    exact = exact.to(got.device)
    err, sep = relmax(got, model), relmax(model, exact)
    assert err < tol, f"{what}: relmax {err:.3e} vs the operand model (bound {tol:.1e})"
    assert sep >= sep_factor * tol and sep >= 20 * err, \
        f"{what}: model vs exact {sep:.3e} cannot separate the bound {tol:.1e} / the error {err:.3e}"
    return err, sep


@pytest.mark.parametrize("nsplit", [3, 1])
@pytest.mark.parametrize("kind,n,cin,cout,h,w", CONV_CASES)
def test_conv_forward(kind, n, cin, cout, h, w, nsplit):
    from swapnet_b200 import ops

    layer, x, wt, bias = make_layer(kind, n, cin, cout, h, w, nsplit)
    oh, ow = L.out_hw(kind, h, w)
    y = torch.full((n, oh, ow, cout + 5), 7.0, device=dev())  # sentinel in the pad channels
    layer.bind_forward(y, y_c_off=2)
    layer.pack()
    layer.forward()
    torch.cuda.synchronize()
    ref = nhwc(ref_forward(kind, x.double(), wt.double(), bias.double()))
    got = y[..., 2:2 + cout].cpu()
    tag = f"conv_fwd[{kind},{n},{cin},{cout},{h}x{w},nsplit={nsplit}]"
    if nsplit == 3:
        # fp16-split x3: operands carry 22 bits; what remains (~3e-6) is the tensor core's fp32
        # accumulation (truncating adds)
        err = relmax(got, ref)
        record(tag, f"{err:.3e}")
        assert err < 1.5e-5, f"{kind} fwd nsplit={nsplit}: relmax {err:.3e}"
    else:
        # single pass: the same fp32-accumulation floor, against the fp64 product of the fp16 hi words it reads
        err, sep = check_single_pass(tag, y[..., 2:2 + cout], model_forward(layer), ref, 1.5e-5, SP_SEP_FP16)
        record(tag, f"{err:.3e} (model vs exact {sep:.3e})")
    assert torch.all(y[..., :2] == 7.0) and torch.all(y[..., 2 + cout:] == 7.0), "wrote outside its channel slice"
    if nsplit == 3 and not getattr(layer, "stacked", False):  # SIMT cross-check of the same descriptors (same split operands)
        y2 = torch.zeros_like(y)
        for spec in L.forward_specs(kind, h, w):
            kw = {}
            if kind == "head":
                p = spec.w_phase
                nt = L.head_neff(p >> 1) * L.head_neff(p & 1)
                kw = dict(w_elem_off=layer.rows_pad * layer.k_pad * L.HEAD_PHASE_OFF[p], w_rows=layer.rows_pad,
                          w_k=nt * layer.k_pad)
            d = ops.tap_gemm_desc(layer.x, spec, layer.wp, layer.k_pad, y2, cout, bias=layer.bias, nsplit=3,
                                  block_n=layer.block_n, out_c_off=2, **kw)
            ops.tap_gemm_simt(d)
        torch.cuda.synchronize()
        assert relmax(y2[..., 2:2 + cout].cpu(), ref) < 5e-6   # fp32 FMA chain over K up to 2048


@pytest.mark.parametrize("kind,n,cin,cout,h,w,nsplit", at_both_nsplits(CONV_CASES))
def test_conv_backward(kind, n, cin, cout, h, w, nsplit):
    from swapnet_b200 import ops

    layer, x, wt, bias = make_layer(kind, n, cin, cout, h, w, nsplit)
    oh, ow = L.out_hw(kind, h, w)
    xr = x.double().requires_grad_()
    wr = wt.double().requires_grad_()
    br = bias.double().requires_grad_()
    yr = ref_forward(kind, xr, wr, br)
    g = torch.Generator().manual_seed(99)
    gy = torch.randn(yr.shape, generator=g)
    if kind == "conv3r":  # compare against the gradient w.r.t. the PADDED input
        xp = F.pad(x.double(), (1, 1, 1, 1), mode="reflect").requires_grad_()
        gx = torch.autograd.grad(F.conv2d(xp, wt.double()), xp, gy.double())[0]
        gw, gb = torch.autograd.grad(yr, (wr, br), gy.double())
    else:
        gx, gw, gb = torch.autograd.grad(yr, (xr, wr, br), gy.double())
    dyc = L.padc(cout) if layer.x.c >= 64 else L.pad64(cout)   # one wgrad operand must carry >= 64 channels
    dy = ops.Planes(n, oh, ow, dyc, dev(), fmt=ops.FMT_BF16)  # gradients travel as bf16-split
    if cout * 33 * 4 > 48 * 1024:   # the NCHW packer stages [c][33] floats in shared memory: wide gradients go NHWC
        ops.pack_planes(nhwc(gy).to(dev()), dy, nhwc=True)
    else:
        ops.pack_planes(gy.to(dev()), dy)
    ih, iw = (h + 2, w + 2) if kind == "conv3r" else (h, w)
    dx = torch.full((n, ih, iw, cin + 3), 5.0, device=dev())
    wg = torch.zeros_like(layer.weight)
    bg = torch.zeros(cout, device=dev())
    layer.bind_backward(dy, dx, wg, bg, dx_c_off=1)
    layer.pack()
    layer.backward()
    torch.cuda.synchronize()
    # the bias gradient is no GEMM: bias_grad_kernel reads hi + lo whatever nsplit is
    e_b = relmax(bg.cpu(), gb)
    assert e_b < 1e-4, f"{kind} bias grad relmax {e_b:.3e}"
    if nsplit == 3:
        e_dx = relmax(dx[..., 1:1 + cin].cpu(), nhwc(gx))
        e_w = relmax(wg.cpu(), gw)
        record(f"conv_bwd[{kind},{n},{cin},{cout},{h}x{w}]", f"dx {e_dx:.3e} w {e_w:.3e} b {e_b:.3e}")
        assert e_dx < 1e-4, f"{kind} dgrad relmax {e_dx:.3e}"
        assert e_w < 1e-4, f"{kind} wgrad relmax {e_w:.3e}"
    else:
        e_dx, s_dx = check_single_pass(f"{kind} dgrad", dx[..., 1:1 + cin], model_dgrad(layer), nhwc(gx), 1.5e-5,
                                       SP_SEP_BF16)
        e_w, s_w = check_single_pass(f"{kind} wgrad", wg, model_wgrad(layer), gw, 1.5e-5, SP_SEP_BF16)
        record(f"conv_bwd[{kind},{n},{cin},{cout},{h}x{w},nsplit=1]",
               f"dx {e_dx:.3e} w {e_w:.3e} b {e_b:.3e} (model vs exact: dx {s_dx:.3e} w {s_w:.3e})")
    assert torch.all(dx[..., 0] == 5.0) and torch.all(dx[..., 1 + cin:] == 5.0)


# BASELINE configs[1] layer shapes (512x512, batch 16 per GPU; App. A of SURVEY.md): the resblock conv (K = 9216 forward,
# 16384-pixel weight-gradient reduction), the PatchGAN stride-1 conv on the 2B batch of the D step (63x63 planes), the
# up-sample+pad head (256x256 -> 512x512, 19 outputs) and the widest decoder ConvTranspose2d.  The checker is torch's
# own fp64 convolution ON THE GPU (cuDNN / native fp64 — test infrastructure only; the same sizes on 16 CPU cores would
# take minutes).
BASELINE_CASES = [
    ("conv3r", 16, 1024, 1024, 32, 32),
    ("conv4s1", 32, 256, 512, 64, 64),
    ("head", 16, 192, 19, 256, 256),
    ("convT4s2", 16, 768, 128, 64, 64),
]


def ref_fwd_bwd(kind, x, wt, bias, gy, chunk=4):
    """fp64 output of ref_forward and its gradients (input, weight, bias) for the output gradient gy, on the GPU,
    `chunk` images at a time: every image is independent and the weight and bias gradients are sums over the images.
    At the 512x512 head shape the autograd graph of the whole batch of 16 exceeds the 80 GB of an H100."""
    d = dev()
    w = wt.to(d).double().requires_grad_()
    b = bias.to(d).double().requires_grad_()
    ys, gxs, gw, gb = [], [], 0, 0
    for i in range(0, x.shape[0], chunk):
        xi = x[i:i + chunk].to(d).double().requires_grad_()
        gyi = gy[i:i + chunk].double()
        yi = ref_forward(kind, xi, w, b)
        if kind == "conv3r":   # gradient w.r.t. the PADDED input (what the engine consumes)
            xp = F.pad(xi.detach(), (1, 1, 1, 1), mode="reflect").requires_grad_()
            gxi = torch.autograd.grad(F.conv2d(xp, w.detach()), xp, gyi)[0]
            gwi, gbi = torch.autograd.grad(yi, (w, b), gyi)
        else:
            gxi, gwi, gbi = torch.autograd.grad(yi, (xi, w, b), gyi)
        ys.append(yi.detach())
        gxs.append(gxi)
        gw, gb = gw + gwi, gb + gbi
    return torch.cat(ys), torch.cat(gxs), gw, gb


@pytest.mark.parametrize("kind,n,cin,cout,h,w,nsplit", at_both_nsplits(BASELINE_CASES))
def test_conv_baseline_shapes_fwd_bwd(kind, n, cin, cout, h, w, nsplit):
    from swapnet_b200 import ops

    layer, x, wt, bias = make_layer(kind, n, cin, cout, h, w, nsplit)
    oh, ow = L.out_hw(kind, h, w)
    d = dev()
    y = torch.zeros(n, oh, ow, cout, device=d)
    layer.bind_forward(y)
    layer.pack()
    layer.forward()
    torch.cuda.synchronize()
    with torch.backends.cudnn.flags(enabled=True, deterministic=True, allow_tf32=False):
        gy = torch.randn((n, cout, oh, ow), generator=torch.Generator().manual_seed(99)).to(d)
        yr, gx, gw, gb = ref_fwd_bwd(kind, x, wt, bias, gy)
        e_f = relmax(y, nhwc(yr))
        if nsplit == 1:
            e_f, s_f = check_single_pass(f"{kind} fwd", y, model_forward(layer), nhwc(yr), 3e-5, SP_SEP_FP16)
        del yr
    dyc = L.padc(cout) if layer.x.c >= 64 else L.pad64(cout)
    dy = ops.Planes(n, oh, ow, dyc, d, fmt=ops.FMT_BF16)
    if cout * 33 * 4 > 48 * 1024:
        ops.pack_planes(nhwc(gy), dy, nhwc=True)
    else:
        ops.pack_planes(gy.contiguous(), dy)
    ih, iw = (h + 2, w + 2) if kind == "conv3r" else (h, w)
    dx = torch.zeros(n, ih, iw, cin, device=d)
    wg = torch.zeros_like(layer.weight)
    bg = torch.zeros(cout, device=d)
    layer.bind_backward(dy, dx, wg, bg)
    layer.pack()
    layer.backward()
    torch.cuda.synchronize()
    e_b = relmax(bg, gb)
    if nsplit == 1:   # the real K (up to 9216) and the 1 M-pixel weight-gradient reductions, single pass
        e_dx, s_dx = check_single_pass(f"{kind} dgrad", dx, model_dgrad(layer), nhwc(gx), 3e-5, SP_SEP_BF16)
        del gx
        e_w, s_w = check_single_pass(f"{kind} wgrad", wg, model_wgrad(layer), gw, 3e-5, SP_SEP_BF16)
        record(f"conv_baseline_shape[{kind},{n},{cin},{cout},{h}x{w},nsplit=1]",
               f"fwd {e_f:.3e} dx {e_dx:.3e} w {e_w:.3e} b {e_b:.3e} "
               f"(model vs exact: fwd {s_f:.3e} dx {s_dx:.3e} w {s_w:.3e})")
        assert e_b < 1e-4, e_b
        return
    e_dx, e_w = relmax(dx, nhwc(gx)), relmax(wg, gw)
    record(f"conv_baseline_shape[{kind},{n},{cin},{cout},{h}x{w}]",
           f"fwd {e_f:.3e} dx {e_dx:.3e} w {e_w:.3e} b {e_b:.3e}")
    # forward: fp16-split x3 operands; the floor is the tensor core's truncating fp32 accumulator (grows with K).
    # weight gradient: bf16-split operands (2^-17 per product) reduced over up to 1 M pixels with fp32 atomics
    assert e_f < 3e-5, f"{kind} fwd relmax {e_f:.3e}"
    assert e_dx < 1e-4 and e_w < 3e-4 and e_b < 1e-4, (e_dx, e_w, e_b)


def test_pack_planes_roundtrip():
    from swapnet_b200 import ops

    x = torch.randn(2, 19, 24, 40)
    p = ops.Planes(2, 24, 40, 128, dev(), c=64, c_off=64)
    ops.pack_planes(x.to(dev()), p)
    torch.cuda.synchronize()
    got = p.dense().cpu()
    assert relmax(got[..., :19], nhwc(x)) < 1e-6
    assert torch.all(got[..., 19:] == 0) and torch.all(p.hi[..., :64] == 0)
    # hi is exactly fp16(x) (default activation format); bf16 planes hold bf16(x)
    assert torch.equal(p.hi[..., 64:64 + 19].view(torch.float16).cpu(), nhwc(x).to(torch.float16))
    pb = ops.Planes(2, 24, 40, 64, dev(), fmt=ops.FMT_BF16)
    ops.pack_planes(x.to(dev()), pb)
    torch.cuda.synchronize()
    assert torch.equal(pb.hi[..., :19].cpu(), nhwc(x).to(torch.bfloat16))
    assert relmax(pb.dense().cpu()[..., :19], nhwc(x)) < 2e-5
    y = torch.randn(2, 24, 40, 32)
    q = ops.Planes(2, 24, 40, 64, dev(), c=24, c_off=8)
    ops.pack_planes(y.to(dev()), q, nhwc=True)
    torch.cuda.synchronize()
    assert relmax(q.dense().cpu(), y[..., :24]) < 1e-6


@pytest.mark.parametrize("c,h,w", [(64, 32, 32), (19, 16, 8), (256, 8, 8), (1, 62, 62), (1024, 4, 4)])
def test_instance_norm_block_fwd_bwd(c, h, w):
    """stats + IN-apply + LeakyReLU + dropout, forward and backward, vs torch autograd (fp64)."""
    from swapnet_b200 import ops

    n = 3
    g = torch.Generator().manual_seed(5)
    y = torch.randn(n, c, h, w, generator=g) * 2.0 + 0.5
    seed, p = 77, 0.5
    mask = ops.dropout_mask(seed, p, n * h * w * c, dev()).cpu().view(n, h, w, c).permute(0, 3, 1, 2).double()
    assert 0.4 < mask.mean().item() < 0.6 or mask.numel() < 2000
    yr = y.double().requires_grad_()
    a_ref = F.leaky_relu(F.instance_norm(yr, eps=1e-5), 0.2) * mask * 2.0
    ga = torch.randn(a_ref.shape, generator=g).double()
    (gy_ref,) = torch.autograd.grad(a_ref, yr, ga)

    yd = nhwc(y).to(dev())
    stats = torch.zeros(n, c, 2, dtype=torch.float64, device=dev())
    ops.plane_stats(yd, c, stats)
    out = ops.Planes(n, h, w, L.pad64(c) + 64, dev(), c=L.pad64(c), c_off=64)
    f32 = torch.zeros(n, h, w, c, device=dev())
    ops.norm_act_fwd(yd, c, stats, ops.ACT_LRELU, 0.2, p, seed, out=out, out_f32=f32)
    torch.cuda.synchronize()
    mean_ref = y.double().mean((2, 3))
    assert relmax(stats[..., 0].cpu(), mean_ref) < 1e-6
    assert relmax(f32.cpu(), nhwc(a_ref.detach())) < 1e-5
    assert relmax(out.dense().cpu()[..., :c], nhwc(a_ref.detach())) < 1e-5

    gad = nhwc(ga.float()).to(dev())
    half = (gad * 0.25).contiguous()
    dy = ops.Planes(n, h, w, L.pad64(c), dev(), fmt=ops.FMT_BF16)
    gst = torch.zeros(n, c, 2, dtype=torch.float64, device=dev())
    # two sources that sum to ga (exercises the multi-source gather)
    ops.norm_act_bwd([ops.GradSrc(half), ops.GradSrc((gad - half).contiguous())], yd, c, stats, ops.ACT_LRELU, dy,
                     gst, 0.2, p, seed)
    torch.cuda.synchronize()
    assert relmax(dy.dense().cpu()[..., :c], nhwc(gy_ref)) < 1e-4


@pytest.mark.parametrize("n,c,h,w", [(1, 64, 256, 256), (1, 512, 63, 63), (2, 512, 63, 63), (2, 128, 128, 128), (16, 64, 256, 256),
                                     (1, 1024, 32, 32)])
def test_instance_norm_block_fwd_bwd_baseline_planes(n, c, h, w):
    """The same block at the plane sizes of the 512x512 networks (up to 65536 pixels per plane), two gradient sources,
    checker = torch fp64 autograd on the GPU."""
    from swapnet_b200 import ops

    d = dev()
    g = torch.Generator(device="cpu").manual_seed(n + c + h)
    y = (torch.randn(n, c, h, w, generator=g) * 2.0 + 0.5).to(d)
    ga = torch.randn(n, c, h, w, generator=g).to(d)
    yr = y.double().requires_grad_()
    a_ref = F.leaky_relu(F.instance_norm(yr, eps=1e-5), 0.2)
    (gy_ref,) = torch.autograd.grad(a_ref, yr, ga.double())
    yd = nhwc(y)
    stats = torch.zeros(n, c, 2, dtype=torch.float64, device=d)
    ops.plane_stats(yd, c, stats)
    out = ops.Planes(n, h, w, L.pad64(c), d)
    ops.norm_act_fwd(yd, c, stats, ops.ACT_LRELU, 0.2, 0.0, 0, out=out)
    gad = nhwc(ga)
    half = (gad * 0.25).contiguous()
    dy = ops.Planes(n, h, w, L.pad64(c), d, fmt=ops.FMT_BF16)
    gst = torch.zeros(n, c, 2, dtype=torch.float64, device=d)
    bg = torch.full((c,), 3.0, device=d) if ops.fused_bias_grad_ok(c) else None    # += semantics: starts at 3
    ops.norm_act_bwd([ops.GradSrc(half), ops.GradSrc((gad - half).contiguous())], yd, c, stats, ops.ACT_LRELU, dy, gst, 0.2,
                     0.0, 0, bias_grad=bg)
    torch.cuda.synchronize()
    e_f = relmax(out.dense()[..., :c], nhwc(a_ref.detach()))
    e_b = relmax(dy.dense()[..., :c], nhwc(gy_ref))
    record(f"instance_norm_block_baseline[{n},{c},{h}x{w}]", f"fwd {e_f:.3e} bwd {e_b:.3e}")
    assert e_f < 1e-5 and e_b < 1e-4, (e_f, e_b)
    if bg is not None:   # the fused bias gradient: per-channel sum of the dy written (~0 behind an InstanceNorm)
        want = dy.dense()[..., :c].double().sum((0, 1, 2))
        assert (bg.double() - 3.0 - want).abs().max().item() < 1e-3 * gy_ref.abs().max().item() * (n * h * w) ** 0.5


@pytest.mark.parametrize("c", [256, 1024])
def test_fused_bias_grad_without_instance_norm(c):
    """norm_act_bwd(bias_grad=...) on a block WITHOUT InstanceNorm (a real, non-zero bias gradient): += sum over pixels."""
    from swapnet_b200 import ops

    d = dev()
    n, h, w = 2, 8, 8
    g = torch.Generator().manual_seed(c)
    y = torch.randn(n, h, w, c, generator=g).to(d)
    ga = torch.randn(n, h, w, c, generator=g).to(d)
    dy = ops.Planes(n, h, w, c, d, fmt=ops.FMT_BF16)
    bg = torch.zeros(c, device=d)
    ops.norm_act_bwd([ops.GradSrc(ga)], y, c, None, ops.ACT_RELU, dy, None, 0.2, 0.0, 0, bias_grad=bg)
    torch.cuda.synchronize()
    ref = (ga.double() * (y > 0)).sum((0, 1, 2))
    assert relmax(bg, ref) < 1e-5


def test_residual_tail_and_reflect_pad():
    """ResidualBlock tail: out = x + IN(y2), written as reflect-padded planes + fp32 stream."""
    from swapnet_b200 import ops

    n, c, h, w = 2, 64, 8, 8
    y = torch.randn(n, c, h, w)
    xres = torch.randn(n, c, h, w)
    ref = xres.double() + F.instance_norm(y.double(), eps=1e-5)
    yd, xd = nhwc(y).to(dev()), nhwc(xres).to(dev())
    stats = torch.zeros(n, c, 2, dtype=torch.float64, device=dev())
    ops.plane_stats(yd, c, stats)
    pl = ops.Planes(n, h + 2, w + 2, 64, dev())
    f32 = torch.zeros(n, h, w, c, device=dev())
    ops.norm_act_fwd(yd, c, stats, ops.ACT_NONE, residual=xd, out=pl, reflect_pad=True, out_f32=f32)
    torch.cuda.synchronize()
    assert relmax(f32.cpu(), nhwc(ref)) < 1e-5
    pad_ref = nhwc(F.pad(ref, (1, 1, 1, 1), mode="reflect"))
    assert relmax(pl.dense().cpu(), pad_ref) < 1e-5
    # adjoint: reflect-padded gradient source folds back onto the interior
    gp = torch.randn(n, c, h + 2, w + 2)
    xin = torch.randn(n, c, h, w).double().requires_grad_()
    (gref,) = torch.autograd.grad(F.pad(xin, (1, 1, 1, 1), mode="reflect"), xin, gp.double())
    dst = torch.zeros(n, h, w, c, device=dev())
    ops.sum_grads([ops.GradSrc(nhwc(gp).to(dev()), 0, True)], n, h, w, c, dst)
    torch.cuda.synchronize()
    assert relmax(dst.cpu(), nhwc(gref)) < 1e-6


def test_tanh_bwd():
    from swapnet_b200 import ops

    n, c, h, w = 2, 19, 16, 16
    z = torch.randn(n, h, w, c).double().requires_grad_()
    out = torch.tanh(z)
    g1, g2 = torch.randn(n, h, w, 24), torch.randn(n, h, w, c)
    (ref,) = torch.autograd.grad(out, z, g1[..., 3:3 + c].double() + g2.double())
    dy = ops.Planes(n, h, w, 64, dev(), fmt=ops.FMT_BF16)
    ops.tanh_bwd([ops.GradSrc(g1.to(dev()), 3), ops.GradSrc(g2.to(dev()))], out.detach().float().to(dev()), c, dy)
    torch.cuda.synchronize()
    assert relmax(dy.dense().cpu()[..., :c], ref) < 1e-4


def test_losses():
    from swapnet_b200 import ops

    n, c, h, w = 2, 19, 32, 32
    g = torch.Generator().manual_seed(3)
    logits = torch.tanh(torch.randn(n, c, h, w, generator=g))
    lab = torch.randint(0, c, (n, h, w), generator=g)
    tgt = torch.zeros(n, c, h, w)
    for k in range(1, c):
        tgt[:, k] = (lab == k).float()  # label 0 -> all-zero vector (argmax tie -> index 0)
    lr = logits.double().requires_grad_()
    loss_ref = F.cross_entropy(lr, tgt.argmax(1)) * 100
    (g_ref,) = torch.autograd.grad(loss_ref, lr)
    acc = torch.zeros(1, dtype=torch.float64, device=dev())
    grad = torch.zeros(n, h, w, c, device=dev())
    ops.ce_loss_fwd_bwd(nhwc(logits).to(dev()), c, tgt.to(dev()), 100.0, acc, grad)
    torch.cuda.synchronize()
    assert abs(acc.item() - loss_ref.item()) / loss_ref.item() < 1e-6
    assert relmax(grad.cpu(), nhwc(g_ref)) < 1e-5

    pred = torch.randn(2 * 4, 1, 30, 30, generator=g) * 3
    pr = pred.double().requires_grad_()
    lf = F.binary_cross_entropy_with_logits(pr[:4], torch.full_like(pr[:4], 0.83))
    lr_ = F.binary_cross_entropy_with_logits(pr[4:], torch.full_like(pr[4:], 1.02))
    (gp,) = torch.autograd.grad(0.5 * (lf + lr_), pr)
    acc2 = torch.zeros(2, dtype=torch.float64, device=dev())
    dp = torch.zeros_like(pred, device=dev())
    ops.bce_logits_fwd_bwd(pred.to(dev()), 2, 0.83, 1.02, 0.5, acc2, dp)
    torch.cuda.synchronize()
    assert abs(acc2[0].item() - lf.item()) < 1e-6 and abs(acc2[1].item() - lr_.item()) < 1e-6
    assert relmax(dp.cpu(), gp) < 1e-5

    a = torch.randn(n, 3, h, w, generator=g)
    b = torch.randn(n, 3, h, w, generator=g)
    ar = a.double().requires_grad_()
    l1 = F.l1_loss(ar, b.double()) * 10
    (ga,) = torch.autograd.grad(l1, ar)
    acc3 = torch.zeros(1, dtype=torch.float64, device=dev())
    g3 = torch.zeros(n, h, w, 3, device=dev())
    ops.l1_loss_fwd_bwd(nhwc(a).to(dev()), 3, b.to(dev()), 10.0, acc3, g3)
    torch.cuda.synchronize()
    assert abs(acc3.item() - l1.item()) / l1.item() < 1e-6
    assert relmax(g3.cpu(), nhwc(ga)) < 1e-6


def test_roi_align_pack_bit_exact():
    """ROI bookkeeping must be bit-exact: values equal the numpy oracle bit for bit."""
    from swapnet_b200 import ops

    S, B = 256, 3
    base = np.concatenate([R.NOTEBOOK_ROIS_256, R.NOTEBOOK_EXTRA_256])
    rois = np.stack([np.roll(base, b, axis=0)[:12] for b in range(B)]).astype(np.float32)
    rois[2, 5] = [-30, -20, 40, 50]
    rois[1, 3] = [S + 5, S + 7, S + 40, S + 50]
    rois[0, 7] = [10.5, 20.25, 11.0, 20.5]
    tex = torch.randn(B, 3, S, S, generator=torch.Generator().manual_seed(0))
    ref = R.roi_align_pack(tex.numpy(), rois, 128)  # [B, 36, 128, 128]
    out = torch.zeros(B, 128, 128, 40, device=dev())
    planes = ops.Planes(B, 128, 128, 64, dev())
    ops.roi_align_pack(tex.to(dev()), torch.from_numpy(rois).to(dev()), 128, out, planes)
    torch.cuda.synchronize()
    got = out[..., :36].permute(0, 3, 1, 2).cpu().numpy()
    assert np.array_equal(got, ref), f"max abs diff {np.abs(got - ref).max()}"
    assert relmax(planes.dense().cpu()[..., :36], torch.from_numpy(ref).permute(0, 2, 3, 1)) < 1e-6


def test_fused_adamw_matches_torch():
    """FusedAdamW (one kernel over flat buffers) vs torch.optim.AdamW as the reference builds it
    (optimizers/__init__.py:48-59), 5 steps, G-like (wd 0) and D-like (wd 0.01) settings; state_dict round trip."""
    from swapnet_b200.optim import FusedAdamW, flatten_parameters

    for lr, wd in ((1e-4, 0.0), (4e-4, 0.01)):
        torch.manual_seed(1)
        shapes = [(64, 3, 4, 4), (19,), (128, 64, 3, 3), (7,)]
        ref_p = [torch.nn.Parameter(torch.randn(s, device=dev())) for s in shapes]
        my_p = [torch.nn.Parameter(p.detach().clone()) for p in ref_p]
        flat = flatten_parameters(my_p)
        ref = torch.optim.AdamW(ref_p, lr=lr, weight_decay=wd, betas=(0.9, 0.999))
        mine = FusedAdamW(my_p, flat, lr=lr, weight_decay=wd, betas=(0.9, 0.999))
        mine.flat_grad = torch.zeros_like(flat)
        off = 0
        views = []
        for p in my_p:
            views.append(mine.flat_grad[off:off + p.numel()].view_as(p))
            off += p.numel()
        for step in range(5):
            for rp, gv in zip(ref_p, views):
                g = torch.randn(rp.shape, device=dev()) * (10.0 ** (-step))
                rp.grad = g.clone()
                gv.copy_(g)
            ref.step()
            mine.step()
            if step == 2:   # state_dict round trip in torch's layout
                sd = mine.state_dict()
                assert set(sd["state"][0]) == {"step", "exp_avg", "exp_avg_sq"}
                mine.load_state_dict(sd)
        torch.cuda.synchronize()
        for rp, mp in zip(ref_p, my_p):
            assert relmax(mp.detach().cpu(), rp.detach().cpu()) < 2e-6, (lr, wd)
        rs = ref.state_dict()["state"]
        ms = mine.state_dict()["state"]
        for i in range(len(shapes)):
            assert relmax(ms[i]["exp_avg_sq"].cpu(), rs[i]["exp_avg_sq"].cpu()) < 1e-5
            assert float(ms[i]["step"]) == float(rs[i]["step"]) == 5.0


# ---------------------------------------------------------------------------------------------
# VGG16 perceptual-loss pieces (modules/losses/perceptual.py)
# ---------------------------------------------------------------------------------------------
def planes_to_float(p):
    return p.dense()


def test_affine_pack():
    from swapnet_b200 import ops

    g = torch.Generator().manual_seed(3)
    a = torch.rand(2, 3, 16, 24, generator=g)
    for nhwc_src in (False, True):
        src = (a.permute(0, 2, 3, 1).contiguous() if nhwc_src else a).to(dev())
        dst = ops.Planes(2, 16, 24, 16, dev())
        dst.hi.fill_(1.0)                                    # stale data must be overwritten
        ops.affine_pack(src, nhwc_src, 2.0, -1.0, dst)
        got = planes_to_float(dst).cpu()
        assert relmax(got[..., :3], nhwc(2.0 * a - 1.0)) < 1e-6
        assert torch.all(got[..., 3:] == 0)


@pytest.mark.parametrize("c,h,w", [(64, 16, 24), (128, 8, 8), (512, 4, 6)])
def test_relu_pool_fwd_bwd(c, h, w):
    from swapnet_b200 import ops

    g = torch.Generator().manual_seed(c + h)
    n = 2
    y = torch.randn(n, c, h, w, generator=g)
    y[0, :, :2, :2] = -1.0                                   # an all-negative window: zero output, zero gradient
    y[1, :, 2:4, 2:4] = 0.75                                 # a tied window: gradient goes to the first element
    gp = torch.randn(n, c, h // 2, w // 2, generator=g)
    gd = torch.randn(n, c, h, w, generator=g)
    yd = nhwc(y).to(dev())
    out = ops.Planes(n, h // 2, w // 2, c, dev())
    ops.relu_pool_fwd(yd, c, out)
    yr = y.double().requires_grad_()
    a = F.relu(yr)
    pooled = F.max_pool2d(a, 2, 2)
    assert relmax(planes_to_float(out).cpu(), nhwc(pooled.detach())) < 1e-6
    (gx,) = torch.autograd.grad([pooled, a], [yr], [gp.double(), gd.double()])
    dy = ops.Planes(n, h, w, c, dev(), fmt=ops.FMT_BF16)
    ops.relu_pool_bwd(yd, c, nhwc(gp).to(dev()), nhwc(gd).to(dev()), dy)
    assert relmax(planes_to_float(dy).cpu(), nhwc(gx)) < 2e-5          # bf16-split: 16 bits
    ops.relu_pool_bwd(yd, c, nhwc(gp).to(dev()), None, dy)
    (gx2,) = torch.autograd.grad([F.max_pool2d(F.relu(yr), 2, 2)], [yr], [gp.double()])
    assert relmax(planes_to_float(dy).cpu(), nhwc(gx2)) < 2e-5


@pytest.mark.parametrize("c", [64, 128, 256, 512])
def test_feat_loss(c):
    """one tap of PerceptualLoss: MSE of L2-normalised ReLU features, value + gradient (perceptual.py:53-57,72-78)"""
    from swapnet_b200 import ops

    g = torch.Generator().manual_seed(c)
    n, h, w = 2, 6, 5
    yo = torch.randn(n, c, h, w, generator=g)
    yt = torch.randn(n, c, h, w, generator=g)
    lam = 20.0
    xo = F.relu(yo.double()).requires_grad_()
    xt = F.relu(yt.double())
    fo = xo / (torch.sqrt(torch.pow(xo, 2).sum(1, keepdim=True)) + 1e-8)
    ft = xt / (torch.sqrt(torch.pow(xt, 2).sum(1, keepdim=True)) + 1e-8)
    loss = F.mse_loss(fo, ft) * lam
    (gx,) = torch.autograd.grad(loss, xo)
    acc = torch.zeros(1, dtype=torch.float64, device=dev())
    dx = torch.zeros(n, h, w, c, device=dev())
    ops.feat_loss_fwd_bwd(nhwc(yo).to(dev()), nhwc(yt).to(dev()), c, lam / yo.numel(), 2.0, acc, dx)
    assert abs(acc.item() - loss.item()) < 1e-5 * abs(loss.item())
    assert relmax(dx.cpu(), 2.0 * nhwc(gx)) < 1e-5


@pytest.mark.parametrize("n,s", [(2, 32), (16, 64), (1, 48)])
def test_gram_rows_style_loss(n, s):
    """5 x MSE(gram(out), gram(tgt)) on raw images viewed as [B*3, H*W] (perceptual.py:6-10,58-63)"""
    from swapnet_b200 import ops

    g = torch.Generator().manual_seed(n + s)
    out = torch.rand(n, 3, s, s, generator=g) * 2 - 1
    tgt = torch.rand(n, 3, s, s, generator=g) * 4.5 - 2
    lam = 1e-8
    o = out.double().requires_grad_()

    def gram(t):
        t = t.reshape(n * 3, s * s)
        return t @ t.t()

    loss = 5 * F.mse_loss(gram(o), gram(tgt.double())) * lam
    (gx,) = torch.autograd.grad(loss, o)
    r = 3 * n
    go = torch.zeros(r, r, dtype=torch.float64, device=dev())
    gt = torch.zeros_like(go)
    m = torch.zeros(r, r, device=dev())
    fk = nhwc(out).to(dev())
    tg = tgt.to(dev())
    ops.gram_rows(fk, fk, True, go)
    ops.gram_rows(tg, tg, False, gt)
    assert relmax(go.cpu(), gram(out.double())) < 1e-5 and relmax(gt.cpu(), gram(tgt.double())) < 1e-5
    acc = torch.zeros(1, dtype=torch.float64, device=dev())
    ops.gram_rows_mse(go, gt, 5 * lam, acc, m)
    assert abs(acc.item() - loss.item()) < 1e-4 * abs(loss.item())
    dx = torch.full((n, s, s, 3), 7.0, device=dev())
    ops.gram_rows_bwd(m, fk, True, dx, accumulate=False)
    assert relmax(dx.cpu(), nhwc(gx)) < 1e-4
    base = torch.randn(n, s, s, 3, generator=g) * gx.abs().max().float()   # same magnitude as the L1 gradient it joins
    dx = base.clone().to(dev())
    ops.gram_rows_bwd(m, fk, True, dx, accumulate=True)
    assert relmax(dx.cpu(), base.double() + nhwc(gx)) < 1e-4


@pytest.mark.parametrize("c,f", [(36, 8), (6, 2), (64, 4)])
def test_upsample_planes(c, f):
    """F.interpolate(scale_factor=f) (nearest) of the encoded textures (swapnet_modules.py:244-247) on split planes."""
    from swapnet_b200 import ops

    g = torch.Generator().manual_seed(c)
    n, h, w = 2, 4, 6
    x = torch.randn(n, c, h, w, generator=g)
    src = ops.Planes(n, h, w, 64, dev(), c=L.padc(c) if c > 8 else 8)
    ops.pack_planes(x.to(dev()), src.slice(0, c))
    dst = ops.Planes(n, h * f, w * f, 128, dev(), c=64, c_off=8)
    ops.upsample_planes(src.slice(0, c), dst.slice(0, c), f)
    torch.cuda.synchronize()
    ref = nhwc(F.interpolate(x, scale_factor=f))
    got = dst.dense().cpu()
    assert relmax(got[..., :c], ref) < 1e-6
    assert torch.all(got[..., c:] == 0)


@pytest.mark.parametrize("n,cin,h,w", [(2, 256, 15, 15), (3, 64, 9, 12), (2, 128, 63, 63), (2, 512, 63, 63), (3, 512, 5, 5)])
def test_to_one_conv_layer(n, cin, h, w):
    """Conv2d(cin, 1, 4, 1, 1) (PatchGAN logits, discriminators.py:131) through layers.ToOneConvLayer (CUDA-core
    streaming kernels of csrc/patch_logits.cu): forward, input gradient, weight and bias gradients vs torch (fp64)."""
    from swapnet_b200 import ops
    from swapnet_b200.layers import ToOneConvLayer

    g = torch.Generator().manual_seed(n * 1000 + cin + h)
    x = torch.randn(n, cin, h, w, generator=g)
    wt = torch.randn(1, cin, 4, 4, generator=g) * (1.0 / (cin * 16) ** 0.5)
    bias = torch.randn(1, generator=g)
    planes = ops.Planes(n, h, w, L.pad64(cin), dev(), dual=True)
    ops.pack_planes(nhwc(x).to(dev()), planes, nhwc=True)
    layer = ToOneConvLayer("conv4s1", wt.to(dev()).contiguous(), bias.to(dev()), planes, nsplit=3, name="logits")
    y = torch.zeros(n, h - 1, w - 1, 1, device=dev())
    layer.bind_forward(y)
    xr, wr, br = x.double().requires_grad_(), wt.double().requires_grad_(), bias.double().requires_grad_()
    yr = F.conv2d(xr, wr, br, 1, 1)
    gy = torch.randn(yr.shape, generator=g)
    gx, gw, gb = torch.autograd.grad(yr, (xr, wr, br), gy.double())
    dy = ops.Planes(n, h - 1, w - 1, 16, dev(), fmt=ops.FMT_BF16)
    ops.pack_planes(gy.to(dev()), dy)
    dx = torch.zeros(n, h, w, cin, device=dev())
    wg = torch.zeros_like(layer.weight)
    bg = torch.zeros(1, device=dev())
    layer.bind_backward(dy, dx, wg, bg)
    layer.pack()
    layer.forward()
    layer.backward()
    layer.backward()           # weight gradients accumulate (+=); dx and the bias gradient are overwritten
    torch.cuda.synchronize()
    e_y = relmax(y.cpu(), nhwc(yr.detach()))
    e_dx, e_w, e_b = relmax(dx.cpu(), nhwc(gx)), relmax(wg.cpu(), 2 * gw), relmax(bg.cpu(), gb)
    record(f"to_one_conv[{n},{cin},{h}x{w}]", f"y {e_y:.3e} dx {e_dx:.3e} w {e_w:.3e} b {e_b:.3e}")
    # forward: fp32 FMA chain over cin*16 products of 22-bit operands; backward: dy carried as bf16-split planes
    assert e_y < 3e-5 and e_dx < 1e-4 and e_w < 1e-4 and e_b < 1e-4, (e_y, e_dx, e_w, e_b)


@pytest.mark.parametrize("kind,n,cin,cout,h,w,fused,nsplit", at_both_nsplits([
    ("conv4s2", 2, 64, 128, 32, 64, True), ("convT4s2", 2, 128, 64, 16, 16, True),
    ("conv3r", 3, 128, 128, 32, 32, True), ("conv4s1", 2, 128, 256, 64, 64, True),
    ("conv4s2", 3, 128, 192, 16, 16, False),
    ("conv4s2", 2, 36, 36, 64, 64, False),   # n_valid % 16 != 0
    ("conv4s2", 2, 55, 64, 64, 64, True)]))
def test_fused_instance_norm_statistics(kind, n, cin, cout, h, w, fused, nsplit):
    """InstanceNorm statistics accumulated by the GEMM epilogue (sn_tap_gemm_desc.stats + sn_stats_finalize) equal the
    per-(image, channel) mean and 1/sqrt(biased variance + eps) of the conv output; planes smaller than a tile (several
    images per tile) are refused by the plan and fall back to sn_plane_stats."""
    from swapnet_b200 import ops

    layer, x, wt, bias = make_layer(kind, n, cin, cout, h, w, nsplit)
    oh, ow = L.out_hw(kind, h, w)
    y = torch.zeros(n, oh, ow, cout, device=dev())
    stats = torch.zeros(n, cout, 2, dtype=torch.float64, device=dev())
    layer.bind_forward(y, stats=stats)
    assert layer.fused_stats == fused
    layer.pack()
    layer.forward()
    layer.forward()                       # the launch zeroes the buffer itself: a second run must not double the sums
    if layer.fused_stats:
        ops.stats_finalize(stats, n * cout, oh * ow)
    else:
        ops.plane_stats(y, cout, stats)
    torch.cuda.synchronize()
    ref = ref_forward(kind, x.double(), wt.double(), bias.double())
    sep = ""
    if nsplit == 1:   # the statistics of the single-pass output: those of the operand model's
        model = model_forward(layer)
        _, s_ = check_single_pass(f"{kind} fwd", y, model, nhwc(ref), 1.5e-5, SP_SEP_FP16)
        ref, sep = model.permute(0, 3, 1, 2).cpu(), f" (model vs exact {s_:.3e})"
    mean = ref.mean((2, 3))
    rstd = (ref.var((2, 3), unbiased=False) + 1e-5).rsqrt()
    e_m = ((stats[..., 0].cpu() - mean).abs().max() / ref.abs().max()).item()
    e_r = relmax(stats[..., 1].cpu(), rstd)
    tag = f"fused_in_stats[{kind},{n},{cin},{cout},{h}x{w}" + ("]" if nsplit == 3 else ",nsplit=1]")
    record(tag, f"fused={layer.fused_stats} mean {e_m:.3e} rstd {e_r:.3e}{sep}")
    assert e_m < 1e-5 and e_r < 1e-5, (e_m, e_r)
    assert relmax(y.cpu(), nhwc(ref)) < 1.5e-5
