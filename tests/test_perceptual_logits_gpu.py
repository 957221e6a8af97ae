"""The perceptual-loss kernels (csrc/perceptual.cu) and the PatchGAN logits kernels (csrc/patch_logits.cu) against plain
fp64 torch of the same operation, at the training shapes and at the edges where their grids and tails change.

- affine_pack, relu_pool_fwd/bwd: exact operations (one fp32 multiply and add; a max; one fp32 add).  Their words must
  be common.cuh's split16 of the restated fp32 value, bit for bit.
- feat_loss, the style term (gram_rows, gram_rows_mse, gram_rows_bwd), to_one_fwd, tap_sum_fwd, to_one_wgrad,
  to_one_dgrad: fp32 sums.  Each entry's error is normalised by the sum of the absolute values of its terms (for the
  Gram matrix by sqrt(G_ii G_jj), which bounds that sum) and must stay under k u, u = 2^-24, with k the length of the
  longest chain of fp32 roundings that forms the entry: the kernel's per-thread chain, its tree or row reduction, and
  its block sums.  These are worst-case bounds; the measured values (in units of u) go to the parity log.
- Operands that arrive as split planes are decoded first (dense_of): the fp64 reference is computed from the values the
  kernel reads, so the bounds measure the kernel's arithmetic, not the 16-bit encoding.
- Every output is prefilled with a sentinel (NaN for fp32, SENT16 for plane words): each valid entry must be written,
  nothing outside the channel slice or pitch may be.
- Every reduction with a _det twin runs in both modes against fp64; the _det result must repeat bit for bit and a slot
  capacity one short must be refused.

The references run in fp64 on the GPU (test infrastructure only).
"""
import itertools
import math

import pytest
import torch
import torch.nn.functional as F

from swapnet_b200 import _lib, ops
from swapnet_b200.layers import ToOneConvLayer
from test_elementwise_gpu import (SENT16, assert_outside_untouched, assert_split_exact, dense_of, fill_sentinel,
                                  split_ref, words)
from test_kernels_gpu import dev, nhwc, record

pytestmark = pytest.mark.gpu

U = 2.0 ** -24          # fp32 unit roundoff
NAN = float("nan")
F16, BF16 = ops.FMT_F16, ops.FMT_BF16
SMS = 132               # SN_NUM_SMS: the grid caps below are multiples of it


def gen(seed):
    return torch.Generator(device=dev()).manual_seed(seed)


def randn(*shape, g):
    return torch.randn(*shape, generator=g, device=dev())


def bounded(name, got, ref, scale, k):
    """max over the entries of |got - ref| / scale must stay under k u.  An entry left NaN fails."""
    err = ((got.double() - ref.double()).abs() / scale.double().clamp_min(1e-300)).max().item()
    record(name, f"{err / U:.2f} u (bound {k:.0f} u)")
    assert err <= k * U, f"{name}: {err / U:.2f} u > {k:.0f} u"


def refused(fn):
    with pytest.raises(_lib.SwapnetB200Error):
        fn()


def split_planes(v, fmt, pitch, c_off):
    """Planes [n,h,w,pitch] holding split16(v) in channels [c_off, c_off + c) and SENT16 elsewhere, and the fp64
    values they decode to."""
    n, h, w, c = v.shape
    p = ops.Planes(n, h, w, pitch, dev(), c=c, c_off=c_off, fmt=fmt)
    fill_sentinel(p)
    hi, lo = split_ref(v, fmt)
    words(p.hi)[..., c_off:c_off + c] = hi
    words(p.lo)[..., c_off:c_off + c] = lo
    return p, dense_of(p.hi, p.lo, fmt, c_off, c_off + c)


def pitched(n, h, w, c, extra, fill):
    """An fp32 NHWC buffer with `extra` channels past c, all set to `fill`, and its [..., :c] view."""
    buf = torch.full((n, h, w, c + extra), fill, device=dev())
    return buf, buf[..., :c]


def _stream():
    return torch.cuda.current_stream().cuda_stream


# =============================================================================================
# perceptual.cu
# =============================================================================================
def run_affine(n, c, h, w, src_nhwc, fmt, seed):
    g = gen(seed)
    a = randn(n, c, h, w, g=g) * 3.0
    a.view(-1)[:6] = torch.tensor([7.0e4, -1.0e5, 0.0, -0.0, 65504.0, 1e-30])   # past the fp16 range, signed zeros
    if src_nhwc:   # the fakes: a channel slice of a wider NHWC buffer
        wide = torch.full((n, h, w, c + 5), 1e30, device=dev())
        wide[..., :c] = nhwc(a)
        src = wide[..., :c]
    else:          # the targets: contiguous NCHW
        src = a
    for mul, add in ((2.0, -1.0), (1.7, -0.3)):
        dst = ops.Planes(n, h, w, 32, dev(), c=16, c_off=8, fmt=fmt)
        fill_sentinel(dst)
        ops.affine_pack(src, src_nhwc, mul, add, dst)
        torch.cuda.synchronize()
        m32 = torch.tensor(mul, dtype=torch.float32, device=dev())
        a32 = torch.tensor(add, dtype=torch.float32, device=dev())
        want = torch.add(torch.mul(nhwc(a), m32), a32)       # fp32 product, then fp32 add: no fused multiply-add
        assert_split_exact(dst, 8, 8 + c, want)
        assert_split_exact(dst, 8 + c, 24, torch.zeros(n, h, w, 16 - c, device=dev()))
        assert_outside_untouched(dst, 8, 24)


@pytest.mark.parametrize("fmt", [F16, BF16])
@pytest.mark.parametrize("src_nhwc", [False, True])
@pytest.mark.parametrize("c", [1, 3, 16])
def test_affine_pack_words(c, src_nhwc, fmt):
    run_affine(2, c, 17, 23, src_nhwc, fmt, seed=c * 10 + src_nhwc)


@pytest.mark.parametrize("src_nhwc", [False, True])
def test_affine_pack_past_grid_cap(src_nhwc):
    """3 x 512 x 512 pixels: more than the 2112 x 256 threads of the capped grid."""
    run_affine(3, 3, 512, 512, src_nhwc, F16, seed=7)


def test_affine_pack_refusals():
    dst = ops.Planes(1, 4, 4, 16, dev())
    refused(lambda: ops.affine_pack(torch.zeros(1, 17, 4, 4, device=dev()), False, 2.0, -1.0, dst))
    odd = ops.Planes(1, 4, 4, 24, dev(), c=16, c_off=4)          # planes not 16-byte aligned
    refused(lambda: ops.affine_pack(torch.zeros(1, 3, 4, 4, device=dev()), False, 2.0, -1.0, odd))


# ---- ReLU + MaxPool2d(2) ----------------------------------------------------------------------------------------
P_TIE = 0.75
POOL_WINDOWS = [(-1.0, -2.0, -0.5, -3.0)]                      # all negative
for _q1, _q2 in itertools.combinations(range(4), 2):            # a positive tie at every pair of window positions
    _v = [0.25, -0.5, 0.5, -0.25]
    _v[_q1] = _v[_q2] = P_TIE
    POOL_WINDOWS.append(tuple(_v))
POOL_WINDOWS += [(P_TIE,) * 4,                                  # a four-way tie
                 (-1.0, 0.0, -2.0, 0.0), (0.0, -1.0, 0.0, -3.0),  # zero ties a negative after the ReLU
                 (-0.0, -1.0, -0.0, -0.5), (-0.0, 0.0, -0.0, 0.0), (-0.0, P_TIE, -0.0, P_TIE)]


def plant_windows(y):
    """Window (0, ow) of row 0 of image 0 holds POOL_WINDOWS[ow] in every channel (positions in row-major order)."""
    for j, v in enumerate(POOL_WINDOWS):
        y[0, :, 0, 2 * j], y[0, :, 0, 2 * j + 1], y[0, :, 1, 2 * j], y[0, :, 1, 2 * j + 1] = v


# (n, c, h, w, output format, gradient format): the five tap shapes of the 512 x 512 texture stage (the first passes
# the 2112-block grid cap), and a small one with c % 8 = 4 and the formats swapped
POOL_CASES = [(1, 64, 512, 512, F16, BF16), (2, 128, 256, 256, F16, BF16), (2, 256, 128, 128, F16, BF16),
              (2, 512, 64, 64, F16, BF16), (2, 512, 32, 32, F16, BF16), (2, 12, 4, 28, BF16, F16)]


@pytest.mark.parametrize("n,c,h,w,ofmt,gfmt", POOL_CASES)
def test_relu_pool_words(n, c, h, w, ofmt, gfmt):
    g = gen(c + h)
    y = randn(n, c, h, w, g=g)
    plant_windows(y)
    ybuf, yv = pitched(n, h, w, c, 4, 1e30)          # a pitched y; the pad channels would win any max they entered
    yv.copy_(nhwc(y))
    relu = torch.where(y > 0, y, 0.0)                 # +0.0 for every y <= 0, -0.0 included
    pooled, idx = F.max_pool2d(relu, 2, 2, return_indices=True)   # torch's rule: the first maximum in the window
    opitch = (c + 8 + 7) // 8 * 8
    out = ops.Planes(n, h // 2, w // 2, opitch, dev(), c=c, c_off=4, fmt=ofmt)
    fill_sentinel(out)
    ops.relu_pool_fwd(yv, c, out)
    torch.cuda.synchronize()
    assert_split_exact(out, 4, 4 + c, nhwc(pooled))
    assert_outside_untouched(out, 4, 4 + c)

    gp = randn(n, c, h // 2, w // 2, g=g)
    gd = randn(n, c, h, w, g=g)
    gpbuf, gpv = pitched(n, h // 2, w // 2, c, 4, 1e30)
    gpv.copy_(nhwc(gp))
    gdbuf, gdv = pitched(n, h, w, c, 8, 1e30)
    gdv.copy_(nhwc(gd))
    routed = torch.zeros(n, c, h * w, device=dev()).scatter_(2, idx.flatten(2), gp.flatten(2)).view(n, c, h, w)
    zero = torch.zeros_like(gd)
    for use_pool, use_direct in ((True, True), (True, False), (False, True)):
        # fp32: g_direct + (g_pool at the first maximum, +0 elsewhere), gated by y > 0
        want = torch.where(y > 0, (gd if use_direct else zero) + (routed if use_pool else zero), 0.0)
        dy = ops.Planes(n, h, w, opitch, dev(), c=c, c_off=4, fmt=gfmt)
        fill_sentinel(dy)
        ops.relu_pool_bwd(yv, c, gpv if use_pool else None, gdv if use_direct else None, dy)
        torch.cuda.synchronize()
        assert_split_exact(dy, 4, 4 + c, nhwc(want))
        assert_outside_untouched(dy, 4, 4 + c)


def test_relu_pool_refusals():
    for h, w, c in ((7, 8, 8), (8, 7, 8), (8, 8, 6)):
        y = torch.zeros(1, h, w, 8, device=dev())
        out = ops.Planes(1, h // 2, w // 2, 8, dev())
        dy = ops.Planes(1, h, w, 8, dev(), fmt=BF16)
        refused(lambda: ops.relu_pool_fwd(y, c, out))
        refused(lambda: ops.relu_pool_bwd(y, c, None, y, dy))


# ---- feature loss ----------------------------------------------------------------------------------------------
def feat_nv(c):
    """float4 registers per lane of feat_loss_kernel (C = 64 runs on half the lanes of NV = 1)."""
    return 1 if c <= 128 else 2 if c <= 256 else 4


def run_feat(n, h, w, c, seed):
    g = gen(seed)
    npix = n * h * w
    yo = randn(n, h, w, c, g=g)
    yt = randn(n, h, w, c, g=g)
    fo_, ft_ = yo.view(npix, c), yt.view(npix, c)
    if npix >= 7:
        neg = -(randn(4, c, g=g).abs() + 0.1)
        fo_[1] = neg[0]                      # output features all zero after the ReLU
        ft_[2] = neg[1]                      # target features all zero
        fo_[npix - 2], ft_[npix - 2] = neg[2], neg[3]   # both
        fo_[npix - 1] = neg[0]
        fo_[npix - 1, c - 1] = 1e-6          # one tiny positive channel: the 1e-8 in the denominator shows
    lam = 20.0
    weight, gscale = lam / (npix * c), 2.0   # PerceptualEngine.content: MSELoss's mean, d(2x - 1)/dx
    acc0 = 0.375

    xo = yo.double().clamp_min(0).requires_grad_()
    xt = yt.double().clamp_min(0)
    # vector_norm's gradient at a zero vector is 0: the kernel's `no > 0` branch
    no = torch.linalg.vector_norm(xo, dim=-1, keepdim=True)
    nt = torch.linalg.vector_norm(xt, dim=-1, keepdim=True)
    fo, ft = xo / (no + 1e-8), xt / (nt + 1e-8)
    lsum = ((fo - ft) ** 2).sum()
    (gx,) = torch.autograd.grad(lsum, xo)
    with torch.no_grad():
        fo, ft, no = fo.detach(), ft.detach(), no.detach()
        d = fo - ft
        unit = torch.where(no > 0, xo.detach() / no.clamp_min(1e-300), 0.0)
        ido = 1.0 / (no + 1e-8)
        # dx_j = 2 w ido [(fo_j - ft_j) - fo_j sum_k (fo_k - ft_k) unit_k]: the absolute values of its terms
        dx_scale = 2 * weight * gscale * ido * (fo.abs() + ft.abs() + fo.abs() * ((fo.abs() + ft.abs()) * unit).sum(-1, keepdim=True))
        loss_ref = weight * lsum.item()
        loss_scale = weight * (d * d + 2 * d.abs() * (fo.abs() + ft.abs())).sum().item()
    # per lane 4 NV squares, a 5-level shuffle tree, for the norm and for the projection, then ~16 single roundings
    k = 2 * (4 * feat_nv(c) + 5) + 16
    blocks = min((npix + 7) // 8, SMS * 8)
    ws = ops.DetWorkspace(dev())
    runs = []
    for det in (False, True, True):
        acc = torch.full((1,), acc0, dtype=torch.float64, device=dev())
        dxb, dxv = pitched(n, h, w, c, 4, NAN)
        yob, yov = pitched(n, h, w, c, 4, 1e30)
        ytb, ytv = pitched(n, h, w, c, 8, 1e30)
        yov.copy_(yo)
        ytv.copy_(yt)
        ops.feat_loss_fwd_bwd(yov, ytv, c, weight, gscale, acc, dxv, ws=ws if det else None)
        torch.cuda.synchronize()
        tag = f"feat_loss[{n}x{h}x{w},c={c},{'det' if det else 'atomic'}]"
        bounded(tag + " dx", dxv, gscale * weight * gx, dx_scale, k)
        assert bool(torch.isnan(dxb[..., c:]).all()), "wrote past its channels"
        err = abs(acc.item() - acc0 - loss_ref) / loss_scale
        record(tag + " loss", f"{err / U:.2f} u (bound {k} u), {blocks} blocks")
        assert err <= k * U + 1e-15 * (acc0 + loss_ref) / loss_scale, (err / U, k)
        runs.append((acc.clone(), dxb.clone()))
    assert torch.equal(runs[1][0], runs[2][0]) and torch.equal(runs[1][1].view(torch.int32), runs[2][1].view(torch.int32)), \
        "feat_loss_det did not repeat bit for bit"


@pytest.mark.parametrize("npix", [1, 7, 8447, 8448, 8449])   # the 1056-block grid strides from 8449 pixels on
@pytest.mark.parametrize("c", [4, 64, 128, 192, 256, 512])
def test_feat_loss(c, npix):
    run_feat(1, 1, npix, c, seed=c + npix)


def test_feat_loss_training_tap():
    """The first tap of the 512 x 512 texture stage at batch 2: 64 channels, 2^19 pixels."""
    run_feat(2, 512, 512, 64, seed=3)


def test_feat_loss_refusals():
    for c, pitch in ((516, 516), (6, 8)):
        t = torch.zeros(1, 1, 4, pitch, device=dev())
        acc = torch.zeros(1, dtype=torch.float64, device=dev())
        refused(lambda: ops.feat_loss_fwd_bwd(t, t, c, 1.0, 1.0, acc, torch.zeros_like(t)))
    for npix in (7, 8449):
        blocks = min((npix + 7) // 8, SMS * 8)
        t = torch.randn(1, 1, npix, 64, device=dev())
        dx = torch.zeros_like(t)
        acc = torch.zeros(1, dtype=torch.float64, device=dev())
        slots = torch.zeros(blocks, dtype=torch.float64, device=dev())

        def call(cap):
            _lib.check(_lib.load().sn_feat_loss_fwd_bwd_det(t.data_ptr(), 64, t.data_ptr(), 64, npix, 64, 1.0, 1.0,
                                                            acc.data_ptr(), dx.data_ptr(), 64, slots.data_ptr(), cap,
                                                            _stream()))
        refused(lambda: call(blocks - 1))
        call(blocks)
        torch.cuda.synchronize()


# ---- Gram matrix and the style term ----------------------------------------------------------------------------
GRAM_P = 128
GRAM_K = GRAM_P + 2     # fp32 chain of one Gram entry: the 128 products of a chunk; the chunk sums are fp64


def gram_source(n, c, npix, src_nhwc, g, lo=-1.0, hi=1.0):
    """(tensor the kernel reads, fp64 rows [n*c, npix])."""
    x = torch.rand(n, c, npix, generator=g, device=dev()) * (hi - lo) + lo
    rows = x.reshape(n * c, npix).double()
    if src_nhwc:
        return x.permute(0, 2, 1).contiguous().view(n, 1, npix, c), rows
    return x.view(n, c, 1, npix), rows


def gram_scale(gm):
    dg = gm.diagonal().abs()
    return torch.sqrt(dg[:, None] * dg[None, :])


@pytest.mark.parametrize("det", [False, True])
def test_gram_rows_style_term_training_shape(det):
    """PerceptualEngine.style at B = 16, S = 512 (R = 48) against fp64 autograd of 5 MSE(X X^T, T T^T) lambda."""
    B, S, lam = 16, 512, 1e-8
    g = gen(16 + det)
    fakes = torch.rand(B, S, S, 3, generator=g, device=dev()) * 2 - 1
    targets = torch.rand(B, 3, S, S, generator=g, device=dev()) * 4.5 - 2
    r, npix = 3 * B, S * S
    xo = fakes.permute(0, 3, 1, 2).reshape(r, npix).double().requires_grad_()
    xt = targets.reshape(r, npix).double()
    go_ref, gt_ref = xo @ xo.T, xt @ xt.T
    loss = 5 * F.mse_loss(go_ref, gt_ref) * lam
    (gx,) = torch.autograd.grad(loss, xo)
    ws = ops.DetWorkspace(dev()) if det else None
    go = torch.full((r, r), NAN, dtype=torch.float64, device=dev())
    gt = torch.full_like(go, NAN)
    m = torch.full((r, r), NAN, device=dev())
    acc0 = 0.25
    acc = torch.full((1,), acc0, dtype=torch.float64, device=dev())
    grad = gx.detach().view(B, 3, S, S).permute(0, 2, 3, 1)
    base = torch.randn(B, S, S, 3, generator=g, device=dev()) * grad.abs().max().float()   # the L1 gradient it joins
    dx = base.clone()
    ops.gram_rows(fakes, fakes, True, go, ws=ws)
    ops.gram_rows(targets, targets, False, gt, ws=ws)
    ops.gram_rows_mse(go, gt, 5.0 * lam, acc, m)
    ops.gram_rows_bwd(m, fakes, True, dx, accumulate=True)
    torch.cuda.synchronize()
    with torch.no_grad():
        dg = GRAM_K * U * (gram_scale(go_ref) + gram_scale(gt_ref))            # |Go error| + |Gt error|, per entry
        d = (go_ref - gt_ref).abs()
        loss_bound = 5 * lam / r ** 2 * (2 * d * dg + dg * dg).sum().item()
        m_ref = 4 * 5 * lam * (go_ref - gt_ref) / r ** 2
        dm = 4 * 5 * lam / r ** 2 * dg + U * m_ref.abs()                  # the Gram errors, then M's fp32 cast
        xabs = xo.detach().abs()
        dx_scale = (dm @ xabs + (r + 2) * U * (m_ref.abs() @ xabs)).view(B, 3, S, S).permute(0, 2, 3, 1)
        dx_scale = dx_scale + U * (base.double().abs() + grad.abs())
    tag = f"style_term[B={B},S={S},{'det' if det else 'atomic'}]"
    lerr = abs(acc.item() - acc0 - loss.item())
    record(tag + " loss", f"{lerr:.3e} (bound {loss_bound:.3e}, loss {loss.item():.3e})")
    assert lerr <= loss_bound + 1e-15 * acc0, (lerr, loss_bound)
    ratio = ((dx.double() - base.double() - grad).abs() / dx_scale).max().item()
    record(tag + " dx", f"{ratio:.3e} of the bound")
    assert ratio <= 1.0, ratio


# =============================================================================================
# patch_logits.cu
# =============================================================================================
def tap_grads(dyd, h, w, pad):
    """dP[n, h, w, 4 kh + kw] = dy[n, h + pad - kh, w + pad - kw] (0 outside) from dy [n, OH, OW] fp64."""
    dyp = F.pad(dyd, (3, 3, 3, 3))
    return torch.stack([dyp[:, 3 + pad - kh:3 + pad - kh + h, 3 + pad - kw:3 + pad - kw + w]
                        for kh in range(4) for kw in range(4)], -1)


def logits_weight(c, g):
    return randn(1, c, 4, 4, g=g) * (1.0 / (c * 16) ** 0.5)


def fwd_k(c):
    """to_one_fwd: a lane's FMA chain over its 8 channels of every 256, then a 5-level shuffle tree."""
    return 8 * ((c + 255) // 256) + 6


def grad_planes(n, oh, ow, g, fmt=BF16):
    """dy as channel 0 of 16-channel planes; channels 1..15 hold SENT16."""
    dy, dyd = split_planes(randn(n, oh, ow, 1, g=g), fmt, 16, 0)
    return dy, dyd[..., 0]


# (c, n, h, w, x format): odd pixel counts, the 528 x 16 = 8448 pixels below which to_one_fwd runs one pass, 264 (not
# a multiple of 256), 1536 (96 KB of weights in shared memory) and the 512 x 512 discriminator's logits at batch 16
FWD_CASES = [(8, 1, 5, 7, F16), (64, 3, 53, 53, F16), (264, 1, 71, 119, BF16), (512, 1, 88, 96, F16),
             (1536, 2, 65, 65, F16), (64, 1, 88, 96, BF16), (8, 2, 65, 65, BF16), (512, 16, 63, 63, F16)]


@pytest.mark.parametrize("c,n,h,w,fmt", FWD_CASES)
def test_to_one_fwd_tap_sum(c, n, h, w, fmt):
    g = gen(c + h)
    x, xd = split_planes(randn(n, h, w, c, g=g), fmt, c + 16, 8)
    wt = logits_weight(c, g)
    pbuf, p = pitched(n, h, w, 16, 8, NAN)
    ops.to_one_fwd(x, wt, p)
    torch.cuda.synchronize()
    wm = wt.double().reshape(c, 16)
    xf = xd.reshape(-1, c)
    k = fwd_k(c)
    bounded(f"to_one_fwd[{c},{n}x{h}x{w},fmt={fmt}]", p.reshape(-1, 16), xf @ wm, xf.abs() @ wm.abs(), k)
    assert bool(torch.isnan(pbuf[..., 16:]).all()), "wrote past the 16 taps"
    bias = randn(1, g=g)
    xn = xd.permute(0, 3, 1, 2)
    for pad in (0, 1, 2):
        mag = F.conv2d(xn.abs(), wt.double().abs(), None, 1, pad)
        for b in (bias, None):
            oh, ow = h + 2 * pad - 3, w + 2 * pad - 3
            ybuf, y = pitched(n, oh, ow, 1, 1, NAN)
            ops.tap_sum_fwd(p, 4, pad, b, y)
            torch.cuda.synchronize()
            ref = F.conv2d(xn, wt.double(), None if b is None else b.double(), 1, pad)
            scale = mag + (0.0 if b is None else b.double().abs())
            bounded(f"tap_sum[{c},{n}x{h}x{w},pad={pad},bias={b is not None}]", y, nhwc(ref), nhwc(scale), k + 17)
            assert bool(torch.isnan(ybuf[..., 1]).all())


def test_to_one_fwd_refuses_1544_channels():
    c = 1544
    x = ops.Planes(1, 4, 4, c + 8, dev(), c=c)
    refused(lambda: ops.to_one_fwd(x, torch.zeros(1, c, 4, 4, device=dev()), torch.zeros(1, 4, 4, 16, device=dev())))


def wgrad_k(npix, c):
    """to_one_wgrad: a thread's chain over its block's pixel rows, the row reduction, the block sums, the += ."""
    blocks = max(1, min(npix // 256, SMS * 4))
    per = (npix + blocks - 1) // blocks
    rows = max(1, 256 // (c // 4))
    return math.ceil(per / rows) + rows + blocks + 3, blocks


def to_one_wgrad_call(x, c, dy, with_lo, pad, dw, slots=None, cap=None):
    args = (x.hi_ptr, x.lo_ptr, x.pitch, x.fmt, x.n, x.h, x.w, c, dy.hi_ptr, dy.lo_ptr if with_lo else None, dy.pitch,
            dy.fmt, 4, pad, dw.data_ptr())
    L = _lib.load()
    if slots is None:
        _lib.check(L.sn_to_one_wgrad(*args, _stream()))
    else:
        _lib.check(L.sn_to_one_wgrad_det(*args, slots.data_ptr(), slots.numel() if cap is None else cap, _stream()))


WG_SHAPES = {"small": (1, 9, 13),      # 117 pixels: one block
             "mid": (3, 37, 41),       # 4551 pixels over 17 blocks of 268 (the last one shorter)
             "big": (2, 261, 263)}     # 137286 pixels > 528 x 256: 528 blocks of 261, the last ones empty
WG_CASES = ([(c, s, 1, F16, True) for c in (4, 12, 64, 192, 512, 1024) for s in WG_SHAPES] +
            [(64, "small", 0, BF16, False), (192, "mid", 2, BF16, True), (12, "mid", 0, F16, False),
             (1024, "mid", 2, BF16, False), (4, "big", 2, BF16, False), (512, "big", 0, F16, False)])


@pytest.mark.parametrize("c,shape,pad,fmt,with_lo", WG_CASES)
def test_to_one_wgrad(c, shape, pad, fmt, with_lo):
    """Block (C/4, 256/(C/4)): C = 4 -> 1 x 256, 12 -> 3 x 85, 192 -> 48 x 5, 1024 -> 256 x 1 (no row reduction)."""
    n, h, w = WG_SHAPES[shape]
    g = gen(c + h + pad)
    pitch = (c + 16 + 7) // 8 * 8
    x, xd = split_planes(randn(n, h, w, c, g=g), fmt, pitch, 8)
    oh, ow = h + 2 * pad - 3, w + 2 * pad - 3
    dy, dyd = grad_planes(n, oh, ow, g)
    if not with_lo:
        dyd = dy.hi[..., 0].float().double()          # bf16 hi words alone
    dp = tap_grads(dyd, h, w, pad).reshape(-1, 16)
    xf = xd.reshape(-1, c)
    npix = n * h * w
    dw0 = randn(1, c, 4, 4, g=g) * npix ** 0.5        # dw += : a gradient of the same magnitude already there
    ref = dw0.double().reshape(c, 16) + xf.T @ dp
    scale = dw0.double().abs().reshape(c, 16) + xf.abs().T @ dp.abs()
    k, blocks = wgrad_k(npix, c)
    slots = torch.empty(blocks * c * 16, dtype=torch.float32, device=dev())
    outs = []
    for det in (False, True, True):
        dw = dw0.clone()
        to_one_wgrad_call(x, c, dy, with_lo, pad, dw, slots if det else None)
        torch.cuda.synchronize()
        bounded(f"to_one_wgrad[{c},{n}x{h}x{w},pad={pad},fmt={fmt},lo={with_lo},{'det' if det else 'atomic'}]",
                dw.reshape(c, 16), ref, scale, k)
        outs.append(dw)
    assert torch.equal(outs[1].view(torch.int32), outs[2].view(torch.int32)), "to_one_wgrad_det did not repeat"


def test_to_one_wgrad_refusals():
    g = gen(1028)
    x = ops.Planes(1, 8, 8, 1032, dev(), c=1028)
    dy, _ = grad_planes(1, 7, 7, g)
    refused(lambda: to_one_wgrad_call(x, 1028, dy, True, 1, torch.zeros(1, 1028, 4, 4, device=dev())))
    x, _ = split_planes(randn(2, 40, 40, 64, g=g), F16, 64, 0)
    dy, _ = grad_planes(2, 39, 39, g)
    _, blocks = wgrad_k(2 * 40 * 40, 64)
    dw = torch.zeros(1, 64, 4, 4, device=dev())
    slots = torch.empty(blocks * 64 * 16, dtype=torch.float32, device=dev())
    refused(lambda: to_one_wgrad_call(x, 64, dy, True, 1, dw, slots, blocks * 64 * 16 - 1))


# (c, n, h, w, pad): c / 4 = 9 and 25 channel quads (a partial pass of the 32 lanes), more than the 1056 x 8 pixels
# one pass of the capped grid covers, and the training shape
DG_CASES = [(36, 2, 37, 29, 0), (36, 3, 61, 59, 2), (100, 2, 37, 29, 2), (100, 3, 61, 59, 0), (512, 16, 63, 63, 1)]


@pytest.mark.parametrize("c,n,h,w,pad", DG_CASES)
def test_to_one_dgrad(c, n, h, w, pad):
    g = gen(c + h + pad)
    wt = logits_weight(c, g)
    dy, dyd = grad_planes(n, h + 2 * pad - 3, w + 2 * pad - 3, g)
    dp = tap_grads(dyd, h, w, pad).reshape(-1, 16)
    wm = wt.double().reshape(c, 16)
    dxb = torch.full((n, h, w, c + 8), NAN, device=dev())
    dx = dxb[..., 4:4 + c]
    ops.to_one_dgrad(dy, wt, pad, dx)
    torch.cuda.synchronize()
    bounded(f"to_one_dgrad[{c},{n}x{h}x{w},pad={pad}]", dx.reshape(-1, c), dp @ wm.T, dp.abs() @ wm.abs().T, 18)
    assert bool(torch.isnan(dxb[..., :4]).all()) and bool(torch.isnan(dxb[..., 4 + c:]).all()), "wrote outside dx"


@pytest.mark.parametrize("det", [False, True])
def test_to_one_layer_training_shape(det):
    """ToOneConvLayer on the 512 x 512 discriminator's logits at batch 16 (63 x 63 x 512 -> 62 x 62): forward, dx,
    dw and db against fp64 from the decoded planes, with and without the deterministic workspace."""
    n, c, h, w = 16, 512, 63, 63
    g = gen(99 + det)
    x, xd = split_planes(randn(n, h, w, c, g=g), F16, c, 0)
    wt = logits_weight(c, g)
    bias = randn(1, g=g)
    layer = ToOneConvLayer("conv4s1", wt, bias, x, nsplit=3, name="logits",
                           det_ws=ops.DetWorkspace(dev()) if det else None)
    y = torch.full((n, h - 1, w - 1, 1), NAN, device=dev())
    layer.bind_forward(y)
    dy, dyd = grad_planes(n, h - 1, w - 1, g)
    dx = torch.full((n, h, w, c), NAN, device=dev())
    wg = torch.zeros(1, c, 4, 4, device=dev())
    bg = torch.full((1,), NAN, device=dev())
    layer.bind_backward(dy, dx, wg, bg)
    layer.pack()
    layer.forward()
    layer.backward()
    torch.cuda.synchronize()
    tag = f"to_one_layer[{n}x{h}x{w}x{c},{'det' if det else 'atomic'}]"
    xn = xd.permute(0, 3, 1, 2)
    wd = wt.double()
    ref = F.conv2d(xn, wd, bias.double(), 1, 1)
    scale = F.conv2d(xn.abs(), wd.abs(), bias.double().abs(), 1, 1)
    bounded(tag + " y", y, nhwc(ref), nhwc(scale), fwd_k(c) + 17)
    dp = tap_grads(dyd, h, w, 1).reshape(-1, 16)
    wm = wd.reshape(c, 16)
    bounded(tag + " dx", dx.reshape(-1, c), dp @ wm.T, dp.abs() @ wm.abs().T, 18)
    xf = xd.reshape(-1, c)
    bounded(tag + " dw", wg.reshape(c, 16), xf.T @ dp, xf.abs().T @ dp.abs(), wgrad_k(n * h * w, c)[0])
    # bias_grad: fp32 runs of 64 pixels, then fp64 sums, an fp32 staging and the final cast
    bounded(tag + " db", bg, dyd.sum().reshape(1), dyd.abs().sum().reshape(1), 68)
