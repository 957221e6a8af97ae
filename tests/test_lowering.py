"""CPU proof that swapnet_b200/lowering.py maps each reference conv layer, its input gradient
and its weight gradient onto the generic tap-GEMM / wgrad-GEMM contractions exactly (fp64)."""
import pytest
import torch
import torch.nn.functional as F

from oracle import emulate as E
from swapnet_b200 import lowering as L

torch.manual_seed(0)


def ref_forward(kind, x, w, b=None):
    """x NCHW fp64 -> NCHW, with torch's own ops exactly as the reference modules call them."""
    if kind == "conv4s2":
        return F.conv2d(x, w, b, 2, 1)
    if kind == "convT4s2":
        return F.conv_transpose2d(x, w, b, 2, 1)
    if kind == "conv3r":
        return F.conv2d(F.pad(x, (1, 1, 1, 1), mode="reflect"), w, b)
    if kind == "conv4s1":
        return F.conv2d(x, w, b, 1, 1)
    if kind == "conv3z":   # torchvision vgg16.features conv (perceptual.py:26)
        return F.conv2d(x, w, b, 1, 1)
    if kind == "head":
        u = F.interpolate(x, scale_factor=2)  # nn.Upsample default = nearest
        u = F.pad(u, (1, 0, 1, 0))            # ZeroPad2d((1,0,1,0))
        return F.conv2d(u, w, b, 1, 1)
    raise ValueError(kind)


CASES = [
    ("conv4s2", 3, 5, 8, 8), ("conv4s2", 4, 6, 12, 16),
    ("convT4s2", 5, 3, 4, 4), ("convT4s2", 6, 4, 6, 8),
    ("conv3r", 4, 5, 6, 6), ("conv3r", 3, 3, 8, 10),
    ("conv4s1", 4, 3, 7, 9), ("conv4s1", 5, 1, 8, 8),
    ("head", 6, 5, 4, 4), ("head", 4, 3, 6, 8),
    ("conv3z", 4, 5, 6, 6), ("conv3z", 3, 2, 8, 10),
]


def nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def to_planes(x_nchw, kind, pitch):
    """layer input NCHW -> dense A [N, H', W', pitch] as the planes buffer would hold it."""
    if kind == "conv3r":
        x_nchw = F.pad(x_nchw, (1, 1, 1, 1), mode="reflect")
    a = nhwc(x_nchw)
    out = a.new_zeros(*a.shape[:3], pitch)
    out[..., : a.shape[3]] = a
    return out


@pytest.mark.parametrize("kind,cin,cout,h,w", CASES)
def test_forward_dgrad_wgrad(kind, cin, cout, h, w):
    N = 2
    k_pad = 8  # emulator has no 64-alignment requirement
    x = torch.randn(N, cin, h, w, dtype=torch.float64, requires_grad=True)
    wshape = (cin, cout, 4, 4) if kind == "convT4s2" else (cout, cin, 3 if kind == "conv3r" else 4,) * 1
    if kind != "convT4s2":
        k = 3 if kind in ("conv3r", "conv3z") else 4
        wshape = (cout, cin, k, k)
    wt = torch.randn(*wshape, dtype=torch.float64, requires_grad=True)
    bias = torch.randn(cout, dtype=torch.float64)
    y = ref_forward(kind, x, wt, bias)
    gy = torch.randn_like(y)
    gx, gw = torch.autograd.grad(y, (x, wt), gy)
    oh, ow = L.out_hw(kind, h, w)
    assert y.shape[2:] == (oh, ow)

    # ---- forward ----
    A = to_planes(x.detach(), kind, pitch=k_pad + 3)
    out = torch.zeros(N, oh, ow, cout, dtype=torch.float64)
    specs = L.forward_specs(kind, h, w)
    if kind == "head":
        mats = E.pack_head_ref(wt.detach(), rows_pad=cout + 2, k_pad=k_pad, dgrad=False)
    else:
        Wp = E.pack_weights_ref(wt.detach(), kind, False, k_pad)
    for s in specs:
        assert s.a_hw == tuple(A.shape[1:3])
        E.emul_tap_gemm(A, s, mats[s.w_phase] if kind == "head" else Wp, k_pad, cout, out, bias=bias)
    torch.testing.assert_close(out, nhwc(y.detach()), rtol=1e-10, atol=1e-10)

    # ---- dgrad ----
    DY = torch.zeros(N, oh, ow, k_pad + 5, dtype=torch.float64)
    DY[..., :cout] = nhwc(gy)
    if kind == "head":
        Wd = E.pack_head_ref(wt.detach(), 0, k_pad, dgrad=True)
    else:
        Wd = E.pack_weights_ref(wt.detach(), kind, True, k_pad)
    ih, iw = (h + 2, w + 2) if kind == "conv3r" else (h, w)
    dx = torch.zeros(N, ih, iw, cin, dtype=torch.float64)
    for s in L.dgrad_specs(kind, h, w):
        assert s.a_hw == (oh, ow)
        E.emul_tap_gemm(DY, s, Wd, k_pad, cin, dx)
    if kind == "conv3r":  # fold the reflect padding back (adjoint of ReflectionPad2d(1))
        xp = F.pad(x.detach(), (1, 1, 1, 1), mode="reflect").requires_grad_()
        ref = torch.autograd.grad(F.conv2d(xp, wt.detach()), xp, gy)[0]
        torch.testing.assert_close(dx, nhwc(ref), rtol=1e-10, atol=1e-10)
    else:
        torch.testing.assert_close(dx, nhwc(gx), rtol=1e-10, atol=1e-10)

    # ---- wgrad ----
    (ws,) = L.wgrad_specs(kind, h, w)
    Xd, Yd = (DY, A) if ws.x_is == "dy" else (A, DY)
    cx, cy = (cout, cin) if ws.x_is == "dy" else (cin, cout)
    G = E.emul_wgrad(Xd, Yd, ws, cx, cy)  # [taps, cx, cy]
    s_row, s_col = L.wgrad_out_strides(kind, cin, cout, ws.x_is == "dy")
    if kind == "head":
        flat = torch.zeros(cout * 25 * cin, dtype=torch.float64)
        tap_off = [t * cin for t in ws.tap_ids]
    else:
        flat = torch.zeros(wt.numel(), dtype=torch.float64)
        tap_off = list(ws.tap_ids)
    r = torch.arange(cx)[:, None] * s_row
    c = torch.arange(cy)[None, :] * s_col
    for t, off in enumerate(tap_off):
        flat.index_add_(0, (r + c + off).reshape(-1), G[t].reshape(-1))
    if kind == "head":
        got = E.fold_head_wgrad_ref(flat.reshape(cout, 25, cin))
    else:
        got = flat.reshape(wt.shape)
    torch.testing.assert_close(got, gw, rtol=1e-9, atol=1e-9)


def test_to_one_factorisation():
    """layers.ToOneConvLayer: Conv2d(cin, 1, 4, 1, 1) = per-tap product image P (a 1-tap GEMM) + shifted sums, and
    its adjoint (dP = shifted dy; dW, dx = 1-tap contractions with dP) — fp64 proof against torch."""
    N, cin, h, w = 2, 5, 7, 9
    x = torch.randn(N, cin, h, w, dtype=torch.float64, requires_grad=True)
    wt = torch.randn(1, cin, 4, 4, dtype=torch.float64, requires_grad=True)
    b = torch.randn(1, dtype=torch.float64)
    y = F.conv2d(x, wt, b, 1, 1)
    gy = torch.randn_like(y)
    gx, gw = torch.autograd.grad(y, (x, wt), gy)
    X = nhwc(x.detach())                                           # [N,h,w,cin]
    Wt = wt.detach().reshape(cin, 16)                              # [c][t]
    P = X @ Wt                                                     # [N,h,w,16]: one 1-tap GEMM
    out = torch.zeros(N, h - 1, w - 1, dtype=torch.float64)
    dP = torch.zeros(N, h, w, 16, dtype=torch.float64)
    GY = gy[:, 0]
    for kh in range(4):
        for kw in range(4):
            t = kh * 4 + kw
            for oh in range(h - 1):
                ih = oh + kh - 1
                if not 0 <= ih < h:
                    continue
                for ow in range(w - 1):
                    iw = ow + kw - 1
                    if 0 <= iw < w:
                        out[:, oh, ow] += P[:, ih, iw, t]          # sn_tap_sum_fwd
                        dP[:, ih, iw, t] = GY[:, oh, ow]           # dP = dy shifted by tap t
    torch.testing.assert_close(out + b, y.detach()[:, 0], rtol=1e-12, atol=1e-12)
    dW = torch.einsum("nhwc,nhwt->ct", X, dP).reshape(1, cin, 4, 4)
    dX = dP @ Wt.t()
    torch.testing.assert_close(dW, gw, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(dX, nhwc(gx), rtol=1e-12, atol=1e-12)


def test_merged_parity_view_addresses():
    """gemm_tc.cu sn_make_act_map(parity, plane_stride): the stride-2 'parity view' with BOTH parities folded into
    the channel coordinate, c' = hp*W*pitch + pw*pitch + c over dims (c', w/2, h/2, n), must address element
    (n, 2*h2 + hp, 2*w2 + pw, c) of the NHWC tensor."""
    import itertools

    N, H, W, pitch = 2, 6, 8, 16
    e = 1                                             # element units
    s_w2, s_h2, s_n = 2 * pitch * e, 2 * W * pitch * e, H * W * pitch * e
    for n, h2, w2, hp, pw, c in itertools.product(range(N), range(H // 2), range(W // 2), range(2), range(2), (0, 5, 15)):
        cprime = hp * W * pitch + pw * pitch + c
        assert cprime < (W + 1) * pitch + pitch       # inside dims[0] of the map
        addr = cprime + w2 * s_w2 + h2 * s_h2 + n * s_n
        want = ((n * H + 2 * h2 + hp) * W + 2 * w2 + pw) * pitch + c
        assert addr == want


def test_head_stacked_phases_equal_the_reference_head():
    """The head forward as ONE 9-tap contraction with the 4 output-parity phases stacked along N (lowering.
    head_stacked_spec + the stacked weight layout of csrc pack_head_stacked_kernel, restated here) reproduces
    Upsample(2) + ZeroPad2d((1,0,1,0)) + Conv2d(k4, p1) of swapnet_modules.py:85-90."""
    import torch
    import torch.nn.functional as F

    from oracle import emulate as EM
    from swapnet_b200 import lowering as L

    g = torch.Generator().manual_seed(3)
    n, cin, cout, h, w = 2, 8, 5, 6, 7
    x = torch.randn(n, cin, h, w, generator=g, dtype=torch.float64)
    wt = torch.randn(cout, cin, 4, 4, generator=g, dtype=torch.float64)
    ref = F.conv2d(F.pad(F.interpolate(x, scale_factor=2), (1, 0, 1, 0)), wt, None, 1, 1)
    eff = EM.head_eff_weights(wt)                     # [cout, 25, cin], phase-major effective taps
    slot, k_pad = L.HEAD_SLOT, cin
    Wp = torch.zeros(4 * slot, 9, k_pad, dtype=torch.float64)
    for p in range(4):
        py, px = p >> 1, p & 1
        for ey in range(L.head_neff(py)):
            for ex in range(L.head_neff(px)):
                te = L.HEAD_PHASE_OFF[p] + ey * L.head_neff(px) + ex
                Wp[p * slot:p * slot + cout, ey * 3 + ex] = eff[:, te]
    spec = L.head_stacked_spec(h, w)
    A = x.permute(0, 2, 3, 1).contiguous()
    acc = torch.zeros(n, h, w, 4 * slot, dtype=torch.float64)
    plain = L.GemmSpec(False, h, w, spec.taps, (1, 1), (0, 0), a_hw=(h, w))
    EM.emul_tap_gemm(A, plain, Wp.reshape(4 * slot, 9 * k_pad), k_pad, 4 * slot, acc)
    out = torch.zeros(n, 2 * h, 2 * w, cout, dtype=torch.float64)
    for p in range(4):
        out[:, (p >> 1)::2, (p & 1)::2] = acc[..., p * slot:p * slot + cout]
    assert torch.allclose(out.permute(0, 3, 1, 2), ref, atol=1e-12)
