"""TEST INFRASTRUCTURE ONLY — CPU emulator of the two generic contractions of libswapnet_b200
(tap GEMM / wgrad GEMM, csrc/gemm_tc.cu) plus torch restatements of the weight packers
(csrc/elementwise.cu pack_weights_multi / pack_head_weights / fold_head_wgrad).

Used by tests/ to (a) prove on the CPU that swapnet_b200/lowering.py maps every reference conv
layer (modules/layers.py:15,31,131-138; swapnet_modules.py:85-90; discriminators.py:111-131)
and its autograd onto those contractions exactly, and (b) check the CUDA kernels against the
same spec on the GPU: the single-pass (nsplit = 1) GEMMs are held to the fp64 contraction of the
16-bit operands they read, computed here on the device (tests/test_kernels_gpu.py model_forward /
model_dgrad / model_wgrad, used by test_conv_forward, test_conv_backward,
test_conv_baseline_shapes_fwd_bwd and test_fused_instance_norm_statistics; by
tests/test_gemm_edges_gpu.py and tests/test_deterministic_gpu.py::test_wgrad_plan_repeats_bit_identically;
and directly by tests/test_single_pass_gemm_gpu.py).  Nothing under swapnet_b200/ imports this file.
"""
from __future__ import annotations

import torch

from swapnet_b200 import lowering as L


def gather_patch(A: torch.Tensor, parity: bool, m_h: int, m_w: int, tap: L.Tap, pitch: int,
                 c_base: int, k: int) -> torch.Tensor:
    """A: [N, H, W, pitch] dense.  Returns [N, m_h, m_w, k] with zero for out-of-range pixels."""
    N, H, W, _ = A.shape
    out = A.new_zeros(N, m_h, m_w, k)
    hs = torch.arange(m_h, device=A.device) + tap.dh
    ws = torch.arange(m_w, device=A.device) + tap.dw
    if parity:
        vh = (hs >= 0) & (hs < H // 2)
        vw = (ws >= 0) & (ws < W // 2)
        sh = 2 * hs + tap.hp
        sw = 2 * ws + tap.pw
    else:
        vh = (hs >= 0) & (hs < H)
        vw = (ws >= 0) & (ws < W)
        sh, sw = hs, ws
    hi = torch.nonzero(vh).flatten()
    wi = torch.nonzero(vw).flatten()
    if hi.numel() == 0 or wi.numel() == 0:
        return out
    src = A[:, sh[hi]][:, :, sw[wi]][..., c_base:c_base + k]
    out[:, hi[:, None], wi[None, :]] = src
    return out


def emul_tap_gemm(A: torch.Tensor, spec: L.GemmSpec, Wp: torch.Tensor, k_pad: int, n_valid: int,
                  out: torch.Tensor, c_base: int = 0, bias=None) -> None:
    """A [N,H,W,pitch] fp32/fp64, Wp [rows, ntaps*k_pad]; writes out[N, OH, OW, >=n_valid] at the
    strided positions of the spec."""
    N = A.shape[0]
    acc = A.new_zeros(N, spec.m_h, spec.m_w, n_valid)
    for tap in spec.taps:
        patch = gather_patch(A, spec.parity, spec.m_h, spec.m_w, tap, A.shape[3], c_base, k_pad)
        wk = Wp[:n_valid, tap.kb * k_pad:(tap.kb + 1) * k_pad]
        acc += patch @ wk.T
    if bias is not None:
        acc += bias[:n_valid]
    mh, mw = spec.out_mul
    oh, ow = spec.out_off
    out[:, oh::mh, ow::mw, :n_valid][:, :spec.m_h, :spec.m_w] = acc


def emul_wgrad(X: torch.Tensor, Y: torch.Tensor, spec: L.WgradSpec, cx: int, cy: int,
               x_base: int = 0, y_base: int = 0) -> torch.Tensor:
    """-> G [ntaps, cx, cy]"""
    G = X.new_zeros(len(spec.xtaps), cx, cy)
    for t, (xt, yt) in enumerate(zip(spec.xtaps, spec.ytaps)):
        xp = gather_patch(X, spec.x_parity, spec.m_h, spec.m_w, xt, X.shape[3], x_base, cx)
        yp = gather_patch(Y, spec.y_parity, spec.m_h, spec.m_w, yt, Y.shape[3], y_base, cy)
        G[t] = xp.reshape(-1, cx).T @ yp.reshape(-1, cy)
    return G


# ---- packers (restating the CUDA packers) ---------------------------------------------------
def pack_weights_ref(weight: torch.Tensor, kind: str, dgrad: bool, k_pad: int) -> torch.Tensor:
    """torch-layout weight -> [rows, taps*k_pad] (fp32/fp64, no bf16 split)."""
    if kind == "convT4s2":
        cin, cout = weight.shape[0], weight.shape[1]
    else:
        cout, cin = weight.shape[0], weight.shape[1]
    s_row, s_k, rows, k_real = L.pack_strides(kind, cin, cout, dgrad)
    t = L.ntaps(kind)
    flat = weight.reshape(-1)
    r = torch.arange(rows)[:, None, None]
    tt = torch.arange(t)[None, :, None]
    k = torch.arange(k_real)[None, None, :]
    vals = flat[r * s_row + k * s_k + tt]
    out = weight.new_zeros(rows, t, k_pad)
    out[:, L.pack_slots(kind, dgrad), :k_real] = vals      # packed slot of each torch tap
    return out.reshape(rows, t * k_pad)


def _head_taps_of(par: int, e: int):
    if par == 0:
        return [2 * e, 2 * e + 1]
    return [[0], [1, 2], [3]][e]


def head_eff_weights(weight: torch.Tensor) -> torch.Tensor:
    """OIHW [cout, cin, 4, 4] -> effective taps [cout, 25, cin] (phase-major, (ey, ex) row-major)."""
    cout, cin = weight.shape[:2]
    eff = weight.new_zeros(cout, 25, cin)
    for py in range(2):
        for px in range(2):
            for ey in range(L.head_neff(py)):
                for ex in range(L.head_neff(px)):
                    te = L.HEAD_PHASE_OFF[2 * py + px] + ey * L.head_neff(px) + ex
                    for ky in _head_taps_of(py, ey):
                        for kx in _head_taps_of(px, ex):
                            eff[:, te] += weight[:, :, ky, kx]
    return eff


def pack_head_ref(weight: torch.Tensor, rows_pad: int, k_pad: int, dgrad: bool):
    """fwd: list of 4 per-phase matrices [rows_pad, ntaps_p*k_pad]; dgrad: [cin, 25*k_pad]."""
    cout, cin = weight.shape[:2]
    eff = head_eff_weights(weight)
    if dgrad:
        out = weight.new_zeros(cin, 25, k_pad)
        out[:, :, :cout] = eff.permute(2, 1, 0)
        return out.reshape(cin, 25 * k_pad)
    mats = []
    for p in range(4):
        nt = L.head_neff(p >> 1) * L.head_neff(p & 1)
        m = weight.new_zeros(rows_pad, nt, k_pad)
        m[:cout, :, :cin] = eff[:, L.HEAD_PHASE_OFF[p]:L.HEAD_PHASE_OFF[p] + nt]
        mats.append(m.reshape(rows_pad, nt * k_pad))
    return mats


def fold_head_wgrad_ref(geff: torch.Tensor) -> torch.Tensor:
    """[cout, 25, cin] -> dW [cout, cin, 4, 4]"""
    cout, _, cin = geff.shape
    dw = geff.new_zeros(cout, cin, 4, 4)
    for py in range(2):
        for px in range(2):
            for ey in range(L.head_neff(py)):
                for ex in range(L.head_neff(px)):
                    te = L.HEAD_PHASE_OFF[2 * py + px] + ey * L.head_neff(px) + ex
                    for ky in _head_taps_of(py, ey):
                        for kx in _head_taps_of(px, ex):
                            dw[:, :, ky, kx] += geff[:, te]
    return dw
