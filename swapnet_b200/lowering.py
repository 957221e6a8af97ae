"""Lowering of the SwapNet conv layers onto the two generic tensor-core contractions of
libswapnet_b200 (tap GEMM / wgrad GEMM, see csrc/gemm_tc.cu).

Pure shape/index arithmetic — no torch, no CUDA — so that every table can be checked on the
CPU against torch's own conv ops (tests/test_lowering.py runs an emulator of the two generic
contractions over these specs).

Layer kinds (reference call sites):
  conv4s2   Conv2d(k4, s2, p1)              layers.py:15, pix2pix_modules.py:217, discriminators.py:111-121
  convT4s2  ConvTranspose2d(k4, s2, p1)     layers.py:31, pix2pix_modules.py:226-247
  conv3r    ReflectionPad2d(1)+Conv2d(k3)   layers.py:130-138
  conv4s1   Conv2d(k4, s1, p1)              discriminators.py:124-131
  conv3z    Conv2d(k3, s1, p1) zero padding  torchvision vgg16.features (modules/losses/perceptual.py:26-42)
  head      Upsample(2)+ZeroPad2d((1,0,1,0))+Conv2d(k4,p1)   swapnet_modules.py:85-90

Each kind provides forward, dgrad (gradient w.r.t. the conv input) and wgrad specs.  A spec is
a list of `GemmSpec`/`WgradSpec`, one per launch (stride-2 transposed structures and the head
split into 4 output-parity phases).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Tuple

KINDS = ("conv4s2", "convT4s2", "conv3r", "conv4s1", "head", "conv3z")

# (c_off_is_pw, kb_off, dw, dh, hp): c_off is given as (pw, cbase) and resolved against the
# operand pitch when the descriptor is bound.
@dataclass
class Tap:
    pw: int      # parity view: w parity (c' offset = pw * pitch); 0 otherwise
    kb: int      # tap index inside the packed weight matrix (K offset = kb * k_pad)
    dw: int
    dh: int
    hp: int = 0


@dataclass
class GemmSpec:
    """One tap-GEMM launch.  Rows = (n, h, w) over m_hw; A is read through `parity` view."""
    parity: bool
    m_h: int
    m_w: int
    taps: List[Tap]
    out_mul: Tuple[int, int] = (1, 1)   # (mul_h, mul_w)
    out_off: Tuple[int, int] = (0, 0)   # (off_h, off_w)
    w_phase: int = 0                    # head only: which per-phase weight matrix
    a_hw: Tuple[int, int] = (0, 0)      # logical H, W of the A operand


@dataclass
class WgradSpec:
    """One wgrad launch: G[row, col, tap] += sum_pixels X[pix + xtap] * Y[pix + ytap]."""
    m_h: int
    m_w: int
    x_parity: bool
    y_parity: bool
    xtaps: List[Tap]
    ytaps: List[Tap]
    # what X / Y are: "dy" or "in"
    x_is: str = "dy"
    # index of the tap in the weight layout for each launch tap (for tap_off)
    tap_ids: List[int] = field(default_factory=list)


def _phase_taps():
    """The 4 output-parity phases of a stride-2 transposed structure (ConvTranspose2d forward, Conv2d
    input-gradient): per phase the (kh, dh) x (kw, dw) pairs.  ho = 2*hi - 1 + kh."""
    out = []
    for py in range(2):
        khs = [(1, 0), (3, -1)] if py == 0 else [(0, 1), (2, 0)]
        for px in range(2):
            kws = [(1, 0), (3, -1)] if px == 0 else [(0, 1), (2, 0)]
            out.append(((py, px), [(kh, dh, kw, dw) for kh, dh in khs for kw, dw in kws]))
    return out


def phase_major_slots() -> List[int]:
    """slot_of_tap[kh*4+kw] for the packed weights of the 4-phase structures: the 4 taps of a phase are
    contiguous in K (needed when 64/k narrow taps share one weight box), phases in (py, px) order."""
    slot = [0] * 16
    for p, (_, taps) in enumerate(_phase_taps()):
        for j, (kh, _, kw, _) in enumerate(taps):
            slot[kh * 4 + kw] = p * 4 + j
    return slot


def pack_slots(kind: str, dgrad: bool) -> List[int]:
    """Packed tap slot of each torch tap for sn_pack_weights_multi (identity except for the 4-phase structures)."""
    if (kind == "convT4s2" and not dgrad) or (kind == "conv4s2" and dgrad):
        return phase_major_slots()
    return list(range(ntaps(kind)))


def _s2_tap(k: int) -> Tuple[int, int]:
    """stride-2, pad-1 gather: source index 2*o - 1 + k  ->  (delta on the half grid, parity)."""
    return ((k - 1) >> 1, (k - 1) & 1)


def out_hw(kind: str, h: int, w: int) -> Tuple[int, int]:
    if kind == "conv4s2":
        return h // 2, w // 2
    if kind == "convT4s2":
        return 2 * h, 2 * w
    if kind in ("conv3r", "conv3z"):
        return h, w
    if kind == "conv4s1":
        return h - 1, w - 1
    if kind == "head":
        return 2 * h, 2 * w
    raise ValueError(kind)


def ntaps(kind: str) -> int:
    return {"conv4s2": 16, "convT4s2": 16, "conv3r": 9, "conv4s1": 16, "head": 25, "conv3z": 9}[kind]


HEAD_PHASE_OFF = (0, 4, 10, 16)


def head_neff(par: int) -> int:
    return 3 if par else 2


# ------------------------------------------------------------------------------------------
# forward
# ------------------------------------------------------------------------------------------
def forward_specs(kind: str, h: int, w: int) -> List[GemmSpec]:
    """h, w = spatial size of the layer INPUT (un-padded)."""
    if kind == "conv4s2":
        taps = []
        for kh in range(4):
            dh, hp = _s2_tap(kh)
            for kw in range(4):
                dw, pw = _s2_tap(kw)
                taps.append(Tap(pw, kh * 4 + kw, dw, dh, hp))
        return [GemmSpec(True, h // 2, w // 2, taps, a_hw=(h, w))]
    if kind == "convT4s2":
        slot = phase_major_slots()
        return [GemmSpec(False, h, w, [Tap(0, slot[kh * 4 + kw], dw, dh) for kh, dh, kw, dw in taps], (2, 2),
                         (py, px), a_hw=(h, w)) for (py, px), taps in _phase_taps()]
    if kind == "conv3r":  # A = reflect-padded planes [h+2, w+2]
        taps = [Tap(0, kh * 3 + kw, kw, kh) for kh in range(3) for kw in range(3)]
        return [GemmSpec(False, h, w, taps, a_hw=(h + 2, w + 2))]
    if kind == "conv4s1":
        taps = [Tap(0, kh * 4 + kw, kw - 1, kh - 1) for kh in range(4) for kw in range(4)]
        return [GemmSpec(False, h - 1, w - 1, taps, a_hw=(h, w))]
    if kind == "conv3z":  # zero padding = TMA out-of-bounds fill
        taps = [Tap(0, kh * 3 + kw, kw - 1, kh - 1) for kh in range(3) for kw in range(3)]
        return [GemmSpec(False, h, w, taps, a_hw=(h, w))]
    if kind == "head":
        specs = []
        for py in range(2):
            for px in range(2):
                taps = []
                for ey in range(head_neff(py)):
                    for ex in range(head_neff(px)):
                        taps.append(Tap(0, ey * head_neff(px) + ex, ex - 1, ey - 1))
                specs.append(GemmSpec(False, h, w, taps, (2, 2), (py, px), w_phase=2 * py + px, a_hw=(h, w)))
        return specs
    raise ValueError(kind)


HEAD_SLOT = 24      # columns per output-parity phase in the stacked head GEMM (19 real + 5 zero): N = 4 * 24 = 96


def head_stacked_spec(h: int, w: int) -> GemmSpec:
    """The head forward as ONE 9-tap GEMM whose N columns are the 4 output-parity phases side by side: the union of
    the phases' effective taps is the 3x3 shift set {-1,0,1}^2 (parity 0 uses shifts -1, 0; parity 1 all three), so the
    input is read 9 times instead of 4+6+6+9 = 25.  Packed weights: ops.pack_head_stacked (zero where a phase has no
    tap at a shift)."""
    taps = [Tap(0, (sy + 1) * 3 + (sx + 1), sx, sy) for sy in (-1, 0, 1) for sx in (-1, 0, 1)]
    return GemmSpec(False, h, w, taps, (2, 2), (0, 0), a_hw=(h, w))


# ------------------------------------------------------------------------------------------
# dgrad: A = dy planes (spatial = layer OUTPUT size), result = gradient w.r.t. layer input
# ------------------------------------------------------------------------------------------
def dgrad_specs(kind: str, h: int, w: int) -> List[GemmSpec]:
    """h, w = spatial size of the layer INPUT (un-padded); dy has out_hw(kind, h, w)."""
    oh, ow = out_hw(kind, h, w)
    if kind == "conv4s2":  # transposed structure over the dy grid, 4 input-parity phases
        slot = phase_major_slots()
        return [GemmSpec(False, oh, ow, [Tap(0, slot[kh * 4 + kw], dw, dh) for kh, dh, kw, dw in taps], (2, 2),
                         (py, px), a_hw=(oh, ow)) for (py, px), taps in _phase_taps()]
    if kind == "convT4s2":  # strided conv of dy (dy is 2h x 2w)
        taps = []
        for kh in range(4):
            dh, hp = _s2_tap(kh)
            for kw in range(4):
                dw, pw = _s2_tap(kw)
                taps.append(Tap(pw, kh * 4 + kw, dw, dh, hp))
        return [GemmSpec(True, h, w, taps, a_hw=(oh, ow))]
    if kind == "conv3r":  # gradient w.r.t. the PADDED input [h+2, w+2]
        taps = [Tap(0, kh * 3 + kw, -kw, -kh) for kh in range(3) for kw in range(3)]
        return [GemmSpec(False, h + 2, w + 2, taps, a_hw=(oh, ow))]
    if kind == "conv4s1":
        taps = [Tap(0, kh * 4 + kw, 1 - kw, 1 - kh) for kh in range(4) for kw in range(4)]
        return [GemmSpec(False, h, w, taps, a_hw=(oh, ow))]
    if kind == "conv3z":
        taps = [Tap(0, kh * 3 + kw, 1 - kw, 1 - kh) for kh in range(3) for kw in range(3)]
        return [GemmSpec(False, h, w, taps, a_hw=(oh, ow))]
    if kind == "head":  # dy is 2h x 2w, read through the parity view
        taps = []
        for py in range(2):
            for px in range(2):
                for ey in range(head_neff(py)):
                    for ex in range(head_neff(px)):
                        te = HEAD_PHASE_OFF[2 * py + px] + ey * head_neff(px) + ex
                        taps.append(Tap(px, te, -(ex - 1), -(ey - 1), py))
        return [GemmSpec(True, h, w, taps, a_hw=(oh, ow))]
    raise ValueError(kind)


# ------------------------------------------------------------------------------------------
# wgrad
# ------------------------------------------------------------------------------------------
def wgrad_specs(kind: str, h: int, w: int) -> List[WgradSpec]:
    """One launch covers every tap (grid.y = tap).  Pixel grid and per-tap offsets:
    X is always the operand WITHOUT tap offsets of its own unless noted."""
    oh, ow = out_hw(kind, h, w)
    zero = Tap(0, 0, 0, 0, 0)
    if kind == "conv4s2":  # pixels = dy grid; in via parity view
        yt = []
        for kh in range(4):
            dh, hp = _s2_tap(kh)
            for kw in range(4):
                dw, pw = _s2_tap(kw)
                yt.append(Tap(pw, 0, dw, dh, hp))
        return [WgradSpec(oh, ow, False, True, [zero] * 16, yt, "dy", list(range(16)))]
    if kind == "convT4s2":  # pixels = input grid; dy via parity view
        yt = []
        for kh in range(4):
            dh, hp = _s2_tap(kh)
            for kw in range(4):
                dw, pw = _s2_tap(kw)
                yt.append(Tap(pw, 0, dw, dh, hp))
        return [WgradSpec(h, w, False, True, [zero] * 16, yt, "in", list(range(16)))]
    if kind == "conv3r":  # pixels = output grid; in = padded planes
        yt = [Tap(0, 0, kw, kh) for kh in range(3) for kw in range(3)]
        return [WgradSpec(h, w, False, False, [zero] * 9, yt, "dy", list(range(9)))]
    if kind == "conv4s1":
        yt = [Tap(0, 0, kw - 1, kh - 1) for kh in range(4) for kw in range(4)]
        return [WgradSpec(oh, ow, False, False, [zero] * 16, yt, "dy", list(range(16)))]
    if kind == "conv3z":
        yt = [Tap(0, 0, kw - 1, kh - 1) for kh in range(3) for kw in range(3)]
        return [WgradSpec(oh, ow, False, False, [zero] * 9, yt, "dy", list(range(9)))]
    if kind == "head":  # pixels = source grid; dy via parity view (x), in with eff-tap offsets (y)
        xt, yt, ids = [], [], []
        for py in range(2):
            for px in range(2):
                for ey in range(head_neff(py)):
                    for ex in range(head_neff(px)):
                        xt.append(Tap(px, 0, 0, 0, py))
                        yt.append(Tap(0, 0, ex - 1, ey - 1))
                        ids.append(HEAD_PHASE_OFF[2 * py + px] + ey * head_neff(px) + ex)
        return [WgradSpec(h, w, True, False, xt, yt, "dy", ids)]
    raise ValueError(kind)


# ------------------------------------------------------------------------------------------
# weight layouts.  torch layouts: conv OIHW [cout][cin][k][k]; convT IOHW [cin][cout][k][k].
# pack_weights_multi reads src[row*s_row + k*s_k + tap].
# ------------------------------------------------------------------------------------------
def pack_strides(kind: str, cin: int, cout: int, dgrad: bool) -> Tuple[int, int, int, int]:
    """-> (s_row, s_k, rows, k_real) for sn_pack_weights_multi (not for 'head')."""
    t = ntaps(kind)
    if kind == "convT4s2":
        if not dgrad:  # rows = co, k = ci
            return t, cout * t, cout, cin
        return cout * t, t, cin, cout  # rows = ci, k = co
    if not dgrad:  # OIHW, rows = co, k = ci
        return cin * t, t, cout, cin
    return t, cin * t, cin, cout


def wgrad_out_strides(kind: str, cin: int, cout: int, x_is_dy: bool) -> Tuple[int, int]:
    """(s_row, s_col) into the torch-layout gradient for X rows / Y cols; tap stride is 1."""
    t = ntaps(kind)
    if kind == "head":  # scratch geff [cout][25][cin]; tap_off = te * cin
        co_s, ci_s = 25 * cin, 1
    elif kind == "convT4s2":
        ci_s, co_s = cout * t, t
    else:
        co_s, ci_s = cin * t, t
    return (co_s, ci_s) if x_is_dy else (ci_s, co_s)


def pad64(c: int) -> int:
    return (c + 63) // 64 * 64


def padc(c: int) -> int:
    """Channel padding of an operand plane: 16 or 32 for narrow tensors (3/19/22-channel images,
    1/3/19-channel gradients: TMA rows of 32 / 64 bytes, SWIZZLE_32B / 64B), else a multiple of 64."""
    if c <= 16:
        return 16
    if c <= 32:
        return 32
    return pad64(c)


def pick_block_n(n_valid: int) -> int:
    """N tile of the tap GEMM: largest of 128/64/32/16 that does not over-pad small outputs."""
    if n_valid >= 128:
        return 128
    for b in (16, 32, 64, 128):
        if n_valid <= b:
            return b
    return 128
