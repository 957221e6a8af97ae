"""Python face of the C ABI: torch tensors in, kernel launches on torch's current stream out.

torch is used for device memory and streams only; every function here ends in a call into
libswapnet_b200.so and raises if that fails (no eager fallback).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Optional, Sequence, Tuple

import torch

from . import _lib
from . import lowering as L

from ._lib import (ACT_LRELU, ACT_NONE, ACT_RELU, ACT_TANH, FMT_BF16, FMT_F16, LAYOUT_LABEL_U8, LAYOUT_MASK_I32,
                   LAYOUT_NCHW, LAYOUT_NHWC, SnGradSrc, SnNormActBwdDesc, SnNormActDesc, SnTap, SnTapGemmDesc,
                   SnWgradDesc, check)

IN_EPS = 1e-5  # nn.InstanceNorm2d default (modules/__init__.py:67-69)


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


# ---------------------------------------------------------------------------------------------
# split-plane operand buffers
# ---------------------------------------------------------------------------------------------
class Planes:
    """A split-bf16 NHWC operand [n, h, w, c] living at channel offset `c_off` of a (possibly
    wider) buffer with `pitch` channels per pixel.  Padding channels stay zero forever."""

    def __init__(self, n: int, h: int, w: int, pitch: int, device, c: Optional[int] = None, c_off: int = 0,
                 hi: Optional[torch.Tensor] = None, lo: Optional[torch.Tensor] = None, fmt: int = FMT_F16,
                 dual: bool = False, twin: Optional["Planes"] = None):
        """fmt: FMT_F16 (activations: 22-bit split) or FMT_BF16 (gradients: fp32 range).  The storage
        dtype is bfloat16 either way — the planes are opaque 16-bit words to torch.
        dual=True also allocates a bf16-split twin of the same geometry (`self.twin`): forward GEMMs
        read the fp16 planes, the weight-gradient GEMM reads the twin (one MMA = one format)."""
        assert pitch % 8 == 0
        self.fmt = fmt
        self.twin = twin
        if dual and twin is None:
            self.twin = Planes(n, h, w, pitch, device, c, c_off, fmt=FMT_BF16)
        self.n, self.h, self.w, self.pitch = n, h, w, pitch
        self.c = pitch if c is None else c
        self.c_off = c_off
        if hi is None:
            # hi and lo live in ONE buffer, a fixed plane stride apart: the GEMM kernels then fetch both planes of
            # a tile with a single TMA box (extra box dimension of 2) — views (slice / batch_slice) keep the stride
            assert lo is None
            buf = torch.zeros(2, n, h, w, pitch, dtype=torch.bfloat16, device=device)
            hi, lo = buf[0], buf[1]
        self.hi, self.lo = hi, lo

    def slice(self, c_off: int, c: int) -> "Planes":
        assert c_off + c <= self.pitch
        return Planes(self.n, self.h, self.w, self.pitch, self.hi.device, c, self.c_off + c_off, self.hi, self.lo,
                      self.fmt, twin=None if self.twin is None else self.twin.slice(c_off, c))

    def batch_slice(self, n0: int, n: int) -> "Planes":
        return Planes(n, self.h, self.w, self.pitch, self.hi.device, self.c, self.c_off, self.hi[n0:n0 + n],
                      self.lo[n0:n0 + n], self.fmt, twin=None if self.twin is None else self.twin.batch_slice(n0, n))

    @property
    def hi_ptr(self) -> int:
        return self.hi.data_ptr() + 2 * self.c_off

    @property
    def lo_ptr(self) -> int:
        return self.lo.data_ptr() + 2 * self.c_off

    def dense(self) -> torch.Tensor:
        """fp32 reconstruction hi + lo of the logical [n,h,w,c] tensor (tests / debugging)."""
        s = slice(self.c_off, self.c_off + self.c)
        if self.fmt == FMT_F16:
            return self.hi[..., s].view(torch.float16).float() + self.lo[..., s].view(torch.float16).float()
        return self.hi[..., s].float() + self.lo[..., s].float()


class PackedWeights:
    """[rows][k_total] split 16-bit weight matrix (K contiguous), fp16-split with an exact
    power-of-two scale (`scale` = device (s, 1/s), set by a PackTable scale item)."""

    def __init__(self, rows: int, k_total: int, device, scale: Optional[torch.Tensor] = None, fmt: int = FMT_F16):
        self.rows, self.k_total = rows, k_total
        self.fmt = fmt
        # bf16-split packs (backward GEMMs) are unscaled; fp16-split packs carry the per-tensor 2^k
        self.scale = scale if (scale is not None and fmt == FMT_F16) else None
        buf = torch.zeros(2, rows, k_total, dtype=torch.bfloat16, device=device)   # one buffer: see Planes
        self.hi, self.lo = buf[0], buf[1]


class DetWorkspace:
    """Slot workspace of the deterministic reductions (the *_det entry points): each block stores its partial sums in a
    slot of its own and a second kernel adds the slots in index order.  Launches on one stream run one after the other
    and may share a workspace; launches that can overlap (the weight-gradient stream and the launching stream) each need
    their own.  It grows to the largest request and is sized by the first (eager) step: a CUDA-graph capture that
    would have to grow it raises."""

    def __init__(self, device):
        self.device = torch.device(device)
        self._buf: Optional[torch.Tensor] = None

    @property
    def nbytes(self) -> int:
        return 0 if self._buf is None else self._buf.numel() * self._buf.element_size()

    def get(self, elems: int, dtype=torch.float64) -> torch.Tensor:
        """A buffer of at least `elems` elements of dtype (float64 or float32) viewing the workspace."""
        nb = elems * torch.tensor([], dtype=dtype).element_size()
        if nb > self.nbytes:
            if self.device.type == "cuda" and torch.cuda.is_current_stream_capturing():
                raise RuntimeError("DetWorkspace: a CUDA-graph capture cannot grow the workspace; run the step eagerly "
                                   "first")
            self._buf = torch.empty((nb + 7) // 8, dtype=torch.float64, device=self.device)
        return self._buf.view(dtype)

    def slots(self, n: int, c: int) -> torch.Tensor:
        """float64 slots enough for a deterministic reduction onto [n][c] per-channel values (or a loss)."""
        return self.get(int(_lib.load().sn_det_slots(n, c)))


class Plan:
    """Owns one sn_plan handle (encoded TMA descriptors + launch geometry)."""

    def __init__(self, handle: int, keep: Sequence, tag=None):
        self.handle = handle
        self.tag = tag
        self._keep = list(keep)  # tensors whose addresses are baked into the plan

    @property
    def workspace_bytes(self) -> int:
        """Device bytes the plan owns beyond its descriptors (the split partials of a deterministic wgrad plan)."""
        return int(_lib.load().sn_plan_workspace_bytes(self.handle))

    @property
    def has_stats(self) -> bool:
        """True when the launch also accumulates the InstanceNorm statistics requested through its descriptor."""
        return bool(_lib.load().sn_plan_has_stats(self.handle))

    # bench.py's roofline pass: when a list is installed here every plan launch is bracketed by CUDA
    # events on the launching stream and (tag, start, end) is appended
    trace = None

    def run(self) -> None:
        if Plan.trace is None:
            check(_lib.load().sn_plan_run(self.handle, _stream()))
            return
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        check(_lib.load().sn_plan_run(self.handle, _stream()))
        e1.record()
        Plan.trace.append((self, e0, e1))

    def __del__(self):
        try:
            if self.handle:
                _lib.load().sn_plan_destroy(self.handle)
        except Exception:
            pass


def _fill_tap(dst: SnTap, tap: L.Tap, pitch: int, k_pad: int, c_base: int = 0) -> None:
    dst.c_off = tap.pw * pitch + c_base
    dst.kb_off = tap.kb * k_pad
    dst.dw, dst.dh, dst.hp = tap.dw, tap.dh, tap.hp


def tap_gemm_desc(a: Planes, spec: L.GemmSpec, w: PackedWeights, k_per_tap: int, out: torch.Tensor,
                  n_valid: int, *, w_row_off: int = 0, w_rows: Optional[int] = None,
                  w_k: Optional[int] = None, w_elem_off: int = 0, bias: Optional[torch.Tensor] = None,
                  act: int = ACT_NONE, nsplit: int = 3, block_n: Optional[int] = None,
                  out_c_off: int = 0, nphase: int = 1, stack_slot: int = 0, stack_c: int = 0,
                  stats: Optional[torch.Tensor] = None) -> SnTapGemmDesc:
    """out: fp32 NHWC tensor [n, OH, OW, pitch_out]; rows (h, w) land on pixel
    (h*mul_h + off_h, w*mul_w + off_w)."""
    assert (a.h, a.w) == tuple(spec.a_hw), f"operand is {a.h}x{a.w}, spec wants {spec.a_hw}"
    assert a.c_off % 8 == 0 and k_per_tap <= a.c
    narrow = k_per_tap < 64
    assert (k_per_tap in (16, 32)) if narrow else (k_per_tap % 64 == 0)
    taps = list(spec.taps)
    if narrow and nphase == 4:
        assert (len(taps) // 4) % (64 // k_per_tap) == 0, "4-phase narrow launch: taps per phase must fill whole stages"
    elif narrow:  # 64/k taps share a pipeline stage: pad with dummy taps whose packed weights are zero
        tps = 64 // k_per_tap
        kb_next = max(t.kb for t in taps) + 1
        while len(taps) % tps:
            taps.append(L.Tap(taps[0].pw, kb_next, taps[0].dw, taps[0].dh, taps[0].hp))
            kb_next += 1
    d = SnTapGemmDesc()
    d.a_chunk = k_per_tap if narrow else 64
    d.a_hi, d.a_lo = a.hi_ptr, a.lo_ptr
    d.a_n, d.a_h, d.a_w, d.a_c, d.a_pitch = a.n, a.h, a.w, a.c, a.pitch
    d.a_parity = 1 if spec.parity else 0
    d.a_fmt, d.b_fmt = a.fmt, w.fmt
    d.b_scale = None if w.scale is None else w.scale.data_ptr()
    d.b_hi = w.hi.data_ptr() + 2 * w_elem_off
    d.b_lo = w.lo.data_ptr() + 2 * w_elem_off
    d.b_rows = w.rows if w_rows is None else w_rows
    d.b_k = w.k_total if w_k is None else w_k
    d.m_n, d.m_h, d.m_w = a.n, spec.m_h, spec.m_w
    d.ntaps, d.k_per_tap = len(taps), k_per_tap
    for i, t in enumerate(taps):
        _fill_tap(d.taps[i], t, a.pitch, k_per_tap)
    assert out.dtype == torch.float32 and out.dim() == 4 and (out.shape[3] == 1 or out.stride(3) == 1)
    d.out = out.data_ptr() + 4 * out_c_off
    d.out_sn, d.out_sh, d.out_sw = out.stride(0), out.stride(1), out.stride(2)
    d.out_mul_h, d.out_mul_w = spec.out_mul
    d.out_off_h, d.out_off_w = spec.out_off
    d.n_valid = n_valid
    d.block_n = block_n or L.pick_block_n(n_valid)
    d.bias = _ptr(bias)
    d.act = act
    d.nsplit = nsplit
    d.nphase = nphase
    d.stack_slot, d.stack_c = stack_slot, stack_c
    if stats is not None:      # fused InstanceNorm statistics [n, n_valid, 2] float64 (see Plan.has_stats)
        assert stats.dtype == torch.float64 and stats.numel() >= a.n * n_valid * 2 and out_c_off == 0
        d.stats = stats.data_ptr()
    return d


def merge_phase_specs(specs) -> Optional[L.GemmSpec]:
    """Four GemmSpecs that differ only by their taps and by the output offset (py, px) — the parity phases
    of a ConvTranspose2d forward / Conv2d input-gradient — become ONE spec whose taps are the 4 groups
    concatenated (phase z = 2*py + px), launched with grid.z = 4."""
    if len(specs) != 4:
        return None
    s0 = specs[0]
    n = len(s0.taps)
    for z, s in enumerate(specs):
        if (s.parity, s.m_h, s.m_w, s.out_mul, s.a_hw, len(s.taps)) != (s0.parity, s0.m_h, s0.m_w, s0.out_mul, s0.a_hw, n):
            return None
        if s.out_off != (z >> 1, z & 1) or s.w_phase != 0:
            return None
    return L.GemmSpec(s0.parity, s0.m_h, s0.m_w, [t for s in specs for t in s.taps], s0.out_mul, (0, 0), 0, s0.a_hw)


def tap_gemm_plan(desc: SnTapGemmDesc, keep: Sequence = ()) -> Plan:
    h = C.c_void_p()
    check(_lib.load().sn_tap_gemm_plan_create(C.byref(desc), C.byref(h)))
    return Plan(h.value, keep)


def tap_gemm_simt(desc: SnTapGemmDesc) -> None:
    check(_lib.load().sn_tap_gemm_simt(C.byref(desc), _stream()))


def wgrad_desc(x: Planes, y: Planes, spec: L.WgradSpec, out: torch.Tensor, s_row: int, s_col: int,
               tap_off: Sequence[int], rows_valid: int, cols_valid: int, *, swap: bool = False,
               nsplit: int = 3, block_n: Optional[int] = None, ksplit: int = 0,
               deterministic: bool = False) -> SnWgradDesc:
    """x / y follow the spec orientation; swap=True exchanges the roles (rows <-> cols).  deterministic: the split-K
    partials are added in split order by a second kernel (bit-identical runs), the split count follows from the shapes."""
    xt, yt = spec.xtaps, spec.ytaps
    xp, yp = spec.x_parity, spec.y_parity
    if swap:
        x, y, xt, yt, xp, yp = y, x, yt, xt, yp, xp
        s_row, s_col = s_col, s_row
        rows_valid, cols_valid = cols_valid, rows_valid
    assert x.c_off % 8 == 0 and y.c_off % 8 == 0
    order = list(range(len(xt)))
    groups = []
    if y.c < 64:
        # narrow N side: taps with the same X tap become column blocks of one accumulator (X read once)
        gmax = 128 // y.c
        key = lambda i: (xt[i].pw, xt[i].dw, xt[i].dh, xt[i].hp)
        order = sorted(order, key=key)           # stable: keeps the tap order inside a group
        i = 0
        while i < len(order):
            j = i
            while j < len(order) and j - i < gmax and key(order[j]) == key(order[i]):
                j += 1
            groups.append((i, j - i))
            i = j
        xt = [xt[i] for i in order]
        yt = [yt[i] for i in order]
        tap_off = [tap_off[i] for i in order]
    d = SnWgradDesc()
    d.x_hi, d.x_lo = x.hi_ptr, x.lo_ptr
    d.x_n, d.x_h, d.x_w, d.x_c, d.x_pitch, d.x_parity = x.n, x.h, x.w, x.c, x.pitch, int(xp)
    d.x_fmt, d.y_fmt = x.fmt, y.fmt
    d.y_hi, d.y_lo = y.hi_ptr, y.lo_ptr
    d.y_n, d.y_h, d.y_w, d.y_c, d.y_pitch, d.y_parity = y.n, y.h, y.w, y.c, y.pitch, int(yp)
    d.m_n, d.m_h, d.m_w = x.n, spec.m_h, spec.m_w
    d.ntaps = len(xt)
    for i in range(len(xt)):
        _fill_tap(d.xtaps[i], xt[i], x.pitch, 0)
        _fill_tap(d.ytaps[i], yt[i], y.pitch, 0)
        d.tap_off[i] = tap_off[i]
    assert out.dtype == torch.float32
    d.out = out.data_ptr()
    d.s_row, d.s_col = s_row, s_col
    d.rows_valid, d.cols_valid = rows_valid, cols_valid
    assert x.c >= 64, "the 128-row operand of a wgrad GEMM must carry >= 64 channels (swap the roles)"
    if y.c < 64:   # narrow N-side operand: one 16/32-channel atom
        assert y.c in (16, 32) and cols_valid <= y.c
        d.y_chunk = y.c
        d.ngroups = len(groups)
        for g, (st, sz) in enumerate(groups):
            d.group_start[g], d.group_size[g] = st, sz
        d.block_n = max(sz for _, sz in groups) * y.c
    else:
        d.y_chunk = 64
        d.block_n = block_n or (128 if cols_valid > 64 else 64)
    d.ksplit = ksplit
    d.nsplit = nsplit
    d.deterministic = int(deterministic)
    return d


def wgrad_ksplit(desc: SnWgradDesc, sm_count: int) -> int:
    """The split-K count a plan of `desc` gets on a device with sm_count SMs (host logic, no device needed)."""
    k = _lib.load().sn_wgrad_ksplit(C.byref(desc), sm_count)
    if k <= 0:
        check(k)
    return int(k)


def wgrad_plan(desc: SnWgradDesc, keep: Sequence = ()) -> Plan:
    h = C.c_void_p()
    check(_lib.load().sn_wgrad_plan_create(C.byref(desc), C.byref(h)))
    return Plan(h.value, keep)


# ---------------------------------------------------------------------------------------------
# packing
# ---------------------------------------------------------------------------------------------
class SegMap:
    """A 0/1-valued [n, c, h, w] segmentation tensor in compact form (SURVEY §8f rank 4): `data` is a uint8 label map
    [n,h,w] (label L > 0 -> channel L one-hot, 0 -> the all-zero vector: datasets/data_utils.py:330-343) or an int32
    bit mask [n,h,w] (bit c = channel c: the independently augmented channels of data_utils.py:346-361).  The kernels
    that consume cloth tensors (pack_concat, pack_planes, ce_loss_fwd_bwd) expand it on the fly."""

    def __init__(self, data: torch.Tensor, channels: int):
        assert data.dim() == 3 and data.dtype in (torch.uint8, torch.int32), "uint8 label map or int32 bit mask [n,h,w]"
        assert channels <= (32 if data.dtype == torch.int32 else 256)
        self.data, self.channels = data.contiguous(), channels
        self.layout = LAYOUT_LABEL_U8 if data.dtype == torch.uint8 else LAYOUT_MASK_I32

    @property
    def shape(self):
        n, h, w = self.data.shape
        return (n, self.channels, h, w)

    @property
    def is_cuda(self):
        return self.data.is_cuda

    def dense(self) -> torch.Tensor:
        """fp32 [n,c,h,w] expansion with torch ops (visuals / tests; the hot path never calls this)."""
        ch = torch.arange(self.channels, device=self.data.device).view(1, -1, 1, 1)
        d = self.data.unsqueeze(1)
        if self.layout == LAYOUT_LABEL_U8:
            return ((d.long() == ch) & (ch > 0)).float()
        return ((d.long() >> ch) & 1).float()

    @staticmethod
    def from_dense(t: torch.Tensor) -> "SegMap":
        """Compress an fp32 0/1 tensor [n,c,h,w] (what the reference's dataset yields): a uint8 label map when it is
        one-hot with an empty channel 0, else an int32 bit mask.  Raises if the tensor is not 0/1-valued."""
        assert t.dim() == 4 and t.shape[1] <= 32
        b = t != 0
        if not torch.equal(b.to(t.dtype), t):
            raise ValueError("SegMap.from_dense: tensor is not 0/1-valued")
        c = t.shape[1]
        if int(b.sum(1).max()) <= 1 and not bool(b[:, 0].any()):
            return SegMap(b.to(torch.uint8).mul(torch.arange(c, dtype=torch.uint8, device=t.device).view(1, -1, 1, 1))
                          .sum(1, dtype=torch.uint8), c)
        w = (1 << torch.arange(c, dtype=torch.int64, device=t.device)).view(1, -1, 1, 1)
        return SegMap((b.long() * w).sum(1).to(torch.int32), c)


def _src_args(t, nhwc: bool):
    """(pointer, layout, pitch, channels, (n, h, w)) of a pack source: fp32 NCHW / NHWC tensor or SegMap."""
    if isinstance(t, SegMap):
        n, h, w = t.data.shape
        return t.data.data_ptr(), t.layout, 0, t.channels, (n, h, w)
    assert t.dtype == torch.float32
    if nhwc:
        n, h, w, c = t.shape
        return t.data_ptr(), LAYOUT_NHWC, _pitch(t), c, (n, h, w)
    assert t.is_contiguous()
    n, c, h, w = t.shape
    return t.data_ptr(), LAYOUT_NCHW, 0, c, (n, h, w)


def pack_planes(src, dst: Planes, *, nhwc: bool = False) -> None:
    """src: fp32 NCHW contiguous [n,c,h,w] (or NHWC [n,h,w,pitch] with nhwc=True, first dst.c channels), or a SegMap."""
    if isinstance(src, SegMap):
        ptr, layout, _, c, (n, h, w) = _src_args(src, False)
        assert c <= dst.c and (n, h, w) == (dst.n, dst.h, dst.w)
        for d_ in ((dst,) if dst.twin is None else (dst, dst.twin)):
            check(_lib.load().sn_pack_planes(ptr, layout, 0, n, c, h, w, d_.hi_ptr, d_.lo_ptr, d_.pitch, 0, d_.fmt,
                                             _stream()))
        return
    assert src.dtype == torch.float32
    if nhwc:
        n, h, w, sp = src.shape
        # dense [n, h, w, sp]: is_contiguous() ignores the strides of size-1 dimensions, which a w = 1 plane may carry
        assert src.is_contiguous()
        c = dst.c
        for d_ in ((dst,) if dst.twin is None else (dst, dst.twin)):
            check(_lib.load().sn_pack_planes(src.data_ptr(), LAYOUT_NHWC, sp, n, c, h, w, d_.hi_ptr, d_.lo_ptr,
                                             d_.pitch, 0, d_.fmt, _stream()))
    else:
        assert src.is_contiguous()
        n, c, h, w = src.shape
        assert c <= dst.c
        for d_ in ((dst,) if dst.twin is None else (dst, dst.twin)):
            check(_lib.load().sn_pack_planes(src.data_ptr(), LAYOUT_NCHW, 0, n, c, h, w, d_.hi_ptr, d_.lo_ptr,
                                             d_.pitch, 0, d_.fmt, _stream()))
    assert (n, h, w) == (dst.n, dst.h, dst.w)


def pack_concat(srcs, dst: Planes, lead: int = 0) -> None:
    """srcs: 1-2 tuples (tensor, nhwc: bool); `lead` zero channels, then the sources' channels concatenated,
    zero-filled to dst.c, written to dst and its twin in one pass.  Replaces cat((zeros, a, b), 1) + the channel
    padding of the operand."""
    assert 1 <= len(srcs) <= 2 and dst.c % 8 == 0 and dst.c_off % 8 == 0 and lead >= 0
    args = [lead]
    for t, nhwc in srcs:
        ptr, layout, pitch, c, nhw = _src_args(t, nhwc)
        args += [ptr, layout, pitch, c]
        assert nhw == (dst.n, dst.h, dst.w)
    if len(srcs) == 1:
        args += [None, 0, 0, 0]
    tw = dst.twin
    check(_lib.load().sn_pack_concat(*args, dst.n, dst.h, dst.w, dst.c, dst.hi.data_ptr(), dst.lo.data_ptr(),
                                     None if tw is None else tw.hi.data_ptr(), None if tw is None else tw.lo.data_ptr(),
                                     dst.pitch, dst.c_off, dst.fmt, FMT_BF16 if tw is None else tw.fmt, _stream()))


class PackTable:
    """All weight-scale and pack launches of one network as TWO launches (sn_weight_scale_multi,
    sn_pack_weights_multi): layers register their tensors once, the item tables live in device memory."""

    def __init__(self, device):
        self.device = device
        self._scales, self._packs, self._keep = [], [], []
        self._dev = None

    def add_scale(self, weight: torch.Tensor, scale: torch.Tensor) -> None:
        """scale <- (s, 1/s) at every run(), s = 2^k with max|w| * s in [2^13, 2^14)."""
        assert weight.is_contiguous() and weight.dtype == torch.float32 and self._dev is None
        assert weight.data_ptr() % 16 == 0, "weight_scale_multi reads float4: the weight must be 16-byte aligned"
        it = _lib.SnScaleItem()
        it.w, it.count, it.scale2 = weight.data_ptr(), weight.numel(), scale.data_ptr()
        self._scales.append(it)
        self._keep += [weight, scale]

    def add_pack(self, weight: torch.Tensor, kind: str, dgrad: bool, k_pad: int, dst: PackedWeights) -> None:
        """dst <- the torch-layout weight of a `kind` conv in its forward (dgrad=False) or input-gradient kernel
        layout, K padded to k_pad, scaled by dst.scale[0] when dst has a scale."""
        assert weight.is_contiguous() and weight.dtype == torch.float32 and self._dev is None
        if kind == "convT4s2":
            cin, cout = weight.shape[0], weight.shape[1]
        else:
            cout, cin = weight.shape[0], weight.shape[1]
        s_row, s_k, rows, k_real = L.pack_strides(kind, cin, cout, dgrad)
        t = L.ntaps(kind)
        assert dst.rows >= rows and dst.k_total >= t * k_pad and k_pad >= k_real and dst.k_total % k_pad == 0 and t <= 16
        it = _lib.SnPackItem()
        it.src, it.s_row, it.s_k = weight.data_ptr(), s_row, s_k
        it.rows, it.taps, it.taps_pitch, it.k_real, it.k_pad, it.fmt = rows, t, dst.k_total // k_pad, k_real, k_pad, dst.fmt
        it.hi, it.lo = dst.hi.data_ptr(), dst.lo.data_ptr()
        it.scale2 = None if dst.scale is None else dst.scale.data_ptr()
        for i, sl in enumerate(L.pack_slots(kind, dgrad)):
            it.slot[i] = sl
        self._packs.append(it)
        self._keep += [weight, dst]

    def _upload(self, items, ctype):
        arr = (ctype * len(items))(*items)
        return torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(self.device)

    def finalize(self) -> None:
        lib = _lib.load()
        rpb, kpb = lib.sn_pack_rows_per_block(), lib.sn_pack_k_per_block()
        begin = 0
        for it in self._packs:
            it.block_begin = begin
            begin += ((it.rows + rpb - 1) // rpb) * ((it.k_pad + kpb - 1) // kpb)
        self._blocks = begin
        self._max_taps = max([it.taps for it in self._packs], default=1)
        self._dev = (self._upload(self._scales, _lib.SnScaleItem) if self._scales else None,
                     self._upload(self._packs, _lib.SnPackItem) if self._packs else None,
                     torch.zeros(2 * max(1, len(self._scales)), dtype=torch.int32, device=self.device))

    def run(self) -> None:
        if self._dev is None:
            self.finalize()
        sc, pk, scratch = self._dev
        lib = _lib.load()
        if sc is not None:
            check(lib.sn_weight_scale_multi(sc.data_ptr(), len(self._scales), scratch.data_ptr(), _stream()))
        if pk is not None:
            check(lib.sn_pack_weights_multi(pk.data_ptr(), len(self._packs), self._blocks, self._max_taps, _stream()))


def pack_head_weights(weight: torch.Tensor, rows_pad: int, k_pad: int, dgrad: bool, dst: PackedWeights) -> None:
    cout, cin = weight.shape[:2]
    assert dst.hi.numel() >= (cin * 25 * k_pad if dgrad else rows_pad * 25 * k_pad)
    taps_pitch = dst.k_total // k_pad if dgrad else 25
    check(_lib.load().sn_pack_head_weights(weight.data_ptr(), cout, cin, rows_pad, k_pad, int(dgrad), taps_pitch,
                                           dst.hi.data_ptr(), dst.lo.data_ptr(), dst.fmt,
                                           None if dst.scale is None else dst.scale.data_ptr(), _stream()))


def pack_head_stacked(weight: torch.Tensor, slot: int, k_pad: int, dst: PackedWeights) -> None:
    """dst [4*slot rows][9 taps * k_pad]: the head's effective taps, output-parity phases stacked along the rows."""
    cout, cin = weight.shape[:2]
    assert dst.rows == 4 * slot and dst.k_total == 9 * k_pad and slot >= cout and k_pad >= cin
    check(_lib.load().sn_pack_head_stacked(weight.data_ptr(), cout, cin, slot, k_pad, dst.hi.data_ptr(),
                                           dst.lo.data_ptr(), dst.fmt,
                                           None if dst.scale is None else dst.scale.data_ptr(), _stream()))


def fold_head_wgrad(geff: torch.Tensor, cout: int, cin: int, dw: torch.Tensor) -> None:
    check(_lib.load().sn_fold_head_wgrad(geff.data_ptr(), cout, cin, dw.data_ptr(), _stream()))


# ---------------------------------------------------------------------------------------------
# InstanceNorm / activation blocks
# ---------------------------------------------------------------------------------------------
def _pitch(t: torch.Tensor) -> int:
    """pixel pitch (elements) of an NHWC fp32 tensor or channel-slice view of one"""
    assert t.dim() == 4 and (t.shape[3] == 1 or t.stride(3) == 1)
    n, h, w, c = t.shape
    if w > 1:
        p = t.stride(2)
    elif h > 1:
        p = t.stride(1)
    elif n > 1:
        p = t.stride(0)
    else:
        p = c
    assert t.stride(1) == w * p or h == 1, "not an NHWC-contiguous pixel grid"
    assert t.stride(0) == h * w * p or n == 1, "not an NHWC-contiguous pixel grid"
    return p


def plane_stats(y: torch.Tensor, c: int, stats: torch.Tensor, eps: float = IN_EPS,
                ws: Optional[DetWorkspace] = None) -> None:
    """y fp32 NHWC [n,h,w,pitch]; stats float64 [n, c, 2] <- (mean, rstd).  ws: deterministic reduction."""
    n, h, w, _ = y.shape
    pitch = _pitch(y)
    assert stats.dtype == torch.float64 and stats.numel() >= n * c * 2
    if ws is not None:
        sl = ws.slots(n, c)
        check(_lib.load().sn_plane_stats_det(y.data_ptr(), pitch, n, h * w, c, eps, stats.data_ptr(), sl.data_ptr(),
                                             sl.numel(), _stream()))
        return
    check(_lib.load().sn_plane_stats(y.data_ptr(), pitch, n, h * w, c, eps, stats.data_ptr(), _stream()))


def stats_finalize(stats: torch.Tensor, count: int, hw: int, eps: float = IN_EPS) -> None:
    """(sum, sum of squares) accumulated by a GEMM launch with fused statistics -> (mean, rstd), in place."""
    check(_lib.load().sn_stats_finalize(stats.data_ptr(), count, hw, eps, _stream()))


def plane_sums(y: torch.Tensor, c: int, stats: torch.Tensor, ws: Optional[DetWorkspace] = None) -> None:
    """y fp32 NHWC [n,h,w,pitch]; stats float64 [n, c, 2] <- (sum, sum of squares) over the plane."""
    n, h, w, _ = y.shape
    assert stats.dtype == torch.float64 and stats.numel() >= n * c * 2
    if ws is not None:
        sl = ws.slots(n, c)
        check(_lib.load().sn_plane_sums_det(y.data_ptr(), _pitch(y), n, h * w, c, stats.data_ptr(), sl.data_ptr(),
                                            sl.numel(), _stream()))
        return
    check(_lib.load().sn_plane_sums(y.data_ptr(), _pitch(y), n, h * w, c, stats.data_ptr(), _stream()))


def bn_finalize(stats: torch.Tensor, n: int, c: int, groups: int, hw: int, bn: "torch.nn.BatchNorm2d") -> None:
    """Train-mode BatchNorm2d statistics: per-(n, c) (sum, sum of squares) -> (mean, rstd) of each sample's group, in
    place; bn's running_mean / running_var / num_batches_tracked (device tensors) are updated group by group."""
    assert stats.dtype == torch.float64 and n % groups == 0
    assert bn.momentum is not None, "BatchNorm2d(momentum=None) (cumulative average) is not provided"
    track = bn.track_running_stats
    check(_lib.load().sn_bn_finalize(stats.data_ptr(), n, c, groups, hw, float(bn.eps), float(bn.momentum),
                                     _ptr(bn.running_mean if track else None), _ptr(bn.running_var if track else None),
                                     _ptr(bn.num_batches_tracked if track else None), _stream()))


def bn_group_sums(stats: torch.Tensor, n: int, c: int, groups: int, hw: int, part: torch.Tensor) -> None:
    """Per-(n, c) pair sums (the forward's (sum, sum of squares) or, after norm_act_bwd(bn_phase=1), the backward's
    (sum g, sum g*xhat)) -> this rank's partials part [groups, c, 3] fp64 = (element count, sum, sum of squares)."""
    assert stats.dtype == part.dtype == torch.float64 and n % groups == 0 and part.numel() >= groups * c * 3
    check(_lib.load().sn_bn_group_sums(stats.data_ptr(), n, c, groups, hw, part.data_ptr(), _stream()))


def bn_finalize_gathered(stats: torch.Tensor, n: int, c: int, groups: int, gathered: torch.Tensor,
                         bn: "torch.nn.BatchNorm2d") -> None:
    """bn_finalize with the statistics of every rank: gathered [world, groups, c, 3] fp64 holds the ranks'
    bn_group_sums partials in rank order; stats [n, c, 2] <- (mean, rstd) of each local sample's global group, and bn's
    running buffers are updated from the global statistics."""
    assert stats.dtype == gathered.dtype == torch.float64 and n % groups == 0
    assert gathered.dim() == 4 and tuple(gathered.shape[1:]) == (groups, c, 3) and gathered.is_contiguous()
    assert bn.momentum is not None, "BatchNorm2d(momentum=None) (cumulative average) is not provided"
    track = bn.track_running_stats
    check(_lib.load().sn_bn_finalize_gathered(stats.data_ptr(), n, c, groups, gathered.data_ptr(), gathered.shape[0],
                                              float(bn.eps), float(bn.momentum),
                                              _ptr(bn.running_mean if track else None),
                                              _ptr(bn.running_var if track else None),
                                              _ptr(bn.num_batches_tracked if track else None), _stream()))


def bn_eval_stats(stats: torch.Tensor, n: int, c: int, bn: "torch.nn.BatchNorm2d") -> None:
    """Eval-mode BatchNorm2d: stats [n, c, 2] <- (running_mean, rstd of running_var)."""
    assert stats.dtype == torch.float64
    check(_lib.load().sn_bn_eval_stats(stats.data_ptr(), n, c, bn.running_mean.data_ptr(), bn.running_var.data_ptr(),
                                       float(bn.eps), _stream()))


def norm_act_fwd(y: torch.Tensor, c: int, stats: Optional[torch.Tensor], act: int, slope: float = 0.2,
                 drop_p: float = 0.0, drop_seed: int = 0, residual: Optional[torch.Tensor] = None,
                 out: Optional[Planes] = None, reflect_pad: bool = False,
                 out_f32: Optional[torch.Tensor] = None, drop_offset: int = 0,
                 seed_dev: Optional[torch.Tensor] = None, stage_id: int = 0,
                 gamma: Optional[torch.Tensor] = None, beta: Optional[torch.Tensor] = None) -> None:
    """drop_offset: element offset of the keep-mask index (global sample index of the first local sample * h*w*c);
    seed_dev (float32[2] on the device: the 32-bit step seed as its exact 16-bit halves (lo, hi), as
    set_step_params writes them) + stage_id: the per-stage seed is derived on the device from the step seed
    stored there (CUDA-graph replay), drop_seed is then ignored.
    gamma, beta (fp32 [c]): BatchNorm's affine, applied before the activation.
    Any c and any row alignment: four channels per thread where c % 4 == 0 and the rows are aligned, else one."""
    n, h, w, _ = y.shape
    pitch = _pitch(y)
    d = SnNormActDesc()
    d.y, d.y_pitch = y.data_ptr(), pitch
    d.n, d.h, d.w, d.c = n, h, w, c
    d.stats = _ptr(stats)
    d.act, d.slope = act, slope
    d.drop_p, d.drop_seed = drop_p, drop_seed
    d.drop_offset, d.drop_step_seed_dev, d.drop_stage_id = drop_offset, _ptr(seed_dev), stage_id
    if residual is not None:
        d.residual, d.res_pitch = residual.data_ptr(), _pitch(residual)
    if out is not None:
        if reflect_pad:
            assert (out.h, out.w) == (h + 2, w + 2)
        else:
            assert (out.h, out.w) == (h, w)
        assert out.c >= c and out.n == n
        d.out_hi, d.out_lo, d.out_pitch, d.out_coff = out.hi.data_ptr(), out.lo.data_ptr(), out.pitch, out.c_off
        d.out_reflect_pad = int(reflect_pad)
        d.out_fmt = out.fmt
        if out.twin is not None:
            d.out2_hi, d.out2_lo, d.out2_fmt = out.twin.hi.data_ptr(), out.twin.lo.data_ptr(), out.twin.fmt
    if out_f32 is not None:
        d.out_f32, d.f32_pitch = out_f32.data_ptr(), _pitch(out_f32)
    d.gamma, d.beta = _ptr(gamma), _ptr(beta)
    check(_lib.load().sn_norm_act_fwd(C.byref(d), _stream()))


@dataclass
class GradSrc:
    t: torch.Tensor          # fp32 NHWC [n, h(+2), w(+2), pitch]
    c_off: int = 0
    reflect_padded: bool = False
    up: int = 1              # >1: t is [n, h*up, w*up, .] (gradient of a nearest-upsampled copy)
    act: int = -1            # activation of THIS consumer (-1: the stage's own)


def _fill_srcs(arr, srcs: Sequence[GradSrc]) -> None:
    assert 1 <= len(srcs) <= _lib.SN_MAX_SRC
    for i, s in enumerate(srcs):
        assert s.t.dtype == torch.float32 and (s.t.shape[3] == 1 or s.t.stride(3) == 1)
        arr[i].ptr = s.t.data_ptr()
        arr[i].pitch = _pitch(s.t)
        arr[i].c_off = s.c_off
        arr[i].reflect_padded = int(s.reflect_padded)
        arr[i].up = s.up
        arr[i].act = s.act


def norm_act_bwd(srcs: Sequence[GradSrc], y: torch.Tensor, c: int, stats: Optional[torch.Tensor], act: int,
                 dy: Planes, gstats: Optional[torch.Tensor] = None, slope: float = 0.2, drop_p: float = 0.0,
                 drop_seed: int = 0, drop_offset: int = 0, seed_dev: Optional[torch.Tensor] = None,
                 stage_id: int = 0, bias_grad: Optional[torch.Tensor] = None,
                 bn: Optional[Tuple[torch.Tensor, torch.Tensor]] = None, bn_groups: int = 1, bn_train: bool = True,
                 bn_grads: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
                 ws: Optional[DetWorkspace] = None, bn_phase: int = 0, bn_gathered: Optional[torch.Tensor] = None,
                 bn_rank: int = 0) -> None:
    """ws: deterministic reduction of the normalisation's gradient statistics (then no fused bias_grad).
    bias_grad (fp32 [c], c in {256, 512, 1024}): += per-channel sums of the dy written — the bias gradient of the
    conv that produced y — inside the apply pass (see fused_bias_grad_ok; operands that take the one-channel
    instantiation, c % 4 != 0 or unaligned rows, allow c in {64, 128, 256} instead).
    Any c and any row alignment: four channels per thread where c % 4 == 0 and the rows are aligned, else one.
    bn = (gamma, beta): BatchNorm backward over `bn_groups` sample groups, with batch (bn_train) or running statistics
    in `stats`; bn_grads = (d gamma, d beta) are accumulated (+=) when given.
    Batch statistics across ranks split the call in two around the gather: bn_phase=1 leaves the per-(n, c)
    (sum g, sum g*xhat) in gstats (for bn_group_sums); bn_phase=2 takes the group means from bn_gathered
    [world, bn_groups, c, 3] and runs the apply pass, adding only rank bn_rank's sums to bn_grads."""
    n, h, w, _ = y.shape
    pitch = _pitch(y)
    d = SnNormActBwdDesc()
    _fill_srcs(d.src, srcs)
    d.nsrc = len(srcs)
    d.y, d.y_pitch = y.data_ptr(), pitch
    d.n, d.h, d.w, d.c = n, h, w, c
    d.stats = _ptr(stats)
    d.act, d.slope = act, slope
    d.drop_p, d.drop_seed = drop_p, drop_seed
    d.drop_offset, d.drop_step_seed_dev, d.drop_stage_id = drop_offset, _ptr(seed_dev), stage_id
    d.gstats = _ptr(gstats)
    assert (dy.n, dy.h, dy.w) == (n, h, w) and dy.c >= c
    d.dy_hi, d.dy_lo, d.dy_pitch, d.dy_coff = dy.hi.data_ptr(), dy.lo.data_ptr(), dy.pitch, dy.c_off
    d.dy_fmt = dy.fmt
    d.bias_grad = _ptr(bias_grad)
    if bn is not None:
        d.gamma, d.beta = bn[0].data_ptr(), bn[1].data_ptr()
        d.bn_groups, d.bn_train = bn_groups, int(bn_train)
        if bn_grads is not None:
            d.gamma_grad, d.beta_grad = bn_grads[0].data_ptr(), bn_grads[1].data_ptr()
    if ws is not None and stats is not None:
        sl = ws.slots(n, c)
        d.det_slots, d.det_slots_cap = sl.data_ptr(), sl.numel()
    d.bn_phase = bn_phase
    if bn_gathered is not None:
        assert bn_gathered.dtype == torch.float64 and bn_gathered.is_contiguous()
        assert bn_gathered.dim() == 4 and tuple(bn_gathered.shape[1:]) == (bn_groups, c, 3)
        d.bn_gathered, d.bn_world, d.bn_rank = bn_gathered.data_ptr(), bn_gathered.shape[0], bn_rank
    check(_lib.load().sn_norm_act_bwd(C.byref(d), _stream()))


def fused_bias_grad_ok(c: int) -> bool:
    """Channel counts for which norm_act_bwd can accumulate the bias gradient itself, given aligned operands (the
    engines' are)."""
    return c in (256, 512, 1024)


def bias_grad(dy: Planes, c: int, scratch: torch.Tensor, db: torch.Tensor, ws: Optional[DetWorkspace] = None) -> None:
    assert scratch.dtype == torch.float64 and scratch.numel() >= c and db.dtype == torch.float32
    if ws is not None:
        sl = ws.slots(1, c)
        check(_lib.load().sn_bias_grad_det(dy.hi.data_ptr(), dy.lo.data_ptr(), dy.pitch, dy.c_off, dy.fmt,
                                           dy.n * dy.h * dy.w, c, scratch.data_ptr(), db.data_ptr(), sl.data_ptr(),
                                           sl.numel(), _stream()))
        return
    check(_lib.load().sn_bias_grad(dy.hi.data_ptr(), dy.lo.data_ptr(), dy.pitch, dy.c_off, dy.fmt, dy.n * dy.h * dy.w, c,
                                   scratch.data_ptr(), db.data_ptr(), _stream()))


def sum_grads(srcs: Sequence[GradSrc], n: int, h: int, w: int, c: int, dst: torch.Tensor) -> None:
    arr = (SnGradSrc * _lib.SN_MAX_SRC)()
    _fill_srcs(arr, srcs)
    check(_lib.load().sn_sum_grads(arr, len(srcs), n, h, w, c, dst.data_ptr(), _pitch(dst), _stream()))


def tanh_bwd(srcs: Sequence[GradSrc], out: torch.Tensor, c: int, dy: Planes) -> None:
    n, h, w, _ = out.shape
    pitch = _pitch(out)
    arr = (SnGradSrc * _lib.SN_MAX_SRC)()
    _fill_srcs(arr, srcs)
    check(_lib.load().sn_tanh_bwd(arr, len(srcs), out.data_ptr(), pitch, n, h, w, c, dy.hi.data_ptr(),
                                  dy.lo.data_ptr(), dy.pitch, dy.c_off, dy.fmt, _stream()))


def upsample_planes(src: Planes, dst: Planes, factor: int) -> None:
    """dst[n,h,w,:src.c] = src[n,h//f,w//f,:] on the 16-bit words (and on the bf16 twins if both have one)."""
    assert (dst.h, dst.w) == (src.h * factor, src.w * factor) and dst.c >= src.c and src.fmt == dst.fmt
    pairs = [(src, dst)]
    if src.twin is not None and dst.twin is not None:
        pairs.append((src.twin, dst.twin))
    for s_, d_ in pairs:
        check(_lib.load().sn_upsample_planes(s_.hi.data_ptr(), s_.lo.data_ptr(), s_.pitch, s_.c_off, dst.n, dst.h,
                                             dst.w, src.c, factor, d_.hi.data_ptr(), d_.lo.data_ptr(), d_.pitch,
                                             d_.c_off, _stream()))


def adamw_step(p: torch.Tensor, g: torch.Tensor, m: torch.Tensor, v: torch.Tensor, lr: float, b1: float, b2: float,
               eps: float, wd: float, step: int) -> None:
    assert p.is_contiguous() and g.is_contiguous() and p.numel() == g.numel() == m.numel() == v.numel()
    check(_lib.load().sn_adamw_step(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), p.numel(), lr, b1, b2, eps,
                                    wd, step, _stream()))


def adamw_hyper(lr: float, b1: float, b2: float, eps: float, wd: float, step: int, gscale: float = 1.0):
    """The 8 fp32 scalars of sn_adamw_step_dev for optimizer step `step` (1-based), as a list of Python floats."""
    out = (C.c_float * 8)()
    _lib.load().sn_adamw_hyper(lr, b1, b2, eps, wd, step, gscale, out)
    return list(out)


def adamw_step_dev(p: torch.Tensor, g: torch.Tensor, m: torch.Tensor, v: torch.Tensor, hyper_dev: torch.Tensor) -> None:
    """AdamW with its scalars read from device memory (hyper_dev: float32[8] view of the step-parameter buffer)."""
    assert p.is_contiguous() and g.is_contiguous() and p.numel() == g.numel() == m.numel() == v.numel()
    assert hyper_dev.dtype == torch.float32 and hyper_dev.numel() >= 8
    check(_lib.load().sn_adamw_step_dev(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), p.numel(),
                                        hyper_dev.data_ptr(), _stream()))


def adabound_step(p: torch.Tensor, g: torch.Tensor, m: torch.Tensor, v: torch.Tensor, lr: float, base_lr: float,
                  b1: float, b2: float, eps: float, wd: float, final_lr: float, gamma: float, step: int) -> None:
    assert p.is_contiguous() and g.is_contiguous() and p.numel() == g.numel() == m.numel() == v.numel()
    check(_lib.load().sn_adabound_step(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), p.numel(), lr, base_lr,
                                       b1, b2, eps, wd, final_lr, gamma, step, _stream()))


def adabound_hyper(lr: float, base_lr: float, b1: float, b2: float, eps: float, wd: float, final_lr: float,
                   gamma: float, step: int, gscale: float = 1.0):
    """The 8 fp32 scalars of sn_adabound_step_dev for optimizer step `step` (1-based), as a list of Python floats."""
    out = (C.c_float * 8)()
    _lib.load().sn_adabound_hyper(lr, base_lr, b1, b2, eps, wd, final_lr, gamma, step, gscale, out)
    return list(out)


def adabound_step_dev(p: torch.Tensor, g: torch.Tensor, m: torch.Tensor, v: torch.Tensor,
                      hyper_dev: torch.Tensor) -> None:
    """AdaBound with its scalars read from device memory (hyper_dev: float32[8] view of the step-parameter buffer)."""
    assert p.is_contiguous() and g.is_contiguous() and p.numel() == g.numel() == m.numel() == v.numel()
    assert hyper_dev.dtype == torch.float32 and hyper_dev.numel() >= 8
    check(_lib.load().sn_adabound_step_dev(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), p.numel(),
                                           hyper_dev.data_ptr(), _stream()))


def set_step_params(dst: torch.Tensor, values) -> None:
    """dst[:len(values)] <- values (<= 64 floats passed by value through one tiny launch)."""
    n = len(values)
    assert dst.dtype == torch.float32 and dst.numel() >= n and n <= 64
    arr = (C.c_float * n)(*values)
    check(_lib.load().sn_set_step_params(dst.data_ptr(), arr, n, _stream()))


def dropout_mask(seed: int, p: float, count: int, device) -> torch.Tensor:
    out = torch.empty(count, dtype=torch.uint8, device=device)
    check(_lib.load().sn_dropout_mask(seed, p, count, out.data_ptr(), _stream()))
    return out


# ---------------------------------------------------------------------------------------------
# losses
# ---------------------------------------------------------------------------------------------
def ce_loss_fwd_bwd(logits: torch.Tensor, c: int, target, weight: float,
                    loss_acc: torch.Tensor, grad: torch.Tensor) -> None:
    """target: fp32 NCHW one-hot [n,c,h,w] (argmax taken in the kernel, first maximum wins) or a uint8-label SegMap."""
    n, h, w, pitch = logits.shape
    if isinstance(target, SegMap):
        assert target.layout == LAYOUT_LABEL_U8 and target.shape == (n, c, h, w), "CE target: a uint8 label map"
        tptr, layout = target.data.data_ptr(), LAYOUT_LABEL_U8
    else:
        assert target.is_contiguous() and target.shape == (n, c, h, w)
        tptr, layout = target.data_ptr(), LAYOUT_NCHW
    check(_lib.load().sn_ce_loss_fwd_bwd(logits.data_ptr(), pitch, tptr, layout, n, h, w, c, weight,
                                         loss_acc.data_ptr(), grad.data_ptr(), grad.shape[3], _stream()))


def ce_tanh_bwd(out: torch.Tensor, c: int, target, weight: float, loss_acc: torch.Tensor,
                extra: Sequence[GradSrc], dy: Planes, ws: Optional[DetWorkspace] = None) -> None:
    """Cross entropy on the tanh head's outputs `out` (NHWC [n,h,w,c]) fused with the head's backward:
    dy <- (weight * dCE/d(out) + sum(extra)) * (1 - out^2); loss_acc += weight * CE."""
    n, h, w, pitch = out.shape
    if isinstance(target, SegMap):
        assert target.layout == LAYOUT_LABEL_U8 and target.shape == (n, c, h, w), "CE target: a uint8 label map"
        tptr, layout = target.data.data_ptr(), LAYOUT_LABEL_U8
    else:
        assert target.is_contiguous() and target.shape == (n, c, h, w)
        tptr, layout = target.data_ptr(), LAYOUT_NCHW
    arr = (SnGradSrc * _lib.SN_MAX_SRC)()
    if extra:
        _fill_srcs(arr, extra)
    assert (dy.n, dy.h, dy.w) == (n, h, w)
    args = (out.data_ptr(), pitch, tptr, layout, arr, len(extra), n, h, w, c, weight, loss_acc.data_ptr(),
            dy.hi.data_ptr(), dy.lo.data_ptr(), dy.pitch, dy.c_off, dy.fmt)
    if ws is not None:
        sl = ws.slots(1, 1)
        check(_lib.load().sn_ce_tanh_bwd_det(*args, sl.data_ptr(), sl.numel(), _stream()))
        return
    check(_lib.load().sn_ce_tanh_bwd(*args, _stream()))


def bce_logits_fwd_bwd(pred: torch.Tensor, halves: int, t0, t1: float, gscale: float,
                       loss_acc: torch.Tensor, dpred: Optional[torch.Tensor]) -> None:
    """t0 may be a device float32 tensor holding the target(s) of the half(s) (step-parameter buffer): t1 is ignored."""
    count = pred.numel() // halves
    if torch.is_tensor(t0):
        assert t0.dtype == torch.float32 and t0.numel() >= halves and t0.is_cuda
        check(_lib.load().sn_bce_logits_fwd_bwd_dev(pred.data_ptr(), count, halves, t0.data_ptr(), gscale,
                                                    loss_acc.data_ptr(), _ptr(dpred), _stream()))
        return
    check(_lib.load().sn_bce_logits_fwd_bwd(pred.data_ptr(), count, halves, t0, t1, gscale, loss_acc.data_ptr(),
                                            _ptr(dpred), _stream()))


# GANLoss objectives (include/swapnet_b200.h SN_GAN_*) and the --gan_mode values that select them
GAN_BCE, GAN_MSE, GAN_WGAN = 0, 1, 2
GAN_OBJECTIVES = {"vanilla": GAN_BCE, "lsgan": GAN_MSE, "wgan": GAN_WGAN}


def gan_loss_fwd_bwd(objective: int, pred: torch.Tensor, halves: int, t, gscale: float, loss_acc: torch.Tensor,
                     dpred: Optional[torch.Tensor], ws: Optional[DetWorkspace] = None) -> None:
    """GANLoss over `halves` (1 or 2) equal consecutive blocks of `pred`, one pass: loss_acc[h] += the unweighted batch
    mean of block h, dpred <- gscale * d(mean)/d(pred).  t holds one scalar per block: the target label of GAN_BCE /
    GAN_MSE, as a device float32 tensor (step-parameter buffer) or a sequence of floats; the sign of GAN_WGAN (+1 for a
    fake block, -1 for a real one) as a sequence of floats."""
    count = pred.numel() // halves
    if torch.is_tensor(t):
        assert objective != GAN_WGAN, "the WGAN signs are constants of the call, passed by value"
        assert t.dtype == torch.float32 and t.numel() >= halves and t.is_cuda
        t0 = t1 = 0.0
        tptr = t.data_ptr()
    else:
        assert len(t) == halves
        t0, t1, tptr = float(t[0]), float(t[-1]), None
    args = (objective, pred.data_ptr(), count, halves, t0, t1, tptr, gscale, loss_acc.data_ptr(), _ptr(dpred))
    if ws is not None:
        sl = ws.slots(1, halves)
        check(_lib.load().sn_gan_loss_fwd_bwd_det(*args, sl.data_ptr(), sl.numel(), _stream()))
        return
    check(_lib.load().sn_gan_loss_fwd_bwd_dev(*args, _stream()))


def l1_loss_fwd_bwd(a: torch.Tensor, c: int, b_nchw: torch.Tensor, weight: float, loss_acc: torch.Tensor,
                    grad: torch.Tensor, ws: Optional[DetWorkspace] = None) -> None:
    n, h, w, pitch = a.shape
    if ws is not None:
        sl = ws.slots(1, 1)
        check(_lib.load().sn_l1_loss_fwd_bwd_det(a.data_ptr(), pitch, b_nchw.data_ptr(), n, h, w, c, weight,
                                                 loss_acc.data_ptr(), grad.data_ptr(), grad.shape[3], sl.data_ptr(),
                                                 sl.numel(), _stream()))
        return
    check(_lib.load().sn_l1_loss_fwd_bwd(a.data_ptr(), pitch, b_nchw.data_ptr(), n, h, w, c, weight,
                                         loss_acc.data_ptr(), grad.data_ptr(), grad.shape[3], _stream()))


def roi_align_pack(tex_nchw: torch.Tensor, rois: torch.Tensor, pool: int, out_f32: Optional[torch.Tensor],
                   out_planes: Optional[Planes]) -> None:
    b, ch, h, w = tex_nchw.shape
    nroi = rois.shape[1]
    assert rois.shape == (b, nroi, 4) and rois.is_contiguous() and tex_nchw.is_contiguous()
    check(_lib.load().sn_roi_align_pack_fwd(
        tex_nchw.data_ptr(), b, ch, h, w, rois.data_ptr(), nroi, pool, _ptr(out_f32),
        0 if out_f32 is None else out_f32.shape[3],
        None if out_planes is None else out_planes.hi.data_ptr(),
        None if out_planes is None else out_planes.lo.data_ptr(),
        0 if out_planes is None else out_planes.pitch, 0 if out_planes is None else out_planes.c_off,
        FMT_F16 if out_planes is None else out_planes.fmt, _stream()))


def augment_channels(src, channels: int, ops_dev: torch.Tensor, op_stride: int, max_ops: int, out: torch.Tensor,
                     tmp: Optional[torch.Tensor]) -> None:
    """Per-channel geometric augmentation (datasets/data_utils.py:346-361) of a uint8 label map [n,h,w] (expanded to
    one-hot on the fly, data_utils.py:330-343) or of a dense fp32 [n,c,h,w] tensor -> out fp32 [n,c,h,w].
    ops_dev: the sn_aug_op table [n*c, op_stride] as bytes on the device (swapnet_b200/data.py builds it)."""
    labels = src.dtype == torch.uint8
    assert src.is_cuda and src.is_contiguous() and out.is_contiguous() and out.dtype == torch.float32
    n, h, w = (src.shape[0], src.shape[-2], src.shape[-1])
    assert (src.dim() == 3) if labels else (src.dtype == torch.float32 and tuple(src.shape) == (n, channels, h, w))
    assert tuple(out.shape) == (n, channels, h, w) and (tmp is None or (tmp.shape == out.shape and tmp.dtype == out.dtype))
    assert ops_dev.is_cuda and ops_dev.dtype == torch.uint8 and ops_dev.numel() == n * channels * op_stride * 72
    check(_lib.load().sn_augment_channels(src.data_ptr() if labels else None, None if labels else src.data_ptr(),
                                          n, channels, h, w, ops_dev.data_ptr(), op_stride, max_ops, out.data_ptr(),
                                          _ptr(tmp), _stream()))


def launch_count() -> int:
    return int(_lib.load().sn_launch_count())


def count_replayed(n: int) -> None:
    """Account for n kernel launches executed by a CUDA-graph replay (they bypass the per-call counter)."""
    _lib.load().sn_count_replayed(int(n))


# ---------------------------------------------------------------------------------------------
# VGG16 perceptual loss pieces (modules/losses/perceptual.py:6-79)
# ---------------------------------------------------------------------------------------------
def affine_pack(src: torch.Tensor, nhwc: bool, mul: float, add: float, dst: Planes) -> None:
    """dst[..., :16] = split(mul * src + add) (channels beyond src's are zero): `x = 2.0 * x - 1.0`."""
    assert src.dtype == torch.float32 and dst.c == 16
    if nhwc:
        n, h, w, c = src.shape
        pitch = _pitch(src)
    else:
        assert src.is_contiguous()
        n, c, h, w = src.shape
        pitch = 0
    assert (n, h, w) == (dst.n, dst.h, dst.w)
    check(_lib.load().sn_affine_pack(src.data_ptr(), LAYOUT_NHWC if nhwc else LAYOUT_NCHW, pitch, n, c, h, w, mul, add,
                                     dst.hi.data_ptr(), dst.lo.data_ptr(), dst.pitch, dst.c_off, dst.fmt, _stream()))


def relu_pool_fwd(y: torch.Tensor, c: int, out: Planes) -> None:
    n, h, w, _ = y.shape
    assert (out.n, out.h, out.w) == (n, h // 2, w // 2) and out.c >= c
    check(_lib.load().sn_relu_pool_fwd(y.data_ptr(), _pitch(y), n, h, w, c, out.hi.data_ptr(), out.lo.data_ptr(),
                                       out.pitch, out.c_off, out.fmt, _stream()))


def relu_pool_bwd(y: torch.Tensor, c: int, g_pool: Optional[torch.Tensor], g_direct: Optional[torch.Tensor],
                  dy: Planes) -> None:
    n, h, w, _ = y.shape
    assert (dy.n, dy.h, dy.w) == (n, h, w) and dy.c >= c
    assert g_pool is None or g_pool.shape[:3] == (n, h // 2, w // 2)
    assert g_direct is None or g_direct.shape[:3] == (n, h, w)
    check(_lib.load().sn_relu_pool_bwd(y.data_ptr(), _pitch(y), _ptr(g_pool), 0 if g_pool is None else _pitch(g_pool),
                                       _ptr(g_direct), 0 if g_direct is None else _pitch(g_direct), n, h, w, c,
                                       dy.hi.data_ptr(), dy.lo.data_ptr(), dy.pitch, dy.c_off, dy.fmt, _stream()))


def feat_loss_fwd_bwd(y_out: torch.Tensor, y_tgt: torch.Tensor, c: int, weight: float, gscale: float,
                      loss_acc: torch.Tensor, dx: torch.Tensor, ws: Optional[DetWorkspace] = None) -> None:
    """loss_acc += weight * sum((f_out - f_tgt)^2), f = relu(y) / (|relu(y)|_2 + 1e-8); dx = gscale * dloss/d relu(y_out)."""
    n, h, w, _ = y_out.shape
    assert y_tgt.shape[:3] == (n, h, w) and dx.shape[:3] == (n, h, w) and loss_acc.dtype == torch.float64
    args = (y_out.data_ptr(), _pitch(y_out), y_tgt.data_ptr(), _pitch(y_tgt), n * h * w, c, weight, gscale,
            loss_acc.data_ptr(), dx.data_ptr(), _pitch(dx))
    if ws is not None:
        sl = ws.slots(1, 1)
        check(_lib.load().sn_feat_loss_fwd_bwd_det(*args, sl.data_ptr(), sl.numel(), _stream()))
        return
    check(_lib.load().sn_feat_loss_fwd_bwd(*args, _stream()))


def _gram_strides(x: torch.Tensor, nhwc: bool):
    if nhwc:
        n, h, w, c = x.shape
        assert x.is_contiguous()
        return n, c, h * w, h * w * c, 1, c
    n, c, h, w = x.shape
    assert x.is_contiguous()
    return n, c, h * w, c * h * w, h * w, 1


def gram_rows(a: torch.Tensor, b: torch.Tensor, nhwc: bool, out: torch.Tensor,
              ws: Optional[DetWorkspace] = None) -> None:
    """out [n_a*c, n_b*c] (float64) = A B^T: the rows (sample, channel) of `a` against those of `b` (same layout and
    image size; b may hold more samples, e.g. every rank's).  With a = b: gram_matrix(a) of perceptual.py:6-10.  Any
    number of rows."""
    na, c, npix, an, ac, ap = _gram_strides(a, nhwc)
    nb, cb, npix_b, bn, bc, bp = _gram_strides(b, nhwc)
    assert (cb, npix_b) == (c, npix) and out.dtype == torch.float64 and out.shape == (na * c, nb * c)
    assert out.is_contiguous()
    args = (a.data_ptr(), an, ac, ap, na, b.data_ptr(), bn, bc, bp, nb, c, npix, out.data_ptr())
    if ws is not None:
        sl = ws.get(int(_lib.load().sn_gram_rows_det_slots(na * c, nb * c)))
        check(_lib.load().sn_gram_rows_det(*args, sl.data_ptr(), sl.numel(), _stream()))
        return
    check(_lib.load().sn_gram_rows(*args, _stream()))


def gram_rows_mse(g_out: torch.Tensor, g_tgt: torch.Tensor, weight: float, loss_acc: torch.Tensor, m: torch.Tensor,
                  gscale: float = 1.0) -> None:
    """For [R_l, R] row blocks: loss_acc += weight * sum((g_out - g_tgt)^2) / R^2; m (fp32 [R_l, R]) = gscale *
    (d/d g_out + transpose) on those rows."""
    rows_l, rows = g_out.shape
    assert g_tgt.shape == g_out.shape and m.dtype == torch.float32 and m.shape == g_out.shape
    assert g_out.is_contiguous() and g_tgt.is_contiguous() and m.is_contiguous() and loss_acc.dtype == torch.float64
    check(_lib.load().sn_gram_rows_mse(g_out.data_ptr(), g_tgt.data_ptr(), rows_l, rows, weight, gscale,
                                       loss_acc.data_ptr(), m.data_ptr(), _stream()))


def gram_rows_bwd(m: torch.Tensor, x: torch.Tensor, nhwc: bool, dx: torch.Tensor, accumulate: bool) -> None:
    """dx (NHWC fp32 [R_l/c, h, w, >=c]) (+)= m @ X, m [R_l, n*c] against the n*c rows X of x."""
    n, c, npix, sn, sc, sp = _gram_strides(x, nhwc)
    rows_l = m.shape[0]
    assert m.dtype == torch.float32 and m.is_contiguous() and m.shape[1] == n * c
    assert dx.shape[0] * c == rows_l and dx.shape[1] * dx.shape[2] == npix
    check(_lib.load().sn_gram_rows_bwd(m.data_ptr(), rows_l, x.data_ptr(), sn, sc, sp, n, c, npix, dx.data_ptr(),
                                       _pitch(dx), 1 if accumulate else 0, _stream()))


# ---------------------------------------------------------------------------------------------
# one-output-channel conv helpers (csrc/patch_logits.cu)
# ---------------------------------------------------------------------------------------------
def tap_sum_fwd(p: torch.Tensor, k: int, pad: int, bias: Optional[torch.Tensor], y: torch.Tensor) -> None:
    n, h, w, _ = p.shape
    assert y.shape[:3] == (n, h + 2 * pad - k + 1, w + 2 * pad - k + 1)
    check(_lib.load().sn_tap_sum_fwd(p.data_ptr(), _pitch(p), n, h, w, k, pad, _ptr(bias), y.data_ptr(), _pitch(y),
                                     _stream()))


def to_one_fwd(x: Planes, weight: torch.Tensor, p: torch.Tensor) -> None:
    """p[n,h,w,t] = sum_c x[n,h,w,c] * weight[0,c,t] (t = 4*kh + kw) on the CUDA cores; x is read once."""
    assert weight.is_contiguous() and weight.shape[0] == 1 and tuple(weight.shape[2:]) == (4, 4)
    assert p.dtype == torch.float32 and p.shape[:3] == (x.n, x.h, x.w) and x.c_off % 8 == 0
    check(_lib.load().sn_to_one_fwd(x.hi_ptr, x.lo_ptr, x.pitch, x.fmt, x.n * x.h * x.w, weight.shape[1],
                                    weight.data_ptr(), 4, p.data_ptr(), _pitch(p), _stream()))


def to_one_wgrad(x: Planes, dy: Planes, pad: int, dw: torch.Tensor, ws: Optional[DetWorkspace] = None) -> None:
    """dw[0,c,kh,kw] += sum_px x[px,c] * dy[px - (kh,kw) + pad] (dy: channel 0 of its planes)."""
    assert dw.is_contiguous() and dw.dtype == torch.float32 and (dy.h, dy.w) == (x.h + 2 * pad - 3, x.w + 2 * pad - 3)
    if ws is not None:
        sl = ws.get(int(_lib.load().sn_to_one_wgrad_det_slots(dw.shape[1])), torch.float32)
        check(_lib.load().sn_to_one_wgrad_det(x.hi_ptr, x.lo_ptr, x.pitch, x.fmt, x.n, x.h, x.w, dw.shape[1], dy.hi_ptr,
                                              dy.lo_ptr, dy.pitch, dy.fmt, 4, pad, dw.data_ptr(), sl.data_ptr(),
                                              sl.numel(), _stream()))
        return
    check(_lib.load().sn_to_one_wgrad(x.hi_ptr, x.lo_ptr, x.pitch, x.fmt, x.n, x.h, x.w, dw.shape[1], dy.hi_ptr,
                                      dy.lo_ptr, dy.pitch, dy.fmt, 4, pad, dw.data_ptr(), _stream()))


def to_one_dgrad(dy: Planes, weight: torch.Tensor, pad: int, dx: torch.Tensor) -> None:
    """dx[n,h,w,c] = sum_t dy[px - off_t] * weight[0,c,t] (fp32 NHWC)."""
    n, h, w, _ = dx.shape
    assert (dy.h, dy.w) == (h + 2 * pad - 3, w + 2 * pad - 3)
    check(_lib.load().sn_to_one_dgrad(dy.hi_ptr, dy.lo_ptr, dy.pitch, dy.fmt, n, h, w, weight.shape[1],
                                      weight.data_ptr(), 4, pad, dx.data_ptr(), _pitch(dx), _stream()))


# ---------------------------------------------------------------------------------------------
# 1x1 PixelGAN discriminator (csrc/pixel_disc.cu)
# ---------------------------------------------------------------------------------------------
def pixel_desc(x: Planes, net, scales: torch.Tensor, nsplit: int, **kw) -> "_lib.SnPixelDesc":
    """Descriptor of the PixelGAN passes over the operand planes x [n, h, w, 16 | 32] (fp16-split; its bf16 twin feeds
    dW1).  net: modules.PixelDiscriminator; scales [2, 2]: (s, 1/s) of net.0 and net.2 weights (weight_scale_multi).
    kw: the remaining sn_pixel_desc fields, tensors or None."""
    d = _lib.SnPixelDesc()
    d.x_hi, d.x_lo = x.hi_ptr, x.lo_ptr
    if x.twin is not None:
        d.xb_hi, d.xb_lo = x.twin.hi_ptr, x.twin.lo_ptr
    d.x_pitch, d.x_c, d.n, d.hw, d.cin = x.pitch, x.c, x.n, x.h * x.w, net.input_nc
    c0, c2, c5 = net.net[0], net.net[2], net.net[5]
    d.w1, d.b1, d.w2, d.b2 = c0.weight.data_ptr(), c0.bias.data_ptr(), c2.weight.data_ptr(), _ptr(c2.bias)
    d.w3, d.b3 = c5.weight.data_ptr(), _ptr(c5.bias)
    d.scale1, d.scale2 = scales[0].data_ptr(), scales[1].data_ptr()
    d.norm, d.nsplit, d.slope, d.eps = int(net.norm == "instance"), nsplit, 0.2, IN_EPS
    for k, v in kw.items():
        setattr(d, k, v.data_ptr() if torch.is_tensor(v) else v)
    return d


def pixel_pass(name: str, d: "_lib.SnPixelDesc", ws: Optional[DetWorkspace] = None) -> None:
    """One PixelGAN pass: name in fwd_stats, fwd, bwd_reduce, bwd_apply.  ws: deterministic reductions."""
    lib = _lib.load()
    if ws is not None:
        sl = ws.get(int(lib.sn_pixel_det_slots(d.n, d.cin)))
        d.slots, d.slots_cap = sl.data_ptr(), sl.numel()
    else:
        d.slots, d.slots_cap = None, 0
    check(getattr(lib, "sn_pixel_" + name)(C.byref(d), _stream()))
