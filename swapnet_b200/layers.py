"""Conv layers of the hot path as bundles of pre-built tensor-core plans.

A `ConvLayer` owns, for one reference conv (kinds in lowering.py), the packed split-bf16 weight
matrices and the sn_plan handles of its forward, input-gradient and weight-gradient launches.
All buffers are allocated once (shapes are static per model/batch), so a training step is a
fixed sequence of launches: `pack()` once per step after the optimizer update, then
`forward()`, `backward()`.
"""
from __future__ import annotations

from typing import List, Optional

import torch

from . import lowering as L
from . import ops
from .ops import ACT_NONE, PackedWeights, Planes


class ConvLayer:
    def __init__(self, kind: str, weight: torch.Tensor, bias: Optional[torch.Tensor], x: Planes, *,
                 nsplit: int = 3, act: int = ACT_NONE, name: str = "", det_ws: Optional[ops.DetWorkspace] = None):
        """x: input operand planes (for 'conv3r' the reflect-padded [h+2, w+2] planes).
        weight / bias: the torch parameters (torch layout, fp32, on the same device).
        det_ws: deterministic weight and bias gradients (bit-identical runs); the bias-gradient reduction uses this
        workspace, so it must not be shared with launches that can overlap this layer's backward()."""
        assert kind in L.KINDS
        self.kind, self.name, self.nsplit, self.act = kind, name, nsplit, act
        self.det_ws = det_ws
        self.weight, self.bias = weight, bias
        self.x = x
        dev = weight.device
        if kind == "convT4s2":
            self.cin, self.cout = weight.shape[0], weight.shape[1]
        else:
            self.cout, self.cin = weight.shape[0], weight.shape[1]
        self.in_h, self.in_w = (x.h - 2, x.w - 2) if kind == "conv3r" else (x.h, x.w)
        self.out_h, self.out_w = L.out_hw(kind, self.in_h, self.in_w)
        self.n = x.n
        self.k_pad = x.c                       # input channels as the planes carry them (16, 32 or 64k)
        assert (self.k_pad % 64 == 0 or self.k_pad in (16, 32)) and self.k_pad >= self.cin, (name, x.c, self.cin)
        self.block_n = L.pick_block_n(self.cout)
        self.t = L.ntaps(kind)
        self.wscale = torch.ones(2, dtype=torch.float32, device=dev)  # (s, 1/s), shared by fwd and dgrad packs
        self.stacked = kind == "head" and self.cout <= L.HEAD_SLOT and self.k_pad % 64 == 0
        if self.stacked:
            self.rows_pad = 4 * L.HEAD_SLOT
            self.wp = PackedWeights(self.rows_pad, 9 * self.k_pad, dev, self.wscale)
        elif kind == "head":
            self.rows_pad = (self.cout + self.block_n - 1) // self.block_n * self.block_n
            self.wp = PackedWeights(self.rows_pad, 25 * self.k_pad, dev, self.wscale)
        else:
            # narrow operands: the tap count is padded to a multiple of 64/k_pad with all-zero K columns
            self.wp = PackedWeights(self.cout, self._tpad(self.t, self.k_pad) * self.k_pad, dev, self.wscale)
        self.fwd_plans: List[ops.Plan] = []
        self.y: Optional[torch.Tensor] = None
        # backward state
        self.wd: Optional[PackedWeights] = None
        self.dy: Optional[Planes] = None
        self.dgrad_plans: List[ops.Plan] = []
        self.wgrad_plan: Optional[ops.Plan] = None
        self.dx: Optional[torch.Tensor] = None
        self.wgrad_out: Optional[torch.Tensor] = None
        self.bgrad_out: Optional[torch.Tensor] = None
        self._geff: Optional[torch.Tensor] = None
        self._bscratch: Optional[torch.Tensor] = None

    @staticmethod
    def _tpad(t: int, k: int) -> int:
        tps = max(1, 64 // k)
        return (t + tps - 1) // tps * tps

    # ---- forward --------------------------------------------------------------------------
    def bind_forward(self, y: torch.Tensor, y_c_off: int = 0, stats: Optional[torch.Tensor] = None) -> None:
        """y: fp32 NHWC [n, out_h, out_w, pitch]; the conv output (+bias, +act) is written to
        channels [y_c_off, y_c_off + cout).  stats (float64 [n, cout, 2]): ask the launch to accumulate the
        InstanceNorm statistics of y as it writes it; `self.fused_stats` says whether it will (single-launch layers whose
        tiles stay inside one image), else the caller runs ops.plane_stats."""
        assert y.shape[:3] == (self.n, self.out_h, self.out_w), (self.name, y.shape, self.out_h, self.out_w)
        self.y = y
        self.fwd_plans = []
        self.fused_stats = False
        if y_c_off != 0 or self.act != ACT_NONE:
            stats = None
        if self.stacked:
            d = ops.tap_gemm_desc(self.x, L.head_stacked_spec(self.in_h, self.in_w), self.wp, self.k_pad, y,
                                  4 * L.HEAD_SLOT, bias=self.bias, act=self.act, nsplit=self.nsplit,
                                  block_n=4 * L.HEAD_SLOT, out_c_off=y_c_off, stack_slot=L.HEAD_SLOT, stack_c=self.cout)
            self.fwd_plans.append(ops.tap_gemm_plan(d, keep=(self.x.hi, self.x.lo, self.wp.hi, self.wp.lo, y)))
            self.fwd_plans[-1].tag = ("fwd", self.name)
            return
        specs = L.forward_specs(self.kind, self.in_h, self.in_w)
        merged = ops.merge_phase_specs(specs)
        if merged is not None and (self.k_pad >= 64 or (len(merged.taps) // 4) % (64 // self.k_pad) == 0):
            d = ops.tap_gemm_desc(self.x, merged, self.wp, self.k_pad, y, self.cout, bias=self.bias, act=self.act,
                                  nsplit=self.nsplit, block_n=self.block_n, out_c_off=y_c_off, nphase=4, stats=stats)
            self.fwd_plans.append(ops.tap_gemm_plan(d, keep=(self.x.hi, self.x.lo, self.wp.hi, self.wp.lo, y)))
            self.fwd_plans[-1].tag = ("fwd", self.name)
            self.fused_stats = stats is not None and self.fwd_plans[-1].has_stats
            specs = []
        for spec in specs:
            kw = {}
            if self.kind == "head":
                p = spec.w_phase
                nt = L.head_neff(p >> 1) * L.head_neff(p & 1)
                kw = dict(w_elem_off=self.rows_pad * self.k_pad * L.HEAD_PHASE_OFF[p], w_rows=self.rows_pad,
                          w_k=nt * self.k_pad)
            one = len(specs) == 1 and self.kind != "head"
            d = ops.tap_gemm_desc(self.x, spec, self.wp, self.k_pad, y, self.cout, bias=self.bias,
                                  act=self.act, nsplit=self.nsplit, block_n=self.block_n, out_c_off=y_c_off,
                                  stats=stats if one else None, **kw)
            self.fwd_plans.append(ops.tap_gemm_plan(d, keep=(self.x.hi, self.x.lo, self.wp.hi, self.wp.lo, y)))
            self.fwd_plans[-1].tag = ("fwd", self.name)
            if one:
                self.fused_stats = stats is not None and self.fwd_plans[-1].has_stats

    def register_packs(self, table: "ops.PackTable") -> bool:
        """Register this layer's scale and generic packs with the network's PackTable; returns True when a separate
        `pack_extra()` call is still needed after the table ran (the head's effective-tap packs)."""
        table.add_scale(self.weight, self.wscale)
        if self.kind == "head":
            return True
        table.add_pack(self.weight, self.kind, False, self.k_pad, self.wp)
        if self.wd is not None and self.dgrad_plans:
            table.add_pack(self.weight, self.kind, True, self.dy.c, self.wd)
        return False

    def pack_extra(self) -> None:
        assert self.kind == "head"
        if self.stacked:
            ops.pack_head_stacked(self.weight, L.HEAD_SLOT, self.k_pad, self.wp)
        else:
            ops.pack_head_weights(self.weight, self.rows_pad, self.k_pad, False, self.wp)
        if self.wd is not None and self.dgrad_plans:
            ops.pack_head_weights(self.weight, 0, self.dy.c, True, self.wd)

    def pack(self) -> None:
        """Re-pack the (updated) torch weights into the kernel layouts: the steps of Engine.pack() with a table of this
        layer alone (tests, single layers).  The table is rebuilt on every call: bind_backward() adds a pack."""
        table = ops.PackTable(self.weight.device)
        extra = self.register_packs(table)
        table.run()
        if extra:
            self.pack_extra()

    def forward(self) -> None:
        for p in self.fwd_plans:
            p.run()

    # ---- backward -------------------------------------------------------------------------
    def bind_backward(self, dy: Planes, dx: Optional[torch.Tensor], wgrad: Optional[torch.Tensor],
                      bgrad: Optional[torch.Tensor] = None, dx_c_off: int = 0) -> None:
        """dy: split planes of dL/d(conv output) [n, out_h, out_w, pad64(cout)].
        dx: fp32 NHWC gradient w.r.t. the input operand ([n, h+2, w+2, .] for conv3r) or None.
        wgrad / bgrad: fp32 tensors in torch layout that receive (+=) the parameter gradients
        (must be zeroed by the caller once per step)."""
        dev = self.weight.device
        assert (dy.n, dy.h, dy.w) == (self.n, self.out_h, self.out_w), (self.name, dy.h, dy.w)
        assert (dy.c % 64 == 0 or dy.c in (16, 32)) and dy.c >= self.cout
        self.dy = dy
        self.dx = dx
        self.dgrad_plans = []
        if dx is not None:
            if self.kind == "head":
                self.wd = PackedWeights(self.cin, self._tpad(25, dy.c) * dy.c, dev, fmt=dy.fmt)
            else:
                self.wd = PackedWeights(self.cin, self._tpad(self.t, dy.c) * dy.c, dev, fmt=dy.fmt)
            bn = L.pick_block_n(self.cin)
            dspecs = L.dgrad_specs(self.kind, self.in_h, self.in_w)
            merged = ops.merge_phase_specs(dspecs)
            if merged is not None and (dy.c >= 64 or (len(merged.taps) // 4) % (64 // dy.c) == 0):
                d = ops.tap_gemm_desc(dy, merged, self.wd, dy.c, dx, self.cin, nsplit=self.nsplit, block_n=bn,
                                      out_c_off=dx_c_off, nphase=4)
                self.dgrad_plans.append(ops.tap_gemm_plan(d, keep=(dy.hi, dy.lo, self.wd.hi, self.wd.lo, dx)))
                self.dgrad_plans[-1].tag = ("dgrad", self.name)
                dspecs = []
            for spec in dspecs:
                d = ops.tap_gemm_desc(dy, spec, self.wd, dy.c, dx, self.cin, nsplit=self.nsplit, block_n=bn,
                                      out_c_off=dx_c_off)
                self.dgrad_plans.append(ops.tap_gemm_plan(d, keep=(dy.hi, dy.lo, self.wd.hi, self.wd.lo, dx)))
                self.dgrad_plans[-1].tag = ("dgrad", self.name)
        self.wgrad_out = wgrad
        self.wgrad_plan = None
        if wgrad is not None:
            assert wgrad.shape == self.weight.shape and wgrad.is_contiguous()
            (ws,) = L.wgrad_specs(self.kind, self.in_h, self.in_w)
            x_is_dy = ws.x_is == "dy"
            # the activation operand must come in the gradient's format: its bf16-split twin
            xin = self.x if self.x.fmt == dy.fmt else self.x.twin
            assert xin is not None, f"{self.name}: wgrad needs a {dy.fmt}-format twin of the input planes (dual=True)"
            xs, ys = (dy, xin) if x_is_dy else (xin, dy)
            cx, cy = (self.cout, self.cin) if x_is_dy else (self.cin, self.cout)
            s_row, s_col = L.wgrad_out_strides(self.kind, self.cin, self.cout, x_is_dy)
            if self.kind == "head":
                self._geff = torch.zeros(self.cout, 25, self.cin, dtype=torch.float32, device=dev)
                out, tap_off = self._geff, [t * self.cin for t in ws.tap_ids]
            else:
                out, tap_off = wgrad, list(ws.tap_ids)
            # the 128-row M side must carry >= 64 channels; otherwise it is the operand with more channels
            if xs.c < 64 or ys.c < 64:
                swap = xs.c < 64
                assert (ys.c if swap else xs.c) >= 64, f"{self.name}: both wgrad operands are narrow"
            else:
                swap = cy > cx
            d = ops.wgrad_desc(xs, ys, ws, out, s_row, s_col, tap_off, cx, cy, swap=swap, nsplit=self.nsplit,
                               deterministic=self.det_ws is not None)
            self.wgrad_plan = ops.wgrad_plan(d, keep=(xs.hi, xs.lo, ys.hi, ys.lo, out))
            self.wgrad_plan.tag = ("wgrad", self.name)
        self.bgrad_out = bgrad
        if bgrad is not None:
            self._bscratch = torch.zeros(self.cout, dtype=torch.float64, device=dev)

    def backward(self, dgrad: bool = True, wgrad: bool = True, bias: bool = True) -> None:
        """bias=False: the caller already accumulated the bias gradient (fused into norm_act_bwd)."""
        if dgrad:
            for p in self.dgrad_plans:
                p.run()
        if wgrad and self.wgrad_plan is not None:
            if self._geff is not None:
                self._geff.zero_()
            self.wgrad_plan.run()
            if self._geff is not None:
                ops.fold_head_wgrad(self._geff, self.cout, self.cin, self.wgrad_out)
        if wgrad and bias and self.bgrad_out is not None:
            ops.bias_grad(self.dy, self.cout, self._bscratch, self.bgrad_out, ws=self.det_ws)


class ToOneConvLayer:
    """Conv2d(cin, 1, k4, s1, p1) — the PatchGAN logits layer (modules/discriminators.py:131) — on the CUDA cores.

    A conv with one output channel is an HBM-bound op (1 GMAC over a 260 MB input at batch 32); a GEMM with N = 1 —
    or N = 16 through the tap factorisation below — leaves the tensor core waiting for its operand loads (round 1:
    forward at 4 TFLOP/s, weight gradient at 2.4).  csrc/patch_logits.cu streams the input once per pass instead:
        P[px, t]   = sum_c x[px, c] W[0, c, t]            ops.to_one_fwd   (fp32 FMAs on the fp16-split input)
        y[o]       = bias + sum_t P[o + off_t, t]         ops.tap_sum_fwd
        dW[0,c,t]  = sum_px x[px, c] dy[px - off_t]       ops.to_one_wgrad
        dx[px, c]  = sum_t dy[px - off_t] W[0, c, t]      ops.to_one_dgrad
    No packed weights: the kernels read the torch parameter itself.  Same interface as ConvLayer."""

    K, PAD = 4, 1

    def __init__(self, kind: str, weight: torch.Tensor, bias: Optional[torch.Tensor], x: Planes, *,
                 nsplit: int = 3, act: int = ACT_NONE, name: str = "", det_ws: Optional[ops.DetWorkspace] = None):
        assert kind == "conv4s1" and weight.shape[0] == 1 and tuple(weight.shape[2:]) == (4, 4) and act == ACT_NONE
        self.kind, self.name, self.nsplit, self.act = kind, name, nsplit, act
        self.det_ws = det_ws
        self.weight, self.bias, self.x = weight, bias, x
        dev = weight.device
        self.cout, self.cin = 1, weight.shape[1]
        self.in_h, self.in_w = x.h, x.w
        self.out_h, self.out_w = L.out_hw(kind, x.h, x.w)
        self.n, self.k_pad, self.t = x.n, x.c, 16
        assert self.cin % 8 == 0 and self.cin <= 1024 and x.c >= self.cin and x.c_off % 8 == 0
        self.p = torch.zeros(self.n, self.in_h, self.in_w, 16, device=dev)         # per-tap products
        self.fwd_plans: List[ops.Plan] = []     # no tensor-core plans: nothing for the GEMM roofline trace
        self.dgrad_plans: List[ops.Plan] = []
        self.wgrad_plan: Optional[ops.Plan] = None
        self.y = self.dy = self.dx = None
        self.wgrad_out = self.bgrad_out = self._bscratch = None

    def bind_forward(self, y: torch.Tensor, y_c_off: int = 0, stats: Optional[torch.Tensor] = None) -> None:
        assert y.shape[:3] == (self.n, self.out_h, self.out_w) and y_c_off == 0
        self.y = y
        self.fused_stats = False

    def register_packs(self, table) -> bool:
        return False            # the kernels read the torch parameter itself

    def pack(self) -> None:
        pass

    def forward(self) -> None:
        ops.to_one_fwd(self.x, self.weight, self.p)
        ops.tap_sum_fwd(self.p, self.K, self.PAD, self.bias, self.y)

    def bind_backward(self, dy: Planes, dx: Optional[torch.Tensor], wgrad: Optional[torch.Tensor],
                      bgrad: Optional[torch.Tensor] = None, dx_c_off: int = 0) -> None:
        assert (dy.n, dy.h, dy.w) == (self.n, self.out_h, self.out_w) and dx_c_off == 0
        assert dx is None or dx.shape[3] == self.cin
        self.dy, self.dx = dy, dx
        self.wgrad_out = wgrad
        if wgrad is not None:
            assert wgrad.shape == self.weight.shape and wgrad.is_contiguous()
        self.bgrad_out = bgrad
        if bgrad is not None:
            self._bscratch = torch.zeros(1, dtype=torch.float64, device=self.weight.device)

    def backward(self, dgrad: bool = True, wgrad: bool = True, bias: bool = True) -> None:
        if dgrad and self.dx is not None:
            ops.to_one_dgrad(self.dy, self.weight, self.PAD, self.dx)
        if wgrad and self.wgrad_out is not None:
            ops.to_one_wgrad(self.x, self.dy, self.PAD, self.wgrad_out, ws=self.det_ws)  # fp16-split planes: no twin
        if wgrad and self.bgrad_out is not None:
            ops.bias_grad(self.dy, 1, self._bscratch, self.bgrad_out, ws=self.det_ws)
