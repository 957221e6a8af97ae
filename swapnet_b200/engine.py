"""Forward/backward engines of the SwapNet networks on the B200 library.

An engine turns one parameter container (swapnet_b200.modules) into a static launch plan for a
fixed (batch, size): every activation buffer, packed weight matrix and TMA-backed sn_plan is
created once; a training step is then a fixed sequence of kernel launches with no allocation
and no host synchronisation.

Dataflow conventions
  * activations that feed a conv live as split-bf16 NHWC `Planes`; the producer stage writes
    straight into the channel slice of the consumer's concat buffer, so torch.cat
    (swapnet_modules.py:131, layers.py:42,61, pix2pix_modules.py:262) never materialises;
  * every stage keeps its raw conv output `y` (fp32 NHWC) + InstanceNorm statistics; the
    normalise/activate/dropout step is one fused kernel forward and two backward;
  * gradients w.r.t. activations are fp32 NHWC tensors; a stage's backward takes a list of
    (tensor, channel offset) sources and sums them on the fly.

Reference graphs: WarpModule.forward swapnet_modules.py:92-151; NLayerDiscriminator
discriminators.py:111-136; TextureModule.forward swapnet_modules.py:231-260 + UnetGenerator
pix2pix_modules.py:113-262.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import torch
from torch import nn

from . import lowering as L
from . import modules as M
from . import ops
from .layers import ConvLayer, ToOneConvLayer
from .ops import ACT_LRELU, ACT_NONE, ACT_RELU, ACT_TANH, FMT_BF16, GradSrc, Planes


def _mix_seed(step_seed: int, stage_id: int) -> int:
    return (step_seed * 0x9E3779B1 + stage_id * 0x85EBCA77 + 0x165667B1) & 0xFFFFFFFFFFFF


class Stage:
    """conv -> [InstanceNorm | BatchNorm] -> activation -> [dropout] (-> + residual), output written as operand
    planes (and/or fp32).  `plain=True`: the conv output itself (after the epilogue activation) is
    the stage output (head conv with tanh, PatchGAN logits).

    norm=True with `bn` (an nn.BatchNorm2d of the container): batch normalisation with bn's weight, bias and running
    buffers, which the stage reads and updates in place.  The batch is `groups` consecutive groups of samples, each
    normalised as a call of its own; Engine.training selects batch (train) or running (eval) statistics."""

    def __init__(self, eng: "Engine", name: str, kind: str, conv: nn.Module, x: Planes, *,
                 out: Optional[Planes] = None, norm: bool = False, act: int = ACT_NONE, slope: float = 0.2,
                 drop_p: float = 0.0, reflect_out: bool = False, residual: Optional[torch.Tensor] = None,
                 out_f32: Optional[torch.Tensor] = None, plain: bool = False, epi_act: int = ACT_NONE,
                 need_dx: bool = True, y: Optional[torch.Tensor] = None, out_relu: Optional[Planes] = None,
                 bn: Optional[nn.BatchNorm2d] = None, groups: int = 1):
        assert bn is None or norm, "a BatchNorm stage is a normalised stage"
        self.eng, self.name, self.kind = eng, name, kind
        self.bn, self.groups = bn, groups
        self.id = len(eng.stages)
        eng.stages.append(self)
        dev = eng.device
        # a stride-1 conv with ONE output channel (the PatchGAN logits) runs as 1-tap GEMMs (layers.ToOneConvLayer)
        to_one = (kind == "conv4s1" and conv.out_channels == 1 and epi_act == ACT_NONE and conv.in_channels % 8 == 0
                  and conv.in_channels <= 1024 and x.c_off % 8 == 0)
        self.layer = (ToOneConvLayer if to_one else ConvLayer)(
            kind, conv.weight.data, None if conv.bias is None else conv.bias.data, x, nsplit=eng.nsplit, act=epi_act,
            name=name, det_ws=eng.det_ws_side)
        self.conv = conv
        ly = self.layer
        self.n, self.oh, self.ow, self.cout = ly.n, ly.out_h, ly.out_w, ly.cout
        self.y = y if y is not None else torch.zeros(self.n, self.oh, self.ow, self.cout, device=dev)
        # InstanceNorm statistics ride on the GEMM epilogue where a tile never spans two images (ConvLayer.fused_stats),
        # except in deterministic mode: the epilogue adds them with atomics, ops.plane_stats can add them in order
        self.stats = torch.zeros(self.n, self.cout, 2, dtype=torch.float64, device=dev) if norm else None
        ly.bind_forward(self.y, stats=None if eng.det_ws is not None else self.stats)
        self.norm, self.act, self.slope, self.drop_p = norm, act, slope, drop_p
        self.out, self.reflect_out, self.residual, self.out_f32 = out, reflect_out, residual, out_f32
        self.plain, self.epi_act, self.need_dx = plain, epi_act, need_dx
        self.out_relu = out_relu   # pix2pix skip: a second consumer reads relu() of the same pre-activation
        self.dy: Optional[Planes] = None
        self.dx: Optional[torch.Tensor] = None
        self.gstats = None
        # batch statistics across ranks: this rank's per-group partials and every rank's, gathered
        self.bn_part = self.bn_gathered = None
        if bn is not None and eng.bn_sync is not None:
            self.bn_part, self.bn_gathered = eng.bn_sync.buffers(groups, self.cout, dev)

    def drop_offset(self) -> int:
        """Keep-mask index of this stage's first element: the masks are indexed by GLOBAL sample (Engine.sample_base =
        global index of local sample 0), so a data-parallel shard, or a batch-1 run of sample i, draws the masks the
        full batch would (SURVEY §8e ii)."""
        return self.eng.sample_base * self.oh * self.ow * self.cout

    def nominal_macs(self) -> int:
        """Dense multiply-accumulates of the reference op for this stage's batch (SURVEY §8d:
        Conv2d out_elems*Cin*k*k, ConvTranspose2d in_elems*Cout*k*k; zero taps of padding and
        up-sampling counted)."""
        ly = self.layer
        k2 = 9 if self.kind in ("conv3r", "conv3z") else 16
        if self.kind == "convT4s2":
            return self.n * ly.in_h * ly.in_w * ly.cin * ly.cout * k2
        return self.n * self.oh * self.ow * ly.cout * ly.cin * k2

    # ---- forward ----
    def _affine(self):
        return (None, None) if self.bn is None else (self.bn.weight.data, self.bn.bias.data)

    def forward(self) -> None:
        self.layer.forward()
        if self.plain:
            return
        fused = getattr(self.layer, "fused_stats", False)
        if self.bn is not None:
            if not self.eng.training:
                ops.bn_eval_stats(self.stats, self.n, self.cout, self.bn)
            else:
                if not fused:
                    ops.plane_sums(self.y, self.cout, self.stats, ws=self.eng.det_ws)
                if self.bn_part is not None:
                    ops.bn_group_sums(self.stats, self.n, self.cout, self.groups, self.oh * self.ow, self.bn_part)
                    self.eng.bn_sync.gather(self.bn_part, self.bn_gathered)
                    ops.bn_finalize_gathered(self.stats, self.n, self.cout, self.groups, self.bn_gathered, self.bn)
                else:
                    ops.bn_finalize(self.stats, self.n, self.cout, self.groups, self.oh * self.ow, self.bn)
        elif self.norm:
            if fused:
                ops.stats_finalize(self.stats, self.n * self.cout, self.oh * self.ow)
            else:
                ops.plane_stats(self.y, self.cout, self.stats, ws=self.eng.det_ws)
        gamma, beta = self._affine()
        p = self.drop_p if self.eng.training else 0.0
        ops.norm_act_fwd(self.y, self.cout, self.stats, self.act, self.slope, p,
                         _mix_seed(self.eng.seed, self.id), residual=self.residual, out=self.out,
                         reflect_pad=self.reflect_out, out_f32=self.out_f32, drop_offset=self.drop_offset(),
                         seed_dev=self.eng.seed_dev, stage_id=self.id, gamma=gamma, beta=beta)
        if self.out_relu is not None:
            ops.norm_act_fwd(self.y, self.cout, self.stats, ACT_RELU, 0.0, 0.0, 0, out=self.out_relu, gamma=gamma,
                             beta=beta)

    # ---- backward ----
    def bind_backward(self, wgrad: bool = True) -> None:
        dev = self.eng.device
        ly = self.layer
        dyc = L.padc(self.cout)
        if dyc < 64 and ly.x.c < 64:   # the weight-gradient GEMM needs one operand with >= 64 channels
            dyc = 64
        self.dy = Planes(self.n, self.oh, self.ow, dyc, dev, fmt=FMT_BF16)  # gradients: fp32 range
        if self.need_dx:
            ih, iw = (ly.in_h + 2, ly.in_w + 2) if self.kind == "conv3r" else (ly.in_h, ly.in_w)
            self.dx = torch.zeros(self.n, ih, iw, (ly.cin + 3) // 4 * 4, device=dev)[..., :ly.cin]
        wg = self.conv.weight.grad if wgrad else None
        bg = self.conv.bias.grad if (wgrad and self.conv.bias is not None) else None
        ly.bind_backward(self.dy, self.dx, wg, bg)
        if self.norm:
            self.gstats = torch.zeros(self.n, self.cout, 2, dtype=torch.float64, device=dev)

    def backward(self, srcs: Optional[Sequence[GradSrc]], wgrad: bool = True) -> None:
        """srcs None: `self.dy` already holds dL/d(conv output) (written by a fused loss kernel, ops.ce_tanh_bwd)."""
        if srcs is None:
            pass
        elif self.plain and self.epi_act == ACT_TANH:
            ops.tanh_bwd(srcs, self.y, self.cout, self.dy)
        else:
            p = 0.0 if self.plain else (self.drop_p if self.eng.training else 0.0)
            # the conv's bias gradient (sum of dy over pixels) rides on the pass that writes dy where it can
            bg = None
            if wgrad and self.conv.bias is not None and self.conv.bias.grad is not None and ops.fused_bias_grad_ok(self.cout) \
                    and self.cout % 4 == 0 and getattr(self.layer, "bgrad_out", None) is not None \
                    and self.eng.det_ws is None:   # the fused bias gradient adds its block sums with atomics
                bg = self.conv.bias.grad
            bn = bn_grads = None
            if self.bn is not None and not self.plain:
                bn = self._affine()
                if wgrad and self.bn.weight.grad is not None:
                    bn_grads = (self.bn.weight.grad, self.bn.bias.grad)
            args = (srcs, self.y, self.cout, None if self.plain else self.stats, ACT_NONE if self.plain else self.act,
                    self.dy, self.gstats, self.slope, p, _mix_seed(self.eng.seed, self.id))
            kw = dict(drop_offset=self.drop_offset(), seed_dev=self.eng.seed_dev, stage_id=self.id, bias_grad=bg, bn=bn,
                      bn_groups=self.groups, bn_train=self.eng.training, bn_grads=bn_grads, ws=self.eng.det_ws)
            if bn is not None and self.bn_part is not None and self.eng.training:
                # the group means of (g, g*xhat) are global: reduce, gather the partials, then group and apply
                ops.norm_act_bwd(*args, **kw, bn_phase=1)
                ops.bn_group_sums(self.gstats, self.n, self.cout, self.groups, self.oh * self.ow, self.bn_part)
                self.eng.bn_sync.gather(self.bn_part, self.bn_gathered)
                ops.norm_act_bwd(*args, **kw, bn_phase=2, bn_gathered=self.bn_gathered, bn_rank=self.eng.bn_sync.rank)
            else:
                ops.norm_act_bwd(*args, **kw)
            if bg is not None:
                self._layer_backward(wgrad, bias=False)
                return
        self._layer_backward(wgrad, bias=True)

    def _layer_backward(self, wgrad: bool, bias: bool) -> None:
        """Input gradient on the launching stream (it is on the critical path of the backward chain); the weight (and
        unfused bias) gradient — tensor-core work nothing downstream waits for — on the engine's second stream, where it
        overlaps the HBM-bound IN/activation backward kernels of the following stages (Engine.join_wgrads() joins)."""
        side = self.eng.wgrad_stream() if wgrad else None
        if side is None:
            self.layer.backward(dgrad=self.need_dx, wgrad=wgrad, bias=bias)
            return
        ready = torch.cuda.Event()
        ready.record()                                   # dy (and everything before it: zero_grad) is complete
        self.layer.backward(dgrad=self.need_dx, wgrad=False)
        side.wait_event(ready)
        with torch.cuda.stream(side):
            self.layer.backward(dgrad=False, wgrad=True, bias=bias)
        self.eng._wgrad_pending = True


class Engine:
    """Common plumbing: stage list, flat gradient buffer, packing."""

    def __init__(self, net: nn.Module, device, nsplit: int, train: bool = True, deterministic: bool = False,
                 bn_sync=None):
        """deterministic: every reduction that spans blocks adds its partial sums in a fixed order instead of with
        floating-point atomics, so a step gives bit-identical results on every run (DESIGN.md §4).
        bn_sync (parallel.BNStatsExchange): train-mode batch norm normalises with the statistics of every rank's
        samples (DESIGN.md §7); None: with this process's samples."""
        self.net, self.device, self.nsplit = net, torch.device(device), nsplit
        self.deterministic = bool(deterministic)
        self.bn_sync = bn_sync
        # slot workspaces of the deterministic reductions: one for the launching stream, one for the weight-gradient
        # stream (the two overlap)
        self.det_ws = ops.DetWorkspace(device) if deterministic else None
        self.det_ws_side = ops.DetWorkspace(device) if deterministic else None
        self.dual = train   # activation planes carry a bf16-split twin for the weight-gradient GEMMs
        self.stages: List[Stage] = []
        self.training = True
        self.seed = 0
        self.seed_dev: Optional[torch.Tensor] = None   # device copy of the step seed (CUDA-graph replay), else host seeds
        self.sample_base = 0        # global index of local sample 0 (dropout masks follow the global sample)
        self._pack_table: Optional[ops.PackTable] = None   # built at the first pack() (after bind_backward)
        self._pack_extra: list = []
        self._wgrad_stream: Optional[torch.cuda.Stream] = None
        self._wgrad_pending = False
        self.flat_grad: Optional[torch.Tensor] = None

    def wgrad_stream(self) -> Optional[torch.cuda.Stream]:
        """Second stream for the weight-gradient GEMMs (None: launch in line, for per-launch tracing)."""
        if ops.Plan.trace is not None:
            return None
        if self._wgrad_stream is None:
            self._wgrad_stream = torch.cuda.Stream(device=self.device)
        return self._wgrad_stream

    def join_wgrads(self) -> None:
        """The launching stream waits for every weight gradient issued so far (before the optimizer, an all-reduce of
        the gradients, or the next overwrite of the operand planes)."""
        if self._wgrad_pending:
            done = torch.cuda.Event()
            done.record(self._wgrad_stream)
            torch.cuda.current_stream(self.device).wait_event(done)
            self._wgrad_pending = False

    def workspace_bytes(self) -> int:
        """Device bytes of the deterministic mode's workspaces: the slot workspaces (sized by the first step) and the
        split-K partials of the weight-gradient plans.  0 in the default mode."""
        if not self.deterministic:
            return 0
        plans = [s.layer.wgrad_plan for s in self.stages if getattr(s.layer, "wgrad_plan", None) is not None]
        return self.det_ws.nbytes + self.det_ws_side.nbytes + sum(p.workspace_bytes for p in plans)

    def planes(self, n: int, h: int, w: int, c: int) -> Planes:
        """fp16-split activation operand (+ bf16 twin when training)."""
        return Planes(n, h, w, c, self.device, dual=self.dual)

    def alloc_grads(self, share_with: Optional["Engine"] = None) -> None:
        """One flat fp32 buffer for all parameter gradients (a single all-reduce under DP);
        p.grad are views into it."""
        if share_with is not None:
            self.flat_grad = share_with.flat_grad
            return
        params = [p for p in self.net.parameters()]
        total = sum(p.numel() for p in params)
        self.flat_grad = torch.zeros(total, device=self.device)
        off = 0
        for p in params:
            p.grad = self.flat_grad[off:off + p.numel()].view_as(p)
            off += p.numel()

    def zero_grad(self) -> None:
        self.flat_grad.zero_()
        # the optimizer may have dropped .grad (zero_grad(set_to_none=True)): re-attach the views
        off = 0
        for p in self.net.parameters():
            if p.grad is None or p.grad.data_ptr() != self.flat_grad.data_ptr() + 4 * off:
                p.grad = self.flat_grad[off:off + p.numel()].view_as(p)
            off += p.numel()

    def pack(self) -> None:
        """Kernel-layout copies of the (updated) torch weights: one scale launch + one pack launch for the whole
        network (ops.PackTable), plus the head's effective-tap packs."""
        if self._pack_table is None:
            self._pack_table = ops.PackTable(self.device)
            self._pack_extra = [s.layer for s in self.stages if s.layer.register_packs(self._pack_table)]
        self._pack_table.run()
        for ly in self._pack_extra:
            ly.pack_extra()

    def bind_backward(self, wgrad: bool = True) -> None:
        for s in self.stages:
            s.bind_backward(wgrad=wgrad)
        self._pack_table = None        # the input-gradient packs exist now: re-register at the next pack()


# =============================================================================================
# WarpModule
# =============================================================================================
class WarpEngine(Engine):
    def __init__(self, net: M.WarpModule, batch: int, size: int, device, nsplit: int = 3, train: bool = True,
                 deterministic: bool = False):
        super().__init__(net, device, nsplit, train, deterministic)
        assert size % 64 == 0 and size >= 64, "WarpModule needs H = W = 64k (cloth_down6 is H/64)"
        B, S, dev = batch, size, self.device
        self.batch, self.size = B, S
        self.cb, self.cc = net.body_channels, net.cloth_channels
        dp = net.dropout
        self.in_body = self.planes(B, S, S, L.padc(self.cb))      # 3 -> 16 channels (32-byte TMA rows)
        self.in_cloth = self.planes(B, S, S, L.padc(self.cc))     # 19 -> 32
        cat3 = self.planes(B, S // 2, S // 2, 192)
        cat2 = self.planes(B, S // 4, S // 4, 384)
        cat1 = self.planes(B, S // 8, S // 8, 768)
        h16 = S // 16
        xpad = [self.planes(B, h16 + 2, h16 + 2, 1024) for _ in range(4)]   # reflect-padded resblock inputs
        xf32 = [torch.zeros(B, h16, h16, 1024, device=dev) for _ in range(5)]  # fp32 residual stream
        a_c4 = self.planes(B, h16, h16, 512)
        a_c5 = self.planes(B, S // 32, S // 32, 1024)
        a_c6 = self.planes(B, S // 64, S // 64, 1024)
        a_u1 = self.planes(B, S // 32, S // 32, 1024)
        x4 = self.planes(B, h16, h16, 1024)
        self.cat3, self.cat2, self.cat1, self.xf32 = cat3, cat2, cat1, xf32
        St = lambda *a, **k: Stage(self, *a, **k)  # noqa: E731
        n = net
        lre = dict(act=ACT_LRELU, slope=0.2)
        self.b1 = St("body_down1", "conv4s2", n.body_down1.model[0], self.in_body, out=cat3.slice(64, 64), need_dx=False, **lre)
        self.b2 = St("body_down2", "conv4s2", n.body_down2.model[0], cat3.slice(64, 64), out=cat2.slice(128, 128), norm=True, **lre)
        self.b3 = St("body_down3", "conv4s2", n.body_down3.model[0], cat2.slice(128, 128), out=cat1.slice(256, 256), norm=True, **lre)
        self.b4 = St("body_down4", "conv4s2", n.body_down4.model[0], cat1.slice(256, 256), out=xpad[0].slice(0, 512),
                     reflect_out=True, out_f32=xf32[0][..., :512], norm=True, drop_p=dp, **lre)
        self.c1 = St("cloth_down1", "conv4s2", n.cloth_down1.model[0], self.in_cloth, out=cat3.slice(128, 64), need_dx=False, **lre)
        self.c2 = St("cloth_down2", "conv4s2", n.cloth_down2.model[0], cat3.slice(128, 64), out=cat2.slice(256, 128), norm=True, **lre)
        self.c3 = St("cloth_down3", "conv4s2", n.cloth_down3.model[0], cat2.slice(256, 128), out=cat1.slice(512, 256), norm=True, **lre)
        self.c4 = St("cloth_down4", "conv4s2", n.cloth_down4.model[0], cat1.slice(512, 256), out=a_c4, norm=True, **lre)
        self.c5 = St("cloth_down5", "conv4s2", n.cloth_down5.model[0], a_c4, out=a_c5, norm=True, drop_p=dp, **lre)
        self.c6 = St("cloth_down6", "conv4s2", n.cloth_down6.model[0], a_c5, out=a_c6, drop_p=dp, **lre)
        self.u1 = St("cloth_up1", "convT4s2", n.cloth_up1.model[0], a_c6, out=a_u1, norm=True, act=ACT_RELU)
        self.u2 = St("cloth_up2", "convT4s2", n.cloth_up2.model[0], a_u1, out=xpad[0].slice(512, 512), reflect_out=True,
                     out_f32=xf32[0][..., 512:], norm=True, act=ACT_RELU)
        self.res: List[Tuple[Stage, Stage]] = []
        for k in range(4):
            blk = n.resblocks[k].conv_block
            p1 = self.planes(B, h16 + 2, h16 + 2, 1024)
            r1 = St(f"resblocks.{k}.conv1", "conv3r", blk[1], xpad[k], out=p1, reflect_out=True, norm=True, act=ACT_RELU,
                    drop_p=dp)
            last = k == 3
            r2 = St(f"resblocks.{k}.conv2", "conv3r", blk[6], p1, out=x4 if last else xpad[k + 1], reflect_out=not last,
                    norm=True, act=ACT_NONE, residual=xf32[k], out_f32=xf32[k + 1])
            self.res.append((r1, r2))
        self.d1 = St("dual_up1", "convT4s2", n.dual_up1.model[0], x4, out=cat1.slice(0, 256), norm=True, act=ACT_RELU)
        self.d2 = St("dual_up2", "convT4s2", n.dual_up2.model[0], cat1, out=cat2.slice(0, 128), norm=True, act=ACT_RELU)
        self.d3 = St("dual_up3", "convT4s2", n.dual_up3.model[0], cat2, out=cat3.slice(0, 64), norm=True, act=ACT_RELU)
        self.fakes = torch.zeros(B, S, S, self.cc, device=dev)   # NHWC; fakes.permute(0,3,1,2) is the NCHW view
        self.head = St("upsample_and_pad", "head", n.upsample_and_pad[2], cat3, plain=True, epi_act=ACT_TANH, y=self.fakes)
        self._fwd_order = [self.b1, self.b2, self.b3, self.b4, self.c1, self.c2, self.c3, self.c4, self.c5, self.c6,
                           self.u1, self.u2] + [s for pair in self.res for s in pair] + [self.d1, self.d2, self.d3, self.head]
        self._dres: List[torch.Tensor] = []

    def forward(self, body: torch.Tensor, cloth: torch.Tensor, training: bool = True, seed: int = 0,
                before_cloth=None) -> torch.Tensor:
        """body [B,cb,S,S], cloth [B,cc,S,S] fp32 NCHW on device -> fakes [B,S,S,cc] (NHWC storage).
        before_cloth(): called after the body branch (body_down1..4, which does not read the cloth) has been
        enqueued and before the cloth is first read — the plugin waits there for the cloth's H2D copy."""
        self.training, self.seed = training, seed
        ops.pack_concat([(body, False)], self.in_body)
        nbody = 4
        assert self._fwd_order[nbody - 1] is self.b4
        for s in self._fwd_order[:nbody]:
            s.forward()
        if before_cloth is not None:
            before_cloth()
        ops.pack_concat([(cloth, False)], self.in_cloth)
        for s in self._fwd_order[nbody:]:
            s.forward()
        return self.fakes

    def bind_backward(self, wgrad: bool = True) -> None:
        super().bind_backward(wgrad)
        h16 = self.size // 16
        self._dres = [torch.zeros(self.batch, h16, h16, 1024, device=self.device) for _ in range(4)]

    def grad_buckets(self):
        """Contiguous [lo, hi) slices of flat_grad in the order backward() completes them."""
        names = [n for n, _ in self.net.named_parameters()]
        sizes = [p.numel() for _, p in self.net.named_parameters()]
        offs = [0]
        for s_ in sizes:
            offs.append(offs[-1] + s_)

        def span(prefixes):
            idx = [i for i, n in enumerate(names) if n.startswith(prefixes)]
            assert idx == list(range(idx[0], idx[-1] + 1)), "bucket is not contiguous in the flat buffer"
            return offs[idx[0]], offs[idx[-1] + 1]

        # in the order backward() retires them: decoder + head; the four resblocks (last first); the four big cloth-branch
        # layers (cloth_up2, cloth_up1, cloth_down6, cloth_down5: 50 M of the branch's 53 M parameters, finished ~4 ms before
        # the backward ends); the small down-path layers of both branches.  Finer buckets start their all-reduce earlier:
        # only the last, 13 MB bucket is issued at the very end of the backward pass.
        return ([span(("dual_up", "upsample_and_pad"))] + [span((f"resblocks.{k}.",)) for k in (3, 2, 1, 0)] +
                [span(("cloth_down5", "cloth_down6", "cloth_up")), span(("body_", "cloth_down1", "cloth_down2", "cloth_down3",
                                                                         "cloth_down4"))])

    def backward(self, srcs: Optional[Sequence[GradSrc]], on_bucket=None) -> None:
        """srcs: gradient(s) w.r.t. fakes (NHWC fp32), or None when the head's dy planes were already written by the
        fused loss kernel (ops.ce_tanh_bwd).  Accumulates parameter grads into flat_grad.
        on_bucket(i): called when bucket i of grad_buckets() has all its gradient launches enqueued."""
        B, h16 = self.batch, self.size // 16

        def done(i):
            """Bucket i is complete once the launches issued so far on BOTH streams have run.  The all-reduce is issued
            from the weight-gradient stream (which first waits for the launching stream's work up to here), so the
            launching stream — the backward chain — never blocks on it."""
            if on_bucket is None:
                return
            side = self._wgrad_stream if self._wgrad_pending else None
            if side is None:
                on_bucket(i)
                return
            here = torch.cuda.Event()
            here.record()
            side.wait_event(here)
            with torch.cuda.stream(side):
                on_bucket(i)

        self.head.backward(srcs)
        g3 = self.head.dx                                     # d cat3 [.,192]
        self.d3.backward([GradSrc(g3, 0)])
        g2 = self.d3.dx                                       # d cat2 [.,384]
        self.d2.backward([GradSrc(g2, 0)])
        g1 = self.d2.dx                                       # d cat1 [.,768]
        self.d1.backward([GradSrc(g1, 0)])
        gx = self.d1.dx                                       # d x4 [.,1024]
        done(0)
        for k in (3, 2, 1, 0):
            r1, r2 = self.res[k]
            r2.backward([GradSrc(gx)])                        # IN(y2) branch; identity branch handled below
            r1.backward([GradSrc(r2.dx, 0, True)])
            ops.sum_grads([GradSrc(gx), GradSrc(r1.dx, 0, True)], B, h16, h16, 1024, self._dres[k])
            gx = self._dres[k]
            done(1 + (3 - k))                                 # resblock k: buckets 1 (k = 3) .. 4 (k = 0)
        self.u2.backward([GradSrc(gx, 512)])
        self.u1.backward([GradSrc(self.u2.dx)])
        self.c6.backward([GradSrc(self.u1.dx)])
        self.c5.backward([GradSrc(self.c6.dx)])
        done(5)
        self.c4.backward([GradSrc(self.c5.dx)])
        self.c3.backward([GradSrc(self.c4.dx), GradSrc(g1, 512)])
        self.c2.backward([GradSrc(self.c3.dx), GradSrc(g2, 256)])
        self.c1.backward([GradSrc(self.c2.dx), GradSrc(g3, 128)])
        self.b4.backward([GradSrc(gx, 0)])
        self.b3.backward([GradSrc(self.b4.dx), GradSrc(g1, 256)])
        self.b2.backward([GradSrc(self.b3.dx), GradSrc(g2, 128)])
        self.b1.backward([GradSrc(self.b2.dx), GradSrc(g3, 64)])
        done(6)
        self.join_wgrads()


# =============================================================================================
# PatchGAN
# =============================================================================================
class PatchGANEngine(Engine):
    """NLayerDiscriminator on a [batch, S, S, pad64(input_nc)] operand (`self.din`).  groups: the batch is that many
    separate D calls stacked (the D step's fake and real halves), which matters to batch norm only."""

    def __init__(self, net: M.NLayerDiscriminator, batch: int, size: int, device, nsplit: int = 3,
                 din: Optional[Planes] = None, input_grad: bool = False, train: bool = True, groups: int = 1,
                 deterministic: bool = False, bn_sync=None):
        super().__init__(net, device, nsplit, train, deterministic, bn_sync)
        B, S, dev = batch, size, self.device
        self.batch, self.size = B, S
        self.din = din if din is not None else self.planes(B, S, S, L.padc(net.input_nc))
        assert (self.din.n, self.din.h, self.din.w) == (B, S, S)
        convs = net.convs()
        bns = net.bns()
        use_norm = net.norm != "none"
        x = self.din
        self.chain: List[Stage] = []
        h = S
        for i, conv in enumerate(convs[:-1]):
            kind = "conv4s2" if conv.stride[0] == 2 else "conv4s1"
            oh = h // 2 if kind == "conv4s2" else h - 1
            out = self.planes(B, oh, oh, L.padc(conv.out_channels))
            st = Stage(self, f"model.{net.conv_index[i]}", kind, conv, x, out=out, norm=use_norm and i > 0,
                       act=ACT_LRELU, slope=0.2, need_dx=(i > 0) or input_grad, bn=bns[i], groups=groups)
            self.chain.append(st)
            x, h = out, oh
        self.last = Stage(self, f"model.{net.conv_index[-1]}", "conv4s1", convs[-1], x, plain=True)
        self.pred = self.last.y                                # [B, S/8-2, S/8-2, 1]

    def forward(self) -> torch.Tensor:
        for s in self.chain:
            s.forward()
        self.last.forward()
        return self.pred

    def backward(self, dpred: torch.Tensor, wgrad: bool = True) -> None:
        self.last.backward([GradSrc(dpred)], wgrad=wgrad)
        g = self.last.dx
        for s in reversed(self.chain):
            s.backward([GradSrc(g)], wgrad=wgrad)
            g = s.dx
        self.join_wgrads()

    @property
    def dx_in(self) -> torch.Tensor:
        return self.chain[0].dx


class PixelGANEngine(Engine):
    """PixelDiscriminator (the 1x1 PatchGAN) on a [batch, S, S, padc(input_nc)] operand (`self.din`), with the surface
    of PatchGANEngine.  Its hidden layers run at full resolution and are never stored: the four passes of
    csrc/pixel_disc.cu recompute them from `din`, so the engine holds only the logits `pred` [batch, S, S], the
    per-(image, channel) statistics and, with input_grad, `dx_in`."""

    def __init__(self, net: M.PixelDiscriminator, batch: int, size: int, device, nsplit: int = 3,
                 din: Optional[Planes] = None, input_grad: bool = False, train: bool = True, groups: int = 1,
                 deterministic: bool = False, bn_sync=None):
        super().__init__(net, device, nsplit, train, deterministic, bn_sync)
        if net.norm == "batch":
            raise NotImplementedError("--discriminator pixel --norm batch: batch statistics couple the samples inside "
                                      "the fused per-pixel passes, which normalise per image; use --norm instance or "
                                      "none")
        B, S, dev = batch, size, self.device
        self.batch, self.size = B, S
        self.din = din if din is not None else self.planes(B, S, S, L.padc(net.input_nc))
        assert (self.din.n, self.din.h, self.din.w) == (B, S, S) and self.din.c in (16, 32)
        self.pred = torch.zeros(B, S, S, device=dev)
        norm = net.norm == "instance"
        self.stats = torch.zeros(B, 128, 2, dtype=torch.float64, device=dev) if norm else None
        self.gstats = torch.zeros_like(self.stats) if norm else None
        self.scales = torch.zeros(2, 2, device=dev)          # (s, 1/s) of net.0 and net.2 weights
        cin = net.input_nc
        self.dx = torch.zeros(B, S, S, (cin + 3) // 4 * 4, device=dev)[..., :cin] if input_grad else None
        self.debug: Optional[torch.Tensor] = None             # [B*S*S, 64 + 128]: z1 and y2 of the forward (tests)

    def workspace_bytes(self) -> int:
        return 0 if self.det_ws is None else self.det_ws.nbytes

    def pack(self) -> None:
        """The power-of-two scales of the (updated) net.0 and net.2 weights; the passes split the weights themselves."""
        if self._pack_table is None:
            self._pack_table = ops.PackTable(self.device)
            self._pack_table.add_scale(self.net.net[0].weight.data, self.scales[0])
            self._pack_table.add_scale(self.net.net[2].weight.data, self.scales[1])
        self._pack_table.run()

    def _desc(self, **kw):
        return ops.pixel_desc(self.din, self.net, self.scales, self.nsplit, stats=self.stats, gstats=self.gstats, **kw)

    def forward(self) -> torch.Tensor:
        if self.stats is not None:
            ops.pixel_pass("fwd_stats", self._desc(), ws=self.det_ws)
        ops.pixel_pass("fwd", self._desc(pred=self.pred, debug=self.debug))
        return self.pred

    def backward(self, dpred: torch.Tensor, wgrad: bool = True) -> None:
        grads = {}
        if wgrad:
            c0, c2, c5 = self.net.net[0], self.net.net[2], self.net.net[5]
            grads = dict(dw1=c0.weight.grad, db1=c0.bias.grad, dw2=c2.weight.grad,
                         db2=None if c2.bias is None else c2.bias.grad, dw3=c5.weight.grad,
                         db3=None if c5.bias is None else c5.bias.grad)
        if self.stats is not None:
            ops.pixel_pass("bwd_reduce", self._desc(dpred=dpred, **grads), ws=self.det_ws)
        dx = dict(dx=self.dx, dx_pitch=self.dx.stride(2)) if self.dx is not None else {}
        ops.pixel_pass("bwd_apply", self._desc(dpred=dpred, **grads, **dx), ws=self.det_ws)

    @property
    def dx_in(self) -> torch.Tensor:
        return self.dx


# =============================================================================================
# pix2pix U-Net (shared by TextureModule and the standalone generator)
# =============================================================================================
class UNetStages:
    """The stages of an M.UnetGenerator on an engine, reading the operand planes `x` and writing `fakes` (fp32 NHWC,
    tanh) — pix2pix_modules.py:113-262; the norm is the container's: instance (bias on every conv), batch (BatchNorm2d,
    no bias but on U_0) or none (no bias but on U_0).

    Bookkeeping (depth j = 0 outermost .. nd-1 innermost; D_j / U_j = its down / up conv):
      L_{j+1} = leaky_relu([IN](D_j(.)))  is both the operand of D_{j+1} and, because the reference's
                LeakyReLU is in place, the skip half of block j+1's output (App. B #1);
      the parent applies ReLU to the whole concat, so U_j reads cat(relu(L_{j+1}), relu(V_{j+1})) with
      V = dropout?(IN(U(.))) — buffer `cu[j]`, written in place by the producing stages.
    Stages are created on `eng` in the order D_0..D_{nd-1}, U_{nd-1}..U_0 (their ids seed the dropout masks)."""

    def __init__(self, eng: Engine, unet: M.UnetGenerator, x: Planes, fakes: torch.Tensor, input_grad: bool = True):
        """input_grad: D_0 computes the gradient w.r.t. `x` (`dx`)."""
        B, S = x.n, x.h
        nd = unet.num_downs
        blocks = unet.blocks()
        assert len(blocks) == nd
        St = lambda *a, **k: Stage(eng, *a, **k)  # noqa: E731
        chans = [blocks[j].down.out_channels for j in range(nd)]          # channels of x_{j+1}
        self.cu = [eng.planes(B, S >> (j + 1), S >> (j + 1), 2 * chans[j]) for j in range(nd - 1)]
        use_norm = unet.norm != "none"
        self.down: List[Stage] = []
        for j in range(nd):
            h = S >> (j + 1)
            last = j == nd - 1
            out = eng.planes(B, h, h, L.padc(chans[j]))
            if last:
                st = St(f"unet.D{j}", "conv4s2", blocks[j].down, x, out=out, norm=False, act=ACT_RELU)
            else:
                st = St(f"unet.D{j}", "conv4s2", blocks[j].down, x, out=out, norm=(j >= 1) and use_norm,
                        act=ACT_LRELU, out_relu=self.cu[j].slice(0, chans[j]), bn=blocks[j].down_bn,
                        need_dx=(j > 0) or input_grad)
            self.down.append(st)
            x = out
        self.up: List[Optional[Stage]] = [None] * nd
        for j in range(nd - 1, 0, -1):
            src = self.down[nd - 1].out if j == nd - 1 else self.cu[j]
            cout = blocks[j].up.out_channels
            drop = 0.5 if (blocks[j].use_dropout and not blocks[j].innermost) else 0.0
            self.up[j] = St(f"unet.U{j}", "convT4s2", blocks[j].up, src, out=self.cu[j - 1].slice(chans[j - 1], cout),
                            norm=use_norm, act=ACT_RELU, drop_p=drop, bn=blocks[j].up_bn)
        self.up[0] = St("unet.U0", "convT4s2", blocks[0].up, self.cu[0], plain=True, epi_act=ACT_TANH, y=fakes)

    def forward(self) -> None:
        for st in self.down:
            st.forward()
        for j in range(len(self.up) - 1, -1, -1):
            self.up[j].forward()

    def backward(self, srcs: Sequence[GradSrc]) -> Optional[torch.Tensor]:
        """srcs: gradient(s) w.r.t. fakes.  Returns d/dx (D_0's `dx`; None without input_grad)."""
        nd = len(self.down)
        self.up[0].backward(srcs)
        g = self.up[0].dx                                           # d cu[0]
        gcu = [None] * (nd - 1)
        gcu[0] = g
        for j in range(1, nd):
            cprev = self.down[j - 1].cout
            self.up[j].backward([GradSrc(gcu[j - 1], cprev)])
            if j < nd - 1:
                gcu[j] = self.up[j].dx
        # innermost down conv: its relu() output only feeds U_{nd-1}
        self.down[nd - 1].backward([GradSrc(self.up[nd - 1].dx)])
        for j in range(nd - 2, -1, -1):
            # L_{j+1} feeds D_{j+1} (as leaky_relu) and the skip slot of cu[j] (as relu)
            self.down[j].backward([GradSrc(self.down[j + 1].dx), GradSrc(gcu[j], 0, act=ACT_RELU)])
        return self.down[0].dx


# =============================================================================================
# TextureModule
# =============================================================================================
class TextureEngine(Engine):
    """ROIAlign+repack -> encode (UNetDown 36->36) -> nearest upsample -> cat cloth -> pix2pix U-Net
    (swapnet_modules.py:231-260; the U-Net is UNetStages; `encode` is always IN)."""

    def __init__(self, net: M.TextureModule, batch: int, size: int, device, nsplit: int = 3, train: bool = True,
                 deterministic: bool = False, bn_sync=None):
        super().__init__(net, device, nsplit, train, deterministic, bn_sync)
        B, S = batch, size
        assert S >= 64 and (S & (S - 1)) == 0, "texture stage: power-of-two size >= 64"
        self.batch, self.size = B, S
        self.ct, self.cc, self.nroi = net.texture_channels, net.cloth_channels, net.num_roi
        ch = self.ct * self.nroi
        self.ch = ch
        self.pool = 128
        self.pooled = self.planes(B, self.pool, self.pool, L.padc(ch))
        self.enc = self.planes(B, self.pool // 2, self.pool // 2, L.padc(ch))
        self.in_unet = self.planes(B, S, S, L.padc(ch + self.cc))
        self.up_factor = S // (self.pool // 2)
        self.encode = Stage(self, "encode", "conv4s2", net.encode.model[0], self.pooled, out=self.enc, norm=True,
                            act=ACT_LRELU, need_dx=False)
        self.fakes = torch.zeros(B, S, S, self.ct, device=self.device)
        self.unet = UNetStages(self, net.unet, self.in_unet, self.fakes)

    def forward(self, tex: torch.Tensor, rois: torch.Tensor, cloth: torch.Tensor, training: bool = True,
                seed: int = 0, before_cloth=None) -> torch.Tensor:
        """tex [B,3,S,S], rois [B,12,4], cloth [B,19,S,S] (fp32, device) -> fakes [B,S,S,3] NHWC."""
        self.training, self.seed = training, seed
        ops.roi_align_pack(tex, rois, self.pool, None, self.pooled.slice(0, self.ch))
        if self.pooled.twin is not None:
            ops.roi_align_pack(tex, rois, self.pool, None, self.pooled.twin.slice(0, self.ch))
        self.encode.forward()
        ops.upsample_planes(self.enc.slice(0, self.ch), self.in_unet.slice(0, self.ch), self.up_factor)
        if before_cloth is not None:       # the plugin waits here for the cloth's H2D copy
            before_cloth()
        ops.pack_planes(cloth, self.in_unet.slice(self.ch, self.cc))
        self.unet.forward()
        return self.fakes

    def backward(self, srcs: Sequence[GradSrc]) -> None:
        dx = self.unet.backward(srcs)
        self.encode.backward([GradSrc(dx, 0, up=self.up_factor)])
        self.join_wgrads()


class UnetEngine(Engine):
    """A bare M.UnetGenerator (the pix2pix generator; `--netG unet_128` of the texture stage) on the operand planes
    `x_in` [batch, S, S, padc(input_nc)], which the caller packs; output `fakes` [batch, S, S, output_nc] (fp32 NHWC,
    tanh).  No input gradient.  S must be a multiple of 2**num_downs: the innermost level is then at least 1 x 1 (the
    reference fails on mismatched skip concatenations otherwise)."""

    def __init__(self, net: M.UnetGenerator, batch: int, size: int, device, nsplit: int = 3, train: bool = True,
                 deterministic: bool = False, bn_sync=None):
        super().__init__(net, device, nsplit, train, deterministic, bn_sync)
        nd = net.num_downs
        if size % (1 << nd) != 0:
            raise ValueError(f"a U-Net with {nd} downsamplings needs an image size divisible by 2**{nd} = {1 << nd}, "
                             f"got {size}: its skip connections would not line up")
        B, S = batch, size
        self.batch, self.size = B, S
        blocks = net.blocks()
        self.x_in = self.planes(B, S, S, L.padc(blocks[0].down.in_channels))
        self.fakes = torch.zeros(B, S, S, blocks[0].up.out_channels, device=self.device)
        self.unet = UNetStages(self, net, self.x_in, self.fakes, input_grad=False)

    def forward(self, training: bool = True, seed: int = 0) -> torch.Tensor:
        """x_in (packed by the caller) -> fakes [B,S,S,output_nc] NHWC."""
        self.training, self.seed = training, seed
        self.unet.forward()
        return self.fakes

    def backward(self, srcs: Sequence[GradSrc]) -> None:
        """srcs: gradient(s) w.r.t. fakes; accumulates the parameter gradients into flat_grad."""
        self.unet.backward(srcs)
        self.join_wgrads()


# =============================================================================================
# VGG16 perceptual loss (modules/losses/perceptual.py:13-79; texture_model.py:68-69,171-176)
# =============================================================================================
class VGGStage(Stage):
    """conv3x3(pad 1)+bias -> ReLU [-> MaxPool2d(2)] of vgg16.features; frozen weights (no wgrad)."""

    def __init__(self, eng: "Engine", name: str, conv: nn.Module, x: Planes, out: Optional[Planes], pool: bool,
                 need_dx: bool):
        super().__init__(eng, name, "conv3z", conv, x, out=out, act=ACT_RELU, need_dx=need_dx)
        self.pool = pool

    def forward(self) -> None:
        self.layer.forward()
        if self.pool:
            ops.relu_pool_fwd(self.y, self.cout, self.out)
        elif self.out is not None:
            ops.norm_act_fwd(self.y, self.cout, None, ACT_RELU, 0.0, 0.0, 0, out=self.out)

    def backward_vgg(self, g_next: Optional[torch.Tensor], g_feat: Optional[torch.Tensor]) -> None:
        """g_next: gradient w.r.t. this stage's output planes (the next conv's dx; pooled size if `pool`);
        g_feat: gradient w.r.t. the un-pooled ReLU output from the feature loss (tap stages)."""
        if self.pool:
            ops.relu_pool_bwd(self.y, self.cout, g_next, g_feat, self.dy)
        else:
            srcs = [GradSrc(g) for g in (g_next, g_feat) if g is not None]
            ops.norm_act_bwd(srcs, self.y, self.cout, None, ACT_RELU, self.dy, None, 0.0, 0.0, 0)
        self.layer.backward(dgrad=self.need_dx, wgrad=False)


class VGGEngine(Engine):
    """vgg16.features[0:30] on a [B,S,S,3] image (already mapped to [-1,1]); keeps every conv output `y`."""

    def __init__(self, net: M.VGG16Features, batch: int, size: int, device, nsplit: int = 3, backward: bool = False):
        super().__init__(net, device, nsplit, train=False)     # frozen weights: no bf16 twins, no wgrad
        assert size % 16 == 0, "VGG16 perceptual loss: H = W = 16k"
        B, S = batch, size
        self.batch, self.size = B, S
        self.x_in = self.planes(B, S, S, 16)
        x, h = self.x_in, S
        self.chain: List[VGGStage] = []
        self.taps: List[VGGStage] = []
        for idx in M.VGG16_CONVS:
            conv = net[idx]
            pool = idx in M.VGG16_POOLED_CONVS
            last = idx == M.VGG16_CONVS[-1]
            oh = h // 2 if pool else h
            out = None if last else self.planes(B, oh, oh, L.padc(conv.out_channels))
            st = VGGStage(self, str(idx), conv, x, out, pool, need_dx=backward)
            self.chain.append(st)
            if idx in M.VGG16_TAP_CONVS:
                self.taps.append(st)
            x, h = out, oh
        if backward:
            self.bind_backward(wgrad=False)
        self.pack()                                            # frozen: packed once

    def forward(self) -> None:
        for s in self.chain:
            s.forward()


class PerceptualEngine:
    """PerceptualLoss(output=fakes, target) value and d/d(fakes) on the device.

    content = sum over 5 taps of MSE(f_out, f_tgt), f = L2-normalised ReLU features of `2x - 1`;
    style   = 5 * MSE(gram(out), gram(tgt)) of the raw images viewed as [B*3, H*W] (perceptual.py:58-63).
    """

    def __init__(self, net: Optional[M.VGG16Features], batch: int, size: int, device, nsplit: int = 3,
                 content: bool = True, deterministic: bool = False):
        """deterministic: the content and style sums add their block partials in a fixed order (bit-identical runs);
        the VGG passes themselves have no cross-block reductions."""
        dev = torch.device(device)
        self.det_ws = ops.DetWorkspace(dev) if deterministic else None
        self.batch, self.size = batch, size
        self.out = self.tgt = None
        self.gfeat: List[torch.Tensor] = []
        if content:
            self.out = VGGEngine(net, batch, size, device, nsplit, backward=True)
            self.tgt = VGGEngine(net, batch, size, device, nsplit, backward=False)
            self.gfeat = [torch.zeros_like(s.y) for s in self.out.taps]
        r = 3 * batch
        if r > 96:   # csrc/perceptual.cu kGramMaxR: the Gram matrix of the style term is held in registers / smem
            raise NotImplementedError(f"style loss: the Gram matrix couples 3 x batch = {r} rows, at most 96 are "
                                      "supported per GPU (batch <= 32); use --lambda_style 0 or a smaller per-GPU batch")
        self.gram_o = torch.zeros(r, r, dtype=torch.float64, device=dev)
        self.gram_t = torch.zeros(r, r, dtype=torch.float64, device=dev)
        self.gram_m = torch.zeros(r, r, dtype=torch.float32, device=dev)

    def workspace_bytes(self) -> int:
        """Device bytes of the deterministic mode's slot workspace (0 in the default mode)."""
        return 0 if self.det_ws is None else self.det_ws.nbytes

    def nominal_macs(self) -> int:
        if self.out is None:
            return 0
        f = sum(s.nominal_macs() for s in self.out.chain)
        return 3 * f            # VGG(fakes) + VGG(targets) + input-gradient of VGG(fakes)

    def content(self, fakes: torch.Tensor, targets: torch.Tensor, lam: float, acc: torch.Tensor) -> torch.Tensor:
        """fakes NHWC [B,S,S,3], targets NCHW [B,3,S,S] (fp32, device).  acc (float64[1]) += lam * content loss.
        Returns d(lam * content)/d(fakes) as an fp32 NHWC [B,S,S,3] view."""
        o, t = self.out, self.tgt
        ops.affine_pack(targets, False, 2.0, -1.0, t.x_in)     # x = 2.0 * x - 1.0 (perceptual.py:70)
        t.forward()
        ops.affine_pack(fakes, True, 2.0, -1.0, o.x_in)
        o.forward()
        for so, st, g in zip(o.taps, t.taps, self.gfeat):
            numel = so.n * so.oh * so.ow * so.cout             # MSELoss: mean over all elements
            ops.feat_loss_fwd_bwd(so.y, st.y, so.cout, lam / numel, 2.0, acc, g, ws=self.det_ws)  # gscale 2: d(2x-1)/dx
        g = None
        ti = len(o.taps) - 1
        for s in reversed(o.chain):
            gf = None
            if ti >= 0 and s is o.taps[ti]:
                gf, ti = self.gfeat[ti], ti - 1
            s.backward_vgg(g, gf)
            g = s.dx
        return g

    def style(self, fakes: torch.Tensor, targets: torch.Tensor, lam: float, acc: torch.Tensor,
              grad_accum: torch.Tensor) -> None:
        """acc += lam * 5 * MSE(gram(fakes), gram(targets)); grad_accum [B,S,S,3] += its gradient."""
        ops.gram(fakes, True, self.gram_o, ws=self.det_ws)
        ops.gram(targets, False, self.gram_t, ws=self.det_ws)
        ops.gram_mse(self.gram_o, self.gram_t, 5.0 * lam, acc, self.gram_m)
        ops.gram_bwd(self.gram_m, fakes, True, grad_accum, accumulate=True)
