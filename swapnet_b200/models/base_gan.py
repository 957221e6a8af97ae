"""GAN training-step framework on the B200 engines.

Keeps the option surface and step order of /root/reference/models/base_gan.py:16-231:
    forward -> zero/backward/step D -> zero/backward/step G        (base_gan.py:194-203)
with G = a generator engine, D = the conditional PatchGAN (define_D 'basic' / 'n_layers',
discriminators.py:45-88) or the 1x1 PixelGAN ('pixel', discriminators.py:138-168; engine.PixelGANEngine), GANLoss
(loss.py:12-130) for --gan_mode vanilla (BCE-with-logits), lsgan (MSE) and wgan
(-mean(pred) for real, +mean(pred) for fake) and torch.optim.AdamW or adabound.AdaBound (--optimizer_G / --optimizer_D,
chosen per network) exactly as optimizers/__init__.py:37-60 builds them.
vanilla and lsgan use the reference's smooth labels (loss.py:65-108, including the "fake target drawn from the real
range" quirk, loss.py:102): three CPU-RNG draws per step, D_fake, D_real, G_gan.  wgan has no target and draws nothing.
The wgan weight "clamp" of texture_model.py:132-135 (`p.data.clamp(...)`, not in place) leaves D unchanged in the
reference and is not reproduced; the warp stage has none.

What runs differently from the eager reference (results unchanged):
  * D's fake and real passes of the D step run as ONE batch of 2B with per-half targets (InstanceNorm is per
    sample; batch norm normalises each half with its own statistics and updates the running buffers fake first);
  * D's weight gradients are not computed in the G step (the reference computes and discards
    them, SURVEY App. B #5);
  * losses stay on the device until get_current_losses() is called.
Unsupported option values raise (there is no eager fallback): --gan_mode wgan-gp / dragan-gp / dragan-lp (the
gradient penalty needs a second derivative through D), --gan_mode mescheder-r1-gp / mescheder-r2-gp (the reference's
GANLoss raises for them too), --gan_label_mode hard (crashes in the reference too), --discriminator pixel with
--norm batch (batch statistics would couple the samples inside its fused per-pixel passes).
--norm batch under data parallelism needs --b200_sync_bn 1: every train-mode BatchNorm2d call then normalises with the
statistics of all ranks' samples (parallel.BNStatsExchange), so that 2 ranks x B/2 samples still reproduce one process
with the full batch B; without the flag it is refused, since per-rank statistics would quietly break that equivalence.
"""
from __future__ import annotations

from abc import ABC, abstractmethod
from argparse import ArgumentParser
from typing import Optional

import gc

import torch

from .. import engine as E
from .. import modules as M
from .. import ops
from .. import parallel
from .base_model import BaseModel, LazyLoss


def adam_modifier(parser: ArgumentParser, *_):
    """optimizers/__init__.py:25-28 (contributed by the options code when the reference's
    `optimizers` package is importable; provided here for standalone use)."""
    parser.add_argument("--b1", type=float, default=0.9, help="Adam b1")
    parser.add_argument("--b2", type=float, default=0.999, help="Adam b2")
    return parser


def adabound_modifier(parser: ArgumentParser, *_):
    """optimizers/__init__.py:31-34: what `--optimizer_G/--optimizer_D AdaBound` reads beyond the Adam flags."""
    parser = adam_modifier(parser)
    parser.add_argument("--final_lr", type=float, default=0.1, help="AdaBound final_lr")
    return parser


def define_optimizer(module, opt, net: str) -> torch.optim.Optimizer:
    """optimizers/__init__.py:37-60 for both of its choices, AdamW and AdaBound, each as one fused kernel over flat
    buffers (swapnet_b200/optim.py); same hyper-parameters, same state_dict layout."""
    from ..optim import FusedAdaBound, FusedAdamW, flatten_parameters

    if net not in ("D", "G"):
        raise ValueError(f"net arg must be 'D' or 'G', received {net}")
    choice = getattr(opt, "optimizer_" + net)
    if choice not in ("AdamW", "AdaBound"):
        raise NotImplementedError(f"optimizer {choice}: only AdamW and AdaBound are available on the B200 plugin")
    lr = opt.d_lr if net == "D" else opt.lr
    wd = opt.d_weight_decay if net == "D" else opt.weight_decay
    params = list(module.parameters())
    flat = flatten_parameters(params)
    if choice == "AdaBound":
        return FusedAdaBound(params, flat, lr=lr, weight_decay=wd, betas=(opt.b1, opt.b2), final_lr=opt.final_lr)
    return FusedAdamW(params, flat, lr=lr, weight_decay=wd, betas=(opt.b1, opt.b2), eps=1e-8)


def deterministic_mode(opt) -> bool:
    """--b200_deterministic when given; otherwise torch.use_deterministic_algorithms() as it stands now."""
    v = getattr(opt, "b200_deterministic", None)
    return torch.are_deterministic_algorithms_enabled() if v is None else bool(v)


def batch_norm_exchange(opt, world: int, batch_norm: Optional[bool] = None) -> Optional[parallel.BNStatsExchange]:
    """The cross-rank statistics exchange of batch norm under data parallelism with --b200_sync_bn 1; None where
    batch statistics stay local (one rank, or no batch norm).  Without the flag the combination is refused: per-rank
    statistics would quietly break the equivalence of 2 ranks x B/2 samples with one process and B samples.
    batch_norm: whether some network of the model has BatchNorm2d layers (default: `--norm batch`; a generator such as
    `--netG unet_128` has them whatever --norm says)."""
    if batch_norm is None:
        batch_norm = opt.norm == "batch"
    if not batch_norm or world <= 1:
        return None
    if not getattr(opt, "b200_sync_bn", 0):
        if opt.norm != "batch":
            raise NotImplementedError("the generator's batch norm under data parallelism needs cross-rank batch "
                                      "statistics: pass --b200_sync_bn 1 or train on one GPU")
        raise NotImplementedError("--norm batch under data parallelism needs cross-rank batch statistics: pass "
                                  "--b200_sync_bn 1, train on one GPU or use --norm instance / none")
    return parallel.BNStatsExchange()


def add_b200_options(parser: ArgumentParser) -> ArgumentParser:
    """The engine switches every GAN plugin accepts, in training and at test time."""
    parser.add_argument("--b200_graph", type=int, default=1, choices=(0, 1),
                        help="1: replay the training step as a captured CUDA graph (single GPU; after two eager "
                             "steps per input shape); 0: launch the kernels one by one")
    parser.add_argument("--b200_deterministic", type=int, default=None, choices=(0, 1),
                        help="1: bit-identical steps on every run (reductions add their partial sums in a fixed "
                             "order instead of with floating-point atomics); 0: the default kernels.  Default: "
                             "torch.are_deterministic_algorithms_enabled() when the model is built")
    parser.add_argument("--b200_sync_bn", type=int, default=0, choices=(0, 1),
                        help="1: under data parallelism, batch norm normalises with the batch statistics of "
                             "every rank's samples (exchanged each call, summed in rank order); no effect on one "
                             "GPU.  0: batch norm with more than one rank is refused")
    parser.add_argument("--b200_precision", default="fp32x3", choices=("fp32x3", "bf16"),
                        help="tensor-core arithmetic of the B200 engines: fp32x3 = split-bf16 3-pass "
                             "(fp32-faithful, parity mode); bf16 = single pass (fast, ~1e-2 relative)")
    return parser


class BaseGAN(BaseModel, ABC):
    @staticmethod
    def modify_commandline_options(parser: ArgumentParser, is_train):
        """Same flags, defaults and aliases as base_gan.py:16-128, plus the engine precision switch."""
        if is_train:
            parser.add_argument("--gan_mode", default="vanilla", help="gan regularization to use",
                                choices=("vanilla", "wgan", "wgan-gp", "lsgan", "dragan-gp", "dragan-lp",
                                         "mescheder-r1-gp", "mescheder-r2-gp"))
            parser.add_argument("--lambda_gan", type=float, default=1.0, help="weight for adversarial loss")
            parser.add_argument("--lambda_discriminator", type=float, default=1.0, help="weight for discriminator loss")
            parser.add_argument("--lambda_gp", type=float, default=10, help="weight parameter for gradient penalty")
            parser.add_argument("--discriminator", default="basic", choices=("basic", "pixel", "n_layers"),
                                help="what discriminator type to use")
            parser.add_argument("--n_layers_D", type=int, default=3, help="only used if discriminator==n_layers")
            parser.add_argument("--norm", type=str, default="instance",
                                help="instance normalization or batch normalization [instance | batch | none]")
            parser.add_argument("--optimizer_G", "--opt_G", "--optim_G", default="AdamW", choices=("AdamW", "AdaBound"),
                                help="optimizer for generator")
            parser.add_argument("--lr", "--g_lr", "--learning_rate", type=float, default=0.0001,
                                help="initial learning rate for generator")
            parser.add_argument("--beta1", type=float, default=0.5, help="momentum term of adam")
            parser.add_argument("--optimizer_D", "--opt_D", "--optim_D", default="AdamW", choices=("AdamW", "AdaBound"),
                                help="optimizer for discriminator")
            parser.add_argument("--d_lr", type=float, default=0.0004, help="initial learning rate for Discriminator")
            parser.add_argument("--d_wt_decay", "--d_weight_decay", dest="d_weight_decay", default=0.01, type=float,
                                help="optimizer L2 weight decay")
            parser.add_argument("--gan_label_mode", default="smooth", choices=("hard", "smooth"),
                                help="whether to use hard (real 1.0 and fake 0.0) or smooth "
                                     "(real [0.7, 1.1] and fake [0., 0.3]) values for labels")
        return add_b200_options(parser)

    def __init__(self, opt):
        super().__init__(opt)
        self.nsplit = 1 if getattr(opt, "b200_precision", "fp32x3") == "bf16" else 3
        self.deterministic = deterministic_mode(opt)
        # slot workspace of the deterministic loss reductions (launched on the step's stream)
        self._det_ws = ops.DetWorkspace(self.device) if self.deterministic else None
        self.net_generator = self.define_G().to(self.device)
        M.init_weights(self.net_generator, opt.init_type, opt.init_gain)
        self.model_names = ["generator"]
        self._eng_G = None          # built lazily for the (batch, size) of the first input
        self._eng_key = None
        self._eng_Dd = self._eng_Dg = None
        self._step = 0
        self._seed_base = int(getattr(opt, "b200_seed", 0))
        self._world = parallel.world_size()
        # smooth-label draws: the CPU default generator like the reference (loss.py:74-77); under DP a
        # dedicated, identically seeded generator so that every rank sees the same label (SURVEY §8e i)
        self._labels = parallel.LabelDraws(1234 if self._world > 1 else None)
        self._bn_sync: Optional[parallel.BNStatsExchange] = None   # cross-rank batch statistics (--b200_sync_bn 1)
        if self.is_train:
            self._gan_obj = self.gan_objective(opt.gan_mode)
            if opt.gan_label_mode != "smooth":
                raise NotImplementedError("--gan_label_mode hard crashes in the reference (loss.py:92,101) and is "
                                          "not provided")
            if opt.discriminator == "pixel" and opt.norm == "batch":
                raise NotImplementedError("--discriminator pixel --norm batch is not provided: batch statistics couple "
                                          "the samples inside the fused per-pixel passes (csrc/pixel_disc.cu), which "
                                          "normalise per image; use --norm instance or none")
            self._bn_sync = batch_norm_exchange(opt, self._world, opt.norm == "batch" or any(
                isinstance(m, torch.nn.BatchNorm2d) for m in self.net_generator.modules()))
            if opt.discriminator == "pixel":     # --n_layers_D is ignored, as in the reference
                self.net_discriminator = M.PixelDiscriminator(self.get_D_inchannels(), 64, opt.norm).to(self.device)
            else:
                n_layers = 3 if opt.discriminator == "basic" else opt.n_layers_D
                self.net_discriminator = M.NLayerDiscriminator(self.get_D_inchannels(), 64, n_layers,
                                                               opt.norm).to(self.device)
            self.init_D_weights(self.net_discriminator)
            self.model_names.append("discriminator")
            if getattr(opt, "lambda_discriminator", 1.0):
                self.loss_names = ["D", "D_real", "D_fake"]
            self.loss_names += ["G"]
            if opt.lambda_gan:
                self.loss_names += ["G_gan"]
            self.optimizer_G, self.optimizer_D = self.define_optimizers()
            self.optimizer_names = ("G", "D")
            self._acc = torch.zeros(8, dtype=torch.float64, device=self.device)  # device-side loss sums
            # per-step scalars read by the kernels from DEVICE memory (one tiny launch per step writes them), so that the
            # whole step is a fixed launch sequence a CUDA graph can replay: [0:3] smooth labels (D_fake, D_real, G_gan),
            # [4:12] optimizer scalars of D, [12:20] of G, [20:22] the dropout step seed as two exact 16-bit halves
            self._sp = torch.zeros(32, dtype=torch.float32, device=self.device)
            self._sp_ready = False          # True inside optimize_parameters(): labels were drawn by the step prologue
            self._graphs = {}               # (batch, size, training, input signature) -> captured step
            self._eager_steps = {}
            self.graph_enabled = bool(getattr(opt, "b200_graph", 1))
            self._acc_host = None                       # host copy of _acc for the current step (one D2H per step)
            lam = self.gan_weight()
            self.loss_D_fake = LazyLoss(lambda: self.loss_values()[0])
            self.loss_D_real = LazyLoss(lambda: self.loss_values()[1])
            self.loss_D = LazyLoss(lambda: 0.5 * (self.loss_values()[0] + self.loss_values()[1]))
            self.loss_G_gan = LazyLoss(lambda: lam * self.loss_values()[2])
            parallel.broadcast_parameters(list(self.net_generator.parameters()) +
                                          list(self.net_discriminator.parameters()))

    # ---- where a plugin departs from the reference's BaseGAN (pix2pix_model.py) ----
    def gan_objective(self, mode: str) -> int:
        """--gan_mode -> the ops.GAN_* objective the loss kernels run."""
        if mode in ("wgan-gp", "dragan-gp", "dragan-lp"):
            raise NotImplementedError(f"--gan_mode {mode}: its gradient penalty needs a second derivative "
                                      "through D, which the engines do not compute (DESIGN.md §1)")
        if mode not in ops.GAN_OBJECTIVES:
            raise NotImplementedError(f"--gan_mode {mode}: the reference's GANLoss does not implement it "
                                      "either (loss.py:61-62)")
        return ops.GAN_OBJECTIVES[mode]

    def gan_weight(self) -> float:
        """Weight of the generator's GAN term."""
        return float(self.opt.lambda_gan)

    def init_D_weights(self, net) -> None:
        M.init_weights(net, self.opt.init_type, self.opt.init_gain)

    def define_optimizers(self):
        """(optimizer_G, optimizer_D)."""
        return define_optimizer(self.net_generator, self.opt, "G"), define_optimizer(self.net_discriminator, self.opt, "D")

    # ---- to be provided by the plugin ----
    @abstractmethod
    def get_D_inchannels(self):
        ...

    @abstractmethod
    def define_G(self):
        ...

    @abstractmethod
    def build_generator_engine(self, batch: int, size: int):
        ...

    @abstractmethod
    def backward_G(self):
        ...

    # ---- engines ----
    ENGINE_CACHE = 2   # plans kept alive: the full batch and the short last batch of an epoch (DataLoader without
                       # drop_last, datasets/__init__.py:69) alternate without re-planning / re-allocating

    def ensure_engines(self, batch: int, size: int) -> None:
        """Engines (buffers + TMA plans) of the current (batch, size); built once per shape and cached (LRU)."""
        key = (batch, size)
        if self._eng_key == key:
            return
        cache = self.__dict__.setdefault("_eng_cache", {})
        if key not in cache:
            while len(cache) >= self.ENGINE_CACHE:           # evict the least recently used shape
                old = next(iter(cache))
                for gk in [k for k in getattr(self, "_graphs", {}) if k[:2] == old]:
                    del self._graphs[gk]                     # captured on the evicted engines' buffers
                for gk in [k for k in getattr(self, "_eager_steps", {}) if k[:2] == old]:
                    del self._eager_steps[gk]
                for eng in cache.pop(old).values():
                    if hasattr(eng, "stages"):
                        for st in eng.stages:                # break the Stage <-> Engine cycle: buffers free now
                            st.eng = None
                        eng.stages.clear()
            # A model is a reference cycle (its loss closures, its stages and engines), so the device buffers of a
            # model the caller has dropped return to the allocator only when the cycle collector runs — which it
            # schedules by object counts, not by device memory.  Collect before allocating tens of GB for this shape.
            gc.collect()
            cache[key] = self._build_engines(batch, size)
        else:
            cache[key] = cache.pop(key)                      # most recently used last
        self._eng_key = key
        e = cache[key]
        self._eng_G, self._eng_Dd, self._eng_Dg = e["G"], e.get("Dd"), e.get("Dg")
        self._dpred_d, self._dpred_g = e.get("dpred_d"), e.get("dpred_g")
        self._eng_extra = e
        if self.is_train:
            self.optimizer_G.flat_grad = self._eng_G.flat_grad
            if self._eng_Dd is not None:
                self.optimizer_D.flat_grad = self._eng_Dd.flat_grad

    def _build_engines(self, batch: int, size: int) -> dict:
        e = {}
        g = e["G"] = self.build_generator_engine(batch, size)
        # dropout masks follow the GLOBAL sample index: rank r holds samples [r*batch, (r+1)*batch)  (SURVEY §8e ii)
        g.sample_base = int(getattr(self.opt, "b200_sample_base", parallel.rank() * batch))
        if self.is_train:
            g.alloc_grads()
            g.bind_backward()
        if self.is_train and hasattr(self, "net_discriminator"):
            dn = self.net_discriminator
            # the D step's fake and real halves are two D calls: with batch norm, two sample groups with their own
            # statistics and running-buffer updates (fake first)
            D = E.PixelGANEngine if isinstance(dn, M.PixelDiscriminator) else E.PatchGANEngine
            dd = e["Dd"] = D(dn, 2 * batch, size, self.device, self.nsplit, groups=2,
                             deterministic=self.deterministic, bn_sync=self._bn_sync)
            dd.alloc_grads()
            dd.bind_backward()
            dg = e["Dg"] = D(dn, batch, size, self.device, self.nsplit, din=dd.din.batch_slice(0, batch), input_grad=True,
                             deterministic=self.deterministic, bn_sync=self._bn_sync)
            dg.alloc_grads(share_with=dd)
            dg.bind_backward(wgrad=False)
            e["dpred_d"] = torch.zeros_like(dd.pred)
            e["dpred_g"] = torch.zeros_like(dg.pred)
        return e

    def loss_values(self):
        """The device-side loss sums of the last step as Python floats: ONE 64-byte D2H copy (and the step's only host
        synchronisation) however many terms train.py:74 / get_current_losses() reads."""
        if self._acc_host is None:
            self._acc_host = self._acc.tolist()
        return self._acc_host

    def step_seed(self) -> int:
        return (self._seed_base * 1000003 + self._step) & 0xFFFFFFFF

    def draw_label(self) -> float:
        """One smooth-label scalar exactly as GANLoss.get_target_tensor computes it (loss.py:65-107):
        fp32 `rand(1) * (1.1 - 0.7) + 0.7`, for real AND fake targets."""
        return self._labels.draw()

    def label_draws(self) -> int:
        """Smooth labels one training step draws: D_fake, D_real, G_gan for vanilla / lsgan; none for wgan, whose loss
        has no target (loss.py:123-127), so the CPU generator is left where the reference leaves it."""
        if not hasattr(self, "net_discriminator") or self._gan_obj == ops.GAN_WGAN:
            return 0
        return 3

    def _targets(self, lo: int, hi: int, wgan_signs) -> object:
        """Per-half scalars of the GAN loss calls lo..hi-1: with wgan the signs (+1 fake, -1 real), constants of the call
        site; otherwise the device view of the smooth-label targets lo..hi-1 of the step-parameter buffer, drawn here
        (reference order) when the phases are run by hand, by the step prologue inside optimize_parameters()."""
        if self._gan_obj == ops.GAN_WGAN:
            return wgan_signs
        if not self._sp_ready:
            ops.set_step_params(self._sp[lo:hi], [self.draw_label() for _ in range(lo, hi)])
        return self._sp[lo:hi]

    def allreduce_grads(self, eng) -> None:
        """Sum over ranks (the 1/world factor is applied by the optimizer kernel as it reads the gradients; code that
        reads flat_grad directly under DP sees the SUM)."""
        parallel.sum_gradients(eng.flat_grad)

    def grad_scale(self) -> float:
        return 1.0 / self._world

    # ---- discriminator phases (conditioning supplied by the plugin through pack_D_inputs) ----
    @abstractmethod
    def pack_D_inputs(self, din_fake: ops.Planes, din_real: Optional[ops.Planes]) -> None:
        """Write the conditioned fake (and real) discriminator inputs into the operand planes."""

    def backward_D(self):
        """D(fake.detach()) and D(real) as one 2B batch; loss_D = 0.5 * (fake + real)
        (warp_model.py:109-139, texture_model.py:127-155)."""
        B = self._eng_key[0]
        d = self._eng_Dd
        d.training = self.training
        d.pack()
        self.pack_D_inputs(d.din.batch_slice(0, B), d.din.batch_slice(B, B))
        pred = d.forward()
        t = self._targets(0, 2, (1.0, -1.0))                     # order: D_fake, D_real (loss.py:117,121)
        ops.gan_loss_fwd_bwd(self._gan_obj, pred, 2, t, 0.5, self._acc[0:2], self._dpred_d, ws=self._det_ws)
        d.backward(self._dpred_d)
        self.allreduce_grads(d)

    def gan_backward_through_D(self) -> torch.Tensor:
        """G phase: D(fake) with the updated D, the GAN objective against a 'real' target, gradient back to the
        discriminator input.  Returns d(loss_G_gan)/d(din) [B,S,S,pad64(cin)] (fp32 NHWC)."""
        g = self._eng_Dg
        g.training = self.training
        g.pack()
        pred = g.forward()
        t = self._targets(2, 3, (-1.0,))
        ops.gan_loss_fwd_bwd(self._gan_obj, pred, 1, t, self.gan_weight(), self._acc[2:3], self._dpred_g,
                             ws=self._det_ws)
        g.backward(self._dpred_g, wgrad=False)
        return g.dx_in

    # ---- the training step: a prologue on the host, then a fixed launch sequence (eager or graph replay) ----
    def input_tensors(self) -> dict:
        """name -> device input of the current step (tensor or ops.SegMap); provided by the plugin."""
        raise NotImplementedError

    def set_input_tensors(self, d: dict) -> None:
        for k, v in d.items():
            setattr(self, k, v)

    def _step_prologue(self, optimizers) -> None:
        """Everything of a step that is decided on the host, written to the device with ONE tiny launch: the smooth
        labels (CPU RNG, reference order; none with wgan), both optimizers' scalars of this step, the dropout step
        seed."""
        vals = [0.0] * 22
        for i in range(self.label_draws()):
            vals[i] = self.draw_label()
        for off, name in ((4, "D"), (12, "G")):
            if name in optimizers:
                vals[off:off + 8] = getattr(self, "optimizer_" + name).advance(self.grad_scale())
        seed = self.step_seed()
        vals[20], vals[21] = float(seed & 0xFFFF), float(seed >> 16)
        ops.set_step_params(self._sp, vals)

    def _step_body(self) -> None:
        """forward -> zero/backward/step D -> zero/backward/step G (base_gan.py:194-203) as device work only."""
        self._acc.zero_()
        self.forward()
        self._eng_Dd.zero_grad()
        self.backward_D()
        self.optimizer_D.launch(self._sp[4:12])
        self._eng_G.zero_grad()
        self.backward_G()
        self.optimizer_G.launch(self._sp[12:20])

    def _run_step(self, optimizers=("D", "G")) -> None:
        self._acc_host = None
        ins = self.input_tensors()
        first = next(iter(ins.values()))
        B, S = first.shape[0], first.shape[-1]
        self.ensure_engines(B, S)
        for eng in (self._eng_G, self._eng_Dd, self._eng_Dg):
            if eng is not None:
                eng.seed_dev = self._sp[20:22]
        self._step_prologue(optimizers)
        self._sp_ready = True
        try:
            sig = tuple((k, str(getattr(v, "data", v).dtype), tuple(v.shape)) for k, v in ins.items())
            key = (B, S, bool(self.training), sig, optimizers)
            use_graph = self.graph_enabled and self._world == 1 and ops.Plan.trace is None
            if not use_graph:
                self._step_body()
            else:
                g = self._graphs.get(key)
                if g is None and self._eager_steps.get(key, 0) < 2:   # warm-up: lazy allocations, attribute calls
                    self._eager_steps[key] = self._eager_steps.get(key, 0) + 1
                    self._step_body()
                else:
                    self.wait_late_copies()                          # H2D of this step's inputs (side stream)
                    if g is None:
                        g = self._graphs[key] = self._capture(ins)
                    static = g["static"]
                    for k, v in ins.items():                          # staging -> the buffers the graph reads
                        getattr(static[k], "data", static[k]).copy_(getattr(v, "data", v))
                    self.set_input_tensors(static)
                    g["graph"].replay()
                    ops.count_replayed(g["launches"])
        finally:
            self._sp_ready = False
            for eng in (self._eng_G, self._eng_Dd, self._eng_Dg):
                if eng is not None:
                    eng.seed_dev = None
        self._step += 1

    def _capture(self, ins: dict) -> dict:
        """Capture _step_body() on static copies of the inputs.  The kernels of the capture pass are recorded, not
        executed: the caller replays the graph for the current step right away."""
        static = {}
        for k, v in ins.items():
            d = getattr(v, "data", v).clone()
            static[k] = ops.SegMap(d, v.channels) if isinstance(v, ops.SegMap) else d
        self.set_input_tensors(static)
        torch.cuda.synchronize(self.device)
        n0 = ops.launch_count()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            self._step_body()
        n = ops.launch_count() - n0
        ops.count_replayed(-n)          # the capture pass recorded the launches, it did not execute them
        return {"graph": graph, "static": static, "launches": n}

    def optimize_parameters(self):
        self._run_step()
