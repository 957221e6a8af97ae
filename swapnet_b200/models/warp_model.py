"""Warp-stage plugin (`--model warp`) on the B200 engines.

Same options, attributes and step semantics as /root/reference/models/warp_model.py:14-183:
generator = WarpModule(body 3ch, cloth 19ch), conditional PatchGAN on cat(body, cloth) (22 ch),
loss_G = lambda_ce * CE(fakes, argmax(targets)) + lambda_gan * GAN (or CE only with
--warp_mode ce).
"""
from __future__ import annotations

from argparse import ArgumentParser

import torch

from .. import engine as E
from .. import modules as M
from .. import ops
from ..ops import GradSrc
from .base_gan import BaseGAN
from .base_model import LazyLoss


class WarpModel(BaseGAN):
    @staticmethod
    def modify_commandline_options(parser: ArgumentParser, is_train):
        if is_train:
            parser.add_argument("--warp_mode", default="gan", choices=("gan", "ce"))
            parser.add_argument("--lambda_ce", type=float, default=100,
                                help="weight for cross entropy loss in final term")
            parser.set_defaults(display_ncols=4)
        return super(WarpModel, WarpModel).modify_commandline_options(parser, is_train)

    def __init__(self, opt):
        self.body_channels = opt.body_channels if opt.body_representation == "labels" else 3
        self.cloth_channels = opt.cloth_channels if opt.cloth_representation == "labels" else 3
        BaseGAN.__init__(self, opt)
        self.visual_names = ["inputs_decoded", "bodys_unnormalized", "fakes_decoded"]
        if self.is_train:
            self.visual_names.append("targets_decoded")
            self.loss_G_ce = LazyLoss(lambda: self.loss_values()[3])
            if opt.warp_mode != "gan":
                self.model_names = ["generator"]
                self.loss_names = "G"   # (sic) warp_model.py:71 — a str; get_current_losses iterates its chars
                del self.net_discriminator
                del self.optimizer_D
                self.optimizer_names = ["G"]
                self.loss_G = self.loss_G_ce
            else:
                self.loss_names += ["G_ce"]
                lam = float(opt.lambda_gan)
                self.loss_G = LazyLoss(lambda: lam * self.loss_values()[2] + self.loss_values()[3])

    # ---- visuals: off the hot path; reuse the reference's helpers when they are importable ----
    def compute_visuals(self):
        from datasets.data_utils import unnormalize
        from util.decode_labels import decode_cloth_labels

        self.inputs_decoded = decode_cloth_labels(self.dense(self.inputs))
        self.bodys_unnormalized = unnormalize(self.bodys, *self.opt.body_norm_stats)
        self.targets_decoded = decode_cloth_labels(self.dense(self.targets))
        self.fakes_decoded = decode_cloth_labels(self.fakes)

    def define_G(self):
        return M.WarpModule(body_channels=self.body_channels, cloth_channels=self.cloth_channels)

    def get_D_inchannels(self):
        return self.cloth_channels + self.body_channels

    def build_generator_engine(self, batch, size):
        return E.WarpEngine(self.net_generator, batch, size, self.device, self.nsplit, train=self.is_train,
                            deterministic=self.deterministic)

    def set_input(self, input):
        # all H2D copies run on a side stream in the order the step needs them: the body (3 ch) first — the
        # body branch and the weight packing run while the 19-channel cloth is still in flight —, the targets
        # last (first needed by the D step, one generator forward later).  No-op for device tensors.
        self.bodys = self.copy_late(input["bodys"], "bodys")
        if "input_labels" in input:
            # a batch of `--dataset warp_b200` (dropin/datasets/warp_b200_dataset.py): uint8 label maps + the drawn op
            # table; the one-hot expansion and the per-channel augmentation (datasets/data_utils.py:330-361) run here,
            # on the device (swapnet_b200/data.py, csrc/augment.cu) — 4 MB + 88 KB of H2D for a 512x512 batch of 16
            from .. import data as D

            if getattr(self, "_augmenter", None) is None:
                self._augmenter = D.ClothAugmenter(None, self.cloth_channels)
            table = D.OpTable.from_collated(input["input_ops"], self.cloth_channels)
            source = input["input_labels"].to(self.device, non_blocking=True)
            self.inputs = self._augmenter.apply(source, table)
            target = input["target_labels"]
            if "resize_iy" in input:
                # the reference's nearest resize + crop AFTER the augmentation (warp_dataset.py:150-174) = one gather per axis
                iy, ix = input["resize_iy"][0], input["resize_ix"][0]
                self.inputs = D.gather_rows_cols(self.inputs, iy.to(self.device), ix.to(self.device))
                target = D.gather_rows_cols(target, iy, ix).contiguous()
            self.targets = self.copy_late(target, "targets", seg_channels=self.cloth_channels)
        else:
            # the cloth tensors may arrive in compact form (uint8 label map / int32 bit mask [B,H,W], ops.SegMap)
            self.inputs = self.copy_late(input["input_cloths"], "inputs", seg_channels=self.cloth_channels)
            self.targets = self.copy_late(input["target_cloths"], "targets", seg_channels=self.cloth_channels)
        self.image_paths = tuple(zip(input["cloth_paths"], input["body_paths"]))

    def forward(self):
        B, _, S, S2 = self.bodys.shape
        assert S == S2, "square inputs expected"
        self.ensure_engines(B, S)
        g = self._eng_G
        g.pack()                      # needs the weights only: overlaps the input copies
        self.wait_copy("bodys")
        out = g.forward(self.bodys, self.inputs, training=self.training and self.is_train, seed=self.step_seed(),
                        before_cloth=lambda: self.wait_copy("inputs"))
        self.fakes = out.permute(0, 3, 1, 2)   # [B,19,S,S] view of the NHWC storage
        self.wait_late_copies()

    def pack_D_inputs(self, din_fake, din_real):
        """conditioned = cat((bodys, cloth), 1): body first (warp_model.py:115,119,157)."""
        ops.pack_concat([(self.bodys, False), (self._eng_G.fakes, True)], din_fake)
        if din_real is not None:
            ops.pack_concat([(self.bodys, False), (self.targets, False)], din_real)

    def backward_G(self):
        """loss_G = lambda_ce * CE(fakes, argmax(targets)) + lambda_gan * GAN (warp_model.py:141-167).  The GAN term's
        gradient w.r.t. the fakes comes back from the discriminator first; the cross entropy, the sum of both gradients and
        the tanh backward of the head are ONE kernel writing the head's dy planes (ops.ce_tanh_bwd)."""
        g = self._eng_G
        extra = []
        if self.opt.warp_mode == "gan":
            extra.append(GradSrc(self.gan_backward_through_D(), self.body_channels))
        ops.ce_tanh_bwd(g.fakes, self.cloth_channels, self.targets, float(self.opt.lambda_ce), self._acc[3:4], extra,
                        g.head.dy, ws=self._det_ws)
        if self._world > 1:
            from .. import parallel
            avg = parallel.BucketedAverager(g.flat_grad, g.grad_buckets(), scale=False)   # 1/world: in the AdamW kernel
            g.backward(None, on_bucket=avg.ready)
            avg.finish()
        else:
            g.backward(None)

    def input_tensors(self):
        return {"bodys": self.bodys, "inputs": self.inputs, "targets": self.targets}

    def _step_body(self):
        if self.opt.warp_mode == "gan":
            return super()._step_body()
        self._acc.zero_()                      # --warp_mode ce: generator only (warp_model.py:175-183)
        self.forward()
        self._eng_G.zero_grad()
        self.backward_G()
        self.optimizer_G.launch(self._sp[12:20])

    def optimize_parameters(self):
        self._run_step(("D", "G") if self.opt.warp_mode == "gan" else ("G",))
