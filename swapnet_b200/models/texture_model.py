"""Texture-stage plugin (`--model texture`) on the B200 engines.

Options, attributes and step semantics of /root/reference/models/texture_model.py:17-180 for both of its
generators: `--netG swapnet` (TextureModule, on engine.TextureEngine) and `--netG unet_128` (a bare 7-level
UnetGenerator with batch norm whatever --norm says and dropout, fed the input texture alone; the rois are unused:
texture_model.py:96-101,121-125; on engine.UnetEngine).  Either way: conditional PatchGAN on cat(cloths, texture)
(cloth FIRST, :138,142,164), loss_G = lambda_gan * GAN + lambda_l1 * L1 (+ perceptual terms).

The VGG16 perceptual terms (texture_model.py:68-69,171-178 -> modules/losses/perceptual.py) run on
engine.PerceptualEngine.  `vgg16(pretrained=True)` needs the torchvision weight file: `--b200_vgg`
selects `pretrained` (default, like the reference; raises when the file cannot be obtained), a path to a
saved state_dict, or `random[:seed]` (seeded torchvision init — what the offline tests and bench use).
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


class TextureModel(BaseGAN):
    @staticmethod
    def modify_commandline_options(parser: ArgumentParser, is_train):
        parser = super(TextureModel, TextureModel).modify_commandline_options(parser, is_train)
        if is_train:
            parser.add_argument("--netG", default="swapnet", choices=["swapnet", "unet_128"])
            parser.add_argument("--lambda_l1", type=float, default=10, help="weight for L1 loss in final term")
            parser.add_argument("--lambda_content", type=float, default=20, help="weight for content loss in final term")
            parser.add_argument("--lambda_style", type=float, default=1e-8, help="weight for style loss in final term")
            parser.add_argument("--b200_vgg", default="pretrained",
                                help="VGG16 weights of the perceptual loss: pretrained | random[:seed] | <state_dict path>")
            parser.set_defaults(display_ncols=5)
        return parser

    def __init__(self, opt):
        # at test time --netG is not an option: it comes from the saved training options (inference.py)
        self.netG = getattr(opt, "netG", "swapnet")
        if self.netG not in ("swapnet", "unet_128"):
            raise ValueError("Cannot find implementation for " + self.netG)
        BaseGAN.__init__(self, opt)
        self.visual_names = ["textures_unnormalized", "cloths_decoded", "fakes", "fakes_scaled"]
        if self.is_train:
            self.visual_names.append("targets_unnormalized")
            self.lam_content = float(getattr(opt, "lambda_content", 0))
            self.lam_style = float(getattr(opt, "lambda_style", 0))
            self.net_vgg = None
            self._eng_P = None
            if self.lam_content != 0:
                # the reference builds PerceptualLoss unconditionally (texture_model.py:68); the frozen VGG is
                # only needed when the content term is on (the style term uses the raw images)
                self.net_vgg = M.load_vgg16_features(getattr(opt, "b200_vgg", "pretrained")).to(self.device)
            lam = float(opt.lambda_gan)
            lv = self.loss_values
            self.loss_G_l1 = LazyLoss(lambda: lv()[3])
            self.loss_G_content = LazyLoss(lambda: lv()[4]) if self.lam_content != 0 else 0.0
            self.loss_G_style = LazyLoss(lambda: lv()[5]) if self.lam_style != 0 else 0.0
            self.loss_G = LazyLoss(lambda: lam * lv()[2] + lv()[3] + lv()[4] + lv()[5])
            for loss in ("l1", "content", "style"):
                if getattr(opt, "lambda_" + loss, 0) != 0:
                    self.loss_names.append("G_" + loss)

    def compute_visuals(self):
        from datasets.data_utils import scale_tensor, unnormalize
        from util.decode_labels import decode_cloth_labels

        self.textures_unnormalized = unnormalize(self.textures, *self.opt.texture_norm_stats)
        try:                                   # texture_model.py:79-81 (needs seaborn through util/draw_rois.py)
            from util.draw_rois import draw_rois_on_texture
        except ImportError:
            draw_rois_on_texture = None
        if draw_rois_on_texture is not None:
            self.textures_unnormalized = draw_rois_on_texture(self.rois, self.textures_unnormalized)
        self.cloths_decoded = decode_cloth_labels(self.dense(self.cloths))
        self.fakes_scaled = scale_tensor(self.fakes, scale_each=True)
        if self.is_train:
            self.targets_unnormalized = unnormalize(self.targets, *self.opt.texture_norm_stats)

    def get_D_inchannels(self):
        return self.opt.texture_channels + self.opt.cloth_channels

    def define_G(self):
        if self.netG == "unet_128":
            ct = self.opt.texture_channels
            return M.UnetGenerator(ct, ct, 7, 64, use_dropout=True, norm="batch")
        return M.TextureModule(texture_channels=self.opt.texture_channels, cloth_channels=self.opt.cloth_channels,
                               num_roi=self.opt.body_channels, img_size=self.opt.crop_size,
                               norm_type=getattr(self.opt, "norm", "instance"))

    def build_generator_engine(self, batch, size):
        if self.netG == "unet_128":
            return E.UnetEngine(self.net_generator, batch, size, self.device, self.nsplit, train=self.is_train,
                                deterministic=self.deterministic, bn_sync=self._bn_sync)
        return E.TextureEngine(self.net_generator, batch, size, self.device, self.nsplit, train=self.is_train,
                               deterministic=self.deterministic, bn_sync=self._bn_sync)

    def _build_engines(self, batch, size):
        e = super()._build_engines(batch, size)
        if self.is_train and (self.lam_content != 0 or self.lam_style != 0):
            e["P"] = E.PerceptualEngine(self.net_vgg, batch, size, self.device, self.nsplit,
                                        content=self.lam_content != 0, deterministic=self.deterministic)
        return e

    def ensure_engines(self, batch, size):
        super().ensure_engines(batch, size)
        self._eng_P = self._eng_extra.get("P")

    def set_input(self, input):
        # side-stream H2D copies in the order the step needs them (see WarpModel.set_input)
        self.textures = self.copy_late(input["input_textures"], "textures")
        self.rois = self.copy_late(input["rois"], "rois")
        self.cloths = self.copy_late(input["cloths"], "cloths", seg_channels=self.opt.cloth_channels)
        self.targets = self.copy_late(input["target_textures"], "targets")
        self.image_paths = tuple(zip(input["cloth_paths"], input["texture_paths"]))

    def input_tensors(self):
        return {"textures": self.textures, "rois": self.rois, "cloths": self.cloths, "targets": self.targets}

    def forward(self):
        B, _, S, S2 = self.textures.shape
        assert S == S2, "square inputs expected"
        self.ensure_engines(B, S)
        g = self._eng_G
        g.pack()                      # needs the weights only: overlaps the input copies
        self.wait_copy("textures")
        training = self.training and self.is_train
        if self.netG == "unet_128":
            ops.pack_concat([(self.textures, False)], g.x_in)
            out = g.forward(training=training, seed=self.step_seed())
        else:
            self.wait_copy("rois")
            out = g.forward(self.textures, self.rois, self.cloths, training=training, seed=self.step_seed(),
                            before_cloth=lambda: self.wait_copy("cloths"))
        self.fakes = out.permute(0, 3, 1, 2)
        self.wait_late_copies()

    def pack_D_inputs(self, din_fake, din_real):
        ops.pack_concat([(self.cloths, False), (self._eng_G.fakes, True)], din_fake)
        if din_real is not None:
            ops.pack_concat([(self.cloths, False), (self.targets, False)], din_real)

    def backward_G(self):
        g = self._eng_G
        B, S = self._eng_key
        ct = self.opt.texture_channels
        if not hasattr(self, "_dl1") or self._dl1.shape[0] != B or self._dl1.shape[1] != S:
            self._dl1 = torch.zeros(B, S, S, ct, device=self.device)
        ops.l1_loss_fwd_bwd(g.fakes, ct, self.targets, float(self.opt.lambda_l1), self._acc[3:4], self._dl1,
                            ws=self._det_ws)
        srcs = [GradSrc(self._dl1)]
        if self.lam_style != 0:      # 5 x MSE of the raw-image Gram matrices (perceptual.py:58-63): adds into _dl1
            self._eng_P.style(g.fakes, self.targets, self.lam_style, self._acc[5:6], self._dl1)
        if self.lam_content != 0:
            srcs.append(GradSrc(self._eng_P.content(g.fakes, self.targets, self.lam_content, self._acc[4:5])))
        dx = self.gan_backward_through_D()
        srcs.append(GradSrc(dx, self.opt.cloth_channels))
        g.backward(srcs)
        self.allreduce_grads(g)
