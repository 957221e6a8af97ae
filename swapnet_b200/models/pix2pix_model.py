"""The pix2pix baseline (`--model pix2pix`) on the B200 engines: /root/reference/models/pix2pix_model.py:11-212.

cloth -> texture with a 7-level UnetGenerator (unet_128) conditioned on real_A = cat(zeros[B, 36, S, S], cloths)
(pix2pix_model.py:158-159) and a conditional discriminator on cat(real_A, texture).  The zero channels are written by
ops.pack_concat's zero lead, in the same pass as the cloth; the dense real_A is built for the visuals only.

Reference semantics kept:
  * options: its own modifier (defaults norm=batch, netG=unet_128; --lambda_l1 10, --beta1 0.5 and its copies of the
    GAN flags), --lr from train_options; --optimizer_G/D, --lambda_gan and --lambda_gp are parsed and ignored;
  * G = UnetGenerator(cloth_channels + 36, texture_channels, 7, 64, --norm, dropout) with init_weights; D = define_D
    with PyTorch's default init (the reference's define_D ignores init_type); constructed G, init G, D;
  * losses: loss_D = (fake + real) * 0.5; loss_G = GAN(D(cat(real_A, fake_B)), real) with no lambda_gan, plus
    lambda_l1 * L1(fake_B, real_B); both optimizers are Adam(lr=--lr, betas=(beta1, 0.999)), no weight decay;
  * checkpoints <epoch>_net_G.pth / <epoch>_net_D.pth, no optimizer files;
  * --gan_mode: what its GANLoss accepts (BCE with logits for vanilla and dragan-gp/lp, MSE for lsgan, the Wasserstein
    mean for wgan and wgan-gp).  pix2pix never computes a gradient penalty, so wgan-gp is plain wgan and dragan-* is
    plain vanilla.  mescheder-* and --gan_label_mode hard are refused, as they fail in the reference.
One deliberate difference: the zero channels take the batch's actual size; the reference's use --batch_size and fail
on a short last batch.
"""
from __future__ import annotations

from argparse import ArgumentParser

import torch

from .. import engine as E
from .. import modules as M
from .. import ops
from ..ops import GradSrc
from .base_gan import BaseGAN, add_b200_options
from .base_model import LazyLoss

ZERO_CHANNELS = 36       # pix2pix_model.py:158: the conditioning's leading zero channels

# --gan_mode -> the loss kernels' objective (loss.py:54-61: GANLoss's choice by name; no penalty is ever added)
PIX2PIX_GAN_OBJECTIVES = {"vanilla": ops.GAN_BCE, "dragan-gp": ops.GAN_BCE, "dragan-lp": ops.GAN_BCE,
                          "lsgan": ops.GAN_MSE, "wgan": ops.GAN_WGAN, "wgan-gp": ops.GAN_WGAN}


class Pix2PixModel(BaseGAN):
    @staticmethod
    def modify_commandline_options(parser: ArgumentParser, is_train=True):
        """pix2pix_model.py:21-103, plus the engine switches."""
        parser.set_defaults(norm="batch", netG="unet_128")
        if is_train:
            parser.add_argument("--lambda_l1", type=float, default=10, help="weight for L1 loss")
            parser.add_argument("--gan_mode", help="gan regularization to use", default="vanilla",
                                choices=("vanilla", "wgan", "wgan-gp", "lsgan", "dragan-gp", "dragan-lp",
                                         "mescheder-r1-gp", "mescheder-r2-gp"))
            parser.add_argument("--lambda_gan", type=float, default=1.0, help="weight for adversarial loss")
            parser.add_argument("--lambda_gp", help="weight parameter for gradient penalty", type=float, default=10)
            parser.add_argument("--discriminator", default="basic", choices=("basic", "pixel", "n_layers"),
                                help="what discriminator type to use")
            parser.add_argument("--n_layers_D", type=int, default=3, help="only used if discriminator==n_layers")
            parser.add_argument("--norm", type=str, default="instance",
                                help="instance normalization or batch normalization [instance | batch | none]")
            parser.add_argument("--optimizer_G", help="optimizer for generator", default="AdamW",
                                choices=("AdamW", "AdaBound"))
            parser.add_argument("--optimizer_D", help="optimizer for discriminator", default="AdamW",
                                choices=("AdamW", "AdaBound"))
            parser.add_argument("--beta1", type=float, default=0.5, help="momentum term of adam")
            parser.add_argument("--gan_label_mode", default="smooth", choices=("hard", "smooth"),
                                help="whether to use hard (real 1.0 and fake 0.0) or smooth "
                                     "(real [0.7, 1.1] and fake [0., 0.3]) values for labels")
            parser.set_defaults(pool_size=0, gan_mode="vanilla")
        return add_b200_options(parser)

    def __init__(self, opt):
        BaseGAN.__init__(self, opt)
        self.net_G = self.net_generator
        self.model_names = ["G"]
        self.visual_names = ["cloth_decoded", "fakes_scaled", "textures_unnormalized"]
        if self.is_train:
            self.net_D = self.net_discriminator
            self.model_names = ["G", "D"]
            self.optimizer_names = []         # the reference saves no optimizer state
            self.loss_names = ["G", "G_GAN", "G_L1", "D_real", "D_fake"]
            lv = self.loss_values
            self.loss_G_GAN = LazyLoss(lambda: lv()[2])
            self.loss_G_L1 = LazyLoss(lambda: lv()[3])
            self.loss_G = LazyLoss(lambda: lv()[2] + lv()[3])

    # ---- where pix2pix departs from BaseGAN ----
    def gan_objective(self, mode: str) -> int:
        if mode not in PIX2PIX_GAN_OBJECTIVES:
            raise NotImplementedError(f"--gan_mode {mode}: the reference's GANLoss does not implement it either "
                                      "(loss.py:61-62)")
        return PIX2PIX_GAN_OBJECTIVES[mode]

    def gan_weight(self) -> float:
        return 1.0                            # loss_G_GAN is not weighted (pix2pix_model.py:198)

    def init_D_weights(self, net) -> None:
        pass                                  # define_D ignores init_type: PyTorch's default init

    def define_optimizers(self):
        from ..optim import FusedAdamW, flatten_parameters

        out = []
        for net in (self.net_generator, self.net_discriminator):
            params = list(net.parameters())
            out.append(FusedAdamW(params, flatten_parameters(params), lr=self.opt.lr, betas=(self.opt.beta1, 0.999),
                                  eps=1e-8, weight_decay=0.0))
        return tuple(out)

    # ---- networks ----
    def get_D_inchannels(self):
        return self.opt.cloth_channels + ZERO_CHANNELS + self.opt.texture_channels

    def define_G(self):
        return M.UnetGenerator(self.opt.cloth_channels + ZERO_CHANNELS, self.opt.texture_channels, 7, 64,
                               use_dropout=True, norm=self.opt.norm)

    def build_generator_engine(self, batch, size):
        return E.UnetEngine(self.net_generator, batch, size, self.device, self.nsplit, train=self.is_train,
                            deterministic=self.deterministic, bn_sync=self._bn_sync)

    # ---- step ----
    def set_input(self, input):
        self.cloths = self.copy_late(input["cloths"], "cloths", seg_channels=self.opt.cloth_channels)
        self.targets = self.copy_late(input["target_textures"], "targets")

    def input_tensors(self):
        return {"cloths": self.cloths, "targets": self.targets}

    @property
    def real_B(self):
        return self.targets

    def forward(self):
        B, _, S, S2 = self.cloths.shape
        assert S == S2, "square inputs expected"
        self.ensure_engines(B, S)
        g = self._eng_G
        g.pack()
        self.wait_copy("cloths")
        ops.pack_concat([(self.cloths, False)], g.x_in, lead=ZERO_CHANNELS)
        out = g.forward(training=self.training and self.is_train, seed=self.step_seed())
        self.fake_B = out.permute(0, 3, 1, 2)
        self.wait_late_copies()

    def pack_D_inputs(self, din_fake, din_real):
        ops.pack_concat([(self.cloths, False), (self._eng_G.fakes, True)], din_fake, lead=ZERO_CHANNELS)
        if din_real is not None:
            ops.pack_concat([(self.cloths, False), (self.targets, False)], din_real, lead=ZERO_CHANNELS)

    def backward_G(self):
        g = self._eng_G
        B, S = self._eng_key
        ct = self.opt.texture_channels
        if not hasattr(self, "_dl1") or self._dl1.shape[0] != B or self._dl1.shape[1] != S:
            self._dl1 = torch.zeros(B, S, S, ct, device=self.device)
        ops.l1_loss_fwd_bwd(g.fakes, ct, self.targets, float(self.opt.lambda_l1), self._acc[3:4], self._dl1,
                            ws=self._det_ws)
        dx = self.gan_backward_through_D()
        g.backward([GradSrc(self._dl1), GradSrc(dx, ZERO_CHANNELS + self.opt.cloth_channels)])
        self.allreduce_grads(g)

    def compute_visuals(self):
        from datasets.data_utils import scale_tensor, unnormalize
        from util.decode_labels import decode_cloth_labels

        cloths = self.dense(self.cloths)
        B, _, S, _ = cloths.shape
        self.real_A = torch.cat((torch.zeros(B, ZERO_CHANNELS, S, S, device=cloths.device), cloths), 1)
        self.cloth_decoded = decode_cloth_labels(self.real_A)
        self.fakes_scaled = scale_tensor(self.fake_B)
        self.textures_unnormalized = unnormalize(self.real_B, *self.opt.texture_norm_stats)
