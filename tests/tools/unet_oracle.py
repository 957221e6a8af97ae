"""TEST INFRASTRUCTURE ONLY — fp64 training-step losses of the two models built on a bare UnetGenerator:
pix2pix (pix2pix_model.py:153-212) and the texture stage with `--netG unet_128` (texture_model.py:96-101,121-180).
Built on norm_oracle.unet_generator / patchgan_forward and gan_modes_oracle's GANLoss; the generator's keys are the
standalone ones (`model.model...`), which unet_generator reads under a prefix.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

import gan_modes_oracle as GM
import norm_oracle as NO
from oracle import nets as ON

ZERO_CHANNELS = 36
NUM_DOWNS = 7
_P = "g"

# pix2pix's --gan_mode -> the GANLoss it computes (no gradient penalty is ever added)
PIX2PIX_MODES = {"vanilla": "vanilla", "dragan-gp": "vanilla", "dragan-lp": "vanilla", "lsgan": "lsgan",
                 "wgan": "wgan", "wgan-gp": "wgan"}


def unet_forward(sdG, x, norm: str, train: bool, drop=None, num_downs: int = NUM_DOWNS):
    """UnetGenerator(x) with `num_downs` downsamplings -> (output, running buffers after the call, keyed like sdG)."""
    psd = {f"{_P}.{k}": v for k, v in sdG.items()}
    bn = NO.BN(psd, norm, train)
    out = NO.unet_generator(psd, _P, x, num_downs, bn, drop)
    return out, {k[len(_P) + 1:]: v for k, v in bn.bufs.items()}


def _l1(fakes, targets, lambda_l1, l1_sign):
    if l1_sign is None:
        return F.l1_loss(fakes, targets) * lambda_l1
    return ((fakes - targets) * l1_sign).mean() * lambda_l1


def real_A(cloth):
    B, _, S, _ = cloth.shape
    return torch.cat((torch.zeros(B, ZERO_CHANNELS, S, S, dtype=cloth.dtype), cloth), 1)


def pix2pix_step_losses(sdG, sdD, cloth, targets, draws, gan_mode: str, norm: str, train: bool, lambda_l1=10.0,
                        drop=None, l1_sign=None):
    """Pix2PixModel.backward_D / backward_G with the same D weights in both phases (no optimizer step between)."""
    mode = PIX2PIX_MODES[gan_mode]
    a = real_A(cloth)
    fakes, bufsG = unet_forward(sdG, a, norm, train, drop)
    bnD = NO.BN(sdD, norm, train)
    o = GM._d_losses(sdD, bnD, a, fakes, targets, draws, mode, 1.0)      # loss_G_GAN carries no lambda_gan
    l1 = _l1(fakes, targets, lambda_l1, l1_sign)
    o.update(fakes=fakes, G=o["G_gan"] + l1, G_GAN=o["G_gan"], G_L1=l1, bufsG=bufsG, bufsD=bnD.bufs)
    return o


def texture_unet_step_losses(sdG, sdD, tex, cloth, targets, draws, gan_mode: str = "vanilla", norm: str = "instance",
                             train: bool = True, lambda_l1=10.0, lambda_gan=1.0, drop=None, l1_sign=None, vgg=None,
                             lambda_content=0.0, lambda_style=0.0):
    """TextureModel with --netG unet_128: G = the batch-norm U-Net on the input texture alone; D (--norm) on
    cat(cloth, texture); L1, content, style and GAN terms as with --netG swapnet."""
    fakes, bufsG = unet_forward(sdG, tex, "batch", train, drop)
    bnD = NO.BN(sdD, norm, train)
    o = GM._d_losses(sdD, bnD, cloth, fakes, targets, draws, gan_mode, lambda_gan)
    l1 = _l1(fakes, targets, lambda_l1, l1_sign)
    content = style = 0.0
    if lambda_content != 0 or lambda_style != 0:
        c, st = ON.perceptual_loss(vgg, fakes, targets, lambda_style != 0)
        content, style = c * lambda_content, st * lambda_style
    o.update(fakes=fakes, G=o["G_gan"] + l1 + content + style, G_l1=l1, G_content=content, G_style=style,
             bufsG=bufsG, bufsD=bnD.bufs)
    return o
