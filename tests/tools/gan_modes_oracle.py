"""TEST INFRASTRUCTURE ONLY — the CPU oracle's training-step losses with the `--gan_mode` objective as a parameter:
GANLoss (modules/loss.py:12-130) for vanilla (BCE with logits), lsgan (MSE) and wgan (-mean for real, +mean for fake),
composed with the `--norm` choice of tests/tools/norm_oracle.py.  With gan_mode='vanilla' and norm='instance' the
losses are those of oracle/nets.py warp_step_losses / texture_step_losses.

vanilla and lsgan take one smooth label per loss call, drawn from the real range for fake targets too (loss.py:102):
`draws` holds the three torch.rand(1) values in reference order (D_fake, D_real, G_gan).  wgan has no target and the
reference draws nothing for it: `draws` is ignored and may be empty.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

import norm_oracle as NO
from oracle import nets as ON

MODES = ("vanilla", "lsgan", "wgan")


def label_draws(gan_mode: str) -> int:
    """CPU-RNG draws of one training step (one per loss call for vanilla / lsgan)."""
    return 0 if gan_mode == "wgan" else 3


def gan_loss(pred, target_is_real: bool, gan_mode: str, draw=None):
    """GANLoss(gan_mode, smooth_labels=True)(pred, target_is_real); draw = the torch.rand(1) of this call (unused by
    wgan)."""
    if gan_mode == "wgan":
        return -pred.mean() if target_is_real else pred.mean()
    t = ON.smooth_label(draw).to(pred.dtype).expand_as(pred)
    if gan_mode == "lsgan":
        return F.mse_loss(pred, t)
    if gan_mode == "vanilla":
        return F.binary_cross_entropy_with_logits(pred, t)
    raise ValueError(gan_mode)


def _d_losses(sdD, bnD, cond, fakes, targets, draws, gan_mode, lambda_gan):
    d = list(draws) if label_draws(gan_mode) else [None] * 3
    loss_D_fake = gan_loss(NO.patchgan_forward(sdD, torch.cat((cond, fakes), 1).detach(), bnD), False, gan_mode, d[0])
    loss_D_real = gan_loss(NO.patchgan_forward(sdD, torch.cat((cond, targets), 1), bnD), True, gan_mode, d[1])
    loss_gan = gan_loss(NO.patchgan_forward(sdD, torch.cat((cond, fakes), 1), bnD), True, gan_mode, d[2]) * lambda_gan
    return dict(D=0.5 * (loss_D_fake + loss_D_real), D_fake=loss_D_fake, D_real=loss_D_real, G_gan=loss_gan)


def warp_step_losses(sdG, sdD, body, inputs, targets, draws, gan_mode: str, norm: str = "instance", train: bool = True,
                     lambda_ce=100.0, lambda_gan=1.0, drop=None):
    """WarpModel losses (warp_model.py:109-160) without the optimizer steps in between: D is evaluated with the same
    weights in the D and G phases, conditioned on the body (body first)."""
    bnD = NO.BN(sdD, norm, train)
    fakes = ON.warp_forward(sdG, body, inputs, drop)
    o = _d_losses(sdD, bnD, body, fakes, targets, draws, gan_mode, lambda_gan)
    loss_ce = F.cross_entropy(fakes, torch.argmax(targets, dim=1)) * lambda_ce
    o.update(fakes=fakes, G=o["G_gan"] + loss_ce, G_ce=loss_ce, bufsD=bnD.bufs)
    return o


def texture_step_losses(sdG, sdD, tex, rois, cloth, targets, draws, gan_mode: str, norm: str = "instance",
                        train: bool = True, lambda_l1=10.0, lambda_gan=1.0, drop=None, l1_sign=None, vgg=None,
                        lambda_content=0.0, lambda_style=0.0):
    """TextureModel losses (texture_model.py:127-180): D conditioned on the cloth (cloth first); perceptual terms when
    lambda_content or lambda_style != 0; l1_sign as in oracle/nets.py texture_step_losses."""
    bnG, bnD = NO.BN(sdG, norm, train), NO.BN(sdD, norm, train)
    fakes = NO.texture_forward(sdG, tex, rois, cloth, bnG, drop)
    o = _d_losses(sdD, bnD, cloth, fakes, targets, draws, gan_mode, lambda_gan)
    if l1_sign is None:
        loss_l1 = F.l1_loss(fakes, targets) * lambda_l1
    else:
        loss_l1 = ((fakes - targets) * l1_sign).mean() * lambda_l1
    loss_content = loss_style = 0.0
    if lambda_content != 0 or lambda_style != 0:
        c, st = ON.perceptual_loss(vgg, fakes, targets, lambda_style != 0)
        loss_content, loss_style = c * lambda_content, st * lambda_style
    o.update(fakes=fakes, G=o["G_gan"] + loss_l1 + loss_content + loss_style, G_l1=loss_l1, G_content=loss_content,
             G_style=loss_style, bufsG=bnG.bufs, bufsD=bnD.bufs)
    return o
