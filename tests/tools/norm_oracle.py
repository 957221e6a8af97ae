"""TEST INFRASTRUCTURE ONLY — the CPU oracle (oracle/nets.py) with the `--norm` choice of the texture U-Net and the
PatchGAN: instance (oracle/nets.py itself), batch or none (modules/__init__.py:53-74 get_norm_layer).

Batch norm is nn.BatchNorm2d(affine=True, track_running_stats=True) restated with F.batch_norm: train mode normalises
with the biased variance of the call and updates the running buffers (momentum 0.1, unbiased variance) and
num_batches_tracked; eval mode uses the running buffers.  The running buffers are taken from the state_dict and the
updated copies are returned in `bufs` (state_dict key -> tensor).  Activations go through oracle/nets.py's _act, so
imposed gates (ON.gate_with) act on gamma * xhat + beta, and recording / dropout hooks work as there.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch
import torch.nn.functional as F

from oracle import nets as ON

EPS, MOMENTUM = 1e-5, 0.1


class BN:
    """Norm state of one network: mode 'instance' | 'batch' | 'none', train (batch statistics) or eval."""

    def __init__(self, sd: Dict[str, torch.Tensor], norm: str, train: bool):
        self.sd, self.norm, self.train = sd, norm, train
        self.bufs = {k: v.detach().clone() for k, v in sd.items()
                     if k.endswith(("running_mean", "running_var", "num_batches_tracked"))}

    def __call__(self, key: str, y: torch.Tensor, groups: int = 1) -> torch.Tensor:
        """key: Sequential prefix of the norm slot (e.g. 'model.3')."""
        if self.norm == "none":
            return y
        if self.norm == "instance":
            return ON._inorm(y)
        w, b = self.sd[key + ".weight"], self.sd[key + ".bias"]
        rm, rv = self.bufs[key + ".running_mean"], self.bufs[key + ".running_var"]
        if not self.train:
            return F.batch_norm(y, rm.to(y.dtype), rv.to(y.dtype), w, b, False, MOMENTUM, EPS)
        outs = []
        for yg in y.chunk(groups, 0):
            # fresh copies per call: autograd saves the running tensors it was given, so a later call must not
            # update those in place
            m, v = rm.to(y.dtype, copy=True), rv.to(y.dtype, copy=True)
            outs.append(F.batch_norm(yg, m, v, w, b, True, MOMENTUM, EPS))
            rm.copy_(m)
            rv.copy_(v)
            self.bufs[key + ".num_batches_tracked"] += 1
        return torch.cat(outs, 0)


def patchgan_forward(sd, x, bn: BN, groups: int = 1):
    """define_D(..., 'basic', 3, norm): convs at model.0/2/5/8/11, norm slots at model.3/6/9."""
    y = ON._rec("model.0.y", F.conv2d(x, sd["model.0.weight"], sd["model.0.bias"], 2, 1))
    y = ON._rec("model.0.a", ON._act("model.0", y, 0.2))
    for idx, stride in ((2, 2), (5, 2), (8, 1)):
        y = ON._rec(f"model.{idx}.y", F.conv2d(y, sd[f"model.{idx}.weight"], sd.get(f"model.{idx}.bias"), stride, 1))
        y = bn(f"model.{idx + 1}", y, groups)
        y = ON._rec(f"model.{idx}.a", ON._act(f"model.{idx}", y, 0.2))
    return ON._rec("model.11.y", F.conv2d(y, sd["model.11.weight"], sd["model.11.bias"], 1, 1))


def unet_generator(sd, p: str, x, num_downs: int, bn: BN, drop=None):
    """oracle/nets.py unet_generator with the norm of `bn`: norm slots of block j at '.2' (down, middle blocks) and
    '.6' (up, middle) / '.4' (up, innermost); convs without bias unless the norm is instance (U_0 keeps its bias)."""
    nd = num_downs
    pre = [p + ".model.model"]
    for j in range(1, nd):
        pre.append(pre[-1] + (".1.model" if j == 1 else ".3.model"))
    dkey = [pre[j] + (".0" if j == 0 else ".1") for j in range(nd)]
    ukey = [pre[j] + (".3" if (j == 0 or j == nd - 1) else ".5") for j in range(nd)]
    nkey_d = [pre[j] + ".2" for j in range(nd)]
    nkey_u = [pre[j] + (".4" if j == nd - 1 else ".6") for j in range(nd)]
    xhat = [None] * nd
    inp = x
    for j in range(nd):
        y = ON._rec(f"unet.D{j}.y", F.conv2d(inp, sd[dkey[j] + ".weight"], sd.get(dkey[j] + ".bias"), 2, 1))
        if 1 <= j <= nd - 2:
            y = bn(nkey_d[j], y)
        xhat[j] = y
        if j < nd - 1:
            inp = ON._act(f"unet.D{j}", y, 0.2)
    v = None
    for j in range(nd - 1, -1, -1):
        if j == nd - 1:
            src = ON._act(f"unet.D{j}", xhat[j], 0.0)
        else:
            src = torch.cat([ON._act(f"unet.D{j}", xhat[j], 0.0), v], 1)
        y = ON._rec(f"unet.U{j}.y", F.conv_transpose2d(src, sd[ukey[j] + ".weight"], sd.get(ukey[j] + ".bias"), 2, 1))
        if j == 0:
            return ON._rec("unet.out", torch.tanh(y))
        y = bn(nkey_u[j], y)
        v = ON._act(f"unet.U{j}", y, 0.0)
        if 4 <= j <= nd - 2:
            v = ON._dr(drop, f"unet.U{j}", v)


def texture_forward(sd, tex, rois, cloth, bn: BN, drop=None):
    from torchvision.ops import roi_align

    B, _, S, _ = tex.shape
    nroi = rois.shape[1]
    bidx = torch.arange(B).repeat_interleave(nroi).to(rois.dtype).unsqueeze(1)
    r5 = torch.cat((bidx, rois.reshape(-1, 4)), 1)
    pooled = roi_align(tex, r5, (128, 128), 1.0, 1).view(B, -1, 128, 128)
    enc = ON._act("encode", ON._inorm(ON._rec("encode.y", F.conv2d(pooled, sd["encode.model.0.weight"], None, 2, 1))),
                  0.2)          # layers.py:12-24: encode always uses InstanceNorm
    up = F.interpolate(enc, scale_factor=S / enc.shape[2])
    x = torch.cat((up, cloth), 1)
    return unet_generator(sd, "unet", x, math.frexp(S)[1] - 1, bn, drop)


def texture_step_losses(sdG, sdD, tex, rois, cloth, targets, draws, norm: str, train: bool, lambda_l1=10.0,
                        lambda_gan=1.0, drop=None, l1_sign: Optional[torch.Tensor] = None, vgg=None,
                        lambda_content=0.0, lambda_style=0.0):
    """oracle/nets.py texture_step_losses with the norm choice.  D is called as the reference calls it: fake, real
    (D step), then fake again (G step); each call has its own batch statistics and running-buffer update.
    Returns the losses plus bufsG / bufsD, the running buffers after the three D calls and the G forward."""
    bnG, bnD = BN(sdG, norm, train), BN(sdD, norm, train)
    fakes = texture_forward(sdG, tex, rois, cloth, bnG, drop)
    t = [ON.smooth_label(d) for d in draws]
    loss_D_fake = ON.gan_loss(patchgan_forward(sdD, torch.cat((cloth, fakes), 1).detach(), bnD), t[0])
    loss_D_real = ON.gan_loss(patchgan_forward(sdD, torch.cat((cloth, targets), 1), bnD), t[1])
    loss_D = 0.5 * (loss_D_fake + loss_D_real)
    loss_gan = ON.gan_loss(patchgan_forward(sdD, torch.cat((cloth, fakes), 1), bnD), t[2]) * lambda_gan
    if l1_sign is None:
        loss_l1 = F.l1_loss(fakes, targets) * lambda_l1
    else:
        loss_l1 = ((fakes - targets) * l1_sign).mean() * lambda_l1
    loss_content = loss_style = 0.0
    if lambda_content != 0 or lambda_style != 0:
        c, st = ON.perceptual_loss(vgg, fakes, targets, lambda_style != 0)
        loss_content, loss_style = c * lambda_content, st * lambda_style
    return dict(fakes=fakes, D=loss_D, D_fake=loss_D_fake, D_real=loss_D_real,
                G=loss_gan + loss_l1 + loss_content + loss_style, G_gan=loss_gan, G_l1=loss_l1,
                G_content=loss_content, G_style=loss_style, bufsG=bnG.bufs, bufsD=bnD.bufs)


def warp_step_losses(sdG, sdD, body, inputs, targets, draws, norm: str, train: bool, lambda_ce=100.0, lambda_gan=1.0,
                     drop=None):
    """oracle/nets.py warp_step_losses with the discriminator's norm choice (the warp generator is always IN)."""
    bnD = BN(sdD, norm, train)
    fakes = ON.warp_forward(sdG, body, inputs, drop)
    t = [ON.smooth_label(d) for d in draws]
    pred_fake = patchgan_forward(sdD, torch.cat((body, fakes), 1).detach(), bnD)
    loss_D_fake = ON.gan_loss(pred_fake, t[0])
    loss_D_real = ON.gan_loss(patchgan_forward(sdD, torch.cat((body, targets), 1), bnD), t[1])
    loss_D = 0.5 * (loss_D_fake + loss_D_real)
    loss_ce = F.cross_entropy(fakes, torch.argmax(targets, dim=1)) * lambda_ce
    loss_gan = ON.gan_loss(patchgan_forward(sdD, torch.cat((body, fakes), 1), bnD), t[2]) * lambda_gan
    return dict(fakes=fakes, D=loss_D, D_fake=loss_D_fake, D_real=loss_D_real, G=loss_gan + loss_ce, G_gan=loss_gan,
                G_ce=loss_ce, bufsD=bnD.bufs)
