"""TEST INFRASTRUCTURE ONLY — the 1x1 PixelGAN discriminator (discriminators.py:138-168) in fp64 torch, with the
LeakyReLU gates optionally imposed (DESIGN §5): z1_gate / y2_gate are boolean [N, 64 | 128, H, W] tensors that replace
`pre-activation > 0`, so that a reference fed the device's gates differentiates the same piecewise-linear function.

sd: the discriminator's state dict (keys net.0.weight, net.0.bias, net.2.weight, [net.2.bias], net.5.weight,
[net.5.bias]); norm: 'instance' (InstanceNorm2d(affine=False), eps 1e-5) or 'none'.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

SLOPE = 0.2


def _lrelu(z, gate):
    if gate is None:
        return F.leaky_relu(z, SLOPE)
    return torch.where(gate, z, z * SLOPE)


def pixel_forward(sd, x, norm: str, z1_gate=None, y2_gate=None, eps: float = 1e-5) -> dict:
    """x [N, cin, H, W] -> dict(z1, a1, z2, y2, a2, pred [N, 1, H, W]) in x's dtype."""
    w = {k: v.to(x.dtype) for k, v in sd.items()}
    z1 = F.conv2d(x, w["net.0.weight"], w["net.0.bias"])
    a1 = _lrelu(z1, z1_gate)
    z2 = F.conv2d(a1, w["net.2.weight"], w.get("net.2.bias"))
    y2 = F.instance_norm(z2, eps=eps) if norm == "instance" else z2
    a2 = _lrelu(y2, y2_gate)
    pred = F.conv2d(a2, w["net.5.weight"], w.get("net.5.bias"))
    return dict(z1=z1, a1=a1, z2=z2, y2=y2, a2=a2, pred=pred)


def pixel_grads(sd, x, norm: str, dpred, z1_gate=None, y2_gate=None) -> dict:
    """fp64 gradients of sum(pred * dpred) w.r.t. every parameter (state-dict keys) and x ('x'), plus the
    intermediates of pixel_forward and dz2 / g1 (d/dz2, d/dz1) for per-entry error bounds."""
    p = {k: v.detach().double().clone().requires_grad_(True) for k, v in sd.items()}
    xx = x.detach().double().clone().requires_grad_(True)
    out = pixel_forward(p, xx, norm, z1_gate, y2_gate)
    out["z1"].retain_grad()
    out["z2"].retain_grad()
    (out["pred"] * dpred.double()).sum().backward()
    g = {k: v.grad for k, v in p.items()}
    g["x"] = xx.grad
    g["dz2"], g["g1"] = out["z2"].grad, out["z1"].grad
    g.update({k: v.detach() for k, v in out.items()})
    return g


def step_state(net):
    """state_dict copies: parameters as leaves that require grad, buffers plain."""
    names = [k for k, _ in net.named_parameters()]
    sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
    for k in names:
        sd[k].requires_grad_()
    return sd, [sd[k] for k in names]


def reference_step(kind: str, G, Dn, batch, label_seed: int, g_gates=None) -> dict:
    """One training step of the reference (warp_model.py:109-160 / texture_model.py:127-180, --gan_mode vanilla,
    --norm instance, dropout off) with the PixelGAN of this module and torch.optim.AdamW, on fresh copies of the
    containers' weights.  batch: the plugin's input dict.  g_gates: (z1_gate, y2_gate) imposed on D in the G step.  Returns the losses, the D gradients of the D step, the G
    gradients of the G step, d G_gan / d(D input) of the G step, the updated state dicts and the SHA-256 of the CPU generator after the step."""
    import hashlib

    import gan_modes_oracle as GO
    import norm_oracle as NO
    from oracle import nets as ON

    sdG, pG = step_state(G)
    sdD, pD = step_state(Dn)
    optG = torch.optim.AdamW(pG, lr=1e-4, weight_decay=0, betas=(0.9, 0.999))
    optD = torch.optim.AdamW(pD, lr=4e-4, weight_decay=0.01, betas=(0.9, 0.999))
    if kind == "texture":
        cond, tgt = batch["cloths"], batch["target_textures"]
        fk = NO.texture_forward(sdG, batch["input_textures"], batch["rois"], cond, NO.BN(sdG, "instance", True))
    else:
        cond, tgt = batch["bodys"], batch["target_cloths"]
        fk = ON.warp_forward(sdG, cond, batch["input_cloths"])
    D = lambda x: pixel_forward(sdD, x, "instance")["pred"]  # noqa: E731
    torch.manual_seed(label_seed)
    d_in = (torch.cat((cond, fk), 1).detach(), torch.cat((cond, tgt), 1))
    lf = GO.gan_loss(D(d_in[0]), False, "vanilla", torch.rand(1))
    lr = GO.gan_loss(D(d_in[1]), True, "vanilla", torch.rand(1))
    lD = 0.5 * (lf + lr)
    lD.backward()
    gD = {k: sdD[k].grad.clone() for k, _ in Dn.named_parameters()}
    sdD0 = {k: v.detach().clone() for k, v in sdD.items()}
    optD.step()
    x_g = torch.cat((cond, fk), 1)
    x_g.retain_grad()
    gan = GO.gan_loss(pixel_forward(sdD, x_g, "instance", *(g_gates or (None, None)))["pred"], True, "vanilla",
                      torch.rand(1))
    if kind == "texture":
        rec, rec_name = F.l1_loss(fk, tgt) * 10, "G_l1"
    else:
        rec, rec_name = F.cross_entropy(fk, torch.argmax(tgt, 1)) * 100, "G_ce"
    (gan + rec).backward()
    gG = {k: sdG[k].grad.clone() for k, _ in G.named_parameters()}
    optG.step()
    losses = {"D": lD.item(), "D_real": lr.item(), "D_fake": lf.item(), "G": (gan + rec).item(), "G_gan": gan.item(),
              rec_name: rec.item()}
    return dict(losses=losses, grads_D=gD, grads_G=gG, sdG=sdG, sdD=sdD, sdD_before=sdD0, d_inputs=d_in, dgan_dx=x_g.grad,
                rng_after=hashlib.sha256(torch.get_rng_state().numpy().tobytes()).hexdigest())
