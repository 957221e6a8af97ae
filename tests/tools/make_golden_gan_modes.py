"""Generate tests/golden/gan_modes_64.pt from the UNMODIFIED reference (needs the reference tree, see
oracle/ref_harness.py).  For each `--gan_mode` in vanilla, lsgan and wgan:
  * GANLoss(gan_mode)(pred, target_is_real) on fixed fp32 predictions of PatchGAN shape, fake and real: the loss and its
    gradient with respect to pred, each call after torch.manual_seed(LOSS_SEED);
  * ONE full reference WarpModel and ONE TextureModel optimize_parameters() at 64 x 64, batch 2, CPU (gpu_id=None),
    --norm instance, the networks in train mode with their nn.Dropout modules in eval mode: the losses, checksums of
    every state_dict entry before and after the step (parameters after the D and G AdamW updates), and the SHA-256 of
    the CPU default generator's state right after torch.manual_seed(LABEL_SEED) and after the step — the smooth-label
    draws are the step's only use of that generator.

    python tests/tools/make_golden_gan_modes.py
"""
import hashlib
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_harness as RH  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "gan_modes_64.pt")
MODES = ("vanilla", "lsgan", "wgan")
PRED_SHAPE, PRED_SEED, LOSS_SEED = (2, 1, 7, 7), 5, 11
STEP_B, STEP_S, STEP_SEED, LABEL_SEED = 2, 64, 0, 123


def checksums(sd):
    return {k: (v.double().sum().item(), v.double().abs().sum().item()) for k, v in sd.items()}


def rng_digest() -> str:
    return hashlib.sha256(torch.get_rng_state().numpy().tobytes()).hexdigest()


def preds():
    return torch.randn(PRED_SHAPE, generator=torch.Generator().manual_seed(PRED_SEED)) * 3.0


def reference_losses(mode):
    """(loss, dloss/dpred) of GANLoss(mode) for target_is_real False and True."""
    from modules.loss import GANLoss

    crit = GANLoss(mode, smooth_labels=True)
    out = {}
    for real in (False, True):
        x = preds().requires_grad_()
        torch.manual_seed(LOSS_SEED)
        loss = crit(x, real)
        loss.backward()
        out[real] = (loss.detach().clone(), x.grad.clone())
    return out


def reference_step(kind, mode):
    """One reference optimize_parameters() with --gan_mode `mode` (see the module doc)."""
    import models as ref_models

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_engine_gpu import synth_texture_batch, synth_warp_batch

    B, S = STEP_B, STEP_S
    torch.manual_seed(STEP_SEED)
    opt = (RH.texture_opt(B, S, gan_mode=mode) if kind == "texture" else RH.warp_opt(B, gan_mode=mode, crop_size=S,
                                                                                      load_size=S))
    import modules.losses.perceptual as P
    import torchvision

    orig = P.vgg16     # TextureModel builds PerceptualLoss unconditionally: no download, the weights are unused here
    P.vgg16 = lambda pretrained=False, **kw: torchvision.models.vgg16(weights=None)
    try:
        model = ref_models.create_model(opt)
    finally:
        P.vgg16 = orig
    model.setup(opt)
    for net in (model.net_generator, model.net_discriminator):
        net.train()
        for m in net.modules():
            if isinstance(m, torch.nn.Dropout):
                m.eval()
    rec = {"init_G": checksums(model.net_generator.state_dict()),
           "init_D": checksums(model.net_discriminator.state_dict())}
    if kind == "texture":
        tex, rois, cloth, tgt = synth_texture_batch(B, S)
        batch = dict(input_textures=tex, rois=rois, cloths=cloth, target_textures=tgt, cloth_paths=["c"] * B,
                     texture_paths=["t"] * B)
    else:
        body, inp, tgt = synth_warp_batch(B, S)
        batch = dict(bodys=body, input_cloths=inp, target_cloths=tgt, cloth_paths=["c"] * B, body_paths=["b"] * B)
    torch.manual_seed(LABEL_SEED)   # GANLoss draws its smooth labels from the CPU default generator
    rec["rng_before"] = rng_digest()
    model.set_input(batch)
    model.optimize_parameters()
    rec["rng_after"] = rng_digest()
    rec["losses"] = {k: float(v) for k, v in model.get_current_losses().items()}
    rec["step_G"] = checksums(model.net_generator.state_dict())
    rec["step_D"] = checksums(model.net_discriminator.state_dict())
    return rec


def main():
    RH.import_reference()
    out = {"preds": preds()}
    for mode in MODES:
        out[mode] = {"loss": reference_losses(mode), "warp_step": reference_step("warp", mode),
                     "texture_step": reference_step("texture", mode)}
    torch.save(out, OUT)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
