"""Generate tests/golden/batchnorm_64.pt from the UNMODIFIED reference (needs the reference tree, see
oracle/ref_harness.py): for `--norm batch` and `--norm none`,
  * state_dict keys and shapes of TextureModule(norm_type=..., img_size=64) and define_D(22, 64, 'basic', norm=...);
  * per-tensor checksums (fp64 sum, sum of |x|) of a seeded init_weights(.., 'normal', 0.02);
  * batch norm only: the PatchGAN output and running buffers after a train-mode call on each half of a seeded batch
    of 4, its eval-mode output, and the texture module's train-mode output (nn.Dropout in eval mode: torch's dropout
    RNG cannot be restated) with the running buffers after it, then its eval-mode output;
  * batch norm only: ONE full reference TextureModel.optimize_parameters() (L1 + GAN) and ONE
    WarpModel.optimize_parameters() with --norm batch, 64 x 64, batch 2, CPU (gpu_id=None), the networks in train mode
    but their nn.Dropout modules in eval mode: the six losses and checksums of every state_dict entry (parameters after
    the D and G AdamW updates, running buffers after the G forward and the three D calls, num_batches_tracked) before
    and after the step.

    python tests/tools/make_golden_batchnorm.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_harness as RH  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "batchnorm_64.pt")
TEX_SEED, D_SEED = 3, 4
STEP_B, STEP_S, STEP_SEED, LABEL_SEED = 2, 64, 0, 123


def checksums(sd):
    return {k: (v.double().sum().item(), v.double().abs().sum().item()) for k, v in sd.items()}


def inputs():
    g = torch.Generator().manual_seed(77)
    x = torch.randn(4, 22, 64, 64, generator=g)
    tex = torch.rand(2, 3, 64, 64, generator=g)
    rois = torch.rand(2, 12, 4, generator=g) * 20
    rois[..., 2:] += 30
    cloth = torch.rand(2, 19, 64, 64, generator=g)
    return x, tex, rois, cloth


def reference_step(kind):
    """One reference optimize_parameters() with --norm batch (see the module doc)."""
    import models as ref_models

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_engine_gpu import synth_texture_batch, synth_warp_batch

    B, S = STEP_B, STEP_S
    torch.manual_seed(STEP_SEED)
    opt = (RH.texture_opt(B, S, norm="batch") if kind == "texture" else RH.warp_opt(B, norm="batch", crop_size=S,
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
    model.set_input(batch)
    model.optimize_parameters()
    rec["losses"] = {k: float(v) for k, v in model.get_current_losses().items()}
    rec["step_G"] = checksums(model.net_generator.state_dict())
    rec["step_D"] = checksums(model.net_discriminator.state_dict())
    return rec


def main():
    RH.import_reference()
    from modules import discriminators as D
    from modules import init_weights
    from modules import swapnet_modules as SM

    x, tex, rois, cloth = inputs()
    out = {}
    for norm in ("batch", "none"):
        torch.manual_seed(TEX_SEED)
        T = SM.TextureModule(3, 19, 12, norm_type=norm, img_size=64)
        init_weights(T, "normal", 0.02)
        torch.manual_seed(D_SEED)
        Dn = D.define_D(22, 64, "basic", 3, norm=norm)
        init_weights(Dn, "normal", 0.02)
        rec = {"tex_keys": [(k, tuple(v.shape)) for k, v in T.state_dict().items()],
               "d_keys": [(k, tuple(v.shape)) for k, v in Dn.state_dict().items()],
               "tex_init": checksums(T.state_dict()), "d_init": checksums(Dn.state_dict())}
        if norm == "batch":
            with torch.no_grad():
                Dn.train()
                rec["d_train"] = torch.cat([Dn(x[:2]), Dn(x[2:])])
                rec["d_train_bufs"] = {k: v.clone() for k, v in Dn.state_dict().items()
                                       if "running" in k or "num_batches" in k}
                Dn.eval()
                rec["d_eval"] = Dn(x)
                T.train()
                for m in T.modules():
                    if isinstance(m, torch.nn.Dropout):
                        m.eval()
                rec["tex_train"] = T(tex, rois, cloth)
                rec["tex_train_bufs"] = {k: v.clone() for k, v in T.state_dict().items()
                                         if "running" in k or "num_batches" in k}
                T.eval()
                rec["tex_eval"] = T(tex, rois, cloth)
        out[norm] = rec
    out["texture_step"] = reference_step("texture")
    out["warp_step"] = reference_step("warp")
    torch.save(out, OUT)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
