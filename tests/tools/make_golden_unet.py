"""Generate tests/golden/pix2pix_128.pt and tests/golden/texture_unet_128.pt from the UNMODIFIED reference (needs the
reference tree, see oracle/ref_harness.py).  On the CPU, 128 x 128, batch 2, --init_type kaiming, under a fixed seed:
  * pix2pix_128:       the reference's Pix2PixModel (--norm batch: G = define_G 'unet_128' + init_weights, D = define_D
                       at PyTorch's default init);
  * texture_unet_128:  the reference's TextureModel with --netG unet_128 (--norm instance for D; the generator's batch
                       norm is fixed), no perceptual terms;
each file holds
  * `init_G` / `init_D`: state_dict keys, shapes and checksums (fp64 sum, sum of |x|, sum of squares) of the seeded
    networks (the parameters themselves, ~45 M per model, are not stored);
  * one step's D phase (backward_D) and G phase (backward_G) with the same D weights (no optimizer step between), the
    networks in train mode with their nn.Dropout modules in eval mode (torch's dropout RNG cannot be restated): the
    losses, and per parameter the gradient's checksums and its first HEAD flat elements;
  * the label draws: the torch.rand(1) values GANLoss drew (CPU default generator seeded with `label_seed` before the
    step) and the smooth labels it made of them, in call order.
The batch is tests/test_engine_gpu.py synth_texture_batch(2, 128) (fp32 one-hot cloth).

    python tests/tools/make_golden_unet.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import ref_harness as RH  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
SEED, LABEL_SEED, B, S, HEAD = 5, 321, 2, 128, 256


def checksums(sd):
    return [(k, tuple(v.shape), v.double().sum().item(), v.double().abs().sum().item(), v.double().square().sum().item())
            for k, v in sd.items()]


def grads(net):
    return {k: dict(sum=p.grad.double().sum().item(), abs=p.grad.double().abs().sum().item(),
                    head=p.grad.detach().reshape(-1)[:HEAD].clone())
            for k, p in net.named_parameters() if p.grad is not None}


def run(kind):
    ref_models, _ = RH.import_reference()
    import modules.loss as RL
    import modules.losses.perceptual as P
    import torchvision
    from test_engine_gpu import synth_texture_batch

    if kind == "pix2pix":
        opt = RH.texture_opt(B, S, model="pix2pix", name="pix2pix", norm="batch", netG="unet_128", beta1=0.5, lr=0.01)
    else:
        opt = RH.texture_opt(B, S, netG="unet_128", norm="instance")
    orig = P.vgg16     # TextureModel builds PerceptualLoss unconditionally: no download, the weights are unused here
    P.vgg16 = lambda pretrained=False, **kw: torchvision.models.vgg16(weights=None)
    torch.manual_seed(SEED)
    try:
        model = ref_models.create_model(opt)
    finally:
        P.vgg16 = orig
    G, D = (model.net_G, model.net_D) if kind == "pix2pix" else (model.net_generator, model.net_discriminator)
    rec = {"seed": SEED, "label_seed": LABEL_SEED, "batch": B, "size": S, "init_type": "kaiming",
           "init_G": checksums(G.state_dict()), "init_D": checksums(D.state_dict())}
    for net in (G, D):
        net.train()
        for m in net.modules():
            if isinstance(m, torch.nn.Dropout):
                m.eval()
    tex, rois, cloth, tgt = synth_texture_batch(B, S)
    if kind == "pix2pix":
        batch = dict(cloths=cloth, target_textures=tgt)
    else:
        batch = dict(input_textures=tex, rois=rois, cloths=cloth, target_textures=tgt, cloth_paths=["c"] * B,
                     texture_paths=["t"] * B)
    draws, labels = [], []
    orig_rb = RL.GANLoss.rand_between

    def rand_between(low, high, normal=False):     # the draw GANLoss makes, and the label it makes of it
        state = torch.get_rng_state()
        draws.append(torch.rand(1))
        torch.set_rng_state(state)
        out = orig_rb(low, high, normal)
        labels.append(out.detach().clone())
        return out

    RL.GANLoss.rand_between = staticmethod(rand_between)
    try:
        model.set_input(batch)
        torch.manual_seed(LABEL_SEED)
        model.forward()
        D.zero_grad()
        model.backward_D()
        rec["grads_D"] = grads(D)
        G.zero_grad()
        model.backward_G()
        rec["grads_G"] = grads(G)
    finally:
        RL.GANLoss.rand_between = orig_rb
    names = ("G", "G_GAN", "G_L1", "D_real", "D_fake") if kind == "pix2pix" else \
        ("D", "D_real", "D_fake", "G", "G_gan", "G_l1")
    rec["losses"] = {n: float(getattr(model, "loss_" + n)) for n in names}
    rec["draws"], rec["labels"] = torch.cat(draws), torch.cat([x.reshape(1) for x in labels])
    return rec


def main():
    for kind, name in (("pix2pix", "pix2pix_128.pt"), ("texture", "texture_unet_128.pt")):
        path = os.path.join(GOLDEN, name)
        torch.save(run(kind), path)
        print("wrote", path)


if __name__ == "__main__":
    main()
