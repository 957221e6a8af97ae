"""`--gan_mode` vanilla / lsgan / wgan on the CPU: the objective-aware oracle (tests/tools/gan_modes_oracle.py) against
the reference's GANLoss and against full reference optimize_parameters() steps — live where the reference tree is
importable, else against tests/golden/gan_modes_64.pt (generated from it by tests/tools/make_golden_gan_modes.py)."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "tools"))

import gan_modes_oracle as GO  # noqa: E402
import make_golden_gan_modes as MG  # noqa: E402
import norm_oracle as NO  # noqa: E402
from oracle import nets as ON  # noqa: E402
from oracle import ref_harness as RH  # noqa: E402
from swapnet_b200 import modules as M  # noqa: E402

GOLD = torch.load(os.path.join(HERE, "golden", "gan_modes_64.pt"))


def oracle_losses(mode):
    out = {}
    for real in (False, True):
        x = MG.preds().requires_grad_()
        torch.manual_seed(MG.LOSS_SEED)
        loss = GO.gan_loss(x, real, mode, torch.rand(1) if GO.label_draws(mode) else None)
        loss.backward()
        out[real] = (loss.detach(), x.grad)
    return out


@pytest.mark.parametrize("mode", GO.MODES)
def test_oracle_gan_loss_is_bit_identical_to_reference(mode):
    """Loss and gradient of GANLoss(mode) for fake and real targets, bit for bit (the golden file, and the reference
    itself when it is importable)."""
    assert torch.equal(MG.preds(), GOLD["preds"])
    got = oracle_losses(mode)
    wants = [GOLD[mode]["loss"]]
    if RH.available():
        RH.import_reference()
        wants.append(MG.reference_losses(mode))
    for want in wants:
        for real in (False, True):
            assert torch.equal(got[real][0], want[real][0]), (mode, real, got[real][0], want[real][0])
            assert torch.equal(got[real][1], want[real][1]), (mode, real)


def test_oracle_vanilla_losses_equal_oracle_nets():
    """gan_mode='vanilla' with norm 'instance' computes exactly what oracle/nets.py computes."""
    from test_engine_gpu import synth_warp_batch

    torch.manual_seed(0)
    G, Dn = M.WarpModule(), M.NLayerDiscriminator(22, 64, 3, "instance")
    M.init_weights(G, "kaiming")
    M.init_weights(Dn, "kaiming")
    body, inp, tgt = synth_warp_batch(1, 64)
    draws = [torch.rand(1) for _ in range(3)]
    sdG, sdD = G.state_dict(), Dn.state_dict()
    with torch.no_grad():
        a = ON.warp_step_losses(sdG, sdD, body, inp, tgt, draws)
        b = GO.warp_step_losses(sdG, sdD, body, inp, tgt, draws, "vanilla")
    for k in ("fakes", "D", "D_fake", "D_real", "G", "G_gan", "G_ce"):
        assert torch.equal(a[k], b[k]), k


def test_wgan_losses_have_the_reference_signs():
    x = torch.randn(3, 1, 5, 5, dtype=torch.float64)
    assert GO.gan_loss(x, True, "wgan") == -x.mean()
    assert GO.gan_loss(x, False, "wgan") == x.mean()
    t = ON.smooth_label(torch.tensor([0.25]))
    assert GO.gan_loss(x, True, "lsgan", torch.tensor([0.25])) == F.mse_loss(x, t.double().expand_as(x))
    with pytest.raises(ValueError):
        GO.gan_loss(x, True, "wgan-gp", torch.tensor([0.25]))


def _step_state(net):
    """state_dict copies: parameters as leaves that require grad, buffers plain."""
    names = [k for k, _ in net.named_parameters()]
    sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
    for k in names:
        sd[k].requires_grad_()
    return sd, [sd[k] for k in names]


@pytest.mark.parametrize("mode", GO.MODES)
@pytest.mark.parametrize("kind", ["warp", "texture"])
def test_full_step_matches_reference_golden(kind, mode):
    """One full reference optimize_parameters() per objective and stage: the oracle plus torch.optim.AdamW reproduce
    the losses and every updated parameter of G and D, and leave the CPU generator where the reference left it — three
    smooth-label draws for vanilla / lsgan, none at all for wgan.  For the texture stage with wgan, the reference's
    parameter "clamp" (texture_model.py:132-135, not in place) runs before the D step: the updated D matching an AdamW
    step from the unclamped weights shows that it changes nothing."""
    from test_engine_gpu import synth_texture_batch, synth_warp_batch
    from test_oracle_cpu import checksums, close_checksums

    g = GOLD[mode][f"{kind}_step"]
    B, S = MG.STEP_B, MG.STEP_S
    torch.manual_seed(MG.STEP_SEED)
    G = M.TextureModule(3, 19, 12, "instance", 0.5, S) if kind == "texture" else M.WarpModule()
    M.init_weights(G, "kaiming")
    Dn = M.NLayerDiscriminator(22, 64, 3, "instance")
    M.init_weights(Dn, "kaiming")
    # the seeded init is bit-identical; the fp64 checksums themselves may differ in the last bits between hosts
    close_checksums(checksums(G.state_dict()), g["init_G"], 1e-12)
    close_checksums(checksums(Dn.state_dict()), g["init_D"], 1e-12)
    if kind == "texture" and mode == "wgan":
        # the clamp would move most weights: kaiming init puts them far outside [-0.01, 0.01]
        assert max(p.abs().max().item() for p in Dn.parameters()) > 0.1
    sdG, pG = _step_state(G)
    sdD, pD = _step_state(Dn)
    bnG, bnD = NO.BN(sdG, "instance", True), NO.BN(sdD, "instance", True)
    optG = torch.optim.AdamW(pG, lr=1e-4, weight_decay=0, betas=(0.9, 0.999))
    optD = torch.optim.AdamW(pD, lr=4e-4, weight_decay=0.01, betas=(0.9, 0.999))
    if kind == "texture":
        tex, rois, cloth, tgt = synth_texture_batch(B, S)
        cond = cloth
    else:
        cond, inp, tgt = synth_warp_batch(B, S)
    torch.manual_seed(MG.LABEL_SEED)
    assert MG.rng_digest() == g["rng_before"]

    def draw():
        return torch.rand(1) if GO.label_draws(mode) else None

    fk = NO.texture_forward(sdG, tex, rois, cloth, bnG) if kind == "texture" else ON.warp_forward(sdG, cond, inp)
    lf = GO.gan_loss(NO.patchgan_forward(sdD, torch.cat((cond, fk), 1).detach(), bnD), False, mode, draw())
    lr = GO.gan_loss(NO.patchgan_forward(sdD, torch.cat((cond, tgt), 1), bnD), True, mode, draw())
    lD = 0.5 * (lf + lr)
    lD.backward()
    grads = {id(sdD): {k: sdD[k].grad.clone() for k, _ in Dn.named_parameters()}}
    optD.step()
    gan = GO.gan_loss(NO.patchgan_forward(sdD, torch.cat((cond, fk), 1), bnD), True, mode, draw())
    if kind == "texture":
        rec = F.l1_loss(fk, tgt) * 10
        got = dict(G_l1=rec.item())
    else:
        rec = F.cross_entropy(fk, torch.argmax(tgt, 1)) * 100
        got = dict(G_ce=rec.item())
    (gan + rec).backward()
    grads[id(sdG)] = {k: sdG[k].grad for k, _ in G.named_parameters()}
    optG.step()
    assert MG.rng_digest() == g["rng_after"]
    if mode == "wgan":
        assert g["rng_after"] == g["rng_before"], "a wgan step draws nothing"
    else:
        assert g["rng_after"] != g["rng_before"]
    got.update(D=lD.item(), D_real=lr.item(), D_fake=lf.item(), G=(gan + rec).item(), G_gan=gan.item())
    assert got.keys() == g["losses"].keys()
    # a wgan loss is a difference of means and may cancel: its bar scales with the larger of the two means
    scale = max(abs(lf.item()), abs(lr.item())) if mode == "wgan" else 0.0
    for k, v in g["losses"].items():
        assert abs(got[k] - v) <= 1e-5 * max(abs(v), scale), (k, got[k], v)
    for sd, want, lr_ in ((sdG, g["step_G"], 1e-4), (sdD, g["step_D"], 4e-4)):
        gr = grads[id(sd)]
        gmax = max(v.abs().max().item() for v in gr.values() if v is not None)
        # a bias in front of an InstanceNorm has an exact gradient of zero: AdamW's first step moves each element by
        # +-lr in the direction of the host's rounding noise, so only that bound is checked for it
        zero = {k for k, v in gr.items() if v is None or v.abs().max().item() < 1e-6 * gmax}
        assert all(k.endswith(".bias") for k in zero), zero
        state = {k: v.detach() for k, v in sd.items()}
        numel = {k: v.numel() for k, v in state.items()}
        got = checksums(state)
        close_checksums({k: got[k] for k in got if k not in zero}, {k: want[k] for k in want if k not in zero}, 5e-6,
                        numel=numel, lr=lr_)
        for k in zero:
            assert all(abs(x - y) <= 2 * lr_ * numel[k] * 1.01 for x, y in zip(got[k], want[k])), k
