"""`--discriminator pixel` without a GPU: the parameter container against the reference's PixelDiscriminator (keys,
shapes, bias rule, seeded init; live where the reference tree is present, else tests/golden/pixel_disc_64.pt), the fp64
oracle of tests/tools/pixel_oracle.py against the reference module, one full reference training step per stage
replayed by that oracle, and the engine's `--norm batch` refusal."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "tools"))

import make_golden_gan_modes as MGM  # noqa: E402
import make_golden_pixel as MG  # noqa: E402
import pixel_oracle as PO  # noqa: E402
from oracle import ref_harness as RH  # noqa: E402
from swapnet_b200 import modules as M  # noqa: E402

GOLDEN = torch.load(os.path.join(HERE, "golden", "pixel_disc_64.pt"))
NORMS = ("instance", "none")


def _ours(norm):
    torch.manual_seed(MG.SEED)
    net = M.PixelDiscriminator(MG.CIN, 64, norm)
    M.init_weights(net, "kaiming", 0.02)
    return net


def _reference(norm):
    """(state dict, fp32 output on x_input()) of the reference's define_D(..., 'pixel'): live, else the fixture."""
    if RH.available():
        RH.import_reference()
        net = MG.reference_net(norm)
        with torch.no_grad():
            return net.state_dict(), net(MG.x_input())
    return GOLDEN[norm]["state_dict"], GOLDEN[norm]["pred"]


@pytest.mark.parametrize("norm", NORMS)
def test_container_matches_reference_keys_shapes_and_seeded_init(norm):
    sd_ref, _ = _reference(norm)
    sd = _ours(norm).state_dict()
    assert list(sd) == list(sd_ref)
    for k, v in sd.items():
        assert v.shape == sd_ref[k].shape and torch.equal(v, sd_ref[k]), k
    # the reference's bias rule: net.2 and net.5 carry a bias only with InstanceNorm2d
    assert ("net.2.bias" in sd) == ("net.5.bias" in sd) == (norm == "instance")


@pytest.mark.parametrize("norm", NORMS)
def test_oracle_is_the_reference_module_at_fp32(norm):
    sd, pred = _reference(norm)
    out = PO.pixel_forward(sd, MG.x_input(), norm)["pred"]
    if RH.available():
        assert torch.equal(out, pred)
    else:
        torch.testing.assert_close(out, pred, rtol=1e-6, atol=1e-7)


@pytest.mark.parametrize("norm", NORMS)
def test_oracle_with_its_own_gates_imposed_is_unchanged(norm):
    sd, _ = _reference(norm)
    x = MG.x_input().double()
    free = PO.pixel_forward(sd, x, norm)
    gated = PO.pixel_forward(sd, x, norm, free["z1"] > 0, free["y2"] > 0)
    assert torch.equal(free["pred"], gated["pred"])


def test_pixel_engine_refuses_batch_norm_with_its_reason():
    from swapnet_b200 import engine as E

    with pytest.raises(NotImplementedError, match="batch statistics couple the samples"):
        E.PixelGANEngine(M.PixelDiscriminator(MG.CIN, 64, "batch"), 2, 64, "cpu")


def _step_batch(kind):
    sys.path.insert(0, HERE)
    from test_engine_gpu import synth_texture_batch, synth_warp_batch

    B, S = MGM.STEP_B, MGM.STEP_S
    if kind == "texture":
        tex, rois, cloth, tgt = synth_texture_batch(B, S)
        return dict(input_textures=tex, rois=rois, cloths=cloth, target_textures=tgt)
    body, inp, tgt = synth_warp_batch(B, S)
    return dict(bodys=body, input_cloths=inp, target_cloths=tgt)


def step_nets(kind):
    """The seeded G and PixelGAN of the reference step (G first, then D, as BaseGAN builds them)."""
    torch.manual_seed(MGM.STEP_SEED)
    G = M.TextureModule(3, 19, 12, "instance", 0.5, MGM.STEP_S) if kind == "texture" else M.WarpModule()
    M.init_weights(G, "kaiming")
    Dn = M.PixelDiscriminator(22, 64, "instance")
    M.init_weights(Dn, "kaiming")
    return G, Dn


@pytest.mark.parametrize("kind", ["warp", "texture"])
def test_step_replay_matches_reference_golden(kind):
    """One full reference optimize_parameters() with --discriminator pixel per stage: the oracle plus
    torch.optim.AdamW reproduce its losses and every updated parameter of G and D, and leave the CPU generator where
    the reference left it (three smooth-label draws)."""
    from test_oracle_cpu import checksums, close_checksums

    g = GOLDEN[f"{kind}_step"]
    G, Dn = step_nets(kind)
    close_checksums(checksums(G.state_dict()), g["init_G"], 1e-12)
    close_checksums(checksums(Dn.state_dict()), g["init_D"], 1e-12)
    torch.manual_seed(MGM.LABEL_SEED)
    assert MGM.rng_digest() == g["rng_before"]
    o = PO.reference_step(kind, G, Dn, _step_batch(kind), MGM.LABEL_SEED)
    assert o["rng_after"] == g["rng_after"] and g["rng_after"] != g["rng_before"]
    assert o["losses"].keys() == g["losses"].keys()
    for k, v in g["losses"].items():
        assert abs(o["losses"][k] - v) <= 1e-5 * abs(v), (k, o["losses"][k], v)
    for sd, grads, want, lr in ((o["sdG"], o["grads_G"], g["step_G"], 1e-4), (o["sdD"], o["grads_D"], g["step_D"], 4e-4)):
        gmax = max(v.abs().max().item() for v in grads.values())
        # a bias in front of an InstanceNorm has an exact gradient of zero: AdamW's first step moves each element by
        # +-lr in the direction of the host's rounding noise, so only that bound is checked for it
        zero = {k for k, v in grads.items() if v.abs().max().item() < 1e-6 * gmax}
        assert all(k.endswith(".bias") for k in zero), zero
        state = {k: v.detach() for k, v in sd.items()}
        numel = {k: v.numel() for k, v in state.items()}
        got = checksums(state)
        close_checksums({k: got[k] for k in got if k not in zero}, {k: want[k] for k in want if k not in zero}, 5e-6,
                        numel=numel, lr=lr)
        for k in zero:
            assert all(abs(x - y) <= 2 * lr * numel[k] * 1.01 for x, y in zip(got[k], want[k])), k
