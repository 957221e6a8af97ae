"""`--norm batch` / `--norm none` on the CPU: the parameter containers (state_dict keys, shapes, seeded init) and the
norm-aware oracle (tests/tools/norm_oracle.py) against the reference — live where the reference tree is importable,
else against tests/golden/batchnorm_64.pt (generated from it by tests/tools/make_golden_batchnorm.py)."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "tools"))

import make_golden_batchnorm as MG  # noqa: E402
import norm_oracle as NO  # noqa: E402
from oracle import ref_harness as RH  # noqa: E402
from swapnet_b200 import modules as M  # noqa: E402

GOLD = torch.load(os.path.join(HERE, "golden", "batchnorm_64.pt"))


def ours(norm):
    torch.manual_seed(MG.TEX_SEED)
    T = M.TextureModule(3, 19, 12, norm_type=norm, img_size=64)
    M.init_weights(T, "normal", 0.02)
    torch.manual_seed(MG.D_SEED)
    Dn = M.NLayerDiscriminator(22, 64, 3, norm)
    M.init_weights(Dn, "normal", 0.02)
    return T, Dn


def reference(norm):
    RH.import_reference()
    from modules import discriminators as D
    from modules import init_weights
    from modules import swapnet_modules as SM

    torch.manual_seed(MG.TEX_SEED)
    T = SM.TextureModule(3, 19, 12, norm_type=norm, img_size=64)
    init_weights(T, "normal", 0.02)
    torch.manual_seed(MG.D_SEED)
    Dn = D.define_D(22, 64, "basic", 3, norm=norm)
    init_weights(Dn, "normal", 0.02)
    return T, Dn


@pytest.mark.parametrize("norm", ["batch", "none"])
def test_containers_match_reference_keys_and_seeded_init(norm):
    T, Dn = ours(norm)
    g = GOLD[norm]
    assert [(k, tuple(v.shape)) for k, v in T.state_dict().items()] == g["tex_keys"]
    assert [(k, tuple(v.shape)) for k, v in Dn.state_dict().items()] == g["d_keys"]
    assert MG.checksums(T.state_dict()) == g["tex_init"]
    assert MG.checksums(Dn.state_dict()) == g["d_init"]
    if norm == "batch":
        assert any(k.endswith("num_batches_tracked") for k, _ in g["d_keys"])
    else:
        assert not any("running" in k for k, _ in g["tex_keys"] + g["d_keys"])
    if RH.available():
        rT, rD = reference(norm)
        for a, b in ((T, rT), (Dn, rD)):
            sa, sb = a.state_dict(), b.state_dict()
            assert list(sa) == list(sb)
            assert all(torch.equal(sa[k], sb[k]) for k in sa)
            a.load_state_dict(sb, strict=True)      # checkpoints load both ways
            b.load_state_dict(sa, strict=True)


def test_use_bias_rule():
    """use_bias = (norm is InstanceNorm2d): with batch / none only U_0 and the PatchGAN's model.0 / logits keep a bias."""
    for norm in ("batch", "none"):
        T, Dn = ours(norm)
        blocks = T.unet.blocks()
        assert all(b.down.bias is None for b in blocks)
        assert blocks[0].up.bias is not None and all(b.up.bias is None for b in blocks[1:])
        assert [c.bias is not None for c in Dn.convs()] == [True, False, False, False, True]
    T, Dn = ours("instance")
    assert all(b.down.bias is not None for b in T.unet.blocks())
    with pytest.raises(NotImplementedError):
        M.NLayerDiscriminator(22, 64, 3, "group")


def _bufs_equal(bufs, want):
    assert set(bufs) == set(want)
    for k in want:
        assert torch.allclose(bufs[k].double(), want[k].double(), rtol=1e-6, atol=1e-7), k


def test_norm_oracle_matches_reference_batch_norm():
    """Train mode (the PatchGAN called on each half, the texture module once; running buffers after the calls) and
    eval mode, against the reference modules' outputs."""
    x, tex, rois, cloth = MG.inputs()
    T, Dn = ours("batch")
    g = GOLD["batch"]
    sd = {k: v.clone() for k, v in Dn.state_dict().items()}
    bn = NO.BN(sd, "batch", True)
    with torch.no_grad():
        out = NO.patchgan_forward(sd, x, bn, groups=2)
    assert torch.allclose(out, g["d_train"], rtol=1e-5, atol=1e-5)
    _bufs_equal(bn.bufs, g["d_train_bufs"])
    sd.update(bn.bufs)
    with torch.no_grad():
        out = NO.patchgan_forward(sd, x, NO.BN(sd, "batch", False))
    assert torch.allclose(out, g["d_eval"], rtol=1e-5, atol=1e-5)
    sd = {k: v.clone() for k, v in T.state_dict().items()}
    bn = NO.BN(sd, "batch", True)
    with torch.no_grad():
        out = NO.texture_forward(sd, tex, rois, cloth, bn)
    assert torch.allclose(out, g["tex_train"], rtol=1e-5, atol=1e-5)
    _bufs_equal(bn.bufs, g["tex_train_bufs"])
    sd.update(bn.bufs)
    with torch.no_grad():
        out = NO.texture_forward(sd, tex, rois, cloth, NO.BN(sd, "batch", False))
    assert torch.allclose(out, g["tex_eval"], rtol=1e-5, atol=1e-5)


@pytest.mark.skipif(not RH.available(), reason="reference tree not present")
@pytest.mark.parametrize("norm", ["batch", "none"])
def test_norm_oracle_is_bit_identical_to_reference_modules(norm):
    x, tex, rois, cloth = MG.inputs()
    rT, rD = reference(norm)
    sd = {k: v.clone() for k, v in rD.state_dict().items()}
    bn = NO.BN(sd, norm, True)
    rD.train()
    with torch.no_grad():
        assert torch.equal(torch.cat([rD(x[:2]), rD(x[2:])]), NO.patchgan_forward(sd, x, bn, groups=2))
        assert all(torch.equal(rD.state_dict()[k], v) for k, v in bn.bufs.items())
        rD.eval()
        sd = dict(rD.state_dict())
        assert torch.equal(rD(x), NO.patchgan_forward(sd, x, NO.BN(sd, norm, False)))
    rT.train()
    for m in rT.modules():
        if isinstance(m, torch.nn.Dropout):
            m.eval()
    sd = {k: v.clone() for k, v in rT.state_dict().items()}
    bn = NO.BN(sd, norm, True)
    with torch.no_grad():
        assert torch.equal(rT(tex, rois, cloth), NO.texture_forward(sd, tex, rois, cloth, bn))
        assert all(torch.equal(rT.state_dict()[k], v) for k, v in bn.bufs.items())
        rT.eval()
        sd = dict(rT.state_dict())
        assert torch.equal(rT(tex, rois, cloth), NO.texture_forward(sd, tex, rois, cloth, NO.BN(sd, norm, False)))


def _step_state(net):
    """state_dict copies: parameters as leaves that require grad, buffers plain."""
    names = [k for k, _ in net.named_parameters()]
    sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
    for k in names:
        sd[k].requires_grad_()
    return sd, [sd[k] for k in names]


@pytest.mark.parametrize("kind", ["texture", "warp"])
def test_full_batch_norm_step_matches_reference_golden(kind):
    """One full reference optimize_parameters() with --norm batch (tests/golden/batchnorm_64.pt): the norm-aware oracle
    plus torch.optim.AdamW reproduce the losses, every updated parameter (BN gamma / beta included, D with weight
    decay), and the running buffers and num_batches_tracked after the G forward and the three D calls — fake and real in
    the D step, then the G step's call with the weights after optimizer_D.step()."""
    import torch.nn.functional as F

    from oracle import nets as ON
    from test_engine_gpu import synth_texture_batch, synth_warp_batch
    from test_oracle_cpu import checksums, close_checksums

    g = GOLD[f"{kind}_step"]
    B, S = MG.STEP_B, MG.STEP_S
    torch.manual_seed(MG.STEP_SEED)
    if kind == "texture":
        G = M.TextureModule(3, 19, 12, "batch", 0.5, S)
    else:
        G = M.WarpModule()
    M.init_weights(G, "kaiming")
    Dn = M.NLayerDiscriminator(22, 64, 3, "batch")
    M.init_weights(Dn, "kaiming")
    close_checksums(checksums(G.state_dict()), g["init_G"], 0.0)
    close_checksums(checksums(Dn.state_dict()), g["init_D"], 0.0)
    sdG, pG = _step_state(G)
    sdD, pD = _step_state(Dn)
    bnG, bnD = NO.BN(sdG, "batch", True), NO.BN(sdD, "batch", True)
    optG = torch.optim.AdamW(pG, lr=1e-4, weight_decay=0, betas=(0.9, 0.999))
    optD = torch.optim.AdamW(pD, lr=4e-4, weight_decay=0.01, betas=(0.9, 0.999))
    if kind == "texture":
        tex, rois, cloth, tgt = synth_texture_batch(B, S)
        cond = cloth
    else:
        cond, inp, tgt = synth_warp_batch(B, S)
    torch.manual_seed(MG.LABEL_SEED)
    fk = NO.texture_forward(sdG, tex, rois, cloth, bnG) if kind == "texture" else ON.warp_forward(sdG, cond, inp)
    t_fake, t_real = ON.smooth_label(torch.rand(1)), ON.smooth_label(torch.rand(1))
    lf = ON.gan_loss(NO.patchgan_forward(sdD, torch.cat((cond, fk), 1).detach(), bnD), t_fake)
    lr = ON.gan_loss(NO.patchgan_forward(sdD, torch.cat((cond, tgt), 1), bnD), t_real)
    lD = 0.5 * (lf + lr)
    lD.backward()
    optD.step()
    gan = ON.gan_loss(NO.patchgan_forward(sdD, torch.cat((cond, fk), 1), bnD), ON.smooth_label(torch.rand(1)))
    if kind == "texture":
        rec = F.l1_loss(fk, tgt) * 10
        got = dict(G_l1=rec.item())
    else:
        rec = F.cross_entropy(fk, torch.argmax(tgt, 1)) * 100
        got = dict(G_ce=rec.item())
    (gan + rec).backward()
    optG.step()
    got.update(D=lD.item(), D_real=lr.item(), D_fake=lf.item(), G=(gan + rec).item(), G_gan=gan.item())
    assert got.keys() == g["losses"].keys()
    for k, v in g["losses"].items():
        assert abs(got[k] - v) <= 1e-5 * abs(v), (k, got[k], v)
    for sd, bn, want, lr_ in ((sdG, bnG, g["step_G"], 1e-4), (sdD, bnD, g["step_D"], 4e-4)):
        state = {k: v.detach() for k, v in sd.items()}
        state.update(bn.bufs)
        numel = {k: v.numel() for k, v in state.items()}
        bufs = [k for k in state if k.endswith(("running_mean", "running_var", "num_batches_tracked"))]
        assert bufs or sd is sdG, "the discriminator has running buffers"
        close_checksums({k: checksums(state)[k] for k in bufs}, {k: want[k] for k in bufs}, 1e-5)
        params = [k for k in state if k not in bufs]
        close_checksums({k: checksums(state)[k] for k in params}, {k: want[k] for k in params}, 5e-6, numel=numel,
                        lr=lr_)
        for k in bufs:
            if k.endswith("num_batches_tracked"):
                assert want[k] == ((3.0, 3.0) if sd is sdD else (1.0, 1.0)), k
