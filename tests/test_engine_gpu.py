"""GPU parity of the engines and of the WarpModel plugin step against the CPU oracle
(oracle/nets.py, itself pinned bit-exactly to the reference modules in tests/test_oracle_cpu.py).

Bar: 1e-3 relative fp32 (north star) — measured as max|err| / max|ref| per tensor; forward outputs
sit around 1e-5.  Parameter gradients are compared against an fp64 evaluation of the oracle
(the fp32 oracle itself is only good to ~3e-4 on this ill-conditioned net, see DESIGN.md)."""
import argparse
import tempfile

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import dropout as OD  # noqa: E402
from oracle import nets as ON  # noqa: E402


def dev():
    return torch.device("cuda:0")


def relmax(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30)).item()


def record(name, value):
    from conftest import record as _r

    _r(name, value)


def stage_gates(eng, n0=0, n1=None):
    """name -> bool NCHW mask (CPU) of the activation gates the device used: xhat > 0 <=> y > mean."""
    out = {}
    for st in eng.stages:
        if st.plain or st.act == 0:
            continue
        y = st.y[n0:n1]
        if st.stats is not None:
            mean = st.stats[n0:n1, :, 0].float()[:, None, None, :]
            m = y > mean
        else:
            m = y > 0
        out[st.name] = m.permute(0, 3, 1, 2).contiguous().cpu()    # NCHW-contiguous (see oracle/nets.py:_act)
    return out


def vgg_pool_winners(eng, tag):
    """name -> flat winner index [B,C,h/2,w/2] of every ReLU+MaxPool2d(2) the device evaluated (first maximum in
    row-major window order of relu(y), as csrc/perceptual.cu and torch both define it)."""
    import torch.nn.functional as F

    out = {}
    for st in eng.chain:
        if st.pool:
            a = F.relu(st.y.permute(0, 3, 1, 2)).cpu()
            out[f"{tag}.{int(st.name) + 2}"] = F.max_pool2d(a, 2, 2, return_indices=True)[1]
    return out


def synth_warp_batch(B, S, seed=1234):
    """SURVEY §8(d): normalised-RGB-like body, 16x16-block one-hot cloth labels (label 0 = all-zero)."""
    g = torch.Generator().manual_seed(seed)
    body = torch.rand(B, 3, S, S, generator=g) * 4.8 - 0.31
    lab = torch.randint(0, 19, (B, S // 16, S // 16), generator=g).repeat_interleave(16, 1).repeat_interleave(16, 2)
    tgt = torch.zeros(B, 19, S, S)
    for c in range(1, 19):
        tgt[:, c] = (lab == c).float()
    inp = torch.roll(tgt, (8, 8), (2, 3))
    return body, inp, tgt


def make_nets(seed=0):
    from swapnet_b200 import modules as M

    torch.manual_seed(seed)
    G = M.WarpModule()
    M.init_weights(G, "kaiming")
    D = M.NLayerDiscriminator(22, 64, 3, "instance")
    M.init_weights(D, "kaiming")
    # non-zero biases so that bias paths are exercised
    g = torch.Generator().manual_seed(7)
    for net in (G, D):
        for n, p in net.named_parameters():
            if n.endswith("bias"):
                p.data.copy_(torch.randn(p.shape, generator=g) * 0.1)
    return G, D


@pytest.mark.parametrize("mode", ["eval", "shared_masks"])
def test_warp_engine_forward(mode):
    from swapnet_b200 import engine as E

    B, S = 2, 64
    G, _ = make_nets()
    body, inp, _ = synth_warp_batch(B, S)
    sd = {k: v.clone() for k, v in G.state_dict().items()}
    Gd = G.to(dev())
    eng = E.WarpEngine(Gd, B, S, dev())
    eng.pack()
    training = mode == "shared_masks"
    out = eng.forward(body.to(dev()), inp.to(dev()), training=training, seed=42)
    torch.cuda.synchronize()
    drop = None
    if training:
        seeds = {s.name: E._mix_seed(42, s.id) for s in eng.stages}
        drop = OD.make_drop(seeds, 0.5)
    with torch.no_grad():
        ref = ON.warp_forward({k: v.double() for k, v in sd.items()}, body.double(), inp.double(), drop)
    err = relmax(out.permute(0, 3, 1, 2).cpu(), ref)
    assert err < 1e-3, f"warp forward ({mode}) relmax {err:.3e}"
    record(f"warp_engine_forward[{mode}]", f"{err:.3e}")


def _opt(B, S, **over):
    d = dict(model="warp", gpu_id=0, is_train=True, checkpoints_dir=tempfile.mkdtemp(prefix="sn_"), name="warp",
             no_confirm=True, body_representation="rgb", body_channels=12, cloth_representation="labels",
             cloth_channels=19, texture_channels=3, init_type="kaiming", init_gain=0.02, discriminator="basic",
             n_layers_D=3, norm="instance", gan_mode="vanilla", gan_label_mode="smooth", lambda_gan=1.0,
             lambda_discriminator=1.0, lambda_gp=10, optimizer_G="AdamW", optimizer_D="AdamW", lr=1e-4, d_lr=4e-4,
             weight_decay=0, d_weight_decay=0.01, b1=0.9, b2=0.999, warp_mode="gan", lambda_ce=100,
             continue_train=False, load_epoch="latest", verbose=False, batch_size=B, crop_size=S, load_size=S,
             b200_precision="fp32x3")
    d.update(over)
    return argparse.Namespace(**d)


@pytest.mark.parametrize("mode", ["eval", "train_shared_masks"])
def test_warp_model_step_matches_oracle(mode):
    """One WarpModel.optimize_parameters(): all six losses and every parameter gradient of G and D
    against the oracle's autograd (fp64).  eval: dropout off.  train_shared_masks: dropout(0.5) active in
    body_down4, cloth_down5/6 and the four resblocks, the oracle applying the library's own masks."""
    _warp_step_vs_oracle(2, 64, mode)


@pytest.mark.parametrize("mode", ["eval", "train_shared_masks"])
def test_warp_model_step_matches_oracle_512(mode):
    """The same gradient-level check at the BENCHMARKED resolution (BASELINE configs[1]: 512x512; one image so
    that the fp64 CPU oracle finishes in ~20 s): K = 9216 / 16384 contractions forward, weight gradients reduced
    over up to 65536 pixels with split-K atomics, input gradients with K up to 16384."""
    _warp_step_vs_oracle(1, 512, mode, tag="_512")


def _warp_step_vs_oracle(B, S, mode, tag=""):
    from swapnet_b200 import engine as E
    from swapnet_b200.models import create_model

    torch.manual_seed(0)
    # the 512 case runs as if the image were global sample 5 of a larger batch (dropout masks follow the global index)
    model = create_model(_opt(B, S, b200_sample_base=5 if tag else 0))
    model.setup(model.opt)
    if mode == "eval":
        model.eval()                  # dropout off; IN has no running stats
    model.is_train = True
    sdG = {k: v.detach().cpu().double().requires_grad_() for k, v in model.net_generator.state_dict().items()}
    sdD = {k: v.detach().cpu().double().requires_grad_() for k, v in model.net_discriminator.state_dict().items()}
    body, inp, tgt = synth_warp_batch(B, S)
    batch = dict(bodys=body, input_cloths=inp, target_cloths=tgt, cloth_paths=["c"] * B, body_paths=["b"] * B)
    torch.manual_seed(123)            # the label draws come from the CPU default generator
    model.set_input(batch)
    # run the phases by hand so that gradients can be read before the optimizer steps
    model._acc.zero_()
    model.forward()
    model._eng_Dd.zero_grad()
    model.backward_D()
    gD = {k: p.grad.detach().cpu().clone() for k, p in model.net_discriminator.named_parameters()}
    model._eng_G.zero_grad()
    model.backward_G()
    torch.cuda.synchronize()
    gG = {k: p.grad.detach().cpu().clone() for k, p in model.net_generator.named_parameters()}
    losses = model.get_current_losses()

    torch.manual_seed(123)
    draws = [torch.rand(1) for _ in range(3)]
    # gradients are compared at the gates the device used (see oracle/nets.py: _GATE); D is called three
    # times by the oracle: fake half, real half (D step), fake again (G step, same weights here)
    gates_G = stage_gates(model._eng_G)
    gates_D = [stage_gates(model._eng_Dd, 0, B), stage_gates(model._eng_Dd, B, 2 * B), stage_gates(model._eng_Dg)]
    calls = {}

    def gate(name, x):
        if name in gates_G:
            return gates_G[name]
        k = calls.get(name, 0)
        calls[name] = k + 1
        return gates_D[k][name]

    ON.gate_with(gate)
    drop = None
    if mode != "eval":
        eng = model._eng_G
        drop = OD.make_drop({s.name: E._mix_seed(eng.seed, s.id) for s in eng.stages}, 0.5, sample_base=eng.sample_base)
    o = ON.warp_step_losses(sdG, sdD, body.double(), inp.double(), tgt.double(), draws, drop=drop)
    stats = dict(ON.GATE_STATS)
    ON.gate_with(None)
    flips = {k: v for k, v in stats.items() if k != "__total__" and v}
    total = stats.get("__total__", 1)
    record(f"warp_step_gate_flips{tag}[{mode}]", f"{sum(flips.values())} of {total} gates differ from the fp64 oracle: {flips}")
    assert sum(flips.values()) <= 2e-5 * total, f"too many activation gates differ: {flips}"
    refD = torch.autograd.grad(o["D"], list(sdD.values()), retain_graph=True)
    refG = torch.autograd.grad(o["G"], list(sdG.values()), allow_unused=True)
    for k in ("D", "D_real", "D_fake", "G", "G_gan", "G_ce"):
        ref = o[k].item()
        assert abs(losses[k] - ref) <= 1e-3 * abs(ref), f"loss_{k}: {losses[k]} vs {ref}"
    err_f = relmax(model.fakes.cpu(), o["fakes"].detach())
    assert err_f < 1e-3, f"fakes relmax {err_f:.3e}"
    worst = {}
    dmax = max(r.abs().max().item() for r in refD)
    for (k, _), r in zip(sdD.items(), refD):
        if r.abs().max().item() < 1e-6 * dmax:   # bias in front of an InstanceNorm: exact gradient is zero
            assert gD[k].abs().max().item() < 1e-4 * dmax, k
            continue
        worst["D." + k] = relmax(gD[k], r)
    gmax = max(r.abs().max().item() for r in refG if r is not None)
    for (k, _), r in zip(sdG.items(), refG):
        if r is None:
            continue
        if r.abs().max().item() < 1e-6 * gmax:
            # bias in front of an InstanceNorm: the exact gradient is zero, the reference only holds noise
            assert gG[k].abs().max().item() < 1e-4 * gmax, k
            continue
        worst["G." + k] = relmax(gG[k], r)
    bad = {k: v for k, v in worst.items() if v >= 1e-3}
    record(f"warp_step_worst_grads{tag}[{mode}]", sorted(worst.items(), key=lambda kv: -kv[1])[:5])
    record(f"warp_step_fakes{tag}[{mode}]", f"{err_f:.3e}")
    assert not bad, f"parameter gradients beyond 1e-3: {bad}"


def test_warp_model_two_steps_run_and_change_weights():
    from swapnet_b200.models import create_model

    B, S = 2, 64
    torch.manual_seed(0)
    model = create_model(_opt(B, S))
    model.setup(model.opt)
    body, inp, tgt = synth_warp_batch(B, S)
    batch = dict(bodys=body, input_cloths=inp, target_cloths=tgt, cloth_paths=["c"] * B, body_paths=["b"] * B)
    w0 = model.net_generator.body_down2.model[0].weight.detach().clone()
    for _ in range(2):
        model.set_input(batch)
        model.optimize_parameters()
    losses = model.get_current_losses()
    assert all(torch.isfinite(torch.tensor(v)) for v in losses.values()), losses
    assert not torch.equal(w0, model.net_generator.body_down2.model[0].weight)
    model.save_checkpoint("latest")
    model.load_checkpoint_dir("latest")


# ------------------------------------------------------------------------------------------------
# texture stage
# ------------------------------------------------------------------------------------------------
def synth_texture_batch(B, S, seed=1234):
    import numpy as np

    from oracle import roi_align as R

    g = torch.Generator().manual_seed(seed)
    tex = torch.rand(B, 3, S, S, generator=g) * 4.5 - 2.0
    tgt = torch.rand(B, 3, S, S, generator=g) * 4.5 - 2.0
    lab = torch.randint(0, 19, (B, S // 16, S // 16), generator=g).repeat_interleave(16, 1).repeat_interleave(16, 2)
    cloth = torch.zeros(B, 19, S, S)
    for c in range(1, 19):
        cloth[:, c] = (lab == c).float()
    base = np.concatenate([R.NOTEBOOK_ROIS_256, R.NOTEBOOK_EXTRA_256])
    rois = torch.from_numpy(np.stack([np.roll(base, b, axis=0)[:12] for b in range(B)]) * (S / 256.0)).float()
    return tex, rois, cloth, tgt


def make_texture_net(S, seed=0):
    from swapnet_b200 import modules as M

    torch.manual_seed(seed)
    T = M.TextureModule(3, 19, 12, "instance", 0.5, S)
    M.init_weights(T, "kaiming")
    g = torch.Generator().manual_seed(9)
    for n, p in T.named_parameters():
        if n.endswith("bias"):
            p.data.copy_(torch.randn(p.shape, generator=g) * 0.1)
    return T


@pytest.mark.parametrize("S", [64, 128])
def test_texture_engine_forward(S):
    from swapnet_b200 import engine as E

    B = 2
    T = make_texture_net(S)
    tex, rois, cloth, _ = synth_texture_batch(B, S)
    sd = {k: v.clone().double() for k, v in T.state_dict().items()}
    eng = E.TextureEngine(T.to(dev()), B, S, dev())
    eng.pack()
    out = eng.forward(tex.to(dev()), rois.to(dev()), cloth.to(dev()), training=False)
    torch.cuda.synchronize()
    with torch.no_grad():
        ref = ON.texture_forward(sd, tex.double(), rois.double(), cloth.double())
    err = relmax(out.permute(0, 3, 1, 2).cpu(), ref)
    record(f"texture_engine_forward[{S}]", f"{err:.3e}")
    assert err < 1e-3, f"texture forward relmax {err:.3e}"


@pytest.mark.parametrize("perceptual", [False, True])
def test_texture_model_step_matches_oracle(perceptual):
    """perceptual=True: the reference's DEFAULT texture losses (lambda_content 20, lambda_style 1e-8,
    texture_model.py:39-48) with seeded-random VGG16 weights (the pretrained file is not obtainable offline)."""
    _texture_step_vs_oracle(2, 128, perceptual)


def test_texture_model_step_matches_oracle_512():
    """BASELINE configs[2] resolution (512x512, num_downs = 9, 12 ROIs) with the reference's default loss set
    (L1 + GAN + VGG16 content + Gram style), one image, against the fp64 oracle."""
    _texture_step_vs_oracle(1, 512, True, tag="_512")


def _texture_step_vs_oracle(B, S, perceptual, tag=""):
    from swapnet_b200.models import create_model

    torch.manual_seed(0)
    lc, ls = (20.0, 1e-8) if perceptual else (0.0, 0.0)
    opt = _opt(B, S, model="texture", name="texture", netG="swapnet", lambda_l1=10, lambda_content=lc, lambda_style=ls,
               b200_vgg="random")
    model = create_model(opt)
    model.setup(opt)
    model.eval()
    g = torch.Generator().manual_seed(9)
    for net in (model.net_generator, model.net_discriminator):
        for n, p in net.named_parameters():
            if n.endswith("bias"):
                p.data.copy_((torch.randn(p.shape, generator=g) * 0.1).to(p.device))
    sdG = {k: v.detach().cpu().double().requires_grad_() for k, v in model.net_generator.state_dict().items()}
    sdD = {k: v.detach().cpu().double().requires_grad_() for k, v in model.net_discriminator.state_dict().items()}
    tex, rois, cloth, tgt = synth_texture_batch(B, S)
    batch = dict(input_textures=tex, rois=rois, cloths=cloth, target_textures=tgt, cloth_paths=["c"] * B,
                 texture_paths=["t"] * B)
    torch.manual_seed(321)
    model.set_input(batch)
    model._acc.zero_()
    model.forward()
    model._eng_Dd.zero_grad()
    model.backward_D()
    gD = {k: p.grad.detach().cpu().clone() for k, p in model.net_discriminator.named_parameters()}
    model._eng_G.zero_grad()
    model.backward_G()
    torch.cuda.synchronize()
    gG = {k: p.grad.detach().cpu().clone() for k, p in model.net_generator.named_parameters()}
    losses = model.get_current_losses()

    torch.manual_seed(321)
    draws = [torch.rand(1) for _ in range(3)]
    gates_G = stage_gates(model._eng_G)
    gates_D = [stage_gates(model._eng_Dd, 0, B), stage_gates(model._eng_Dd, B, 2 * B), stage_gates(model._eng_Dg)]
    calls = {}

    gates_P, vgg_sd = {}, None
    if perceptual:
        gates_P = {"vgg_o." + k: v for k, v in stage_gates(model._eng_P.out).items()}
        gates_P.update({"vgg_t." + k: v for k, v in stage_gates(model._eng_P.tgt).items()})
        vgg_sd = {k: v.detach().cpu().double() for k, v in model.net_vgg.state_dict().items()}

    def gate(name, x):
        if name in gates_G:
            return gates_G[name]
        if name in gates_P:
            return gates_P[name]
        k = calls.get(name, 0)
        calls[name] = k + 1
        return gates_D[k][name]

    ON.gate_with(gate)
    if perceptual:
        winners = vgg_pool_winners(model._eng_P.out, "vgg_o")
        ON.pool_with(lambda name, x: winners.get(name))
    d = model.fakes.detach() - tgt.to(dev())                     # same fp32 subtraction as the L1 kernel
    l1_sign = torch.sign(d).cpu().double()
    o = ON.texture_step_losses(sdG, sdD, tex.double(), rois.double(), cloth.double(), tgt.double(), draws,
                               l1_sign=l1_sign, vgg=vgg_sd, lambda_content=lc, lambda_style=ls)
    ref_sign = torch.sign(o["fakes"].detach() - tgt.double())
    record(f"texture_step_l1_sign_flips{tag}", f"{int((ref_sign != l1_sign).sum())} of {l1_sign.numel()}")
    stats = dict(ON.GATE_STATS)
    ON.gate_with(None)
    ON.pool_with(None)
    pool_flips = {k: stats.pop(k) for k in list(stats) if k.startswith("pool:")}
    if perceptual:
        record(f"texture_step_pool_winner_flips{tag}", pool_flips)
    flips = {k: v for k, v in stats.items() if k != "__total__" and v}
    record(f"texture_step_gate_flips{tag}[perceptual={perceptual}]", f"{sum(flips.values())} of {stats.get('__total__', 1)}: {flips}")
    refD = torch.autograd.grad(o["D"], list(sdD.values()), retain_graph=True)
    refG = torch.autograd.grad(o["G"], list(sdG.values()), allow_unused=True)
    for k in ("D", "D_real", "D_fake", "G", "G_gan", "G_l1") + (("G_content", "G_style") if perceptual else ()):
        ref = o[k].item()
        assert abs(losses[k] - ref) <= 1e-3 * abs(ref), f"loss_{k}: {losses[k]} vs {ref}"
        if perceptual:
            record(f"texture_step_perceptual_loss{tag}_{k}", f"{losses[k]:.9g} vs {ref:.9g}")
    err_f = relmax(model.fakes.cpu(), o["fakes"].detach())
    assert err_f < 1e-3, f"fakes relmax {err_f:.3e}"
    worst = {}
    for name, got, sd, refs in (("D.", gD, sdD, refD), ("G.", gG, sdG, refG)):
        mx = max(r.abs().max().item() for r in refs if r is not None)
        for (k, _), r in zip(sd.items(), refs):
            if r is None:
                continue
            if r.abs().max().item() < 1e-6 * mx:
                assert got[k].abs().max().item() < 1e-4 * mx, k
                continue
            worst[name + k] = relmax(got[k], r)
    record(f"texture_step_worst_grads{tag}[perceptual={perceptual}]", sorted(worst.items(), key=lambda kv: -kv[1])[:5])
    record(f"texture_step_fakes{tag}", f"{err_f:.3e}")
    bad = {k: v for k, v in worst.items() if v >= 1e-3}
    assert not bad, f"parameter gradients beyond 1e-3: {bad}"
    assert sum(flips.values()) <= 2e-5 * stats.get("__total__", 1), f"too many activation gates differ: {flips}"


def test_warp_forward_full_size_512():
    """BASELINE size (512x512, the K = 9216 / 16384 convolutions) against the fp64 oracle on one image:
    the tensor core's truncating fp32 accumulator makes the per-layer error grow with K, so the bar is
    checked where it is hardest."""
    from swapnet_b200 import engine as E

    B, S = 1, 512
    G, _ = make_nets()
    body, inp, _ = synth_warp_batch(B, S)
    sd = {k: v.clone().double() for k, v in G.state_dict().items()}
    eng = E.WarpEngine(G.to(dev()), B, S, dev(), train=False)
    eng.pack()
    out = eng.forward(body.to(dev()), inp.to(dev()), training=False)
    torch.cuda.synchronize()
    torch.set_num_threads(max(1, min(64, torch.get_num_threads())))
    rec = {}
    ON.record_into(rec)
    with torch.no_grad():
        ref = ON.warp_forward(sd, body.double(), inp.double())
    ON.record_into(None)
    err = relmax(out.permute(0, 3, 1, 2).cpu(), ref)
    per_layer = {st.name: relmax(st.y.cpu(), rec[st.name + ".y"].permute(0, 2, 3, 1)) for st in eng.stages}
    worst = sorted(per_layer.items(), key=lambda kv: -kv[1])[:4]
    record("warp_forward_512", f"fakes {err:.3e}; worst conv outputs {[(k, f'{v:.2e}') for k, v in worst]}")
    assert err < 1e-3, f"512x512 forward relmax {err:.3e}"


@pytest.mark.parametrize("B,S", [(1, 192), (3, 128)])
def test_warp_forward_other_shapes(B, S):
    """Non-power-of-two planes (192 -> 96, 48, 24, 12, 6, 3) and odd batch sizes."""
    from swapnet_b200 import engine as E

    G, _ = make_nets()
    body, inp, _ = synth_warp_batch(B, S) if S % 16 == 0 else (None, None, None)
    sd = {k: v.clone().double() for k, v in G.state_dict().items()}
    eng = E.WarpEngine(G.to(dev()), B, S, dev(), train=False)
    eng.pack()
    out = eng.forward(body.to(dev()), inp.to(dev()), training=False)
    torch.cuda.synchronize()
    with torch.no_grad():
        ref = ON.warp_forward(sd, body.double(), inp.double())
    err = relmax(out.permute(0, 3, 1, 2).cpu(), ref)
    record(f"warp_forward_shape[{B},{S}]", f"{err:.3e}")
    assert err < 1e-3


def test_warp_model_ce_mode_and_checkpoint_roundtrip():
    """--warp_mode ce (no discriminator, warp_model.py:69-74,175-183) and a save/load round trip through the
    reference's checkpoint file names."""
    import os

    from swapnet_b200.models import create_model

    B, S = 2, 64
    torch.manual_seed(0)
    opt = _opt(B, S, warp_mode="ce")
    model = create_model(opt)
    model.setup(opt)
    assert not hasattr(model, "net_discriminator") and model.optimizer_names == ["G"]
    body, inp, tgt = synth_warp_batch(B, S)
    batch = dict(bodys=body, input_cloths=inp, target_cloths=tgt, cloth_paths=["c"] * B, body_paths=["b"] * B)
    model.set_input(batch)
    model.optimize_parameters()
    l0 = float(model.loss_G)
    for _ in range(3):
        model.set_input(batch)
        model.optimize_parameters()
    assert float(model.loss_G) < l0, "cross-entropy did not decrease over 4 AdamW steps on a fixed batch"
    model.save_checkpoint("latest")
    assert os.path.exists(os.path.join(model.save_dir, "latest_net_generator.pth"))
    assert os.path.exists(os.path.join(model.save_dir, "latest_optim_G.pth"))
    w = model.net_generator.dual_up3.model[0].weight.detach().clone()
    model.net_generator.dual_up3.model[0].weight.data.zero_()
    model.load_checkpoint_dir("latest")
    assert torch.equal(w, model.net_generator.dual_up3.model[0].weight)
    model.set_input(batch)
    model.optimize_parameters()     # engines keep working on the re-loaded storage


def test_texture_forward_full_size_512():
    """BASELINE config 3 size (512x512, num_downs = 9, ROI pooling at 128x128 -> x8 nearest up-sampling)."""
    from swapnet_b200 import engine as E

    B, S = 1, 512
    T = make_texture_net(S)
    tex, rois, cloth, _ = synth_texture_batch(B, S)
    sd = {k: v.clone().double() for k, v in T.state_dict().items()}
    eng = E.TextureEngine(T.to(dev()), B, S, dev(), train=False)
    eng.pack()
    out = eng.forward(tex.to(dev()), rois.to(dev()), cloth.to(dev()), training=False)
    torch.cuda.synchronize()
    with torch.no_grad():
        ref = ON.texture_forward(sd, tex.double(), rois.double(), cloth.double())
    err = relmax(out.permute(0, 3, 1, 2).cpu(), ref)
    record("texture_forward_512", f"{err:.3e}")
    assert err < 1e-3


@pytest.mark.parametrize("B,S", [(2, 64), (1, 128)])
def test_perceptual_engine_matches_oracle(B, S):
    """PerceptualLoss(fakes, targets) * (lambda_content, lambda_style) and its gradient w.r.t. fakes
    (modules/losses/perceptual.py:49-79) — seeded-random VGG16, gates imposed from the device."""
    from swapnet_b200 import engine as E
    from swapnet_b200 import modules as M

    vgg = M.load_vgg16_features("random").to(dev())
    g = torch.Generator().manual_seed(B * 100 + S)
    fakes = torch.rand(B, 3, S, S, generator=g) * 2 - 1            # tanh range
    tgt = torch.rand(B, 3, S, S, generator=g) * 4.5 - 2.0          # normalised-RGB range
    lc, ls = 20.0, 1e-8
    P = E.PerceptualEngine(vgg, B, S, dev())
    acc = torch.zeros(2, dtype=torch.float64, device=dev())
    fk = fakes.permute(0, 2, 3, 1).contiguous().to(dev())
    td = tgt.to(dev())
    dstyle = torch.zeros(B, S, S, 3, device=dev())
    P.style(fk, td, ls, acc[1:2], dstyle)
    dcontent = P.content(fk, td, lc, acc[0:1])
    torch.cuda.synchronize()
    gates = {"vgg_o." + k: v for k, v in stage_gates(P.out).items()}
    gates.update({"vgg_t." + k: v for k, v in stage_gates(P.tgt).items()})
    winners = vgg_pool_winners(P.out, "vgg_o")
    ON.gate_with(lambda name, x: gates.get(name))
    ON.pool_with(lambda name, x: winners.get(name))
    sd = {k: v.detach().cpu().double() for k, v in vgg.state_dict().items()}
    f64 = fakes.double().requires_grad_()
    c, st = ON.perceptual_loss(sd, f64, tgt.double(), True)
    stats = dict(ON.GATE_STATS)
    ON.gate_with(None)
    ON.pool_with(None)
    pool_flips = {k: stats.pop(k) for k in list(stats) if k.startswith("pool:")}
    record(f"perceptual_engine_pool_winner_flips[{B},{S}]", pool_flips)
    (gc,) = torch.autograd.grad(c * lc, f64, retain_graph=True)
    (gs,) = torch.autograd.grad(st * ls, f64)
    flips = sum(v for k, v in stats.items() if k != "__total__")
    record(f"perceptual_engine[{B},{S}]",
           f"content {acc[0].item():.9g} vs {(c * lc).item():.9g}; style {acc[1].item():.9g} vs {(st * ls).item():.9g}; "
           f"gate flips {flips} of {stats.get('__total__', 0)}")
    assert abs(acc[0].item() - (c * lc).item()) <= 1e-3 * abs((c * lc).item())
    assert abs(acc[1].item() - (st * ls).item()) <= 1e-3 * abs((st * ls).item())
    ec = relmax(dcontent.cpu(), gc.permute(0, 2, 3, 1))
    es = relmax(dstyle.cpu(), gs.permute(0, 2, 3, 1))
    record(f"perceptual_engine_grads[{B},{S}]", f"content {ec:.3e} style {es:.3e}")
    assert ec < 1e-3 and es < 1e-3
    assert flips <= 2e-5 * stats.get("__total__", 1)


def _run_phases(model, batch, seed):
    """forward, D phase, G phase by hand (no optimizer step) -> (losses, flat D grads, flat G grads) on the CPU."""
    torch.manual_seed(seed)            # the smooth-label draws come from the CPU default generator
    model.set_input(batch)
    model._acc.zero_()
    model.forward()
    model._eng_Dd.zero_grad()
    model.backward_D()
    gD = model._eng_Dd.flat_grad.detach().cpu().clone()
    model._eng_G.zero_grad()
    model.backward_G()
    torch.cuda.synchronize()
    gG = model._eng_G.flat_grad.detach().cpu().clone()
    return dict(model.get_current_losses()), gD, gG


@pytest.mark.parametrize("mode", ["eval", "train"])
def test_warp_batch16_equals_mean_of_16_single_image_steps_512(mode):
    """Self-consistency at the BENCHMARKED configuration (BASELINE configs[1]: 512x512, batch 16): every op on the
    path is per-sample and every loss a batch mean (SURVEY §8e), so the batch-16 gradients must equal the mean of the
    16 single-image gradients (same weights, same label draws, dropout masks of global sample i).  Ties the
    batch-16 training step that bench.py times to the single-image step pinned against the fp64 oracle above."""
    from swapnet_b200.models import create_model

    B, S = 16, 512
    torch.manual_seed(0)
    model = create_model(_opt(B, S))
    model.setup(model.opt)
    if mode == "eval":
        model.eval()
    model.is_train = True
    body, inp, tgt = synth_warp_batch(B, S)
    full = dict(bodys=body, input_cloths=inp, target_cloths=tgt, cloth_paths=["c"] * B, body_paths=["b"] * B)
    l16, gD16, gG16 = _run_phases(model, full, 777)
    sums = None
    lsum = {k: 0.0 for k in l16}
    for i in range(B):
        one = dict(bodys=body[i:i + 1], input_cloths=inp[i:i + 1], target_cloths=tgt[i:i + 1], cloth_paths=["c"],
                   body_paths=["b"])
        model.ensure_engines(1, S)
        model._eng_G.sample_base = i
        l1, gD1, gG1 = _run_phases(model, one, 777)
        sums = [gD1.double(), gG1.double()] if sums is None else [sums[0] + gD1, sums[1] + gG1]
        for k in lsum:
            lsum[k] += l1[k] / B
    eD = relmax(gD16, sums[0] / B)
    eG = relmax(gG16, sums[1] / B)
    el = max(abs(l16[k] - lsum[k]) / abs(lsum[k]) for k in l16)
    record(f"warp_b16_vs_16xb1_512[{mode}]", f"flat grad D {eD:.3e} G {eG:.3e}; losses {el:.3e}")
    assert eD < 1e-4 and eG < 1e-4 and el < 1e-5, (eD, eG, el)


def test_dropped_model_buffers_are_reused_by_the_next_model():
    """A model is a reference cycle (loss closures, stages <-> engines): building a model's engines collects dropped
    models first, so their device buffers are reused instead of piling up (at 512x512, batch 16 one model holds tens of
    GB of the 80 GB).  Automatic collection is off here so that only the model's own collection can free them."""
    import gc

    from swapnet_b200.models import create_model

    def build():
        torch.manual_seed(0)
        m = create_model(_opt(2, 128))
        m.setup(m.opt)
        m.ensure_engines(2, 128)
        return m

    was_enabled = gc.isenabled()
    gc.collect()
    gc.disable()
    try:
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        model = build()
        one = torch.cuda.memory_allocated() - base
        del model
        model = build()
        two = torch.cuda.memory_allocated() - base
        del model
    finally:
        if was_enabled:
            gc.enable()
        gc.collect()
    assert two < 1.5 * one, (one, two)


def test_train_loop_protocol():
    """The calls train.py:31-116 makes, in its order, on a two-epoch run whose last batch of each epoch is short (the
    reference's DataLoader has no drop_last, datasets/__init__.py:69): set_input / optimize_parameters /
    get_current_losses per iteration, save_checkpoint('latest') + save_checkpoint(epoch) per epoch, then a
    --continue_train reload.  Checks the loss keys (loss_names), the checkpoint file names (base_model.py:161-173) and
    that the state_dict keys are the reference's (golden list generated from the reference modules)."""
    import os

    from swapnet_b200.models import create_model

    S = 64
    torch.manual_seed(0)
    opt = _opt(2, S)
    model = create_model(opt)
    model.setup(opt)
    body, inp, tgt = synth_warp_batch(3, S)

    def batch(i0, i1):
        n = i1 - i0
        return dict(bodys=body[i0:i1], input_cloths=inp[i0:i1], target_cloths=tgt[i0:i1], cloth_paths=["c"] * n,
                    body_paths=["b"] * n)

    loader = [batch(0, 2), batch(2, 3)]              # 3 samples, batch_size 2 -> a short last batch
    engines = set()
    for epoch in (1, 2):
        for data in loader:
            model.set_input(data)
            model.optimize_parameters()
            engines.add(id(model._eng_G))
            losses = model.get_current_losses()
            assert list(losses) == ["D", "D_real", "D_fake", "G", "G_gan", "G_ce"]
            assert all(isinstance(v, float) and v == v for v in losses.values())
        model.save_checkpoint("latest")
        model.save_checkpoint(epoch)
    assert len(engines) == 2, "the (batch, size) engine cache re-planned inside the run"
    files = sorted(os.listdir(model.save_dir))
    for prefix in ("latest", "1", "2"):
        for f in (f"{prefix}_net_generator.pth", f"{prefix}_net_discriminator.pth", f"{prefix}_optim_G.pth",
                  f"{prefix}_optim_D.pth"):
            assert f in files, (f, files)
    sd = torch.load(os.path.join(model.save_dir, "latest_net_generator.pth"))
    g = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "warp_64.pt"))
    assert list(sd.keys()) == list(g["init_checksums_G"].keys())          # the reference WarpModule's state_dict keys
    sdd = torch.load(os.path.join(model.save_dir, "latest_net_discriminator.pth"))
    assert list(sdd.keys()) == list(g["init_checksums_D"].keys())
    # --continue_train: a fresh model picks the files up (base_model.py:56-59,193-212) and keeps training
    opt2 = _opt(2, S, continue_train=True, checkpoints_dir=opt.checkpoints_dir)
    m2 = create_model(opt2)
    m2.setup(opt2)
    for k, v in m2.net_generator.state_dict().items():
        assert torch.equal(v.cpu(), sd[k]), k
    assert m2.optimizer_G._step == 4
    m2.set_input(loader[0])
    m2.optimize_parameters()
    assert all(v == v for v in m2.get_current_losses().values())


def test_compact_cloth_inputs_equal_dense_inputs():
    """SURVEY §8f rank 4: the cloth tensors fed as a uint8 label map (targets) and an int32 bit mask (independently
    augmented input channels: not one-hot any more) give the step the dense fp32 tensors give — the planes the
    kernels expand on the device are identical, so only the atomics' summation order differs."""
    from swapnet_b200.models import create_model
    from swapnet_b200.ops import SegMap

    B, S = 2, 128
    torch.manual_seed(0)
    model = create_model(_opt(B, S))
    model.setup(model.opt)
    model.is_train = True
    body, inp, tgt = synth_warp_batch(B, S)
    for c in (3, 7, 11):                       # per-channel augmentation: channels overlap, channel 0 stays empty
        inp[:, c] = torch.roll(inp[:, c], (c, 2 * c), (1, 2))
    dense = dict(bodys=body, input_cloths=inp, target_cloths=tgt, cloth_paths=["c"] * B, body_paths=["b"] * B)
    sm_in, sm_tgt = SegMap.from_dense(inp), SegMap.from_dense(tgt)
    assert sm_in.data.dtype == torch.int32 and sm_tgt.data.dtype == torch.uint8
    assert torch.equal(sm_in.dense(), inp) and torch.equal(sm_tgt.dense(), tgt)
    compact = dict(dense, input_cloths=sm_in.data, target_cloths=sm_tgt.data)    # raw [B,H,W] tensors, as a loader yields
    l0, gD0, gG0 = _run_phases(model, dense, 5)
    f0 = model.fakes.clone()
    l1, gD1, gG1 = _run_phases(model, compact, 5)
    assert torch.equal(f0, model.fakes), "forward differs between dense and compact inputs"
    assert relmax(gD1, gD0) < 1e-5 and relmax(gG1, gG0) < 1e-5
    assert all(abs(l0[k] - l1[k]) <= 1e-6 * abs(l0[k]) for k in l0), (l0, l1)
    assert torch.equal(model.dense(model.targets).cpu(), tgt)


def test_graph_replayed_steps_match_eager_steps():
    """SURVEY §8f rank 2: after two eager steps per input shape the training step is replayed as ONE captured CUDA
    graph (labels, AdamW bias corrections and the dropout seed are read from a device buffer the step prologue
    refreshes).  Five steps with the graph must track five eager steps of an identically seeded model, with fresh
    dropout masks and label draws every step."""
    from swapnet_b200 import ops
    from swapnet_b200.models import create_model

    B, S = 2, 64
    body, inp, tgt = synth_warp_batch(B, S)
    batch = dict(bodys=body, input_cloths=inp, target_cloths=tgt, cloth_paths=["c"] * B, body_paths=["b"] * B)
    runs = {}
    for graph in (1, 0):
        torch.manual_seed(0)
        model = create_model(_opt(B, S, b200_graph=graph))
        model.setup(model.opt)
        torch.manual_seed(99)
        hist, launches = [], []
        for _ in range(5):
            n0 = ops.launch_count()
            model.set_input(batch)
            model.optimize_parameters()
            hist.append(dict(model.get_current_losses()))
            launches.append(ops.launch_count() - n0)
        assert (len(model._graphs) == 1) == bool(graph)
        runs[graph] = (hist, launches, model.net_generator.dual_up3.model[0].weight.detach().clone(),
                       model.optimizer_G._step)
    (hg, lg, wg, sg), (he, le, we, se) = runs[1], runs[0]
    assert sg == se == 5
    assert lg == le, (lg, le)     # replayed launches are accounted for; the capture pass itself is not counted
    for a, b in zip(hg, he):
        for k in a:
            assert abs(a[k] - b[k]) <= 2e-3 * abs(b[k]), (k, a[k], b[k])
    assert hg[3]["G_ce"] != hg[4]["G_ce"]
    # AdamW's first steps move every weight by ~lr per step (sign-like update): a near-zero gradient whose sign differs
    # between the runs (atomics' summation order) moves its weight the other way
    assert (wg - we).abs().max().item() < 6e-4, (wg - we).abs().max().item()   # 5 steps x lr 1e-4: a sign flip moves 2 lr / step
    record("graph_vs_eager_5_steps", f"max |dW| {(wg - we).abs().max().item():.2e}; launches/step graph {lg} eager {le}")


def packed_ref(layer, dgrad):
    """Unscaled fp32 contents of layer.wd (dgrad) or layer.wp: the host restatements of the packed layouts in
    oracle/emulate.py, zero in the padding rows and tap slots."""
    from oracle import emulate as EM
    from swapnet_b200 import lowering as L

    w = layer.weight.detach().cpu()
    pw, k_pad = (layer.wd, layer.dy.c) if dgrad else (layer.wp, layer.k_pad)
    if layer.kind != "head":
        m = EM.pack_weights_ref(w, layer.kind, dgrad, k_pad)
    elif dgrad:
        m = EM.pack_head_ref(w, 0, k_pad, True)
    elif layer.stacked:       # [phase * HEAD_SLOT + co][3 x 3 shifts][ci], zero where a phase has no tap at a shift
        eff, S = EM.head_eff_weights(w), L.HEAD_SLOT
        m = w.new_zeros(4 * S, 9, k_pad)
        for p in range(4):
            for ey in range(L.head_neff(p >> 1)):
                for ex in range(L.head_neff(p & 1)):
                    m[p * S:p * S + layer.cout, ey * 3 + ex, :layer.cin] = \
                        eff[:, L.HEAD_PHASE_OFF[p] + ey * L.head_neff(p & 1) + ex]
        m = m.reshape(4 * S, 9 * k_pad)
    else:                     # the four per-phase matrices one after the other
        m = torch.cat([x.reshape(-1) for x in EM.pack_head_ref(w, layer.rows_pad, k_pad, False)]).view(pw.rows, -1)
    out = torch.zeros(pw.rows, pw.k_total)
    out[:m.shape[0], :m.shape[1]] = m
    return out


def check_layer_packs(layer):
    """layer.wscale and the layer's packed copies, bit for bit against the host reference: s = 2^(14 - e) with
    max|w| = f * 2^e, f in [0.5, 1) (1 for an all-zero weight); fp16-split packs hold the weights times s, saturated
    at the fp16 range, bf16-split packs the weights themselves; hi = rn16(v), lo = rn16(v - hi) (split16 in
    csrc/common.cuh)."""
    import math

    from swapnet_b200 import ops

    m = layer.weight.detach().abs().max().item()
    s = 1.0 if m == 0 else 2.0 ** (14 - math.frexp(m)[1])
    assert torch.equal(layer.wscale.cpu(), torch.tensor([s, 1 / s])), (layer.name, layer.wscale, s)
    for dgrad, pw in ((False, layer.wp), (True, layer.wd)):
        if dgrad and not layer.dgrad_plans:
            continue
        v = packed_ref(layer, dgrad)
        if pw.fmt == ops.FMT_F16:
            v, t = (v * (1.0 if pw.scale is None else s)).clamp(-65504, 65504), torch.float16
        else:
            assert pw.scale is None
            t = torch.bfloat16
        hi = v.to(t)
        lo = (v - hi.float()).to(t)
        assert torch.equal(pw.hi.cpu().view(torch.int16), hi.view(torch.int16)), (layer.name, dgrad, "hi")
        assert torch.equal(pw.lo.cpu().view(torch.int16), lo.view(torch.int16)), (layer.name, dgrad, "lo")


def test_engine_pack_equals_host_reference():
    """Engine.pack() (one multi-tensor scale launch, one multi-tensor pack launch, the head's effective-tap packs)
    writes exactly the scales and split planes of the host reference: forward and input-gradient layouts of every
    conv layer of the warp generator and the PatchGAN."""
    from swapnet_b200 import engine as E
    from swapnet_b200.layers import ConvLayer

    G, D = make_nets()
    for net, mk in ((G, lambda n: E.WarpEngine(n, 1, 64, dev())), (D, lambda n: E.PatchGANEngine(n, 2, 64, dev(), input_grad=True))):
        eng = mk(net.to(dev()))
        eng.alloc_grads()
        eng.bind_backward()
        layers = [st.layer for st in eng.stages if isinstance(st.layer, ConvLayer)]
        for _ in range(2):    # the scale launch resets its scratch words: a second run on cleared outputs is identical
            for ly in layers:
                ly.wscale.zero_()
                for pw in (ly.wp, ly.wd):
                    if pw is not None:
                        pw.hi.zero_()
                        pw.lo.zero_()
            eng.pack()
            torch.cuda.synchronize()
            for ly in layers:
                check_layer_packs(ly)


# kind, cin, cout, input channels (forward K), gradient channels (input-gradient K; None: no input gradient)
PACK_EDGE_CASES = {
    "tail": ("conv3z", 3, 3, 16, None),        # 81 floats: the largest |w| is the last, after the 20 float4 loads
    "zero": ("conv4s2", 19, 64, 32, 64),       # all-zero weight: scale 1, zero planes
    "pow2": ("convT4s2", 64, 3, 64, 16),       # max |w| = 2^-1 exactly (frexp boundary: max|w| * s = 2^13)
    "head27": ("head", 64, 27, 64, None),      # more outputs than HEAD_SLOT: the unstacked forward pack
}


@pytest.mark.parametrize("case", sorted(PACK_EDGE_CASES))
def test_layer_pack_edges(case):
    """ConvLayer.pack() (a pack table of one layer) on what the engines' weights do not show: a count that is not a
    multiple of 4, all zeros, a power-of-two maximum, K padded to 16 and 32 channels, the unstacked head."""
    from swapnet_b200 import lowering as L
    from swapnet_b200 import ops
    from swapnet_b200.layers import ConvLayer

    kind, cin, cout, xc, dyc = PACK_EDGE_CASES[case]
    n, h, w = 1, 16, 16
    k = 3 if kind == "conv3z" else 4
    g = torch.Generator().manual_seed(5)
    wt = torch.randn((cin, cout, k, k) if kind == "convT4s2" else (cout, cin, k, k), generator=g) * 0.1
    if case == "tail":
        wt.view(-1)[-1] = -3 * wt.abs().max()
    elif case == "zero":
        wt.zero_()
    elif case == "pow2":
        wt = wt.clamp(-0.25, 0.25)
        wt.view(-1)[100] = -0.5
    layer = ConvLayer(kind, wt.to(dev()), None, ops.Planes(n, h, w, xc, dev()), name=case)
    if dyc is not None:
        oh, ow = L.out_hw(kind, h, w)
        layer.bind_backward(ops.Planes(n, oh, ow, dyc, dev(), fmt=ops.FMT_BF16),
                            torch.zeros(n, h, w, cin, device=dev()), None)
        assert layer.dgrad_plans
    layer.pack()
    torch.cuda.synchronize()
    check_layer_packs(layer)
