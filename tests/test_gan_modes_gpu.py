"""GPU parity of `--gan_mode lsgan` and `--gan_mode wgan` (vanilla is covered by test_engine_gpu / test_batchnorm_gpu):
the GAN-loss kernel per objective against fp64 torch, plugin steps of both stages against the objective-aware fp64
oracle (tests/tools/gan_modes_oracle.py) at the 1e-3 bar of tests/test_engine_gpu.py, a whole step with AdamW, graph
replay, the CPU generator's state after a step, the refused modes and 2-rank data parallelism.

A wgan loss is a difference of means and may cancel, so its bar is taken relative to the larger of |loss| and the
step's mean |pred|."""
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "tools"))

import gan_modes_oracle as GO  # noqa: E402
import norm_oracle as NO  # noqa: E402
from oracle import dropout as OD  # noqa: E402
from oracle import nets as ON  # noqa: E402
from test_batchnorm_gpu import _check_step, _param_sd, _randomise_affine, bn_stage_gates  # noqa: E402
from test_engine_gpu import _opt, record, relmax, stage_gates, synth_texture_batch, synth_warp_batch  # noqa: E402

NEW_MODES = ("lsgan", "wgan")


def dev():
    return torch.device("cuda:0")


# ---------------------------------------------------------------------------------------------
# kernel
# ---------------------------------------------------------------------------------------------
def _kernel_cases():
    for mode in GO.MODES:
        for halves in (1, 2):
            for count in (1, 961, 2 * 16 * 62 * 62):
                for device_t in ((False, True) if mode != "wgan" else (False,)):
                    yield mode, halves, count, device_t


@pytest.mark.parametrize("mode,halves,count,device_t", list(_kernel_cases()))
def test_gan_loss_kernel_matches_fp64(mode, halves, count, device_t):
    """ops.gan_loss_fwd_bwd per objective: one half (G step) or two (the D step's [fake | real] batch), targets by value
    or from device memory, gscale != 1.  dpred within 1e-6 of max|dpred|; each half's loss within 1e-6 of
    max(|loss|, mean|pred|)."""
    from swapnet_b200 import ops

    g = torch.Generator().manual_seed(count * 2 + halves)
    pred = torch.randn(halves, count, generator=g) * 2.0 + 0.3
    if mode == "wgan":
        t = [1.0, -1.0] if halves == 2 else [-1.0]
    else:
        t = [0.83, 1.02][:halves] if halves == 2 else [0.91]
    gscale = 0.7
    acc = torch.zeros(halves, dtype=torch.float64, device=dev())
    dp = torch.full((halves, count), float("nan"), device=dev())
    arg = torch.tensor(t, dtype=torch.float32, device=dev()) if device_t else t
    ops.gan_loss_fwd_bwd(ops.GAN_OBJECTIVES[mode], pred.to(dev()), halves, arg, gscale, acc, dp)
    torch.cuda.synchronize()

    x = pred.double().requires_grad_()
    refs = []
    for h in range(halves):
        th = torch.tensor(t[h], dtype=torch.float32).double()
        if mode == "wgan":
            refs.append(th * x[h].mean())
        elif mode == "lsgan":
            refs.append(F.mse_loss(x[h], th.expand_as(x[h])))
        else:
            refs.append(F.binary_cross_entropy_with_logits(x[h], th.expand_as(x[h])))
    (ref_dp,) = torch.autograd.grad(sum(refs) * gscale, x)
    err_dp = relmax(dp.cpu(), ref_dp)
    assert err_dp < 1e-6, f"dpred relmax {err_dp:.3e}"
    for h in range(halves):
        ref = refs[h].item()
        scale = max(abs(ref), pred[h].abs().mean().item())
        assert abs(acc[h].item() - ref) <= 1e-6 * scale, (h, acc[h].item(), ref)


def test_gan_loss_kernel_refuses_wgan_device_targets():
    from swapnet_b200 import ops
    from swapnet_b200._lib import SwapnetB200Error

    pred = torch.zeros(8, device=dev())
    acc = torch.zeros(1, dtype=torch.float64, device=dev())
    with pytest.raises(AssertionError):
        ops.gan_loss_fwd_bwd(ops.GAN_WGAN, pred, 1, torch.ones(1, device=dev()), 1.0, acc, None)
    with pytest.raises(SwapnetB200Error, match="unknown objective"):
        ops.gan_loss_fwd_bwd(7, pred, 1, (1.0,), 1.0, acc, None)


# ---------------------------------------------------------------------------------------------
# plugin steps against the oracle
# ---------------------------------------------------------------------------------------------
def _pred_scale(model):
    """mean |pred| of the step's D calls (the wgan loss scale)."""
    return max(model._eng_Dd.pred.abs().mean().item(), model._eng_Dg.pred.abs().mean().item())


def _check_losses(model, o, losses, keys, gan_mode, tag):
    scale = _pred_scale(model) if gan_mode == "wgan" else 0.0
    for k in keys:
        ref = o[k].item()
        assert abs(losses[k] - ref) <= 1e-3 * max(abs(ref), scale), f"loss_{k}: {losses[k]} vs {ref} (scale {scale})"
    record(f"gan_mode_step_losses{tag}", {k: f"{losses[k]:.7g} vs {o[k].item():.7g}" for k in keys})


def _run_phases(model, batch, seed):
    """The D and G phases of one step by hand, so that gradients can be read before the optimizer steps; the labels
    (if the objective has any) are drawn from the CPU generator seeded with `seed`."""
    torch.manual_seed(seed)
    state0 = torch.get_rng_state()
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
    if model.opt.gan_mode == "wgan":
        assert torch.equal(torch.get_rng_state(), state0), "a wgan step must not draw labels"
    torch.manual_seed(seed)
    draws = [torch.rand(1) for _ in range(GO.label_draws(model.opt.gan_mode))]
    return gD, gG, dict(model.get_current_losses()), draws


def _gate_fn(gates_G, gates_D, gates_P=None):
    calls = {}

    def gate(name, x):
        if name in gates_G:
            return gates_G[name]
        if gates_P and name in gates_P:
            return gates_P[name]
        k = calls.get(name, 0)
        calls[name] = k + 1
        return gates_D[k][name]

    return gate


def _warp_step(B, S, mode, gan_mode, tag):
    from swapnet_b200 import engine as E
    from swapnet_b200.models import create_model

    torch.manual_seed(0)
    model = create_model(_opt(B, S, gan_mode=gan_mode, b200_sample_base=5 if S == 512 else 0))
    model.setup(model.opt)
    if mode == "eval":
        model.eval()
    model.is_train = True
    sdG, namesG = _param_sd(model.net_generator)
    sdD, namesD = _param_sd(model.net_discriminator)
    body, inp, tgt = synth_warp_batch(B, S)
    batch = dict(bodys=body, input_cloths=inp, target_cloths=tgt, cloth_paths=["c"] * B, body_paths=["b"] * B)
    gD, gG, losses, draws = _run_phases(model, batch, 123)
    gates_D = [bn_stage_gates(model._eng_Dd, 0, B), bn_stage_gates(model._eng_Dd, B, 2 * B),
               bn_stage_gates(model._eng_Dg)]
    ON.gate_with(_gate_fn(bn_stage_gates(model._eng_G), gates_D))
    drop = None
    if mode != "eval":
        eng = model._eng_G
        drop = OD.make_drop({s.name: E._mix_seed(eng.seed, s.id) for s in eng.stages}, 0.5, sample_base=eng.sample_base)
    try:
        o = GO.warp_step_losses(sdG, sdD, body.double(), inp.double(), tgt.double(), draws, gan_mode, drop=drop)
        stats = dict(ON.GATE_STATS)
    finally:
        ON.gate_with(None)
    flips = {k: v for k, v in stats.items() if k != "__total__" and v}
    record(f"gan_mode_warp_gate_flips{tag}", f"{sum(flips.values())} of {stats.get('__total__', 1)}: {flips}")
    assert sum(flips.values()) <= 2e-5 * stats.get("__total__", 1), f"too many activation gates differ: {flips}"
    keys = ("D", "D_real", "D_fake", "G", "G_gan", "G_ce")
    _check_losses(model, o, losses, keys, gan_mode, tag)
    o["bufsG"] = {}
    _check_step(model, o, sdG, namesG, sdD, namesD, gG, gD, losses, (), {}, mode != "eval", tag)


@pytest.mark.parametrize("mode", ["eval", "train_shared_masks"])
@pytest.mark.parametrize("gan_mode", NEW_MODES)
def test_warp_step_matches_oracle(gan_mode, mode):
    """WarpModel D and G phases: all six losses and every parameter gradient of G and D against the fp64 oracle, in
    eval mode and in training with the library's dropout masks."""
    _warp_step(2, 64, mode, gan_mode, f"[warp,{gan_mode},{mode}]")


@pytest.mark.parametrize("gan_mode", NEW_MODES)
def test_warp_step_matches_oracle_512(gan_mode):
    """One image at the benchmarked 512 x 512: the loss sees 62 x 62 predictions per call."""
    _warp_step(1, 512, "eval", gan_mode, f"[warp512,{gan_mode}]")


def _texture_step(B, S, gan_mode, norm, perceptual, train, tag):
    from swapnet_b200 import engine as E
    from swapnet_b200.models import create_model

    torch.manual_seed(0)
    lc, ls = (20.0, 1e-8) if perceptual else (0.0, 0.0)
    opt = _opt(B, S, model="texture", name="texture", netG="swapnet", lambda_l1=10, lambda_content=lc,
               lambda_style=ls, b200_vgg="random", norm=norm, gan_mode=gan_mode)
    model = create_model(opt)
    model.setup(opt)
    if not train:
        model.eval()
    _randomise_affine((model.net_generator, model.net_discriminator))
    bufs0 = {p + k: b.detach().cpu().clone() for p, net in (("G.", model.net_generator), ("D.", model.net_discriminator))
             for k, b in net.named_buffers()}
    sdG, namesG = _param_sd(model.net_generator)
    sdD, namesD = _param_sd(model.net_discriminator)
    tex, rois, cloth, tgt = synth_texture_batch(B, S)
    batch = dict(input_textures=tex, rois=rois, cloths=cloth, target_textures=tgt, cloth_paths=["c"] * B,
                 texture_paths=["t"] * B)
    gD, gG, losses, draws = _run_phases(model, batch, 321)
    gates_D = [bn_stage_gates(model._eng_Dd, 0, B), bn_stage_gates(model._eng_Dd, B, 2 * B),
               bn_stage_gates(model._eng_Dg)]
    gates_P, vgg_sd = {}, None
    if perceptual:
        from test_engine_gpu import vgg_pool_winners

        gates_P = {"vgg_o." + k: v for k, v in stage_gates(model._eng_P.out).items()}
        gates_P.update({"vgg_t." + k: v for k, v in stage_gates(model._eng_P.tgt).items()})
        vgg_sd = {k: v.detach().cpu().double() for k, v in model.net_vgg.state_dict().items()}
        winners = vgg_pool_winners(model._eng_P.out, "vgg_o")
        ON.pool_with(lambda name, x: winners.get(name))
    ON.gate_with(_gate_fn(bn_stage_gates(model._eng_G), gates_D, gates_P))
    drop = None
    if train:
        eng = model._eng_G
        drop = OD.make_drop({s.name: E._mix_seed(eng.seed, s.id) for s in eng.stages}, 0.5, sample_base=eng.sample_base)
    l1_sign = torch.sign(model.fakes.detach() - tgt.to(dev())).cpu().double()
    try:
        o = GO.texture_step_losses(sdG, sdD, tex.double(), rois.double(), cloth.double(), tgt.double(), draws, gan_mode,
                                   norm, train, drop=drop, l1_sign=l1_sign, vgg=vgg_sd, lambda_content=lc,
                                   lambda_style=ls)
        stats = dict(ON.GATE_STATS)
    finally:
        ON.gate_with(None)
        ON.pool_with(None)
    flips = {k: v for k, v in stats.items() if k != "__total__" and not k.startswith("pool:") and v}
    record(f"gan_mode_texture_gate_flips{tag}", f"{sum(flips.values())} of {stats.get('__total__', 1)}: {flips}")
    assert sum(flips.values()) <= 2e-5 * stats.get("__total__", 1), f"too many activation gates differ: {flips}"
    keys = ("D", "D_real", "D_fake", "G", "G_gan", "G_l1") + (("G_content", "G_style") if perceptual else ())
    _check_losses(model, o, losses, keys, gan_mode, tag)
    _check_step(model, o, sdG, namesG, sdD, namesD, gG, gD, losses, (), bufs0, train, tag)


@pytest.mark.parametrize("perceptual", [False, True])
@pytest.mark.parametrize("gan_mode", NEW_MODES)
def test_texture_step_matches_oracle(gan_mode, perceptual):
    """TextureModel D and G phases in eval mode, with the perceptual terms off and on (seeded-random VGG16)."""
    _texture_step(2, 128, gan_mode, "instance", perceptual, False, f"[texture,{gan_mode},perceptual={perceptual}]")


def test_texture_step_lsgan_batch_norm_matches_oracle():
    """lsgan with --norm batch in training: the D step's halves normalised with their own statistics, running buffers
    updated fake, real, then by the G step's call."""
    _texture_step(2, 128, "lsgan", "batch", False, True, "[texture,lsgan,batch]")


# ---------------------------------------------------------------------------------------------
# a whole step, graph replay, the CPU generator
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gan_mode,norm", [("lsgan", "batch"), ("wgan", "instance")])
def test_full_texture_step_matches_oracle_and_adamw(gan_mode, norm):
    """One whole optimize_parameters() (D step, optimizer_D.step(), G step through the UPDATED D, optimizer_G.step())
    against the fp64 oracle driven the same way with torch.optim.AdamW: losses, running buffers and every updated
    parameter.  As in test_batchnorm_gpu, at most max(8, 1e-3 * numel) elements per tensor may differ by more than 5 %
    of lr (AdamW's first update is ~lr * sign(g)).  Parameters whose exact gradient is zero (the biases in front of an
    InstanceNorm) are held to the bound of one AdamW step instead."""
    from swapnet_b200 import engine as E
    from swapnet_b200.models import create_model

    B, S = 2, 64
    torch.manual_seed(0)
    model = create_model(_opt(B, S, model="texture", name="texture", netG="swapnet", lambda_l1=10, lambda_content=0,
                              lambda_style=0, norm=norm, gan_mode=gan_mode))
    model.setup(model.opt)
    _randomise_affine((model.net_generator, model.net_discriminator))
    nets = (("G.", model.net_generator), ("D.", model.net_discriminator))
    before = {p + k: v.detach().cpu().clone() for p, net in nets for k, v in net.state_dict().items()}

    def affine(net, pre):
        return {id(m): (before[pre + n + ".weight"], before[pre + n + ".bias"]) for n, m in net.named_modules()
                if isinstance(m, torch.nn.BatchNorm2d)}

    tex, rois, cloth, tgt = synth_texture_batch(B, S)
    batch = dict(input_textures=tex, rois=rois, cloths=cloth, target_textures=tgt, cloth_paths=["c"] * B,
                 texture_paths=["t"] * B)
    torch.manual_seed(321)
    model.set_input(batch)
    model.optimize_parameters()
    torch.cuda.synchronize()
    losses = model.get_current_losses()
    scale = _pred_scale(model) if gan_mode == "wgan" else 0.0
    affD = affine(model.net_discriminator, "D.")
    gates_D = [bn_stage_gates(model._eng_Dd, 0, B, affD), bn_stage_gates(model._eng_Dd, B, 2 * B, affD),
               bn_stage_gates(model._eng_Dg)]      # the G step's call: D's weights after optimizer_D.step()
    gate = _gate_fn(bn_stage_gates(model._eng_G, affine=affine(model.net_generator, "G.")), gates_D)
    eng = model._eng_G
    drop = OD.make_drop({s.name: E._mix_seed(eng.seed, s.id) for s in eng.stages}, 0.5, sample_base=eng.sample_base)
    l1_sign = torch.sign(model.fakes.detach() - tgt.to(dev())).cpu().double()
    sd, params = {}, {}
    for pre, net in nets:
        names = [k for k, _ in net.named_parameters()]
        sd[pre] = {k: before[pre + k].double() for k, _ in net.state_dict().items()}
        for k in names:
            sd[pre][k].requires_grad_()
        params[pre] = names
    bnG, bnD = NO.BN(sd["G."], norm, True), NO.BN(sd["D."], norm, True)
    optG = torch.optim.AdamW([sd["G."][k] for k in params["G."]], lr=1e-4, weight_decay=0, betas=(0.9, 0.999), eps=1e-8)
    optD = torch.optim.AdamW([sd["D."][k] for k in params["D."]], lr=4e-4, weight_decay=0.01, betas=(0.9, 0.999),
                             eps=1e-8)
    torch.manual_seed(321)
    draws = [torch.rand(1) for _ in range(GO.label_draws(gan_mode))] or [None] * 3
    ON.gate_with(gate)
    try:
        fk = NO.texture_forward(sd["G."], tex.double(), rois.double(), cloth.double(), bnG, drop)
        c64, tgt64 = cloth.double(), tgt.double()
        lf = GO.gan_loss(NO.patchgan_forward(sd["D."], torch.cat((c64, fk), 1).detach(), bnD), False, gan_mode, draws[0])
        lr = GO.gan_loss(NO.patchgan_forward(sd["D."], torch.cat((c64, tgt64), 1), bnD), True, gan_mode, draws[1])
        lD = 0.5 * (lf + lr)
        lD.backward()
        grads = {"D.": {k: sd["D."][k].grad.clone() for k in params["D."]}}
        optD.step()
        gan = GO.gan_loss(NO.patchgan_forward(sd["D."], torch.cat((c64, fk), 1), bnD), True, gan_mode, draws[2])
        l1 = ((fk - tgt64) * l1_sign).mean() * 10
        (gan + l1).backward()
        grads["G."] = {k: sd["G."][k].grad for k in params["G."]}
        optG.step()
        stats = dict(ON.GATE_STATS)
    finally:
        ON.gate_with(None)
    flips = {k: v for k, v in stats.items() if k != "__total__" and v}
    assert sum(flips.values()) <= 2e-5 * stats.get("__total__", 1), f"too many activation gates differ: {flips}"
    ref = dict(D=lD.item(), D_real=lr.item(), D_fake=lf.item(), G=(gan + l1).item(), G_gan=gan.item(), G_l1=l1.item())
    for k, v in ref.items():
        assert abs(losses[k] - v) <= 1e-3 * max(abs(v), scale), (k, losses[k], v, scale)
    moved, zero_grad = {}, []
    for (pre, net), bn, lr_ in zip(nets, (bnG, bnD), (1e-4, 4e-4)):
        gmax = max(g.abs().max().item() for g in grads[pre].values() if g is not None)
        for k, v in net.state_dict().items():
            g = grads[pre].get(k, 0)
            if k in grads[pre] and (g is None or g.abs().max().item() < 1e-6 * gmax):
                # a bias in front of an InstanceNorm: the exact gradient is zero and AdamW's first step turns the
                # rounding noise of either side into +-lr moves, so only the bound of a single step is checked
                zero_grad.append(pre + k)
                assert (v.detach().cpu().double() - sd[pre][k].detach()).abs().max().item() <= 2.01 * lr_, k
                continue
            got = v.detach().cpu()
            if k.endswith("num_batches_tracked"):
                assert int(got) == int(bn.bufs[k]) == int(before[pre + k]) + (1 if pre == "G." else 3), k
            elif k.endswith(("running_mean", "running_var")):
                assert relmax(got, bn.bufs[k]) < 1e-3, k
            else:
                far = int(((got.double() - sd[pre][k].detach()).abs() > 0.05 * lr_).sum())
                moved[pre + k] = far
                assert far <= max(8, 1e-3 * got.numel()), (k, far, got.numel())
    record(f"gan_mode_full_step_params_off_by_more_than_5pct_lr[{gan_mode},{norm}]", {k: v for k, v in moved.items() if v})
    record(f"gan_mode_full_step_zero_gradient_params[{gan_mode},{norm}]", zero_grad)


@pytest.mark.parametrize("gan_mode", NEW_MODES)
def test_graph_replayed_steps_match_eager_steps(gan_mode):
    """Five warp steps with graph replay (steps 3-5 replay one captured graph) equal five eager steps of an identically
    seeded model: the objective and its per-half scalars (device labels for lsgan, constant signs for wgan) are part of
    the captured launch sequence.  The learning rates are 0, so both runs evaluate the same weights and only the
    summation order of atomics separates them (AdamW's sign-like first steps would turn that into lr-sized weight
    differences; test_engine_gpu covers the replayed weight updates).  Each step draws new dropout masks and, with
    lsgan, new labels: D_real changes from step to step with lsgan only."""
    from swapnet_b200 import ops
    from swapnet_b200.models import create_model

    B, S = 2, 64
    body, inp, tgt = synth_warp_batch(B, S)
    batch = dict(bodys=body, input_cloths=inp, target_cloths=tgt, cloth_paths=["c"] * B, body_paths=["b"] * B)
    runs = {}
    for graph in (1, 0):
        torch.manual_seed(0)
        model = create_model(_opt(B, S, b200_graph=graph, gan_mode=gan_mode, lr=0.0, d_lr=0.0))
        model.setup(model.opt)
        torch.manual_seed(99)
        hist, launches, scales = [], [], []
        for _ in range(5):
            n0 = ops.launch_count()
            model.set_input(batch)
            model.optimize_parameters()
            hist.append(dict(model.get_current_losses()))
            launches.append(ops.launch_count() - n0)
            scales.append(_pred_scale(model) if gan_mode == "wgan" else 0.0)
        assert (len(model._graphs) == 1) == bool(graph)
        runs[graph] = (hist, launches, scales)
    (hg, lg, sg), (he, le, se) = runs[1], runs[0]
    assert lg == le, (lg, le)
    worst = 0.0
    for a, b, sc in zip(hg, he, se):
        for k in a:
            err = abs(a[k] - b[k]) / max(abs(b[k]), sc)
            worst = max(worst, err)
            assert err <= 1e-5, (k, a[k], b[k], sc)
    assert hg[3]["G_ce"] != hg[4]["G_ce"] and hg[3]["D_fake"] != hg[4]["D_fake"]
    real_moves = abs(hg[3]["D_real"] - hg[4]["D_real"]) > 1e-4 * abs(hg[4]["D_real"])
    assert real_moves == (gan_mode == "lsgan"), [h["D_real"] for h in hg]
    record(f"gan_mode_graph_vs_eager[{gan_mode}]", f"worst loss difference {worst:.2e}")


@pytest.mark.parametrize("gan_mode", GO.MODES)
def test_step_leaves_cpu_generator_where_the_reference_does(gan_mode):
    """torch.get_rng_state() after optimize_parameters(): unchanged by a wgan step, three rand(1) draws further after a
    vanilla or lsgan step (GANLoss draws one smooth label per call from the CPU default generator)."""
    from swapnet_b200.models import create_model

    B, S = 2, 64
    body, inp, tgt = synth_warp_batch(B, S)
    batch = dict(bodys=body, input_cloths=inp, target_cloths=tgt, cloth_paths=["c"] * B, body_paths=["b"] * B)
    torch.manual_seed(0)
    model = create_model(_opt(B, S, gan_mode=gan_mode))
    model.setup(model.opt)
    for step in range(3):            # eager, eager, then the captured graph
        torch.manual_seed(5 + step)
        model.set_input(batch)
        model.optimize_parameters()
        after = torch.get_rng_state()
        torch.manual_seed(5 + step)
        for _ in range(GO.label_draws(gan_mode)):
            torch.rand(1)
        assert torch.equal(after, torch.get_rng_state()), (gan_mode, step)
    assert model._graphs and GO.label_draws(gan_mode) == (0 if gan_mode == "wgan" else 3)


@pytest.mark.parametrize("gan_mode,why", [("wgan-gp", "second derivative"), ("dragan-gp", "second derivative"),
                                          ("dragan-lp", "second derivative"), ("mescheder-r1-gp", "GANLoss"),
                                          ("mescheder-r2-gp", "GANLoss")])
def test_unsupported_gan_modes_are_refused(gan_mode, why):
    from swapnet_b200.models import create_model

    for model in ("warp", "texture"):
        with pytest.raises(NotImplementedError, match=why):
            create_model(_opt(2, 64, model=model, name=model, netG="swapnet", lambda_l1=10, lambda_content=0,
                              lambda_style=0, gan_mode=gan_mode))


# ---------------------------------------------------------------------------------------------
# data parallelism
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gan_mode", NEW_MODES)
def test_two_rank_cuda_gradients_equal_full_batch(gan_mode):
    """tests/tools/dp_equiv.py (training mode, 256 x 256, 2 images per rank) with the objective set on both models."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    env = dict(os.environ, SN_DP_MODE="train", SN_DP_SIZE="256", SN_DP_PER_RANK="2", SN_DP_GAN_MODE=gan_mode)
    port = 29600 + (os.getpid() + 7) % 300
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.join(HERE, "tools", "dp_equiv_gan_modes.py")]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("DP_EQUIV")]
    record(f"dp2_cuda_equivalence[{gan_mode}]", line[-1] if line else f"rc={r.returncode}")
    assert r.returncode == 0 and line and " OK " in line[-1], (r.stdout[-2000:], r.stderr[-3000:])
