"""GPU parity of `--norm batch` / `--norm none` (texture U-Net and PatchGAN): the BatchNorm kernels against fp64
F.batch_norm, and plugin steps against the norm-aware fp64 oracle (tests/tools/norm_oracle.py, built on oracle/nets.py)
at the 1e-3 bar of tests/test_engine_gpu.py."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "tools"))

from oracle import dropout as OD  # noqa: E402
from oracle import nets as ON  # noqa: E402
import norm_oracle as NO  # noqa: E402
from test_engine_gpu import _opt, record, relmax, synth_texture_batch, synth_warp_batch  # noqa: E402


def dev():
    return torch.device("cuda:0")


# ---------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("n,h,c,groups", [(2, 8, 64, 1), (4, 63, 64, 2), (1, 2, 512, 1), (4, 4, 512, 2),
                                          (2, 63, 256, 2), (2, 8, 19, 1), (2, 3, 3100, 2), (2, 3, 3102, 2)])
def test_bn_kernels_match_batch_norm(n, h, c, groups, train):
    """sn_plane_sums + sn_bn_finalize (or sn_bn_eval_stats), the affine norm/activation forward and its backward
    against fp64 F.batch_norm per sample group: output, dL/dy, d gamma, d beta, running buffers, the batch counter.
    c = 19 takes the one-channel (V = 1) instantiations; c = 3100 (V = 4) and c = 3102 (V = 1) two channel slices of the
    forward (3072 per block) and of the apply pass (2048)."""
    from swapnet_b200 import ops

    g = torch.Generator().manual_seed(n * 1000 + h * 10 + c + groups)
    y = (torch.randn(n, h, h, c, generator=g) * 1.7 + 0.3).to(dev())
    up = torch.randn(n, h, h, c, generator=g).to(dev())
    bn = torch.nn.BatchNorm2d(c).to(dev())
    with torch.no_grad():
        bn.weight.copy_(1.0 + 0.3 * torch.randn(c, generator=g))
        bn.bias.copy_(0.2 * torch.randn(c, generator=g))
        bn.running_mean.copy_(0.1 * torch.randn(c, generator=g))
        bn.running_var.copy_(1.0 + 0.5 * torch.rand(c, generator=g))
    rm0, rv0 = bn.running_mean.double().cpu(), bn.running_var.double().cpu()
    stats = torch.zeros(n, c, 2, dtype=torch.float64, device=dev())
    if train:
        ops.plane_sums(y, c, stats)
        ops.bn_finalize(stats, n, c, groups, h * h, bn)
    else:
        ops.bn_eval_stats(stats, n, c, bn)
    out = torch.zeros(n, h, h, c, device=dev())
    ops.norm_act_fwd(y, c, stats, ops.ACT_LRELU, 0.2, out_f32=out, gamma=bn.weight.data, beta=bn.bias.data)
    dy = ops.Planes(n, h, h, (c + 7) // 8 * 8, dev(), c=c, fmt=ops.FMT_BF16)
    gst = torch.zeros(n, c, 2, dtype=torch.float64, device=dev())
    dgam, dbet = torch.zeros(c, device=dev()), torch.zeros(c, device=dev())
    ops.norm_act_bwd([ops.GradSrc(up)], y, c, stats, ops.ACT_LRELU, dy, gst, 0.2, bn=(bn.weight.data, bn.bias.data),
                     bn_groups=groups, bn_train=train, bn_grads=(dgam, dbet))
    torch.cuda.synchronize()

    y64 = y.cpu().double().permute(0, 3, 1, 2).requires_grad_()
    w64 = bn.weight.detach().cpu().double().requires_grad_()
    b64 = bn.bias.detach().cpu().double().requires_grad_()
    rm, rv = rm0.clone(), rv0.clone()
    if train:
        z = torch.cat([F.batch_norm(yg, rm, rv, w64, b64, True, 0.1, 1e-5) for yg in y64.chunk(groups, 0)], 0)
    else:
        z = F.batch_norm(y64, rm, rv, w64, b64, False, 0.1, 1e-5)
    gate = (out > 0).cpu().permute(0, 3, 1, 2)           # the device's gates (fp32 rounding near z = 0)
    ref = torch.where(gate, z, 0.2 * z)
    (ref * up.cpu().double().permute(0, 3, 1, 2)).sum().backward()
    flips = int((gate != (z > 0)).sum())
    assert flips <= max(2, 1e-4 * z.numel()), flips
    assert relmax(out.cpu().permute(0, 3, 1, 2), ref.detach()) < 1e-5
    assert relmax(dy.dense()[..., :c].cpu().permute(0, 3, 1, 2), y64.grad) < 1e-3
    assert relmax(dgam.cpu(), w64.grad) < 1e-4
    assert relmax(dbet.cpu(), b64.grad) < 1e-4
    if train:
        assert relmax(bn.running_mean.cpu(), rm) < 1e-5 and relmax(bn.running_var.cpu(), rv) < 1e-5
        assert int(bn.num_batches_tracked) == groups
    else:
        assert torch.equal(bn.running_mean.cpu().double(), rm0) and torch.equal(bn.running_var.cpu().double(), rv0)
        assert int(bn.num_batches_tracked) == 0


# ---------------------------------------------------------------------------------------------
# plugin steps against the oracle
# ---------------------------------------------------------------------------------------------
def bn_stage_gates(eng, n0=0, n1=None, affine=None):
    """name -> bool NCHW gate mask (CPU) the device used: the normalised value (gamma * xhat + beta with batch norm,
    xhat with InstanceNorm, y without norm) > 0.  affine: id(BatchNorm2d) -> (gamma, beta) the call used, when the
    module's weights have been updated since."""
    out = {}
    for st in eng.stages:
        if st.plain or st.act == 0:
            continue
        y = st.y[n0:n1].double()
        if st.stats is not None:
            z = (y - st.stats[n0:n1, None, None, :, 0]) * st.stats[n0:n1, None, None, :, 1]
            if st.bn is not None:
                w, b = (st.bn.weight, st.bn.bias) if affine is None else affine[id(st.bn)]
                z = z * w.to(z.device).double() + b.to(z.device).double()
            m = z > 0
        else:
            m = y > 0
        out[st.name] = m.permute(0, 3, 1, 2).contiguous().cpu()
    return out


def _param_sd(net):
    names = {k for k, _ in net.named_parameters()}
    sd = {k: v.detach().cpu().double() for k, v in net.state_dict().items()}
    return {k: (v.requires_grad_() if k in names else v) for k, v in sd.items()}, names


def _randomise_affine(nets):
    g = torch.Generator().manual_seed(9)
    for net in nets:
        for n, p in net.named_parameters():
            if n.endswith("bias"):
                p.data.copy_((torch.randn(p.shape, generator=g) * 0.1).to(p.device))
        for n, b in net.named_buffers():
            if n.endswith("running_mean"):
                b.copy_((torch.randn(b.shape, generator=g) * 0.1).to(b.device))
            elif n.endswith("running_var"):
                b.copy_((1.0 + 0.5 * torch.rand(b.shape, generator=g)).to(b.device))


def _check_step(model, o, sdG, namesG, sdD, namesD, gG, gD, losses, loss_keys, bufs0, train, tag):
    for k in loss_keys:
        ref = o[k].item()
        assert abs(losses[k] - ref) <= 1e-3 * abs(ref), f"loss_{k}: {losses[k]} vs {ref}"
    err_f = relmax(model.fakes.cpu(), o["fakes"].detach())
    assert err_f < 1e-3, f"fakes relmax {err_f:.3e}"
    worst = {}
    for pre, got, sd, names, loss in (("D.", gD, sdD, namesD, o["D"]), ("G.", gG, sdG, namesG, o["G"])):
        keys = [k for k in sd if k in names]
        refs = torch.autograd.grad(loss, [sd[k] for k in keys], retain_graph=True, allow_unused=True)
        mx = max(r.abs().max().item() for r in refs if r is not None)
        for k, r in zip(keys, refs):
            if r is None:
                continue
            if r.abs().max().item() < 1e-6 * mx:
                assert got[k].abs().max().item() < 1e-4 * mx, k
                continue
            worst[pre + k] = relmax(got[k], r)
    record(f"bn_step_worst_grads{tag}", sorted(worst.items(), key=lambda kv: -kv[1])[:5])
    bad = {k: v for k, v in worst.items() if v >= 1e-3}
    assert not bad, f"parameter gradients beyond 1e-3: {bad}"
    # running buffers and counters: D is called three times per train step (fake, real, G step), G once
    for pre, net, ref_bufs, calls in (("G.", model.net_generator, o.get("bufsG", {}), 1),
                                      ("D.", model.net_discriminator, o["bufsD"], 3)):
        for k, b in net.state_dict().items():
            if k.endswith("num_batches_tracked"):
                assert int(b) == int(bufs0[pre + k]) + (calls if train else 0), k
                assert int(b) == int(ref_bufs[k]), k
            elif k.endswith(("running_mean", "running_var")):
                assert relmax(b.cpu(), ref_bufs[k]) < 1e-3, k


def _texture_step(B, S, norm, perceptual, train, tag=""):
    from swapnet_b200 import engine as E
    from swapnet_b200.models import create_model

    torch.manual_seed(0)
    lc, ls = (20.0, 1e-8) if perceptual else (0.0, 0.0)
    opt = _opt(B, S, model="texture", name="texture", netG="swapnet", lambda_l1=10, lambda_content=lc,
               lambda_style=ls, b200_vgg="random", norm=norm)
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
    gates_G = bn_stage_gates(model._eng_G)
    gates_D = [bn_stage_gates(model._eng_Dd, 0, B), bn_stage_gates(model._eng_Dd, B, 2 * B),
               bn_stage_gates(model._eng_Dg)]
    gates_P, vgg_sd = {}, None
    if perceptual:
        from test_engine_gpu import stage_gates, vgg_pool_winners

        gates_P = {"vgg_o." + k: v for k, v in stage_gates(model._eng_P.out).items()}
        gates_P.update({"vgg_t." + k: v for k, v in stage_gates(model._eng_P.tgt).items()})
        vgg_sd = {k: v.detach().cpu().double() for k, v in model.net_vgg.state_dict().items()}
        winners = vgg_pool_winners(model._eng_P.out, "vgg_o")
        ON.pool_with(lambda name, x: winners.get(name))
    calls = {}

    def gate(name, x):
        if name in gates_G:
            return gates_G[name]
        if name in gates_P:
            return gates_P[name]
        k = calls.get(name, 0)
        calls[name] = k + 1
        return gates_D[k][name]

    ON.gate_with(gate)
    drop = None
    if train:
        eng = model._eng_G
        drop = OD.make_drop({s.name: E._mix_seed(eng.seed, s.id) for s in eng.stages}, 0.5, sample_base=eng.sample_base)
    l1_sign = torch.sign(model.fakes.detach() - tgt.to(dev())).cpu().double()
    try:
        o = NO.texture_step_losses(sdG, sdD, tex.double(), rois.double(), cloth.double(), tgt.double(), draws, norm,
                                   train, drop=drop, l1_sign=l1_sign, vgg=vgg_sd, lambda_content=lc, lambda_style=ls)
        stats = dict(ON.GATE_STATS)
    finally:
        ON.gate_with(None)
        ON.pool_with(None)
    flips = {k: v for k, v in stats.items() if k != "__total__" and not k.startswith("pool:") and v}
    record(f"bn_texture_gate_flips{tag}", f"{sum(flips.values())} of {stats.get('__total__', 1)}: {flips}")
    assert sum(flips.values()) <= 2e-5 * stats.get("__total__", 1), f"too many activation gates differ: {flips}"
    keys = ("D", "D_real", "D_fake", "G", "G_gan", "G_l1") + (("G_content", "G_style") if perceptual else ())
    _check_step(model, o, sdG, namesG, sdD, namesD, gG, gD, losses, keys, bufs0, train, tag)


@pytest.mark.parametrize("norm,perceptual,train", [("batch", False, True), ("batch", True, True),
                                                   ("batch", False, False), ("none", False, True)])
def test_texture_step_with_norm_matches_oracle(norm, perceptual, train):
    _texture_step(2, 128, norm, perceptual, train, tag=f"[{norm},perceptual={perceptual},train={train}]")


def test_texture_step_batch_norm_512_matches_oracle():
    """One image at 512 x 512: the U-Net's innermost batch norm sees 2 x 2 planes of a single sample."""
    _texture_step(1, 512, "batch", True, True, tag="[512]")


@pytest.mark.parametrize("train", [True, False])
def test_warp_step_with_batch_norm_discriminator_matches_oracle(train):
    from swapnet_b200 import engine as E
    from swapnet_b200.models import create_model

    B, S = 2, 64
    torch.manual_seed(0)
    model = create_model(_opt(B, S, norm="batch"))
    model.setup(model.opt)
    if not train:
        model.eval()
    _randomise_affine((model.net_discriminator,))
    bufs0 = {"D." + k: b.detach().cpu().clone() for k, b in model.net_discriminator.named_buffers()}
    sdG, namesG = _param_sd(model.net_generator)
    sdD, namesD = _param_sd(model.net_discriminator)
    body, inp, tgt = synth_warp_batch(B, S)
    batch = dict(bodys=body, input_cloths=inp, target_cloths=tgt, cloth_paths=["c"] * B, body_paths=["b"] * B)
    torch.manual_seed(123)
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

    torch.manual_seed(123)
    draws = [torch.rand(1) for _ in range(3)]
    gates_G = bn_stage_gates(model._eng_G)
    gates_D = [bn_stage_gates(model._eng_Dd, 0, B), bn_stage_gates(model._eng_Dd, B, 2 * B),
               bn_stage_gates(model._eng_Dg)]
    calls = {}

    def gate(name, x):
        if name in gates_G:
            return gates_G[name]
        k = calls.get(name, 0)
        calls[name] = k + 1
        return gates_D[k][name]

    ON.gate_with(gate)
    drop = None
    if train:
        eng = model._eng_G
        drop = OD.make_drop({s.name: E._mix_seed(eng.seed, s.id) for s in eng.stages}, 0.5, sample_base=eng.sample_base)
    try:
        o = NO.warp_step_losses(sdG, sdD, body.double(), inp.double(), tgt.double(), draws, "batch", train, drop=drop)
        stats = dict(ON.GATE_STATS)
    finally:
        ON.gate_with(None)
    flips = {k: v for k, v in stats.items() if k != "__total__" and v}
    assert sum(flips.values()) <= 2e-5 * stats.get("__total__", 1), f"too many activation gates differ: {flips}"
    o["bufsG"] = {}
    _check_step(model, o, sdG, namesG, sdD, namesD, gG, gD, losses, ("D", "D_real", "D_fake", "G", "G_gan", "G_ce"),
                {**bufs0, **{"G." + k: v for k, v in model.net_generator.state_dict().items()}}, train,
                f"[warp,train={train}]")


# ---------------------------------------------------------------------------------------------
# graph replay, checkpoints, data parallelism
# ---------------------------------------------------------------------------------------------
def test_graph_replayed_batch_norm_steps_match_eager_steps():
    """Three texture steps with --norm batch: the third is a captured CUDA graph replay.  Losses and every running
    buffer track three eager steps of an identically seeded model.  The learning rates are 0 so that the running
    statistics see the same weights in both runs (AdamW's sign-like first steps turn last-bit gradient differences of
    the weight-gradient atomics into lr-sized weight differences); test_engine_gpu covers the replayed weight updates."""
    from swapnet_b200.models import create_model

    B, S = 2, 64
    tex, rois, cloth, tgt = synth_texture_batch(B, S)
    batch = dict(input_textures=tex, rois=rois, cloths=cloth, target_textures=tgt, cloth_paths=["c"] * B,
                 texture_paths=["t"] * B)
    runs = {}
    for graph in (1, 0):
        torch.manual_seed(0)
        model = create_model(_opt(B, S, model="texture", name="texture", netG="swapnet", lambda_l1=10,
                                  lambda_content=0, lambda_style=0, norm="batch", b200_graph=graph, lr=0.0,
                                  d_lr=0.0))
        model.setup(model.opt)
        torch.manual_seed(99)
        hist = []
        for _ in range(3):
            model.set_input(batch)
            model.optimize_parameters()
            hist.append(dict(model.get_current_losses()))
        assert (len(model._graphs) == 1) == bool(graph)
        bufs = {p + k: b.detach().cpu().clone() for p, net in (("G.", model.net_generator),
                                                               ("D.", model.net_discriminator))
                for k, b in net.named_buffers()}
        runs[graph] = (hist, bufs)
    (hg, bg), (he, be) = runs[1], runs[0]
    for a, b in zip(hg, he):
        for k in a:
            assert abs(a[k] - b[k]) <= 2e-3 * abs(b[k]), (k, a[k], b[k])
    for k in be:
        if k.endswith("num_batches_tracked"):
            assert int(bg[k]) == int(be[k]) == (9 if k.startswith("D.") else 3), k
        else:
            assert relmax(bg[k], be[k]) < 1e-5, k


def test_batch_norm_checkpoint_round_trip_to_inference_model():
    """save_checkpoint -> a fresh is_train=False model (norm from the saved options, as inference.py restores them from
    args.json) -> load_checkpoint_dir -> eval() -> test(): the output is the oracle's eval forward on the saved running
    statistics, and the saved keys are the reference's."""
    from swapnet_b200.models import create_model

    B, S = 2, 64
    torch.manual_seed(0)
    opt = _opt(B, S, model="texture", name="texture", netG="swapnet", lambda_l1=10, lambda_content=0, lambda_style=0,
               norm="batch")
    model = create_model(opt)
    model.setup(opt)
    tex, rois, cloth, tgt = synth_texture_batch(B, S)
    batch = dict(input_textures=tex, rois=rois, cloths=cloth, target_textures=tgt, cloth_paths=["c"] * B,
                 texture_paths=["t"] * B)
    for _ in range(2):
        model.set_input(batch)
        model.optimize_parameters()
    model.save_checkpoint("latest")
    saved = torch.load(os.path.join(model.save_dir, "latest_net_generator.pth"))
    # the reference's TextureModule(norm_type='batch', img_size=64) key list (tests/tools/make_golden_batchnorm.py)
    gold = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "batchnorm_64.pt"))
    assert [(k, tuple(v.shape)) for k, v in saved.items()] == gold["batch"]["tex_keys"]
    assert any(k.endswith("running_var") for k in saved) and any(k.endswith("num_batches_tracked") for k in saved)

    iopt = _opt(1, S, model="texture", name="texture", is_train=False, norm="batch", load_epoch="latest",
                checkpoints_dir=opt.checkpoints_dir)
    inf = create_model(iopt)
    inf.setup(iopt)                       # is_train=False: loads the generator checkpoint
    inf.eval()
    inf.compute_visuals = lambda: None    # visuals need the reference's helpers
    inf.set_input(dict(input_textures=tex[:1], rois=rois[:1], cloths=cloth[:1], target_textures=tgt[:1],
                       cloth_paths=["c"], texture_paths=["t"]))
    inf.test()
    torch.cuda.synchronize()
    sd = {k: v.double() for k, v in saved.items()}
    with torch.no_grad():
        ref = NO.texture_forward(sd, tex[:1].double(), rois[:1].double(), cloth[:1].double(), NO.BN(sd, "batch", False))
    err = relmax(inf.fakes.cpu(), ref)
    record("bn_checkpoint_eval_forward", f"{err:.3e}")
    assert err < 1e-3, err


def test_batch_norm_under_data_parallelism_is_refused(monkeypatch):
    from swapnet_b200 import parallel
    from swapnet_b200.models import create_model

    monkeypatch.setattr(parallel, "world_size", lambda: 2)
    with pytest.raises(NotImplementedError, match="cross-rank batch statistics"):
        create_model(_opt(2, 64, model="texture", name="texture", netG="swapnet", lambda_l1=10, lambda_content=0,
                          lambda_style=0, norm="batch"))


def test_full_texture_step_with_batch_norm_matches_oracle_and_adamw():
    """One whole optimize_parameters() with --norm batch (D step, optimizer_D.step(), G step through the UPDATED D,
    optimizer_G.step()) against the fp64 oracle driven the same way with torch.optim.AdamW: losses, running buffers
    after the G forward and the three D calls, num_batches_tracked, and every updated parameter including the BN
    gamma / beta and the discriminator's weight decay.  AdamW's first update is ~lr * sign(g), so an element whose
    gradient is within rounding of zero may move the other way: at most max(8, 1e-3 * numel) elements per tensor may
    differ by more than 5 % of lr."""
    from swapnet_b200 import engine as E
    from swapnet_b200.models import create_model

    B, S = 2, 64
    torch.manual_seed(0)
    model = create_model(_opt(B, S, model="texture", name="texture", netG="swapnet", lambda_l1=10, lambda_content=0,
                              lambda_style=0, norm="batch"))
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
    gates_G = bn_stage_gates(model._eng_G, affine=affine(model.net_generator, "G."))
    affD = affine(model.net_discriminator, "D.")
    gates_D = [bn_stage_gates(model._eng_Dd, 0, B, affD), bn_stage_gates(model._eng_Dd, B, 2 * B, affD),
               bn_stage_gates(model._eng_Dg)]      # the G step's call: D's weights after optimizer_D.step()
    calls = {}

    def gate(name, x):
        if name in gates_G:
            return gates_G[name]
        k = calls.get(name, 0)
        calls[name] = k + 1
        return gates_D[k][name]

    eng = model._eng_G
    drop = OD.make_drop({s.name: E._mix_seed(eng.seed, s.id) for s in eng.stages}, 0.5, sample_base=eng.sample_base)
    l1_sign = torch.sign(model.fakes.detach() - tgt.to(dev())).cpu().double()
    sd = {}
    params = {}
    for pre, net in nets:
        names = [k for k, _ in net.named_parameters()]
        sd[pre] = {k: before[pre + k].double() for k, _ in net.state_dict().items()}
        for k in names:
            sd[pre][k].requires_grad_()
        params[pre] = names
    bnG, bnD = NO.BN(sd["G."], "batch", True), NO.BN(sd["D."], "batch", True)
    optG = torch.optim.AdamW([sd["G."][k] for k in params["G."]], lr=1e-4, weight_decay=0, betas=(0.9, 0.999), eps=1e-8)
    optD = torch.optim.AdamW([sd["D."][k] for k in params["D."]], lr=4e-4, weight_decay=0.01, betas=(0.9, 0.999),
                             eps=1e-8)
    torch.manual_seed(321)
    t = [ON.smooth_label(torch.rand(1)) for _ in range(3)]
    ON.gate_with(gate)
    try:
        fk = NO.texture_forward(sd["G."], tex.double(), rois.double(), cloth.double(), bnG, drop)
        c64, tgt64 = cloth.double(), tgt.double()
        lf = ON.gan_loss(NO.patchgan_forward(sd["D."], torch.cat((c64, fk), 1).detach(), bnD), t[0])
        lr = ON.gan_loss(NO.patchgan_forward(sd["D."], torch.cat((c64, tgt64), 1), bnD), t[1])
        lD = 0.5 * (lf + lr)
        lD.backward()
        optD.step()
        gan = ON.gan_loss(NO.patchgan_forward(sd["D."], torch.cat((c64, fk), 1), bnD), t[2])
        l1 = ((fk - tgt64) * l1_sign).mean() * 10
        (gan + l1).backward()
        optG.step()
        stats = dict(ON.GATE_STATS)
    finally:
        ON.gate_with(None)
    flips = {k: v for k, v in stats.items() if k != "__total__" and v}
    assert sum(flips.values()) <= 2e-5 * stats.get("__total__", 1), f"too many activation gates differ: {flips}"
    ref = dict(D=lD.item(), D_real=lr.item(), D_fake=lf.item(), G=(gan + l1).item(), G_gan=gan.item(), G_l1=l1.item())
    for k, v in ref.items():
        assert abs(losses[k] - v) <= 1e-3 * abs(v), (k, losses[k], v)
    moved = {}
    for (pre, net), bn, lr_ in zip(nets, (bnG, bnD), (1e-4, 4e-4)):
        for k, v in net.state_dict().items():
            got = v.detach().cpu()
            if k.endswith("num_batches_tracked"):
                assert int(got) == int(bn.bufs[k]) == int(before[pre + k]) + (1 if pre == "G." else 3), k
            elif k.endswith(("running_mean", "running_var")):
                assert relmax(got, bn.bufs[k]) < 1e-3, k
            else:
                far = int(((got.double() - sd[pre][k].detach()).abs() > 0.05 * lr_).sum())
                moved[pre + k] = far
                assert far <= max(8, 1e-3 * got.numel()), (k, far, got.numel())
    record("bn_full_step_params_off_by_more_than_5pct_lr", {k: v for k, v in moved.items() if v})
