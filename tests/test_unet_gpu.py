"""GPU parity of the standalone U-Net models: `--model pix2pix` and `--model texture --netG unet_128`.

* ops.pack_concat with a leading run of zero channels, bit-equal to packing torch.cat((zeros, *sources), 1);
* engine.UnetEngine forward and backward against the fp64 oracle (tests/tools/unet_oracle.py) for every norm;
* plugin steps (D phase, G phase) against the oracle: every loss and every parameter gradient at the 1e-3 bar of
  tests/test_batchnorm_gpu.py, with the device's activation gates imposed on the oracle (at most 2e-5 of them may
  differ), and the optimizers against torch.optim.Adam;
* graph replay, checkpoints and the 2-rank sync-BN equivalence.
"""
import os
import socket
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "tools"))

from oracle import dropout as OD  # noqa: E402
from oracle import nets as ON  # noqa: E402
import unet_oracle as UO  # noqa: E402
from test_batchnorm_gpu import _check_step, _param_sd, _randomise_affine, bn_stage_gates  # noqa: E402
from test_engine_gpu import _opt, record, relmax, synth_texture_batch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def dev():
    return torch.device("cuda:0")


# ---------------------------------------------------------------------------------------------
# pack_concat with a zero lead
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c_fill,lead,kinds", [(16, 5, ("nchw",)), (16, 3, ("nhwc", "nchw")), (32, 7, ("seg",)),
                                               (32, 1, ("nchw", "nhwc")), (64, 36, ("seg",)),
                                               (64, 36, ("seg", "nhwc")), (64, 36, ("nchw", "nchw")),
                                               (64, 40, ("nhwc",))])
@pytest.mark.parametrize("h,w", [(3, 37), (2, 200)])
def test_pack_concat_zero_lead_equals_cat(c_fill, lead, kinds, h, w):
    """Both kernels (thread-per-pixel for c_fill 16/32, shared-memory tile for 64), every source kind, widths that do
    not divide the pixel run; the fp16 planes and the bf16 twin bit-equal to packing the dense concatenation."""
    from swapnet_b200 import ops

    n = 2
    g = torch.Generator().manual_seed(c_fill * 100 + lead + h)
    chans = {"nchw": 3, "nhwc": 3, "seg": 19}
    srcs, dense = [], [torch.zeros(n, lead, h, w)]
    for k in kinds:
        c = chans[k]
        if k == "seg":
            lab = torch.randint(0, c, (n, h, w), generator=g, dtype=torch.uint8)
            s = ops.SegMap(lab.to(dev()), c)
            srcs.append((s, False))
            dense.append(s.dense().cpu())
        else:
            x = torch.randn(n, c, h, w, generator=g) * 3.0
            dense.append(x)
            srcs.append((x.permute(0, 2, 3, 1).contiguous().to(dev()), True) if k == "nhwc" else (x.to(dev()), False))
    total = sum(d.shape[1] for d in dense)
    assert total <= c_fill
    got = ops.Planes(n, h, w, c_fill, dev(), dual=True)
    ref = ops.Planes(n, h, w, c_fill, dev(), dual=True)
    for p in (got, ref):               # stale content the packs must overwrite
        for t in (p.hi, p.lo, p.twin.hi, p.twin.lo):
            t.fill_(1.0)
    ops.pack_concat(srcs, got, lead=lead)
    ops.pack_concat([(torch.cat(dense, 1).contiguous().to(dev()), False)], ref)
    torch.cuda.synchronize()
    for a, b in ((got.hi, ref.hi), (got.lo, ref.lo), (got.twin.hi, ref.twin.hi), (got.twin.lo, ref.twin.lo)):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    assert not got.dense()[..., :lead].any()


# ---------------------------------------------------------------------------------------------
# UnetEngine against the oracle
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("norm,B,S", [("instance", 2, 128), ("batch", 2, 128), ("none", 2, 128), ("instance", 1, 512),
                                      ("batch", 1, 512), ("none", 1, 512)])
def test_unet_engine_matches_oracle(norm, B, S):
    """pix2pix's generator on its 36-zero + cloth operand, train mode (dropout in the two inner blocks): fakes and
    every parameter gradient for a random upstream gradient."""
    from swapnet_b200 import engine as E
    from swapnet_b200 import modules as M
    from swapnet_b200 import ops

    torch.manual_seed(0)
    net = M.UnetGenerator(55, 3, 7, 64, use_dropout=True, norm=norm).to(dev())
    M.init_weights(net, "kaiming", 0.02)
    _randomise_affine((net,))
    sd, names = _param_sd(net)
    eng = E.UnetEngine(net, B, S, dev())
    eng.alloc_grads()
    eng.bind_backward()
    eng.pack()
    _, _, cloth, _ = synth_texture_batch(B, S)
    g = torch.Generator().manual_seed(5)
    up = torch.randn(B, S, S, 3, generator=g)
    eng.zero_grad()
    ops.pack_concat([(cloth.to(dev()), False)], eng.x_in, lead=36)
    eng.forward(training=True, seed=77)
    eng.backward([ops.GradSrc(up.to(dev()))])
    torch.cuda.synchronize()
    got = {k: p.grad.detach().cpu().clone() for k, p in net.named_parameters()}
    gates = bn_stage_gates(eng)
    ON.gate_with(lambda name, x: gates[name])
    drop = OD.make_drop({s.name: E._mix_seed(eng.seed, s.id) for s in eng.stages}, 0.5)
    try:
        out, _ = UO.unet_forward(sd, UO.real_A(cloth.double()), norm, True, drop)
        stats = dict(ON.GATE_STATS)
    finally:
        ON.gate_with(None)
    flips = sum(v for k, v in stats.items() if k != "__total__")
    assert flips <= 2e-5 * stats.get("__total__", 1), stats
    assert relmax(eng.fakes.cpu().permute(0, 3, 1, 2), out.detach()) < 1e-3
    keys = [k for k in sd if k in names]
    refs = torch.autograd.grad((out * up.double().permute(0, 3, 1, 2)).sum(), [sd[k] for k in keys])
    mx = max(r.abs().max().item() for r in refs)
    worst = {}
    for k, r in zip(keys, refs):
        if r.abs().max().item() < 1e-6 * mx:     # a conv bias followed by InstanceNorm: its gradient is zero
            assert got[k].abs().max().item() < 1e-4 * mx, k
            continue
        worst[k] = relmax(got[k], r)
    record(f"unet_engine_worst_grads[{norm},{S}]", sorted(worst.items(), key=lambda kv: -kv[1])[:3])
    assert max(worst.values()) < 1e-3, worst


def test_unet_engine_refuses_sizes_its_skips_cannot_join():
    from swapnet_b200 import engine as E
    from swapnet_b200 import modules as M

    net = M.UnetGenerator(3, 3, 7, 64, use_dropout=True, norm="batch").to(dev())
    with pytest.raises(ValueError, match="divisible by 2\\*\\*7 = 128"):
        E.UnetEngine(net, 1, 64, dev())


# ---------------------------------------------------------------------------------------------
# plugin steps against the oracle
# ---------------------------------------------------------------------------------------------
def pix2pix_opt(B, S, **over):
    d = dict(model="pix2pix", name="pix2pix", norm="batch", netG="unet_128", lambda_l1=10.0, beta1=0.5, lr=0.01)
    d.update(over)
    return _opt(B, S, **d)


def texture_unet_opt(B, S, **over):
    d = dict(model="texture", name="texture", netG="unet_128", lambda_l1=10, lambda_content=0.0, lambda_style=0.0,
             b200_vgg="random")
    d.update(over)
    return _opt(B, S, **d)


def _phases(model, batch):
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
    return gD, gG, model.get_current_losses()


def _imposed_gates(model, B):
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
    return gate


def _unet_step(kind, B, S, norm="batch", gan_mode="vanilla", train=True, perceptual=False, tag=""):
    from swapnet_b200 import engine as E
    from swapnet_b200.models import create_model

    torch.manual_seed(0)
    lc, ls = (20.0, 1e-8) if perceptual else (0.0, 0.0)
    if kind == "pix2pix":
        opt = pix2pix_opt(B, S, norm=norm, gan_mode=gan_mode)
    else:
        opt = texture_unet_opt(B, S, norm=norm, gan_mode=gan_mode, lambda_content=lc, lambda_style=ls)
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
    if kind == "pix2pix":
        batch = dict(cloths=cloth, target_textures=tgt)
    else:
        batch = dict(input_textures=tex, rois=rois, cloths=cloth, target_textures=tgt, cloth_paths=["c"] * B,
                     texture_paths=["t"] * B)
    torch.manual_seed(321)
    gD, gG, losses = _phases(model, batch)
    draws = UO.GM.label_draws(UO.PIX2PIX_MODES[gan_mode])
    torch.manual_seed(321)
    draws = [torch.rand(1) for _ in range(draws)]
    assert model.label_draws() == len(draws)
    fakes = model.fake_B if kind == "pix2pix" else model.fakes
    gate = _imposed_gates(model, B)
    gates_P, vgg_sd = {}, None
    if perceptual:
        from test_engine_gpu import stage_gates, vgg_pool_winners

        gates_P = {"vgg_o." + k: v for k, v in stage_gates(model._eng_P.out).items()}
        gates_P.update({"vgg_t." + k: v for k, v in stage_gates(model._eng_P.tgt).items()})
        vgg_sd = {k: v.detach().cpu().double() for k, v in model.net_vgg.state_dict().items()}
        winners = vgg_pool_winners(model._eng_P.out, "vgg_o")
        ON.pool_with(lambda name, x: winners.get(name))
    ON.gate_with(lambda name, x: gates_P[name] if name in gates_P else gate(name, x))
    drop = None
    if train:
        eng = model._eng_G
        drop = OD.make_drop({s.name: E._mix_seed(eng.seed, s.id) for s in eng.stages}, 0.5, sample_base=eng.sample_base)
    l1_sign = torch.sign(fakes.detach() - tgt.to(dev())).cpu().double()
    try:
        if kind == "pix2pix":
            o = UO.pix2pix_step_losses(sdG, sdD, cloth.double(), tgt.double(), draws, gan_mode, norm, train,
                                       drop=drop, l1_sign=l1_sign)
        else:
            o = UO.texture_unet_step_losses(sdG, sdD, tex.double(), cloth.double(), tgt.double(), draws, gan_mode,
                                            norm, train, drop=drop, l1_sign=l1_sign, vgg=vgg_sd, lambda_content=lc,
                                            lambda_style=ls)
        stats = dict(ON.GATE_STATS)
    finally:
        ON.gate_with(None)
        ON.pool_with(None)
    flips = {k: v for k, v in stats.items() if k != "__total__" and not k.startswith("pool:") and v}
    record(f"unet_step_gate_flips[{kind}{tag}]", f"{sum(flips.values())} of {stats.get('__total__', 1)}")
    assert sum(flips.values()) <= 2e-5 * stats.get("__total__", 1), f"too many activation gates differ: {flips}"
    if kind == "pix2pix":
        keys = ("D_fake", "D_real", "G", "G_GAN", "G_L1")
        assert list(losses) == ["G", "G_GAN", "G_L1", "D_real", "D_fake"]
        model.fakes = fakes
    else:
        keys = ("D", "D_real", "D_fake", "G", "G_gan", "G_l1") + (("G_content", "G_style") if perceptual else ())
    _check_step(model, o, sdG, namesG, sdD, namesD, gG, gD, losses, keys, bufs0, train, f"[{kind}{tag}]")
    return model


@pytest.mark.parametrize("norm,train,gan_mode", [("batch", True, "vanilla"), ("batch", False, "vanilla"),
                                                 ("instance", True, "vanilla"), ("instance", False, "vanilla"),
                                                 ("none", True, "vanilla"), ("none", False, "vanilla"),
                                                 ("batch", True, "lsgan"), ("batch", True, "wgan"),
                                                 ("instance", True, "wgan-gp")])
def test_pix2pix_step_matches_oracle(norm, train, gan_mode):
    _unet_step("pix2pix", 2, 128, norm, gan_mode, train, tag=f"[{norm},{gan_mode},train={train}]")


def test_pix2pix_step_512_matches_oracle():
    _unet_step("pix2pix", 1, 512, "batch", tag="[512]")


@pytest.mark.parametrize("B,S,perceptual", [(2, 128, False), (2, 128, True), (1, 512, True)])
def test_texture_unet_128_step_matches_oracle(B, S, perceptual):
    _unet_step("texture", B, S, "instance", perceptual=perceptual, tag=f"[{S},perceptual={perceptual}]")


def test_pix2pix_optimizers_are_adam():
    """optimizer_G / optimizer_D over three steps against torch.optim.Adam(lr=--lr, betas=(beta1, 0.999), eps=1e-8), no
    weight decay, on the same parameters and gradients: the step's own gradients, then two more made from them with
    random per-element factors and signs.  Adam's first step is lr * sign(g) whatever the betas; the later ones are
    not, so these pin beta1 = 0.5 and beta2 = 0.999."""
    torch.manual_seed(0)
    from swapnet_b200.models import create_model

    B, S = 2, 128
    model = create_model(pix2pix_opt(B, S, lr=2e-3))
    model.setup(model.opt)
    _, _, cloth, tgt = synth_texture_batch(B, S)
    _phases(model, dict(cloths=cloth, target_textures=tgt))
    gen = torch.Generator().manual_seed(11)
    for net, optim in ((model.net_D, model.optimizer_D), (model.net_G, model.optimizer_G)):
        params = list(net.parameters())
        before = [p.detach().cpu().double().clone() for p in params]
        g0 = [p.grad.detach().cpu().double().clone() for p in params]
        ps = [p.clone().requires_grad_() for p in before]
        ref = torch.optim.Adam(ps, lr=2e-3, betas=(0.5, 0.999), eps=1e-8)
        for step in range(3):
            for p, q, g in zip(ps, params, g0):
                f = 1.0 if step == 0 else (torch.rand(g.shape, generator=gen, dtype=torch.float64) * 1.6 + 0.2) * \
                    torch.where(torch.rand(g.shape, generator=gen) < 0.3, -1.0, 1.0).double()
                gs = (g * f).float()
                q.grad.copy_(gs.to(q.device))          # the optimizer reads the engine's flat gradient buffer
                p.grad = gs.double()
            ref.step()
            optim.step()
            torch.cuda.synchronize()
            for p0, p, q in zip(before, ps, params):
                assert relmax(q.detach().cpu().double() - p0, p.detach() - p0) < 1e-4, step


def _kind_opt(kind, B, S, **over):
    return pix2pix_opt(B, S, **over) if kind == "pix2pix" else texture_unet_opt(B, S, **over)


def _kind_batch(kind, tex, rois, cloth, tgt):
    if kind == "pix2pix":
        return dict(cloths=cloth, target_textures=tgt)
    B = tgt.shape[0]
    return dict(input_textures=tex, rois=rois, cloths=cloth, target_textures=tgt, cloth_paths=["c"] * B,
                texture_paths=["t"] * B)


@pytest.mark.parametrize("kind", ["pix2pix", "texture_unet_128"])
def test_graph_replay_is_bit_identical_to_eager_steps(kind):
    """--b200_deterministic 1: three steps, the third a CUDA-graph replay, give the same losses and parameters bit for
    bit as three eager steps (uint8 cloth label maps; for unet_128 the texture is packed and the rois are copied but
    not read)."""
    from swapnet_b200 import ops
    from swapnet_b200.models import create_model

    B, S = 2, 128
    tex, rois, cloth, tgt = synth_texture_batch(B, S)
    batch = _kind_batch(kind, tex, rois, ops.SegMap.from_dense(cloth), tgt)
    runs = {}
    for graph in (1, 0):
        torch.manual_seed(0)
        model = create_model(_kind_opt(kind, B, S, b200_graph=graph, b200_deterministic=1, lr=2e-4))
        model.setup(model.opt)
        torch.manual_seed(99)
        hist = []
        for _ in range(3):
            model.set_input(batch)
            model.optimize_parameters()
            hist.append(dict(model.get_current_losses()))
        assert (len(model._graphs) == 1) == bool(graph)
        runs[graph] = (hist, {p + k: v.detach().cpu().clone()
                              for p, net in (("G.", model.net_generator), ("D.", model.net_discriminator))
                              for k, v in net.state_dict().items()})
    assert runs[1][0] == runs[0][0]
    for k, v in runs[0][1].items():
        assert torch.equal(runs[1][1][k], v), k


@pytest.mark.parametrize("kind", ["pix2pix", "texture_unet_128"])
def test_checkpoint_round_trip_to_inference_model(kind):
    """The reference's file names and keys (pix2pix: <epoch>_net_G.pth / <epoch>_net_D.pth and no optimizer files;
    the texture stage: net_generator / net_discriminator and both optimizers); an is_train=False model (netG and norm
    from the saved options, as inference.py restores them) loads G only, and its eval forward is the oracle's on the
    saved weights and running statistics."""
    from swapnet_b200.models import create_model

    B, S = 2, 128
    torch.manual_seed(0)
    opt = _kind_opt(kind, B, S, lr=1e-4)
    model = create_model(opt)
    model.setup(opt)
    tex, rois, cloth, tgt = synth_texture_batch(B, S)
    for _ in range(2):
        model.set_input(_kind_batch(kind, tex, rois, cloth, tgt))
        model.optimize_parameters()
    model.save_checkpoint("latest")
    if kind == "pix2pix":
        files, g_file, iopt = ["latest_net_D.pth", "latest_net_G.pth"], "latest_net_G.pth", \
            dict(model="pix2pix", name="pix2pix", norm="batch")
    else:
        files = ["latest_net_discriminator.pth", "latest_net_generator.pth", "latest_optim_D.pth", "latest_optim_G.pth"]
        g_file, iopt = "latest_net_generator.pth", dict(model="texture", name="texture", netG="unet_128",
                                                         norm="instance")
    assert sorted(os.listdir(model.save_dir)) == files
    saved = torch.load(os.path.join(model.save_dir, g_file))
    assert list(saved) == list(model.net_generator.state_dict())
    assert next(iter(saved)) == "model.model.0.weight"
    iopt = _opt(1, S, is_train=False, load_epoch="latest", checkpoints_dir=opt.checkpoints_dir, **iopt)
    inf = create_model(iopt)
    assert not hasattr(inf, "net_discriminator") and len(inf.model_names) == 1
    inf.setup(iopt)
    inf.eval()
    inf.compute_visuals = lambda: None    # visuals need the reference's helpers
    inf.set_input(_kind_batch(kind, tex[:1], rois[:1], cloth[:1], tgt[:1]))
    inf.test()
    torch.cuda.synchronize()
    sd = {k: v.double() for k, v in saved.items()}
    x = UO.real_A(cloth[:1].double()) if kind == "pix2pix" else tex[:1].double()
    with torch.no_grad():
        ref, _ = UO.unet_forward(sd, x, "batch", False)
    err = relmax((inf.fake_B if kind == "pix2pix" else inf.fakes).cpu(), ref)
    record(f"unet_checkpoint_eval_forward[{kind}]", f"{err:.3e}")
    assert err < 1e-3, err


def test_two_rank_gloo_sync_bn_equals_full_batch():
    """pix2pix (--norm batch) and --netG unet_128 (--norm instance: the generator's batch norm alone) with
    --b200_sync_bn 1: two ranks on halves of a batch against one process on the whole batch (tests/tools/
    unet_dp_equiv.py, both ranks on cuda:0 over gloo)."""
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    env = dict(os.environ, SN_SBN_BACKEND="gloo", PYTHONPATH=os.pathsep.join([ROOT, os.environ.get("PYTHONPATH", "")]))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(ROOT, "tests", "tools", "unet_dp_equiv.py")]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("SYNC_BN_EQUIV")]
    for ln in lines:
        record("unet_sync_bn_equivalence", ln)
    ok = r.returncode == 0 and len(lines) == 2 and all(" OK " in ln for ln in lines)
    assert ok, "\n".join(lines) + "\n--- stderr ---\n" + r.stderr[-8000:]
