"""`--discriminator pixel` on the device: each pass of csrc/pixel_disc.cu against fp64 torch with the device's LeakyReLU
gates imposed (from the debug pre-activations of the forward pass), the deterministic mode, CUDA-graph replay, the
bf16 precision mode, whole training steps of both stages, and the memory the fused passes save."""
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "tools"))

import pixel_oracle as PO  # noqa: E402
from test_engine_gpu import _opt, synth_texture_batch, synth_warp_batch  # noqa: E402

CIN = 22


def _net(norm, cin=CIN, seed=0):
    from swapnet_b200 import modules as M

    torch.manual_seed(seed)
    net = M.PixelDiscriminator(cin, 64, norm)
    M.init_weights(net, "kaiming", 0.02)
    with torch.no_grad():   # non-zero biases, so that every bias path is exercised
        for m in net.modules():
            if isinstance(m, torch.nn.Conv2d) and m.bias is not None:
                m.bias.normal_(0.0, 0.1)
    return net.cuda()


def _run_engine(net, n, s, *, input_grad=True, wgrad=True, deterministic=False, nsplit=3, seed=1):
    """One forward + backward of a fresh PixelGANEngine on seeded inputs; returns (engine, x NCHW, dpred)."""
    from swapnet_b200 import engine as E
    from swapnet_b200 import ops

    g = torch.Generator().manual_seed(seed)
    x = (torch.rand(n, net.input_nc, s, s, generator=g) * 2 - 1).cuda()
    dpred = (torch.randn(n, s, s, generator=g) / (n * s * s) ** 0.5).cuda()
    eng = E.PixelGANEngine(net, n, s, "cuda", nsplit, input_grad=input_grad, deterministic=deterministic)
    eng.alloc_grads()
    eng.bind_backward()
    eng.debug = torch.zeros(n * s * s, 192, device="cuda")
    ops.pack_concat([(x, False)], eng.din)
    eng.zero_grad()
    eng.pack()
    eng.forward()
    eng.backward(dpred, wgrad=wgrad)
    torch.cuda.synchronize()
    return eng, x, dpred


def _gates(eng, n, s):
    dbg = eng.debug.view(n, s, s, 192).permute(0, 3, 1, 2).double().cpu()
    return dbg[:, :64] > 0, dbg[:, 64:] > 0


def _check(name, dev, ref, bound, tol):
    dev, ref, bound = dev.double().cpu(), ref.double().cpu(), bound.double().cpu()
    err = (dev - ref).abs()
    worst = (err / (bound + 1e-30)).max().item()
    assert worst <= tol, f"{name}: error {err.max().item():.3e}, {worst:.3e} of the per-entry bound (tol {tol})"


@pytest.mark.parametrize("norm", ["instance", "none"])
@pytest.mark.parametrize("n,s", [(2, 1), (2, 63), (2, 64), (2, 512), (32, 128)])
@pytest.mark.parametrize("input_grad", [True, False])
def test_passes_match_fp64_with_imposed_gates(norm, n, s, input_grad):
    if s == 1 and norm == "instance":
        pytest.skip("InstanceNorm2d refuses a 1x1 plane (one value per channel)")
    net = _net(norm)
    eng, x, dpred = _run_engine(net, n, s, input_grad=input_grad)
    z1g, y2g = _gates(eng, n, s)
    sd = {k: v.detach().cpu() for k, v in net.state_dict().items()}
    r = PO.pixel_grads(sd, x.cpu().double(), norm, dpred.cpu().double().unsqueeze(1), z1g, y2g)
    ab = lambda t: t.abs()  # noqa: E731
    w3 = sd["net.5.weight"].double().view(1, 128, 1, 1)
    # forward: the logits within the split-fp16 products' error, relative to sum |w3| |a2| (+ |b3|)
    pb = (ab(w3) * ab(r["a2"])).sum(1) + (ab(sd["net.5.bias"]).double() if "net.5.bias" in sd else 0)
    _check("pred", eng.pred, r["pred"][:, 0], pb, 1e-4)
    # weight gradients: per entry, relative to the sum of |products| the reduction adds (bf16-split backward)
    dp = ab(dpred.cpu().double())
    bounds = {
        "net.5.weight": torch.einsum("nhw,nchw->c", dp, ab(r["a2"])).view(1, 128, 1, 1),
        "net.5.bias": dp.sum().view(1),
        "net.2.weight": torch.einsum("nahw,nbhw->ab", ab(r["dz2"]), ab(r["a1"])).view(128, 64, 1, 1),
        "net.2.bias": ab(r["dz2"]).sum((0, 2, 3)),
        "net.0.weight": torch.einsum("nahw,nbhw->ab", ab(r["g1"]), ab(x.cpu().double())).view(64, CIN, 1, 1),
        "net.0.bias": ab(r["g1"]).sum((0, 2, 3)),
    }
    params = dict(net.named_parameters())
    for k, p in params.items():
        # dz2 itself carries the InstanceNorm backward's fp32 rounding: a looser bar with normalisation
        # g1 and dz2 can cancel, which these bounds do not see: a loose bar here, and the separation of the split and
        # hi-only products is checked on its own (test_split_products_are_an_order_of_magnitude_closer_than_hi_only)
        _check(k, p.grad, r[k], bounds[k] + 1e-6 * bounds[k].max(), 2e-3)
    if input_grad:
        w1 = sd["net.0.weight"].double().view(64, CIN)
        xb = torch.einsum("nahw,ac->nchw", ab(r["g1"]), ab(w1))
        _check("dx", eng.dx_in.permute(0, 3, 1, 2), r["x"], xb + 1e-6 * xb.max(), 2e-3)


def test_split_products_are_an_order_of_magnitude_closer_than_hi_only():
    """Every GEMM honours nsplit: the three-product split beats the hi x hi product by far on every gradient."""
    errs = {}
    for nsplit in (1, 3):
        net = _net("none")
        eng, x, dpred = _run_engine(net, 2, 64, nsplit=nsplit)
        z1g, y2g = _gates(eng, 2, 64)
        sd = {k: v.detach().cpu() for k, v in net.state_dict().items()}
        r = PO.pixel_grads(sd, x.cpu().double(), "none", dpred.cpu().double().unsqueeze(1), z1g, y2g)
        errs[nsplit] = {k: ((p.grad.double().cpu() - r[k]).abs().max() / r[k].abs().max()).item()
                        for k, p in net.named_parameters()}
        errs[nsplit]["dx"] = ((eng.dx_in.permute(0, 3, 1, 2).double().cpu() - r["x"]).abs().max() /
                              r["x"].abs().max()).item()
    from conftest import record

    record("pixel_disc_nsplit_relmax", errs)
    for k in errs[3]:
        assert errs[3][k] * 10 < errs[1][k], (k, errs[3][k], errs[1][k])


@pytest.mark.parametrize("norm", ["instance", "none"])
def test_forward_only_engine_has_no_gradient_side_effects(norm):
    """The G-step engine (input gradient, no weight gradients) leaves .grad untouched."""
    net = _net(norm)
    eng, _, _ = _run_engine(net, 2, 64, input_grad=True, wgrad=False)
    assert all(p.grad.abs().max().item() == 0 for p in net.parameters())
    assert eng.dx_in.abs().max().item() > 0


_DET_STEP = """
import hashlib, sys
sys.path.insert(0, {tests!r}); sys.path.insert(0, {tools!r})
import test_pixel_disc_gpu as T
m, opt = T._model({model!r}, "pixel", {norm!r}, "vanilla", deterministic=1)
m.set_input(T._inputs({model!r}, opt))
m.optimize_parameters()
import torch
torch.cuda.synchronize()
h = hashlib.sha256()
for t in [m._eng_Dd.flat_grad, m._eng_G.flat_grad, m._eng_Dg.dx_in.contiguous(), torch.tensor(m.loss_values())] + \\
        [p.detach() for p in list(m.net_discriminator.parameters()) + list(m.net_generator.parameters())]:
    h.update(t.detach().cpu().contiguous().numpy().tobytes())
print("STEP_SHA", h.hexdigest())
"""


@pytest.mark.parametrize("model,norm", [("warp", "instance"), ("texture", "none")])
def test_deterministic_steps_are_bit_identical_across_fresh_processes(model, norm):
    import subprocess

    code = _DET_STEP.format(tests=HERE, tools=os.path.join(HERE, "tools"), model=model, norm=norm)
    shas = []
    for _ in range(2):
        r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600,
                           cwd=os.path.dirname(HERE))
        lines = [ln for ln in r.stdout.splitlines() if ln.startswith("STEP_SHA")]
        assert r.returncode == 0 and lines, r.stderr[-4000:]
        shas.append(lines[-1])
    assert shas[0] == shas[1]


@pytest.mark.parametrize("norm", ["instance", "none"])
def test_deterministic_passes_agree_with_default(norm):
    net = _net(norm)
    eng, _, _ = _run_engine(net, 4, 128, deterministic=True)
    det = (eng.pred.clone(), eng.dx_in.clone(), eng.flat_grad.clone())
    net = _net(norm)
    eng, _, _ = _run_engine(net, 4, 128)
    for a, b in zip(det, (eng.pred, eng.dx_in, eng.flat_grad)):
        assert (a - b).abs().max().item() <= 1e-5 * b.abs().max().item()


@pytest.mark.parametrize("model", ["warp", "texture"])
def test_bf16_precision_option_trains_within_1e2(model):
    out = {}
    for prec in ("fp32x3", "bf16"):
        m, opt = _model(model, "pixel", "instance", "vanilla", precision=prec)
        m.set_input(_inputs(model, opt))
        torch.manual_seed(7)
        m.optimize_parameters()
        torch.cuda.synchronize()
        out[prec] = (torch.tensor(m.loss_values()[:3]), m._eng_Dd.flat_grad.detach().clone())
    assert m.nsplit == 1
    for a, b in zip(out["fp32x3"], out["bf16"]):
        assert (a - b.cpu() if a.device != b.device else a - b).abs().max().item() <= 1e-2 * a.abs().max().item()


def _model(model, disc, norm, gan_mode, deterministic=None, graph=0, batch=2, size=64, precision="fp32x3"):
    from swapnet_b200.models import create_model

    extra = {} if model == "warp" else dict(name="texture", netG="swapnet", lambda_l1=10, lambda_content=0,
                                            lambda_style=0)
    opt = _opt(batch, size, model=model, discriminator=disc, norm=norm, gan_mode=gan_mode, b200_graph=graph,
               b200_deterministic=deterministic, b200_precision=precision, **extra)
    torch.manual_seed(0)
    m = create_model(opt)
    m.setup(opt)
    return m, opt


def _inputs(model, opt, seed=3):
    B, S = opt.batch_size, opt.crop_size
    if model == "warp":
        body, inp, tgt = synth_warp_batch(B, S, seed)
        return dict(bodys=body, input_cloths=inp, target_cloths=tgt, cloth_paths=["c"] * B, body_paths=["b"] * B)
    tex, rois, cloth, tgt = synth_texture_batch(B, S, seed)
    return dict(input_textures=tex, rois=rois, cloths=cloth, target_textures=tgt, cloth_paths=["c"] * B,
                texture_paths=["t"] * B)


@pytest.mark.parametrize("model", ["warp", "texture"])
@pytest.mark.parametrize("norm", ["instance", "none"])
@pytest.mark.parametrize("gan_mode", ["vanilla", "lsgan", "wgan"])
def test_training_step_runs_and_d_gradients_match_fp64(model, norm, gan_mode):
    """A whole training step with the PixelGAN: finite losses, and the D step's gradient equals the fp64 oracle's for the
    discriminator inputs the step packed (fakes and reals, gates imposed)."""
    m, opt = _model(model, "pixel", norm, gan_mode, deterministic=1)
    m.set_input(_inputs(model, opt))
    sdD = {k: v.detach().cpu().clone() for k, v in m.net_discriminator.state_dict().items()}
    d = None
    from swapnet_b200 import engine as E

    orig = E.PixelGANEngine.backward

    def spy(self, dpred, wgrad=True):
        nonlocal d
        orig(self, dpred, wgrad)
        if wgrad and d is None:
            torch.cuda.synchronize()
            d = (self.din.dense()[..., :self.net.input_nc].permute(0, 3, 1, 2).double().cpu(),
                 dpred.double().cpu(), {k: p.grad.detach().double().cpu().clone()
                                        for k, p in self.net.named_parameters()})

    E.PixelGANEngine.backward = spy
    try:
        m.ensure_engines(opt.batch_size, opt.crop_size)
        m._eng_Dd.debug = torch.zeros(m._eng_Dd.din.n * opt.crop_size ** 2, 192, device="cuda")
        m.optimize_parameters()
    finally:
        E.PixelGANEngine.backward = orig
    losses = m.get_current_losses()
    assert all(v == v and abs(v) < 1e3 for v in losses.values()), losses
    x, dpred, grads = d
    n, s = x.shape[0], x.shape[-1]
    dbg = m._eng_Dd.debug.view(n, s, s, 192).permute(0, 3, 1, 2).double().cpu()
    r = PO.pixel_grads(sdD, x, norm, dpred.unsqueeze(1), dbg[:, :64] > 0, dbg[:, 64:] > 0)
    for k, g in grads.items():
        # net.2.bias under InstanceNorm has a zero gradient in exact arithmetic: measured against sum |dz2| instead
        scale = r["dz2"].abs().sum((0, 2, 3)).max().item() if k == "net.2.bias" and norm == "instance" else \
            r[k].abs().max().item()
        err = (g - r[k]).abs().max().item() / max(scale, 1e-12)
        assert err < 1e-3, (k, err)


@pytest.mark.parametrize("model", ["warp", "texture"])
def test_graph_replayed_deterministic_steps_equal_eager_steps(model):
    states = []
    for graph in (0, 1):
        m, opt = _model(model, "pixel", "instance", "vanilla", deterministic=1, graph=graph)
        torch.manual_seed(5)
        for i in range(4):
            m.set_input(_inputs(model, opt, seed=10 + i))
            m.optimize_parameters()
        torch.cuda.synchronize()
        states.append([p.detach().clone() for p in list(m.net_discriminator.parameters()) +
                       list(m.net_generator.parameters())] + [torch.tensor(m.loss_values())])
    assert all(torch.equal(a, b) for a, b in zip(*states))


def test_checkpoint_round_trip_with_reference_keys(tmp_path):
    m, opt = _model("warp", "pixel", "none", "vanilla")
    keys = set(m.net_discriminator.state_dict())
    assert keys == {"net.0.weight", "net.0.bias", "net.2.weight", "net.5.weight"}
    m.set_input(_inputs("warp", opt))
    m.optimize_parameters()
    sd = {k: v.detach().cpu().clone() for k, v in m.net_discriminator.state_dict().items()}
    torch.save(sd, tmp_path / "d.pth")
    m2, _ = _model("warp", "pixel", "none", "vanilla")
    m2.net_discriminator.load_state_dict(torch.load(tmp_path / "d.pth"))
    assert all(torch.equal(v.cpu(), sd[k]) for k, v in m2.net_discriminator.state_dict().items())


def _peak_step_bytes(disc):
    import gc

    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    m, opt = _model("warp", disc, "instance", "vanilla", graph=0, batch=16, size=512)
    m.set_input(_inputs("warp", opt))
    m.optimize_parameters()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    del m
    gc.collect()
    torch.cuda.empty_cache()
    return peak


def test_warp_step_memory_at_512_batch_16_stays_with_basic():
    """The reason for the fused design: the PixelGAN's full-resolution hidden layers are never stored, so a warp step
    at 512^2, batch 16 peaks within 256 MB of the same step with the basic PatchGAN."""
    from conftest import record

    basic = _peak_step_bytes("basic")
    pixel = _peak_step_bytes("pixel")
    record("pixel_disc_peak_bytes_basic_vs_pixel", f"{basic} {pixel}")
    assert pixel <= basic + 256 * 2 ** 20, (basic, pixel)


def _model_opt(disc, norm, **over):
    return _opt(2, 64, discriminator=disc, norm=norm, **over)


def test_pixel_with_batch_norm_is_refused_with_its_reason():
    from swapnet_b200.models import create_model

    with pytest.raises(NotImplementedError, match="batch statistics couple the samples"):
        create_model(_model_opt("pixel", "batch"))


@pytest.mark.parametrize("norm", ["instance", "none"])
def test_pixel_model_builds_the_pixel_container_and_ignores_n_layers(norm):   # models refuse a CPU device
    from swapnet_b200 import modules as M
    from swapnet_b200.models import create_model

    m = create_model(_model_opt("pixel", norm, n_layers_D=5))
    assert isinstance(m.net_discriminator, M.PixelDiscriminator)
    assert m.net_discriminator.input_nc == m.get_D_inchannels()


@pytest.mark.parametrize("disc,n_layers", [("basic", 3), ("n_layers", 4)])
def test_basic_and_n_layers_are_unaffected(disc, n_layers):
    from swapnet_b200 import modules as M
    from swapnet_b200.models import create_model

    m = create_model(_model_opt(disc, "instance", n_layers_D=n_layers))
    assert isinstance(m.net_discriminator, M.NLayerDiscriminator)
    assert m.net_discriminator.n_layers == n_layers


@pytest.mark.parametrize("kind", ["warp", "texture"])
def test_full_step_matches_the_reference(kind):
    """The whole device step against the reference step of tests/golden/pixel_disc_64.pt (same seeds, inputs, label
    draws, dropout off): every loss, every D gradient of the D step and the input gradient the PixelGAN passes to G
    within the 1e-3 parity bar of the oracle replay that reproduces that step (tests/test_pixel_disc_cpu.py); the CPU
    generator ends where the reference leaves it; the PixelGAN's LeakyReLU gates that disagree with the oracle's are
    counted apart."""
    import make_golden_gan_modes as MGM
    from conftest import record
    from test_pixel_disc_cpu import GOLDEN, _step_batch, step_nets

    g = GOLDEN[f"{kind}_step"]
    m, opt = _model(kind, "pixel", "instance", "vanilla", deterministic=1)
    G, Dn = step_nets(kind)       # the reference step's seeded weights (pinned to the fixture by the CPU suite)
    m.net_generator.load_state_dict(G.state_dict())
    m.net_discriminator.load_state_dict(Dn.state_dict())
    m.eval()                       # dropout off, as in the reference step; InstanceNorm is per sample either way
    m.is_train = True
    B = opt.batch_size
    batch = dict(_step_batch(kind), **({"cloth_paths": ["c"] * B, "body_paths": ["b"] * B} if kind == "warp" else
                                       {"cloth_paths": ["c"] * B, "texture_paths": ["t"] * B}))
    m.set_input(batch)
    m.ensure_engines(B, opt.crop_size)
    S = opt.crop_size
    m._eng_Dd.debug = torch.zeros(2 * B * S * S, 192, device="cuda")
    m._eng_Dg.debug = torch.zeros(B * S * S, 192, device="cuda")
    torch.manual_seed(MGM.LABEL_SEED)
    m.optimize_parameters()
    torch.cuda.synchronize()
    assert MGM.rng_digest() == g["rng_after"]
    losses = m.get_current_losses()
    for k, v in g["losses"].items():
        assert abs(losses[k] - v) <= 1e-3 * abs(v), (k, losses[k], v)
    gD = {k: p.grad.detach().double().cpu() for k, p in m.net_discriminator.named_parameters()}
    gG = {k: p.grad.detach().double().cpu() for k, p in m.net_generator.named_parameters()}
    # a gate of the G step's PixelGAN flips one pixel's input gradient outright: the device's gates are imposed there
    dbg_g = m._eng_Dg.debug.view(B, S, S, 192).permute(0, 3, 1, 2).double().cpu()
    o = PO.reference_step(kind, G, Dn, _step_batch(kind), MGM.LABEL_SEED, (dbg_g[:, :64] > 0, dbg_g[:, 64:] > 0))
    free = PO.pixel_forward(o["sdD"], o["d_inputs"][0].double(), "instance")
    flips_g = int(((dbg_g[:, :64] > 0) != (free["z1"] > 0)).sum() + ((dbg_g[:, 64:] > 0) != (free["y2"] > 0)).sum())
    record(f"pixel_disc_full_step_gate_flips_G_step[{kind}]", f"{flips_g} of {dbg_g.numel()}")
    assert flips_g <= 1e-4 * dbg_g.numel(), flips_g
    # what the PixelGAN hands back to G: d G_gan / d(D input) of the G step, in the layout the plugins read (dpred
    # scale, [B, S, S, cin] pitch-24 dx_in)
    dx = m._eng_Dg.dx_in.permute(0, 3, 1, 2).double().cpu()
    e_dx = ((dx - o["dgan_dx"].double()).abs().max() / o["dgan_dx"].abs().max()).item()
    record(f"pixel_disc_full_step_dgan_dx[{kind}]", e_dx)
    assert e_dx < 1e-3, e_dx
    # G's own gradients also carry the generator's ReLU / LeakyReLU gates, which this oracle does not impose (the
    # generator's gated parity is tests/test_gan_modes_gpu.py's): recorded, not asserted
    gworst = {k: ((gG[k] - r.double()).abs().max() / r.double().abs().max().clamp_min(1e-30)).item()
              for k, r in o["grads_G"].items()}
    record(f"pixel_disc_full_step_ungated_G_grads[{kind}]", sorted(gworst.items(), key=lambda kv: -kv[1])[:5])
    worst = {}
    for dev, ref in ((gD, o["grads_D"]),):
        gmax = max(v.abs().max().item() for v in ref.values())
        for k, r in ref.items():
            if r.abs().max().item() < 1e-6 * gmax:     # exact zero (a bias before an InstanceNorm): noise on both
                assert dev[k].abs().max().item() < 1e-4 * gmax, k
                continue
            worst[k] = ((dev[k] - r.double()).abs().max() / r.double().abs().max()).item()
    record(f"pixel_disc_full_step_worst_grads[{kind}]", sorted(worst.items(), key=lambda kv: -kv[1])[:5])
    assert max(worst.values()) < 1e-3, sorted(worst.items(), key=lambda kv: -kv[1])[:5]
    # gates of the PixelGAN in the D step: device pre-activations against the oracle's on the oracle's D inputs
    dbg = m._eng_Dd.debug.view(2 * B, S, S, 192).permute(0, 3, 1, 2).double().cpu()
    ref = PO.pixel_forward(o["sdD_before"], torch.cat(o["d_inputs"], 0).double(), "instance")
    flips = int(((dbg[:, :64] > 0) != (ref["z1"] > 0)).sum() + ((dbg[:, 64:] > 0) != (ref["y2"] > 0)).sum())
    total = dbg.numel()
    record(f"pixel_disc_full_step_gate_flips[{kind}]", f"{flips} of {total}")
    assert flips <= 1e-4 * total, (flips, total)


def test_two_rank_gloo_on_one_gpu_equals_full_batch():
    """2 ranks x B/2 give the D and G gradients of one process with B (tests/tools/pixel_dp_equiv.py, gloo)."""
    import subprocess

    from conftest import record

    port = 29600 + os.getpid() % 300
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.join(HERE, "tools", "pixel_dp_equiv.py")]
    r = subprocess.run(cmd, env=dict(os.environ, SN_PIX_BACKEND="gloo"), capture_output=True, text=True, timeout=900)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("PIXEL_DP_EQUIV")]
    for ln in lines:
        record("pixel_dp_equivalence[gloo]", ln)
    assert r.returncode == 0 and len(lines) == 2 and all(" OK " in ln for ln in lines), \
        "\n".join(lines) + "\n--- stderr ---\n" + r.stderr[-8000:]
