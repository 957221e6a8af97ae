"""--b200_deterministic: bit-identical training steps.

With the mode on, every reduction that spans blocks stores per-block partial sums in slots and adds them in slot order
(csrc/common.cuh det_sum_slots, the weight-gradient GEMM's split workspace) instead of with floating-point atomics, so
two identically seeded runs — eager or graph-replayed — agree to the last bit.  The default mode's run-to-run
differences are recorded to parity.log as evidence of what the mode removes."""
import contextlib
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

from test_engine_gpu import (_opt, _texture_step_vs_oracle, _warp_step_vs_oracle, dev, record, relmax,  # noqa: E402
                             synth_texture_batch, synth_warp_batch)
from test_kernels_gpu import SP_SEP_BF16, at_both_nsplits, check_single_pass, model_wgrad  # noqa: E402


@contextlib.contextmanager
def torch_deterministic(on: bool):
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(on, warn_only=True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def _warp_batch(B, S):
    body, inp, tgt = synth_warp_batch(B, S)
    return dict(bodys=body, input_cloths=inp, target_cloths=tgt, cloth_paths=["c"] * B, body_paths=["b"] * B)


def _texture_batch(B, S):
    tex, rois, cloth, tgt = synth_texture_batch(B, S)
    return dict(input_textures=tex, rois=rois, cloths=cloth, target_textures=tgt, cloth_paths=["c"] * B,
                texture_paths=["t"] * B)


def _texture_opt(B, S, **over):
    d = dict(model="texture", name="texture", netG="swapnet", lambda_l1=10, lambda_content=0, lambda_style=0)
    d.update(over)
    return _opt(B, S, **d)


def _run(opt, batch, steps, seed=0):
    """Build an identically seeded model, run `steps` optimize_parameters() calls; returns (losses per step, state)."""
    from swapnet_b200.models import create_model

    torch.manual_seed(seed)
    model = create_model(opt)
    model.setup(opt)
    torch.manual_seed(99)
    losses = []
    for _ in range(steps):
        model.set_input(batch)
        model.optimize_parameters()
        losses.append(model._acc.detach().cpu().clone())
    torch.cuda.synchronize()
    state = {}
    for tag, net, optim in (("G", model.net_generator, model.optimizer_G), ("D", model.net_discriminator,
                                                                            model.optimizer_D)):
        for k, v in net.state_dict().items():
            state[f"{tag}.{k}"] = v.detach().cpu().clone()
        for k, v in optim.state_dict()["state"].items():
            for name, t in v.items():
                if torch.is_tensor(t):
                    state[f"{tag}.adam.{k}.{name}"] = t.detach().cpu().clone()
        state[f"{tag}.flat_grad"] = model._eng_G.flat_grad.detach().cpu().clone() if tag == "G" else \
            model._eng_Dd.flat_grad.detach().cpu().clone()
    return losses, state, model


def _assert_identical(a, b, what):
    (la, sa, _), (lb, sb, _) = a, b
    for i, (x, y) in enumerate(zip(la, lb)):
        assert torch.equal(x, y), f"{what}: losses of step {i} differ: {x} vs {y}"
    assert sa.keys() == sb.keys()
    bad = [k for k in sa if not torch.equal(sa[k], sb[k])]
    assert not bad, f"{what}: {len(bad)} tensors differ, e.g. {bad[:5]}"


def _differences(a, b):
    (la, sa, _), (lb, sb, _) = a, b
    nl = sum(int(not torch.equal(x, y)) for x, y in zip(la, lb))
    nt = sum(int(not torch.equal(sa[k], sb[k])) for k in sa)
    dmax = max(((sa[k].double() - sb[k].double()).abs().max().item() for k in sa if sa[k].is_floating_point()),
               default=0.0)
    return f"{nl} of {len(la)} loss vectors and {nt} of {len(sa)} tensors differ, max |diff| {dmax:.2e}"


def _conv_layers(model):
    """Every conv layer of every engine of a model: G, Dd, Dg and, for the perceptual loss, both VGG16 engines."""
    from swapnet_b200 import engine as E

    engines = {}
    for key, e in model._eng_extra.items():
        if isinstance(e, E.PerceptualEngine):
            engines.update({f"{key}.out": e.out, f"{key}.tgt": e.tgt})
        elif isinstance(e, E.Engine):
            engines[key] = e
    return {f"{k}.{s.name}": s.layer for k, e in engines.items() if e is not None for s in e.stages}


def _check_bf16_precision(case, run, mk, batch):
    """`--b200_precision bf16`: every conv layer of every engine runs single-pass (an engine that ignored the option
    would run nsplit = 3), one step's losses and gradients are finite and its losses within 1e-2 of the fp32x3 step's.
    The gradients' distance from fp32x3 is recorded, not asserted: a 2^-8 operand rounding flips LeakyReLU and max-pool
    gates, which spreads it over 1e-2 .. 1e-1 (DESIGN.md section 2)."""
    from swapnet_b200.layers import ConvLayer

    layers = _conv_layers(run[2])
    convs = {k: ly for k, ly in layers.items() if isinstance(ly, ConvLayer)}
    assert convs and all(ly.nsplit == 1 for ly in layers.values()), \
        [k for k, ly in layers.items() if ly.nsplit != 1]
    engines = sorted({k.split(".")[0] for k in convs})
    assert engines == (["Dd", "Dg", "G", "P"] if "perceptual" in case else ["Dd", "Dg", "G"]), engines
    one = {prec: _run(mk(1, prec), batch, 1) for prec in ("fp32x3", "bf16")}
    lf, lb = one["fp32x3"][0][0], one["bf16"][0][0]
    assert torch.isfinite(lb).all(), lb
    assert (lb - lf).abs().max().item() <= 1e-2 * lf.abs().max().item(), (lb, lf)
    rel = {}
    for k in ("G.flat_grad", "D.flat_grad"):
        gb, gf = one["bf16"][1][k], one["fp32x3"][1][k]
        assert torch.isfinite(gb).all(), k
        rel[k] = relmax(gb, gf)
    record(f"bf16_precision_step_vs_fp32x3[{case}]", f"{len(convs)} conv layers at nsplit 1, losses max|diff| "
           f"{(lb - lf).abs().max().item():.3e}, grads relmax " + " ".join(f"{k} {v:.3e}" for k, v in rel.items()))


# ------------------------------------------------------------------------------------------------
# whole steps
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case,precision", [
    pytest.param("warp512", "fp32x3", id="warp512"),
    pytest.param("texture_perceptual128", "fp32x3", id="texture_perceptual128"),
    pytest.param("texture_batchnorm128", "fp32x3", id="texture_batchnorm128"),
    pytest.param("warp512", "bf16", id="warp512-bf16"),
    pytest.param("texture_perceptual128", "bf16", id="texture_perceptual128-bf16"),
])
def test_identically_seeded_runs_are_bit_identical(case, precision):
    """Four steps (two eager, two graph replays) at the default learning rates: every loss, parameter, AdamW moment,
    BatchNorm buffer and gradient is bit-identical between two fresh, identically seeded models.  With
    `--b200_precision bf16` too (the default PatchGAN and the VGG16 perceptual engines single-pass)."""
    if case == "warp512":
        B, S = 2, 512
        batch = _warp_batch(B, S)
        mk = lambda det, prec=precision: _opt(B, S, b200_deterministic=det, b200_precision=prec)  # noqa: E731
    elif case == "texture_perceptual128":     # the texture model's default loss weights, seeded-random VGG16
        B, S = 2, 128
        batch = _texture_batch(B, S)
        mk = lambda det, prec=precision: _texture_opt(B, S, lambda_content=20, lambda_style=1e-8,  # noqa: E731
                                                      b200_vgg="random", b200_deterministic=det, b200_precision=prec)
    else:
        B, S = 2, 128
        batch = _texture_batch(B, S)
        mk = lambda det, prec=precision: _texture_opt(B, S, norm="batch", b200_deterministic=det,  # noqa: E731
                                                      b200_precision=prec)
    a = _run(mk(1), batch, 4)
    assert a[2].deterministic and len(a[2]._graphs) == 1
    assert a[2].nsplit == (1 if precision == "bf16" else 3)
    b = _run(mk(1), batch, 4)
    _assert_identical(a, b, case)
    if precision == "bf16":
        _check_bf16_precision(case, a, mk, batch)
    del a, b
    # evidence: the default mode on the same setup
    c, d = _run(mk(0), batch, 4), _run(mk(0), batch, 4)
    record(f"deterministic_default_mode_run_to_run[{case}{'' if precision == 'fp32x3' else ',' + precision}]",
           _differences(c, d))


def _graph_vs_eager(precision):
    B, S = 2, 64
    batch = _warp_batch(B, S)
    g = _run(_opt(B, S, b200_graph=1, b200_deterministic=1, b200_precision=precision), batch, 5)
    e = _run(_opt(B, S, b200_graph=0, b200_deterministic=1, b200_precision=precision), batch, 5)
    assert len(g[2]._graphs) == 1 and not e[2]._graphs
    assert g[2].nsplit == e[2].nsplit == (1 if precision == "bf16" else 3)
    _assert_identical(g, e, f"graph vs eager ({precision})")


def test_graph_replay_is_bit_identical_to_eager_steps():
    """With non-zero learning rates, five steps with b200_graph=1 (two eager, three replays) equal five eager steps."""
    _graph_vs_eager("fp32x3")


def test_graph_replay_is_bit_identical_to_eager_steps_at_bf16_precision():
    """The same with `--b200_precision bf16`: the single-pass plans replay bit for bit."""
    _graph_vs_eager("bf16")


def test_agrees_with_the_default_mode():
    """One step from the same weights: losses and gradients within 1e-5 relative of the default mode."""
    B, S = 2, 64
    batch = _warp_batch(B, S)
    d = _run(_opt(B, S, b200_deterministic=1, lr=0.0, d_lr=0.0), batch, 1)
    n = _run(_opt(B, S, b200_deterministic=0, lr=0.0, d_lr=0.0), batch, 1)
    assert d[2].deterministic and not n[2].deterministic
    ld, ln = d[0][0], n[0][0]
    assert ((ld - ln).abs() <= 1e-5 * ln.abs()).all(), (ld, ln)
    for k in ("G.flat_grad", "D.flat_grad"):
        assert relmax(d[1][k], n[1][k]) < 1e-5, (k, relmax(d[1][k], n[1][k]))


def test_torch_flag_selects_the_mode_and_the_option_overrides_it():
    from swapnet_b200.models import create_model

    B, S = 1, 64
    with torch_deterministic(True):
        assert create_model(_opt(B, S)).deterministic
        assert not create_model(_opt(B, S, b200_deterministic=0)).deterministic
    with torch_deterministic(False):
        assert not create_model(_opt(B, S)).deterministic
        assert create_model(_opt(B, S, b200_deterministic=1)).deterministic


# ------------------------------------------------------------------------------------------------
# parity with the fp64 oracle (the existing protocol, with the mode selected through torch's flag)
# ------------------------------------------------------------------------------------------------
def _models_built(monkeypatch):
    """Record every model create_model() builds (the oracle protocols build their own)."""
    import swapnet_b200.models as SM

    built, real = [], SM.create_model

    def create(opt):
        m = real(opt)
        built.append(m)
        return m

    monkeypatch.setattr(SM, "create_model", create)
    return built


def test_warp_step_parity_in_deterministic_mode(monkeypatch):
    built = _models_built(monkeypatch)
    with torch_deterministic(True):
        _warp_step_vs_oracle(2, 64, "eval", tag="_deterministic")
    assert built and all(m.deterministic for m in built)


@pytest.mark.parametrize("perceptual", [False, True])
def test_texture_step_parity_in_deterministic_mode(monkeypatch, perceptual):
    built = _models_built(monkeypatch)
    with torch_deterministic(True):
        _texture_step_vs_oracle(2, 64, perceptual, tag="_deterministic")
    assert built and all(m.deterministic for m in built)


@pytest.mark.parametrize("model", ["warp", "texture_perceptual"])
def test_strict_torch_flag_runs_eager_and_replayed_steps(model):
    """torch.use_deterministic_algorithms(True) without warn_only — the flag users set — selects the mode, and no torch
    op of the step raises under it, in the eager steps or the graph capture."""
    from swapnet_b200.models import create_model

    B, S = 2, 64
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        if model == "warp":
            opt, batch = _opt(B, S), _warp_batch(B, S)
        else:
            opt = _opt(B, S, model="texture", name="texture", netG="swapnet", lambda_l1=10, lambda_content=20,
                       lambda_style=1e-8, b200_vgg="random")
            batch = _texture_batch(B, S)
        torch.manual_seed(0)
        m = create_model(opt)
        m.setup(opt)
        assert m.deterministic
        for _ in range(3):
            m.set_input(batch)
            m.optimize_parameters()
        assert len(m._graphs) == 1
        losses = m.get_current_losses()
        assert all(v == v for v in losses.values()), losses
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


# ------------------------------------------------------------------------------------------------
# kernel level: each converted reduction, launched repeatedly on the same inputs
# ------------------------------------------------------------------------------------------------
def _repeat(fn, out, times=4):
    res = []
    for _ in range(times):
        out.zero_()
        fn()
        torch.cuda.synchronize()
        res.append(out.detach().clone())
    for r in res[1:]:
        assert torch.equal(r, res[0])
    return res[0]


def _planes(n, h, w, c, fmt, g, scale=1.0):
    """(split planes [n,h,w,c] of a seeded random fp32 tensor, that NHWC tensor on the CPU)"""
    from swapnet_b200 import ops

    src = torch.randn(n, h, w, c, generator=g) * scale
    p = ops.Planes(n, h, w, c, dev(), fmt=fmt)
    ops.pack_planes(src.to(dev()), p, nhwc=True)
    return p, src


@pytest.mark.parametrize("kind,cin,cout,hw,n,nsplit", at_both_nsplits([("conv4s2", 64, 64, 128, 4),
                                                                        ("conv4s2", 32, 64, 128, 2),
                                                                        ("conv3r", 128, 16, 32, 2)]))
def test_wgrad_plan_repeats_bit_identically(kind, cin, cout, hw, n, nsplit):
    """A deterministic weight-gradient plan (split-K >= 8; two cases with the narrow grouped-Y layout) gives the same bits
    on every launch, stays within test_kernels_gpu's 1e-4 bound of the fp64 product, and within 1e-5 of the default
    (atomic) plan.  Single-pass (nsplit = 1): within 1.5e-5 of the fp64 product of the bf16 operands it reads."""
    import torch.nn.functional as F

    from swapnet_b200 import lowering as L
    from swapnet_b200 import ops
    from swapnet_b200.layers import ConvLayer

    g = torch.Generator().manual_seed(3)
    in_h = hw + 2 if kind == "conv3r" else hw
    x = ops.Planes(n, in_h, in_h, L.padc(cin), dev(), dual=True)
    xsrc = torch.randn(n, L.padc(cin), in_h, in_h, generator=g)
    ops.pack_planes(xsrc.to(dev()), x)
    w = (torch.randn(cout, cin, 3 if kind == "conv3r" else 4, 3 if kind == "conv3r" else 4, generator=g) * 0.05).to(dev())
    outs = {}
    for det in (True, False):
        ly = ConvLayer(kind, w, None, x, nsplit=nsplit, det_ws=ops.DetWorkspace(dev()) if det else None)
        dyc = max(L.padc(cout), 64 if x.c < 64 else 16)
        dy, dysrc = _planes(n, ly.out_h, ly.out_w, dyc, ops.FMT_BF16, torch.Generator().manual_seed(5))
        gw = torch.zeros_like(w)
        ly.bind_backward(dy, None, gw)
        if det:
            geo = (ctypes.c_int * 6)()
            ops._lib.load().sn_plan_geometry(ly.wgrad_plan.handle, geo)
            ks, y_chunk = geo[3], geo[5]
            assert ly.wgrad_plan.workspace_bytes > 0
            # the narrow cases must take the grouped narrow-Y store path (16/32-channel Y rows)
            assert (y_chunk < 64) == (cin < 64 or cout < 64), (y_chunk, cin, cout)
        outs[det] = _repeat(lambda: ly.backward(dgrad=False, wgrad=True, bias=False), gw, 4 if det else 1)
    xr = xsrc[:, :cin].double()
    dyr = dysrc[..., :cout].permute(0, 3, 1, 2).double()
    wr = w.cpu().double().requires_grad_()
    yr = F.conv2d(xr, wr) if kind == "conv3r" else F.conv2d(xr, wr, stride=2, padding=1)
    (gw64,) = torch.autograd.grad(yr, wr, dyr)
    e64 = relmax(outs[True].cpu(), gw64)
    tag = f"det_wgrad[{kind},{cin},{cout},{hw}" + ("]" if nsplit == 3 else ",nsplit=1]")
    if nsplit == 3:
        record(tag, f"ksplit {ks}, y_chunk {y_chunk}, vs fp64 {e64:.2e}, "
               f"vs default relmax {relmax(outs[True], outs[False]):.2e}")
        assert e64 < 1e-4, e64
    else:   # ly: the atomic plan's layer, bound to the same operand values
        e_m, sep = check_single_pass(tag, outs[True], model_wgrad(ly), gw64, 1.5e-5, SP_SEP_BF16)
        record(tag, f"ksplit {ks}, y_chunk {y_chunk}, vs operand model {e_m:.2e} (model vs exact {sep:.2e}), "
               f"vs default relmax {relmax(outs[True], outs[False]):.2e}")
    assert relmax(outs[True], outs[False]) < 1e-5
    if kind == "conv4s2" and cin == 64:
        assert ks >= 8


def test_reductions_repeat_bit_identically():
    """plane statistics, the norm backward reduction, both bias-gradient kernels, the loss sums, the one-channel
    logits' weight gradient and the style term's Gram rows: repeated launches with a workspace give the same bits, close
    to the atomic versions."""
    from swapnet_b200 import ops

    g = torch.Generator().manual_seed(11)
    ws = ops.DetWorkspace(dev())
    n, h, w, c = 4, 64, 64, 64
    y = torch.randn(n, h, w, c, generator=g).to(dev())
    st = torch.zeros(n, c, 2, dtype=torch.float64, device=dev())
    a = _repeat(lambda: ops.plane_stats(y, c, st, ws=ws), st)
    assert relmax(a, _repeat(lambda: ops.plane_stats(y, c, st), st, 1)) < 1e-12
    a = _repeat(lambda: ops.plane_sums(y, c, st, ws=ws), st)
    assert relmax(a, _repeat(lambda: ops.plane_sums(y, c, st), st, 1)) < 1e-12
    # norm backward reduce (V = 4 and V = 1 instantiations: c = 64 and c = 19)
    for cc in (64, 19):
        yy = y[..., :cc].contiguous() if cc % 4 == 0 else torch.randn(n, h, w, cc, generator=g).to(dev())
        s2 = torch.zeros(n, cc, 2, dtype=torch.float64, device=dev())
        ops.plane_stats(yy, cc, s2)
        src = torch.randn(n, h, w, cc, generator=g).to(dev())
        dy = ops.Planes(n, h, w, 64, dev(), fmt=ops.FMT_BF16)
        gs = torch.zeros(n, cc, 2, dtype=torch.float64, device=dev())
        outs = []
        for wsx in (ws, None):
            res = []
            for _ in range(3):
                ops.norm_act_bwd([ops.GradSrc(src)], yy, cc, s2, ops.ACT_LRELU, dy, gs, ws=wsx)
                torch.cuda.synchronize()
                res.append((gs.clone(), dy.hi.clone(), dy.lo.clone()))
            if wsx is not None:
                for r in res[1:]:
                    assert all(torch.equal(u, v) for u, v in zip(r, res[0])), f"norm_act_bwd c={cc}"
            outs.append(res[0][0])
        assert relmax(outs[0], outs[1]) < 1e-9
    # bias gradient: the V = 8 instantiation (c = 64) and the V = 1 one (odd channel offset)
    dyp, _ = _planes(n, h, w, 64, ops.FMT_BF16, g)
    scratch = torch.zeros(64, dtype=torch.float64, device=dev())
    for view, cc in ((dyp, 64), (dyp.slice(4, 19), 19)):
        db = torch.zeros(cc, device=dev())
        a = _repeat(lambda: ops.bias_grad(view, cc, scratch, db, ws=ws), db)
        assert relmax(a, _repeat(lambda: ops.bias_grad(view, cc, scratch, db), db, 1)) < 1e-6
    # losses
    acc = torch.zeros(2, dtype=torch.float64, device=dev())
    pred = torch.randn(2 * 3 * 30 * 30, generator=g).to(dev())
    dpred = torch.zeros_like(pred)
    for obj in (ops.GAN_BCE, ops.GAN_MSE, ops.GAN_WGAN):
        t = (1.0, -1.0) if obj == ops.GAN_WGAN else (0.1, 0.9)
        a = _repeat(lambda: ops.gan_loss_fwd_bwd(obj, pred, 2, t, 0.5, acc, dpred, ws=ws), acc)
        assert relmax(a, _repeat(lambda: ops.gan_loss_fwd_bwd(obj, pred, 2, t, 0.5, acc, dpred), acc, 1)) < 1e-12
    fk = torch.randn(n, h, w, 3, generator=g).to(dev())
    tg = torch.randn(n, 3, h, w, generator=g).to(dev())
    gr = torch.zeros(n, h, w, 3, device=dev())
    a = _repeat(lambda: ops.l1_loss_fwd_bwd(fk, 3, tg, 10.0, acc[:1], gr, ws=ws), acc)
    assert relmax(a, _repeat(lambda: ops.l1_loss_fwd_bwd(fk, 3, tg, 10.0, acc[:1], gr), acc, 1)) < 1e-12
    logits = torch.tanh(torch.randn(n, h, w, 19, generator=g)).to(dev())
    lab = ops.SegMap(torch.randint(0, 19, (n, h, w), generator=g).to(torch.uint8).to(dev()), 19)
    hd = ops.Planes(n, h, w, 32, dev(), fmt=ops.FMT_BF16)
    a = _repeat(lambda: ops.ce_tanh_bwd(logits, 19, lab, 100.0, acc[:1], [], hd, ws=ws), acc)
    assert relmax(a, _repeat(lambda: ops.ce_tanh_bwd(logits, 19, lab, 100.0, acc[:1], [], hd), acc, 1)) < 1e-12
    # the PatchGAN logits' weight gradient (one output channel, csrc/patch_logits.cu)
    x, _ = _planes(n, 31, 31, 512, ops.FMT_F16, g)
    dyl, _ = _planes(n, 30, 30, 16, ops.FMT_F16, g)
    dw = torch.zeros(1, 512, 4, 4, device=dev())
    a = _repeat(lambda: ops.to_one_wgrad(x, dyl, 1, dw, ws=ws), dw)
    assert relmax(a, _repeat(lambda: ops.to_one_wgrad(x, dyl, 1, dw), dw, 1)) < 1e-5
    # perceptual losses: the content term of one VGG tap and the style term's Gram matrices (NHWC fakes, NCHW targets)
    yo, yt = torch.randn(n, 32, 32, 256, generator=g).to(dev()), torch.randn(n, 32, 32, 256, generator=g).to(dev())
    gf = torch.zeros(n, 32, 32, 256, device=dev())
    a = _repeat(lambda: ops.feat_loss_fwd_bwd(yo, yt, 256, 20.0 / yo.numel(), 2.0, acc[:1], gf, ws=ws), acc)
    assert relmax(a, _repeat(lambda: ops.feat_loss_fwd_bwd(yo, yt, 256, 20.0 / yo.numel(), 2.0, acc[:1], gf),
                             acc, 1)) < 1e-12
    for img, nhwc in ((torch.randn(8, 256, 256, 3, generator=g), True), (torch.randn(8, 3, 256, 256, generator=g), False)):
        img = img.to(dev())
        gm = torch.zeros(24, 24, dtype=torch.float64, device=dev())
        a = _repeat(lambda: ops.gram_rows(img, img, nhwc, gm, ws=ws), gm)
        assert relmax(a, _repeat(lambda: ops.gram_rows(img, img, nhwc, gm), gm, 1)) < 1e-9
        x64 = (img.permute(0, 3, 1, 2) if nhwc else img).reshape(24, -1).double()
        assert relmax(a, x64 @ x64.T) < 1e-6
    record("det_slot_workspace_bytes[kernel tests]", ws.nbytes)
