"""`--optimizer_G / --optimizer_D AdaBound` on the GPU: the fused kernel against the fp64 restatement of the update
(tests/tools/adabound_oracle.py), its three clamp regimes, whole plugin steps of both stages whose optimizer launches are
checked against the oracle on the step's own gradients, graph replay against eager steps bit for bit, and a checkpoint
round trip in the `adabound` package's state_dict layout."""
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "tools"))

import adabound_oracle as AO  # noqa: E402
from test_deterministic_gpu import _assert_identical, _run, _texture_batch, _texture_opt, _warp_batch  # noqa: E402
from test_engine_gpu import _opt, dev, record, relmax  # noqa: E402

BETAS = (0.9, 0.999)


def _hyper_dev(*args):
    from swapnet_b200 import ops

    return torch.tensor(ops.adabound_hyper(*args), dtype=torch.float32, device=dev())


# ---------------------------------------------------------------------------------------------
# kernel
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gscale", [1.0, 0.5])
@pytest.mark.parametrize("wd", [0.0, 0.01])
@pytest.mark.parametrize("n", [1, 3, 4, 1027, 4 * 10 ** 6 + 5])
def test_kernel_matches_fp64_oracle(n, wd, gscale):
    """Five consecutive steps on random gradients, the learning rate moved off base_lr after the second: p, m and v
    within 1e-6 (relative to the largest element) of the oracle run in fp64 from the same fp32 start.  The vector body
    and the scalar tail are both covered (n % 4 in {0, 1, 3}); with gscale = 1 the entry point that takes its scalars by
    value leaves the same bits as the one that reads them from device memory."""
    from swapnet_b200 import ops

    g = torch.Generator().manual_seed(n % 1000 + int(wd * 100) + int(gscale * 10))
    p0 = torch.randn(n, generator=g)
    base_lr, final_lr = 4e-4, 0.1
    bufs = {k: [p0.to(dev()), torch.zeros(n, device=dev()), torch.zeros(n, device=dev())] for k in ("dev", "val")}
    P, M, V = p0.double(), torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64)
    worst = 0.0
    for t in range(1, 6):
        lr = base_lr if t <= 2 else 0.5 * base_lr
        grad = torch.randn(n, generator=g) * (2.0 / gscale)
        gd = grad.to(dev())
        p, m, v = bufs["dev"]
        ops.adabound_step_dev(p, gd, m, v, _hyper_dev(lr, base_lr, *BETAS, AO.EPS, wd, final_lr, AO.GAMMA, t, gscale))
        AO.step(P, grad.double(), M, V, t, lr, BETAS, final_lr, weight_decay=wd, base_lr=base_lr, gscale=gscale)
        torch.cuda.synchronize()
        for name, got, want in (("p", p, P), ("m", m, M), ("v", v, V)):
            err = relmax(got.cpu(), want)
            worst = max(worst, err)
            assert err < 1e-6, f"{name} after step {t}: relmax {err:.3e}"
        if gscale == 1.0:
            pv, mv, vv = bufs["val"]
            ops.adabound_step(pv, gd, mv, vv, lr, base_lr, *BETAS, AO.EPS, wd, final_lr, AO.GAMMA, t)
            torch.cuda.synchronize()
            assert torch.equal(pv, p) and torch.equal(mv, m) and torch.equal(vv, v), f"entry points differ at step {t}"
    record(f"adabound_kernel_vs_fp64[n={n},wd={wd},gscale={gscale}]", f"{worst:.3e}")


def test_kernel_clamps_to_both_bounds():
    """gamma = 0.1 at step 1 puts the bounds at 0.0091 and 1.1 around a raw step size of 0.01 / |g|: gradients above
    1.1 are lifted to `lower`, gradients below 0.0091 are cut to `upper`, the rest pass.  Starting from p = 0 the step
    size each element got is -p / m."""
    from swapnet_b200 import ops

    n, lr, final_lr, gamma = 8192, 1e-3, 0.1, 0.1
    g = torch.Generator().manual_seed(5)
    grad = torch.randn(n, generator=g)
    grad[::7] *= 1e-2
    step_size, lower, upper = AO.scalars(1, lr, lr, BETAS, final_lr, gamma)
    P, M, V = (torch.zeros(n, dtype=torch.float64) for _ in range(3))
    eta = AO.step(P, grad.double(), M, V, 1, lr, BETAS, final_lr, gamma)
    raw = step_size / (V.sqrt() + AO.EPS)
    at_lower, at_upper = raw < lower * (1 - 1e-4), raw > upper * (1 + 1e-4)
    free = (raw > lower * (1 + 1e-4)) & (raw < upper * (1 - 1e-4))
    counts = (int(at_lower.sum()), int(at_upper.sum()), int(free.sum()))
    record("adabound_clamp_regimes[lower,upper,neither]", counts)
    assert min(counts) >= 50 and sum(counts) >= n - 8, counts
    p, m, v = (torch.zeros(n, device=dev()) for _ in range(3))
    ops.adabound_step(p, grad.to(dev()), m, v, lr, lr, *BETAS, AO.EPS, 0.0, final_lr, gamma, 1)
    torch.cuda.synchronize()
    got = (-p / m).cpu().double()
    assert torch.allclose(got[at_lower], torch.full_like(got[at_lower], lower), rtol=1e-6, atol=0)
    assert torch.allclose(got[at_upper], torch.full_like(got[at_upper], upper), rtol=1e-6, atol=0)
    assert torch.allclose(got[free], raw[free], rtol=2e-6, atol=0)
    assert torch.allclose(got, eta, rtol=2e-6, atol=0)
    assert got.min().item() >= lower * (1 - 1e-6) and got.max().item() <= upper * (1 + 1e-6)


def test_fused_adabound_steps_per_tensor_like_the_oracle():
    """FusedAdaBound.step() over four parameters of one flat buffer against the oracle run tensor by tensor, four steps
    with a scheduler halving the rate after the second; at step 2 the state_dict moves into a second instance, which
    carries on and ends on the same bits."""
    from swapnet_b200.optim import FusedAdaBound, flatten_parameters

    def make(values):
        params = [torch.nn.Parameter(v.clone().to(dev())) for v in values]
        o = FusedAdaBound(params, flatten_parameters(params), lr=4e-4, weight_decay=0.01, final_lr=0.05)
        o.flat_grad = torch.zeros_like(o.flat_param)
        return o

    g = torch.Generator().manual_seed(2)
    start = [torch.randn(s, generator=g) for s in ((64, 3, 4, 4), (19,), (128, 64, 3, 3), (7,))]
    mine, twin = make(start), None
    ref = [(p.double(), torch.zeros_like(p, dtype=torch.float64), torch.zeros_like(p, dtype=torch.float64)) for p in start]
    for t in range(1, 5):
        lr = 4e-4 if t <= 2 else 2e-4
        grads = [torch.randn(p.shape, generator=g) * 10.0 ** (1 - t) for p in start]
        flat_g = torch.cat([x.reshape(-1) for x in grads]).to(dev())
        for o in (mine, twin):
            if o is not None:
                o.param_groups[0]["lr"] = lr
                o.flat_grad.copy_(flat_g)
                o.step()
        for (P, M, V), grad, p in zip(ref, grads, mine.param_groups[0]["params"]):
            AO.step(P, grad.double(), M, V, t, lr, BETAS, 0.05, weight_decay=0.01, base_lr=4e-4)
            st = mine.state[p]
            assert st["step"] == t and relmax(p.detach().cpu(), P) < 1e-6
            assert relmax(st["exp_avg"].cpu(), M) < 1e-6 and relmax(st["exp_avg_sq"].cpu(), V) < 1e-6
        if t == 2:
            twin = make([p.detach().cpu() for p in mine.param_groups[0]["params"]])
            twin.load_state_dict(mine.state_dict())
            assert twin._step == 2 and torch.equal(twin.exp_avg_sq, mine.exp_avg_sq)
    for name in ("flat_param", "exp_avg", "exp_avg_sq"):
        assert torch.equal(getattr(mine, name), getattr(twin, name)), name


# ---------------------------------------------------------------------------------------------
# plugin steps
# ---------------------------------------------------------------------------------------------
def _spy(optimizer, log):
    """Snapshot (p, g, m, v) right before every launch of `optimizer` (eager steps only: a replay does not call it)."""
    real = optimizer.launch

    def launch(hyper_dev):
        log.append(tuple(t.detach().clone() for t in (optimizer.flat_param, optimizer.flat_grad, optimizer.exp_avg,
                                                      optimizer.exp_avg_sq)))
        real(hyper_dev)

    optimizer.launch = launch


def _expected(kind, snap, t, lr, wd, final_lr):
    p, g, m, v = (x.cpu().double() for x in snap)
    if kind == "AdaBound":
        AO.step(p, g, m, v, t, lr, BETAS, final_lr, weight_decay=wd)
        return p, m, v
    p.requires_grad_()
    opt = torch.optim.AdamW([p], lr=lr, betas=BETAS, eps=1e-8, weight_decay=wd)
    opt.state[p] = {"step": torch.tensor(float(t - 1)), "exp_avg": m, "exp_avg_sq": v}
    p.grad = g
    opt.step()
    return p.detach(), m, v


@pytest.mark.parametrize("optG,optD", [("AdaBound", "AdaBound"), ("AdamW", "AdaBound"), ("AdaBound", "AdamW")])
@pytest.mark.parametrize("stage", ["warp", "texture"])
def test_step_updates_match_oracle_on_the_steps_own_gradients(stage, optG, optD):
    """Two optimize_parameters() calls at 64 x 64, batch 2.  Each optimizer launch of each step is checked on its own
    inputs: the parameters and both moments it leaves equal the oracle's update (fp64 AdaBound, or torch.optim.AdamW for
    the network that keeps AdamW) of the parameters, gradients and moments it found, within 1e-6."""
    from swapnet_b200.models import create_model
    from swapnet_b200.optim import FusedAdaBound, FusedAdamW

    B, S, final_lr = 2, 64, 0.05
    over = dict(optimizer_G=optG, optimizer_D=optD, final_lr=final_lr)
    opt, batch = (_opt(B, S, **over), _warp_batch(B, S)) if stage == "warp" else \
        (_texture_opt(B, S, **over), _texture_batch(B, S))
    torch.manual_seed(0)
    model = create_model(opt)
    model.setup(opt)
    cls = {"AdaBound": FusedAdaBound, "AdamW": FusedAdamW}
    assert type(model.optimizer_G) is cls[optG] and type(model.optimizer_D) is cls[optD]
    logs = {"G": [], "D": []}
    _spy(model.optimizer_G, logs["G"])
    _spy(model.optimizer_D, logs["D"])
    torch.manual_seed(11)
    worst = 0.0
    for t in (1, 2):
        model.set_input(batch)
        model.optimize_parameters()
        torch.cuda.synchronize()
        for net, kind, lr, wd in (("G", optG, opt.lr, opt.weight_decay), ("D", optD, opt.d_lr, opt.d_weight_decay)):
            o = getattr(model, "optimizer_" + net)
            assert len(logs[net]) == t and logs[net][-1][1].abs().max().item() > 0
            want = _expected(kind, logs[net][-1], t, lr, wd, final_lr)
            for name, got, ref in zip("pmv", (o.flat_param, o.exp_avg, o.exp_avg_sq), want):
                err = relmax(got.cpu(), ref)
                worst = max(worst, err)
                assert err < 1e-6, f"{net}.{name} after step {t}: relmax {err:.3e}"
            moved = (o.flat_param - logs[net][-1][0]).abs().max().item()
            assert moved > 0.1 * lr, (net, t, moved)
            steps = [st["step"] for st in o.state_dict()["state"].values()]
            assert all(int(s) == t and (type(s) is int) == (kind == "AdaBound") for s in steps)
    assert not model._graphs
    losses = model.get_current_losses()
    assert all(v == v for v in losses.values()), losses
    record(f"adabound_step_vs_oracle[{stage},G={optG},D={optD}]", f"{worst:.3e}")


def test_default_options_keep_adamw_and_other_names_are_refused():
    from swapnet_b200.models import create_model
    from swapnet_b200.optim import FusedAdamW

    model = create_model(_opt(1, 64))
    assert type(model.optimizer_G) is FusedAdamW and type(model.optimizer_D) is FusedAdamW
    with pytest.raises(NotImplementedError, match="SGD"):
        create_model(_opt(1, 64, optimizer_G="SGD"))


@pytest.mark.parametrize("optG", ["AdaBound", "AdamW"])
def test_graph_replay_is_bit_identical_to_eager_steps(optG):
    """Three steps with --b200_graph 1 (eager, eager, replay) equal three eager steps under --b200_deterministic 1, and
    a second graph run repeats the first: the AdaBound launch is part of the captured sequence and takes the current
    step's bounds from the step-parameter buffer."""
    B, S = 2, 64
    batch = _warp_batch(B, S)
    over = dict(optimizer_G=optG, optimizer_D="AdaBound", final_lr=0.1, b200_deterministic=1)
    g = _run(_opt(B, S, b200_graph=1, **over), batch, 3)
    e = _run(_opt(B, S, b200_graph=0, **over), batch, 3)
    assert len(g[2]._graphs) == 1 and not e[2]._graphs
    assert any(k.startswith("D.adam.") and k.endswith("exp_avg_sq") for k in g[1])
    _assert_identical(g, e, "graph vs eager")
    _assert_identical(g, _run(_opt(B, S, b200_graph=1, **over), batch, 3), "graph run to run")
    assert {st["step"] for st in g[2].optimizer_D.state_dict()["state"].values()} == {3}


def test_checkpoint_round_trip_continues_the_run(tmp_path):
    """Two steps, save_checkpoint, a fresh differently seeded model, load_checkpoint_dir, one step: the same bits as the
    third step of the uninterrupted run (dropout off, --b200_deterministic 1).  The saved optimizer files have the
    adabound package's layout."""
    from swapnet_b200.models import create_model

    B, S = 2, 64
    batch = _texture_batch(B, S)

    def make(seed):
        opt = _texture_opt(B, S, optimizer_G="AdaBound", optimizer_D="AdaBound", final_lr=0.1, b200_deterministic=1,
                           b200_graph=0, checkpoints_dir=str(tmp_path))
        torch.manual_seed(seed)
        m = create_model(opt)
        m.setup(opt)
        return m.eval()

    def step(m, seed):
        torch.manual_seed(seed)        # the smooth labels of this step
        m.set_input(batch)
        m.optimize_parameters()
        torch.cuda.synchronize()

    a = make(0)
    step(a, 1)
    step(a, 2)
    a.save_checkpoint("latest")
    saved = torch.load(os.path.join(a.save_dir, "latest_optim_D.pth"))
    (group,) = saved["param_groups"]
    assert {k: group[k] for k in group if k != "params"} == dict(lr=4e-4, betas=BETAS, final_lr=0.1, gamma=1e-3,
                                                                 eps=1e-8, weight_decay=0.01, amsbound=False)
    assert all(sorted(st) == ["exp_avg", "exp_avg_sq", "step"] and st["step"] == 2 and type(st["step"]) is int
               for st in saved["state"].values())
    step(a, 3)
    b = make(5)
    assert not torch.equal(b.optimizer_G.flat_param, a.optimizer_G.flat_param)
    b.load_checkpoint_dir("latest")
    assert b.optimizer_D._step == 2 and b.optimizer_D.exp_avg.abs().max().item() > 0
    step(b, 3)
    for net in ("G", "D"):
        oa, ob = getattr(a, "optimizer_" + net), getattr(b, "optimizer_" + net)
        for name in ("flat_param", "exp_avg", "exp_avg_sq"):
            assert torch.equal(getattr(oa, name), getattr(ob, name)), (net, name)
        assert oa._step == ob._step == 3
    assert a.get_current_losses() == b.get_current_losses()
