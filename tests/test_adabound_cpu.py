"""`--optimizer_G / --optimizer_D AdaBound` on the CPU: the plain-torch restatement of the update
(tests/tools/adabound_oracle.py) against a trajectory computed by hand and against its two limits, the host half of the
fused optimizer (`sn_adabound_hyper`, the argument checks of the launch functions) against it, the `state_dict()` layout
of the `adabound` package, and the options."""
import argparse
import math
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "tools"))

import adabound_oracle as AO  # noqa: E402
from swapnet_b200 import _lib, ops  # noqa: E402
from swapnet_b200.optim import FusedAdaBound, FusedAdamW, flatten_parameters  # noqa: E402


# ---------------------------------------------------------------------------------------------
# the oracle
# ---------------------------------------------------------------------------------------------
def test_oracle_follows_a_hand_computed_trajectory():
    """Three steps of a 2-element parameter in Python floats, straight from the formulas.  gamma = 1 and b2 = 0.1 so
    that the bounds [F t/(t+1), F (t+1)/t] and the second moment move fast: at step 1 element 0 (large gradient) is
    lifted to `lower` and element 1 (small gradient) is cut to `upper`; at steps 2 and 3 neither is clipped."""
    lr, (b1, b2), F, gamma, eps, wd = 0.01, (0.5, 0.1), 0.1, 1.0, 1e-8, 0.1
    grads = [[0.4, 0.25], [-0.05, 0.3], [0.0, 0.1]]
    p, m, v = [1.0, -2.0], [0.0, 0.0], [0.0, 0.0]
    P = torch.tensor(p, dtype=torch.float64)
    M, V = torch.zeros_like(P), torch.zeros_like(P)
    clipped = []
    for t, g in enumerate(grads, 1):
        step_size = lr * math.sqrt(1 - b2 ** t) / (1 - b1 ** t)
        lower, upper = F * (1 - 1 / (gamma * t + 1)), F * (1 + 1 / (gamma * t))
        assert lower == pytest.approx(F * t / (t + 1)) and upper == pytest.approx(F * (t + 1) / t)
        for i in range(2):
            gi = g[i] + wd * p[i]
            m[i] = b1 * m[i] + (1 - b1) * gi
            v[i] = b2 * v[i] + (1 - b2) * gi * gi
            raw = step_size / (math.sqrt(v[i]) + eps)
            clipped.append("lower" if raw < lower else "upper" if raw > upper else None)
            p[i] -= min(max(raw, lower), upper) * m[i]
        AO.step(P, torch.tensor(g, dtype=torch.float64), M, V, t, lr, (b1, b2), F, gamma, eps, wd)
        assert P.tolist() == pytest.approx(p, rel=1e-14) and M.tolist() == pytest.approx(m, rel=1e-14)
        assert V.tolist() == pytest.approx(v, rel=1e-14)
        if t == 1:     # in closed form: g' = g + wd p = (0.5, 0.05), m = g'/2, eta = (lower, upper) = (0.05, 0.2)
            assert p == pytest.approx([1.0 - 0.05 * 0.25, -2.0 - 0.2 * 0.025], rel=1e-15)
    assert clipped == ["lower", "upper", None, None, None, None]


@pytest.mark.parametrize("eps", [1e-8, 0.0])
@pytest.mark.parametrize("wd", [0.0, 0.01])
def test_oracle_without_bounds_is_adam_with_l2_decay(wd, eps):
    """gamma -> 0 opens the bounds to [0, inf): what is left is Adam with the decay folded into the gradient
    (`torch.optim.Adam(weight_decay=wd)`), up to where eps sits (Adam divides it by sqrt(1 - b2^t), 31 times larger at
    t = 1): parameters within 1e-7 with eps = 1e-8, and within rounding of a step with eps = 0.  A large final_lr alone
    does not do that: it raises `lower` as well."""
    g = torch.Generator().manual_seed(3)
    p0 = torch.randn(257, dtype=torch.float64, generator=g)
    ref = p0.clone().requires_grad_()
    adam = torch.optim.Adam([ref], lr=2e-3, betas=(0.9, 0.999), eps=eps, weight_decay=wd)
    p, m, v = p0.clone(), torch.zeros_like(p0), torch.zeros_like(p0)
    for t in range(1, 6):
        grad = torch.randn(257, dtype=torch.float64, generator=g)
        before = p.clone()
        ref.grad = grad.clone()
        adam.step()
        eta = AO.step(p, grad, m, v, t, 2e-3, final_lr=0.1, gamma=1e-30, eps=eps, weight_decay=wd)
        lo, up = AO.scalars(t, 2e-3, 2e-3, (0.9, 0.999), 0.1, 1e-30)[1:]
        assert lo == 0.0 and up > 1e28 and eta.max().item() < up
        err = (p - ref.detach()).abs().max().item()
        assert err <= (1e-7 if eps else 1e-12 * (p - before).abs().max().item()), (t, err)
    big = p0.clone()
    AO.step(big, torch.ones_like(p0), torch.zeros_like(p0), torch.zeros_like(p0), 1, 2e-3, final_lr=1e6)
    assert (p0 - big).min().item() > 50.0       # lower = 1e6 * (1 - 1/1.001) ~ 999 times m = 0.1


def test_oracle_tends_to_sgd_with_momentum_at_final_lr():
    """For large t both bounds meet at final_lr * lr / base_lr: the step is that rate times the first moment."""
    g = torch.Generator().manual_seed(4)
    p0, grad = torch.randn(64, dtype=torch.float64, generator=g), torch.randn(64, dtype=torch.float64, generator=g)
    m, v = torch.randn(64, dtype=torch.float64, generator=g), torch.rand(64, dtype=torch.float64, generator=g) * 1e4
    p = p0.clone()
    AO.step(p, grad, m, v, 10 ** 9, 5e-4, final_lr=0.1, base_lr=1e-3)     # lr halved by a scheduler: F = 0.05
    lo, up = AO.scalars(10 ** 9, 5e-4, 1e-3, (0.9, 0.999), 0.1)[1:]
    assert 0.05 * (1 - 2e-6) < lo < 0.05 < up < 0.05 * (1 + 2e-6)
    assert torch.allclose(p0 - p, 0.05 * m, rtol=2e-6, atol=0)


# ---------------------------------------------------------------------------------------------
# the host half of the fused optimizer
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t", [1, 2, 1000])
def test_hyper_scalars_match_the_oracle(t):
    """sn_adabound_hyper: { 1 - b1, 1 - b2, eps, wd, step_size, lower, upper, gscale } formed in double and rounded to
    fp32 once, with a learning rate that a scheduler moved away from the one the optimizer was created with."""
    _lib.load(build_if_missing=True)
    lr, base_lr, betas, final_lr, gamma = 3e-4, 4e-4, (0.9, 0.999), 0.05, 1e-3
    got = ops.adabound_hyper(lr, base_lr, betas[0], betas[1], 1e-8, 0.01, final_lr, gamma, t, 0.5)
    step_size, lower, upper = AO.scalars(t, lr, base_lr, betas, final_lr, gamma)
    want = [1 - betas[0], 1 - betas[1], 1e-8, 0.01, step_size, lower, upper, 0.5]
    assert got == [torch.tensor(x, dtype=torch.float64).float().item() for x in want]
    assert lower < final_lr * lr / base_lr < upper
    # (float)(1 - b2), not 1.f - (float)b2: the latter is 1.3e-5 away
    assert abs(got[1] / 1e-3 - 1) < 1e-7 < abs((1.0 - torch.tensor(0.999).item()) / 1e-3 - 1)


def test_launch_functions_check_their_arguments():
    """Null or misaligned buffers, step 0, gamma <= 0, final_lr < 0 and base_lr <= 0 come back as an error code and a
    message before anything is launched (so this runs without a device)."""
    lib = _lib.load(build_if_missing=True)
    buf = torch.zeros(16)
    a = buf.data_ptr()
    assert a % 16 == 0
    ok = dict(lr=1e-3, base_lr=1e-3, b1=0.9, b2=0.999, eps=1e-8, wd=0.0, final_lr=0.1, gamma=1e-3, step=1)

    def call(p=a, n=8, **over):
        k = {**ok, **over}
        rc = lib.sn_adabound_step(p, a, a, a, n, k["lr"], k["base_lr"], k["b1"], k["b2"], k["eps"], k["wd"],
                                  k["final_lr"], k["gamma"], k["step"], None)
        return rc, lib.sn_last_error()

    for over, msg in ((dict(p=None), b"bad adabound arguments"), (dict(n=0), b"bad adabound arguments"),
                      (dict(step=0), b"bad adabound arguments"), (dict(gamma=0.0), b"gamma > 0"),
                      (dict(final_lr=-0.1), b"final_lr >= 0"), (dict(base_lr=0.0), b"base_lr > 0"),
                      (dict(p=a + 4), b"16-B aligned")):
        rc, err = call(**over)
        assert rc != 0 and msg in err, (over, rc, err)
    assert lib.sn_adabound_step_dev(a, a, a, a, 8, None, None) != 0 and b"bad adabound" in lib.sn_last_error()
    assert lib.sn_adabound_step_dev(a + 4, a, a, a, 8, a, None) != 0 and b"16-B aligned" in lib.sn_last_error()


# ---------------------------------------------------------------------------------------------
# state_dict layout
# ---------------------------------------------------------------------------------------------
def _flat_optimizer(cls, **kw):
    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Linear(3, 4), torch.nn.Linear(4, 2))
    params = list(net.parameters())
    return cls(params, flatten_parameters(params), **kw), params


def test_state_dict_has_the_package_layout():
    opt, params = _flat_optimizer(FusedAdaBound, lr=4e-4, betas=(0.9, 0.999), final_lr=0.05, weight_decay=0.01)
    assert opt.base_lrs == [4e-4]
    sd = opt.state_dict()
    (group,) = sd["param_groups"]
    assert group == dict(lr=4e-4, betas=(0.9, 0.999), final_lr=0.05, gamma=1e-3, eps=1e-8, weight_decay=0.01,
                         amsbound=False, params=[0, 1, 2, 3])
    assert sorted(sd["state"]) == [0, 1, 2, 3]
    for i, p in enumerate(params):
        st = sd["state"][i]
        assert sorted(st) == ["exp_avg", "exp_avg_sq", "step"]
        assert type(st["step"]) is int and st["step"] == 0
        assert st["exp_avg"].shape == p.shape and st["exp_avg_sq"].dtype == torch.float32
    _lib.load(build_if_missing=True)
    opt.param_groups[0]["lr"] = 2e-4                         # a scheduler's doing: base_lrs stays
    hyper = opt.advance(0.5)
    assert all(type(st["step"]) is int and st["step"] == 1 for st in opt.state_dict()["state"].values())
    assert hyper == ops.adabound_hyper(2e-4, 4e-4, 0.9, 0.999, 1e-8, 0.01, 0.05, 1e-3, 1, 0.5)
    # AdamW keeps torch's layout: a float tensor
    adamw, _ = _flat_optimizer(FusedAdamW, lr=1e-4)
    assert all(torch.is_tensor(st["step"]) for st in adamw.state_dict()["state"].values())
    assert sorted(adamw.state_dict()["param_groups"][0]) == ["betas", "eps", "lr", "params", "weight_decay"]


def test_a_state_dict_in_the_package_layout_loads():
    """A dict written the way adabound.AdaBound.state_dict() writes it (Python int steps, per-parameter moments): the
    moments land in the flat buffers, the step count carries on, and saving again gives the same dict back."""
    opt, params = _flat_optimizer(FusedAdaBound, lr=1e-3)
    g = torch.Generator().manual_seed(1)
    state = {i: {"step": 7, "exp_avg": torch.randn(p.shape, generator=g), "exp_avg_sq": torch.rand(p.shape, generator=g)}
             for i, p in enumerate(params)}
    group = dict(lr=5e-4, betas=(0.5, 0.99), final_lr=0.2, gamma=2e-3, eps=1e-7, weight_decay=0.02, amsbound=False,
                 params=[0, 1, 2, 3])
    opt.load_state_dict({"state": state, "param_groups": [group]})
    assert torch.equal(opt.exp_avg, torch.cat([state[i]["exp_avg"].reshape(-1) for i in range(4)]))
    assert torch.equal(opt.exp_avg_sq, torch.cat([state[i]["exp_avg_sq"].reshape(-1) for i in range(4)]))
    for p in params:       # the exposed moments are views of the flat buffers again
        lo, hi = opt.exp_avg.data_ptr(), opt.exp_avg.data_ptr() + 4 * opt.exp_avg.numel()
        assert lo <= opt.state[p]["exp_avg"].data_ptr() < hi
    again = opt.state_dict()
    assert again["param_groups"] == [group]
    for i in range(4):
        assert again["state"][i]["step"] == 7 and type(again["state"][i]["step"]) is int
        assert torch.equal(again["state"][i]["exp_avg"], state[i]["exp_avg"])
    _lib.load(build_if_missing=True)
    assert opt.base_lrs == [1e-3]                            # not part of the dict, as in the package
    assert opt.advance() == ops.adabound_hyper(5e-4, 1e-3, 0.5, 0.99, 1e-7, 0.02, 0.2, 2e-3, 8, 1.0)
    group["amsbound"] = True
    with pytest.raises(NotImplementedError, match="AMSBound"):
        opt.load_state_dict({"state": state, "param_groups": [group]})


def test_constructor_refuses_rates_the_update_cannot_use():
    for kw in (dict(lr=0.0), dict(final_lr=-1.0), dict(gamma=0.0)):
        with pytest.raises(ValueError, match="AdaBound needs"):
            _flat_optimizer(FusedAdaBound, **kw)


# ---------------------------------------------------------------------------------------------
# options
# ---------------------------------------------------------------------------------------------
def test_options_select_adabound_per_network():
    from swapnet_b200.models import base_gan

    parser = argparse.ArgumentParser()
    parser.add_argument("--weight_decay", type=float, default=0)
    base_gan.BaseGAN.modify_commandline_options(parser, True)
    base_gan.adabound_modifier(parser)
    opt = parser.parse_args(["--optimizer_D", "AdaBound", "--final_lr", "0.05"])
    assert (opt.optimizer_G, opt.optimizer_D, opt.final_lr, opt.b1, opt.b2) == ("AdamW", "AdaBound", 0.05, 0.9, 0.999)
    assert parser.parse_args([]).final_lr == 0.1 and parser.parse_args([]).optimizer_D == "AdamW"
    with pytest.raises(SystemExit):
        parser.parse_args(["--optimizer_G", "SGD"])

    torch.manual_seed(0)
    G, Dn = torch.nn.Linear(3, 4), torch.nn.Linear(4, 2)
    optG, optD = base_gan.define_optimizer(G, opt, "G"), base_gan.define_optimizer(Dn, opt, "D")
    assert type(optG) is FusedAdamW and type(optD) is FusedAdaBound
    gd = optD.param_groups[0]
    assert (gd["lr"], gd["weight_decay"], gd["betas"], gd["final_lr"]) == (4e-4, 0.01, (0.9, 0.999), 0.05)
    assert (gd["gamma"], gd["eps"], gd["amsbound"]) == (1e-3, 1e-8, False)
    assert Dn.weight.data_ptr() == optD.flat_param.data_ptr()
    opt.optimizer_G = "SGD"
    with pytest.raises(NotImplementedError, match="SGD"):
        base_gan.define_optimizer(G, opt, "G")


def test_launcher_parses_adabound_options_through_the_reference_parser(tmp_path):
    """`python -m swapnet_b200.run <script> --optimizer_D AdaBound --final_lr 0.05`: the reference's option code accepts
    the choice through the plugin's parser and its own `optimizers.get_options_modifier` contributes --final_lr."""
    import json

    from test_dropin_launcher import REF, make_dataset, run

    if not os.path.isfile(os.path.join(REF, "train.py")):
        pytest.skip("the reference checkout is not mounted")
    probe = tmp_path / "probe.py"
    probe.write_text(
        "import json\n"
        "from options.train_options import TrainOptions\n"
        "opt = TrainOptions().parse()\n"
        "print('PROBE', json.dumps({k: getattr(opt, k) for k in ('optimizer_G', 'optimizer_D', 'final_lr', 'b1', 'b2')}))\n")
    data = tmp_path / "data"
    make_dataset(str(data))
    r = run([sys.executable, "-m", "swapnet_b200.run", str(probe), "--name", "p", "--model", "warp", "--dataroot",
             str(data), "--checkpoints_dir", str(tmp_path / "ck"), "--no_confirm", "--optimizer_D", "AdaBound",
             "--final_lr", "0.05"], cwd=REF, extra_path=[REF])
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("PROBE ")]
    assert r.returncode == 0 and line, (r.stdout[-2000:], r.stderr[-3000:])
    assert json.loads(line[-1][6:]) == dict(optimizer_G="AdamW", optimizer_D="AdaBound", final_lr=0.05, b1=0.9, b2=0.999)
