"""`--model pix2pix` and `--model texture --netG unet_128` without a GPU: the option surface against the reference's
parser, the registry, the networks' keys and seeded inits and the fp64 oracle's training step against the reference
(tests/golden/pix2pix_128.pt, tests/golden/texture_unet_128.pt), the --gan_mode mapping, the label-draw counts and the
refusals."""
import os
import sys
from argparse import ArgumentParser, Namespace

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import ref_harness as RH  # noqa: E402
from swapnet_b200 import modules as M  # noqa: E402
from swapnet_b200 import ops  # noqa: E402
from swapnet_b200.models import base_gan  # noqa: E402
from swapnet_b200.models.pix2pix_model import PIX2PIX_GAN_OBJECTIVES, Pix2PixModel  # noqa: E402

# the reference's Pix2PixModel and TextureModel(--netG unet_128): seeded inits and one step (tests/tools/make_golden_unet.py)
GOLD = {kind: torch.load(os.path.join(ROOT, "tests", "golden", f"{kind}.pt"))
        for kind in ("pix2pix_128", "texture_unet_128")}


def parse(modifier, is_train, args=()):
    p = ArgumentParser()
    p.add_argument("--lr", type=float, default=0.01)          # train_options.py:101-106
    return modifier(p, is_train).parse_args(list(args))


def test_pix2pix_options_and_defaults():
    o = parse(Pix2PixModel.modify_commandline_options, True)
    assert (o.norm, o.netG, o.lambda_l1, o.beta1, o.lr, o.gan_mode, o.pool_size) == \
        ("instance", "unet_128", 10, 0.5, 0.01, "vanilla", 0)     # --norm's own default wins in training, as there
    for flag in ("d_lr", "d_weight_decay", "lambda_discriminator"):
        assert not hasattr(o, flag)
    assert (o.b200_graph, o.b200_sync_bn, o.b200_precision) == (1, 0, "fp32x3")
    t = parse(Pix2PixModel.modify_commandline_options, False)
    assert (t.norm, t.netG) == ("batch", "unet_128") and not hasattr(t, "gan_mode")


@pytest.mark.skipif(not RH.available(), reason="reference tree not mounted")
@pytest.mark.parametrize("is_train", [True, False])
def test_pix2pix_options_match_the_reference_parser(is_train):
    RH.import_reference()
    from models.pix2pix_model import Pix2PixModel as Ref

    args = ["--gan_mode", "lsgan", "--lambda_l1", "3", "--discriminator", "n_layers"] if is_train else []
    ours = vars(parse(Pix2PixModel.modify_commandline_options, is_train, args))
    ref = vars(parse(Ref.modify_commandline_options, is_train, args))
    assert {k: v for k, v in ours.items() if not k.startswith("b200_")} == ref


def test_registry_through_dropin_models():
    sys.path.insert(0, os.path.join(ROOT, "dropin"))
    try:
        import models as dropin_models
    finally:
        sys.path.remove(os.path.join(ROOT, "dropin"))
    if not dropin_models.__file__.startswith(os.path.join(ROOT, "dropin")):
        pytest.skip("another `models` package is already imported")
    assert dropin_models.find_model_using_name("pix2pix") is Pix2PixModel
    assert sys.modules["models.pix2pix_model"].Pix2PixModel is Pix2PixModel
    assert dropin_models.get_options_modifier("pix2pix") == Pix2PixModel.modify_commandline_options


def _checksums(sd):
    return [(k, tuple(v.shape), v.double().sum().item(), v.double().abs().sum().item(),
             v.double().square().sum().item()) for k, v in sd.items()]


def _same(ours, gold):
    assert [(k, s) for k, s, *_ in ours] == [(k, s) for k, s, *_ in gold]
    for (k, _, *a), (_, _, *b) in zip(ours, gold):
        assert a == pytest.approx(b, rel=1e-12, abs=1e-12), k


def _networks(kind):
    """The golden model's G and D as the plugins build them: construction order G, init_weights(G), D
    (+ init_weights(D) for the texture stage only: pix2pix's define_D ignores init_type), under the golden's seed."""
    gold = GOLD[kind]
    torch.manual_seed(gold["seed"])
    if kind == "pix2pix_128":
        g = M.UnetGenerator(19 + 36, 3, 7, 64, use_dropout=True, norm="batch")
        M.init_weights(g, gold["init_type"], 0.02)
        d = M.NLayerDiscriminator(19 + 36 + 3, 64, 3, "batch")
    else:
        g = M.UnetGenerator(3, 3, 7, 64, use_dropout=True, norm="batch")
        M.init_weights(g, gold["init_type"], 0.02)
        d = M.NLayerDiscriminator(22, 64, 3, "instance")
        M.init_weights(d, gold["init_type"], 0.02)
    return g, d


@pytest.mark.parametrize("kind", ["pix2pix_128", "texture_unet_128"])
def test_keys_and_seeded_inits_equal_the_reference(kind):
    g, d = _networks(kind)
    _same(_checksums(g.state_dict()), GOLD[kind]["init_G"])
    _same(_checksums(d.state_dict()), GOLD[kind]["init_D"])


def _oracle_step(kind, dtype):
    """(losses, {"D": grads, "G": grads}) of tests/tools/unet_oracle.py on the golden's networks, batch and draws."""
    import unet_oracle as UO
    from test_engine_gpu import synth_texture_batch

    gold = GOLD[kind]
    g, d = _networks(kind)
    sdG = {k: v.detach().to(dtype).requires_grad_(k in dict(g.named_parameters())) for k, v in g.state_dict().items()}
    sdD = {k: v.detach().to(dtype).requires_grad_(k in dict(d.named_parameters())) for k, v in d.state_dict().items()}
    tex, _, cloth, tgt = synth_texture_batch(gold["batch"], gold["size"])
    tex, cloth, tgt = tex.to(dtype), cloth.to(dtype), tgt.to(dtype)
    draws = list(gold["draws"].reshape(-1, 1))
    if kind == "pix2pix_128":
        o = UO.pix2pix_step_losses(sdG, sdD, cloth, tgt, draws, "vanilla", "batch", True)
    else:
        o = UO.texture_unet_step_losses(sdG, sdD, tex, cloth, tgt, draws, "vanilla", "instance", True)
    grads = {}
    for phase, loss, sd in (("D", o["D"], sdD), ("G", o["G"], sdG)):
        keys = [k for k in sd if sd[k].requires_grad]
        grads[phase] = dict(zip(keys, (x.double() for x in torch.autograd.grad(loss, [sd[k] for k in keys],
                                                                               retain_graph=True))))
    return {k: o[k].item() for k in gold["losses"]}, grads


@pytest.mark.parametrize("kind", ["pix2pix_128", "texture_unet_128"])
def test_oracle_reproduces_the_reference_step(kind):
    """tests/tools/unet_oracle.py, which every GPU parity test of the two models compares against, on the golden's
    networks, batch and label draws.  The smooth labels, every loss, and every parameter gradient of the D phase and the
    G phase must equal the reference's fp32 CPU run.  Losses: within 2e-5.  Gradients (sum, sum of |g|, first elements):
    within 1e-3 of the tensor's scale, or within 4x what the same oracle computed in fp32 differs from its fp64 result,
    whichever is larger.  The second bound matters for the texture stage's unet_128: its dense input meets batch norm
    over 8 values per channel on the 2 x 2 innermost planes, where fp32 rounding alone moves single gradient elements
    by a few percent."""
    from oracle import nets as ON

    gold = GOLD[kind]
    draws = list(gold["draws"].reshape(-1, 1))
    assert len(draws) == 3                       # D_fake, D_real, G_gan: vanilla draws one label per loss call
    assert torch.equal(torch.cat([ON.smooth_label(x).float().reshape(1) for x in draws]), gold["labels"])
    torch.manual_seed(gold["label_seed"])        # the draws are the CPU generator's, seeded as in the golden
    assert torch.equal(torch.cat([torch.rand(1) for _ in range(3)]), gold["draws"])
    losses, got = _oracle_step(kind, torch.float64)
    _, got32 = _oracle_step(kind, torch.float32)
    for k, v in gold["losses"].items():
        assert abs(losses[k] - v) <= 2e-5 * abs(v), (k, losses[k], v)
    for phase in ("D", "G"):
        ref = gold["grads_" + phase]
        assert sorted(got[phase]) == sorted(ref), phase
        mean_abs = max(r["abs"] / got[phase][k].numel() for k, r in ref.items())
        for k, r in ref.items():
            x, x32 = got[phase][k], got32[phase][k]
            if r["abs"] / x.numel() < 1e-6 * mean_abs:   # a conv bias followed by InstanceNorm: the gradient is zero
                assert x.abs().sum().item() / x.numel() < 1e-6 * mean_abs, (phase, k)
                continue
            head = r["head"].double()
            n = head.numel()
            for what, a, b, a32, scale in (
                    ("abs", x.abs().sum().item(), r["abs"], x32.abs().sum().item(), r["abs"]),
                    ("sum", x.sum().item(), r["sum"], x32.sum().item(), r["abs"]),
                    ("head", x.reshape(-1)[:n], head, x32.reshape(-1)[:n], head.abs().max().item())):
                err = float(torch.as_tensor(a - b).abs().max())
                noise = float(torch.as_tensor(a32 - a).abs().max())
                assert err <= max(1e-3 * scale, 4 * noise), (phase, k, what, err, scale, noise)


@pytest.mark.parametrize("mode,objective,draws", [("vanilla", ops.GAN_BCE, 3), ("dragan-gp", ops.GAN_BCE, 3),
                                                  ("dragan-lp", ops.GAN_BCE, 3), ("lsgan", ops.GAN_MSE, 3),
                                                  ("wgan", ops.GAN_WGAN, 0), ("wgan-gp", ops.GAN_WGAN, 0)])
def test_pix2pix_gan_mode_mapping_and_label_draws(mode, objective, draws):
    m = Pix2PixModel.__new__(Pix2PixModel)
    assert m.gan_objective(mode) == objective == PIX2PIX_GAN_OBJECTIVES[mode]
    m._gan_obj, m.net_discriminator = objective, object()
    assert m.label_draws() == draws
    assert m.gan_weight() == 1.0


@pytest.mark.parametrize("mode", ["mescheder-r1-gp", "mescheder-r2-gp"])
def test_pix2pix_refuses_what_the_reference_cannot_run(mode):
    m = Pix2PixModel.__new__(Pix2PixModel)
    with pytest.raises(NotImplementedError, match="GANLoss does not implement it"):
        m.gan_objective(mode)


def test_texture_stage_still_refuses_gradient_penalties():
    from swapnet_b200.models.texture_model import TextureModel

    m = TextureModel.__new__(TextureModel)
    with pytest.raises(NotImplementedError, match="second derivative"):
        m.gan_objective("wgan-gp")


def test_data_parallel_batch_norm_needs_sync_bn():
    """pix2pix (--norm batch by default) and --netG unet_128 (batch norm in the generator whatever --norm says) under
    data parallelism without --b200_sync_bn 1 are refused; with it, or on one rank, they are not."""
    with pytest.raises(NotImplementedError, match="cross-rank batch statistics.*--b200_sync_bn 1"):
        base_gan.batch_norm_exchange(Namespace(norm="batch", b200_sync_bn=0), 2)
    with pytest.raises(NotImplementedError, match="generator's batch norm.*--b200_sync_bn 1"):
        base_gan.batch_norm_exchange(Namespace(norm="instance", b200_sync_bn=0), 2, batch_norm=True)
    assert base_gan.batch_norm_exchange(Namespace(norm="instance", b200_sync_bn=0), 1, batch_norm=True) is None
    assert base_gan.batch_norm_exchange(Namespace(norm="instance", b200_sync_bn=0), 2, batch_norm=False) is None


def test_unet_engine_refuses_sizes_not_divisible_by_2_pow_7():
    from swapnet_b200 import engine as E

    net = M.UnetGenerator(3, 3, 7, 64, use_dropout=True, norm="batch")
    for S in (64, 192 + 32, 96):
        with pytest.raises(ValueError, match="divisible by 2\\*\\*7 = 128"):
            E.UnetEngine(net, 1, S, "cpu")


def test_registry_in_a_fresh_interpreter():
    """The drop-in `models` package resolves `--model pix2pix` to the plugin (also when the reference's own package
    was imported first in this process, which the test above then skips)."""
    import subprocess

    code = ("import models, sys; from swapnet_b200.models.pix2pix_model import Pix2PixModel; "
            "assert models.find_model_using_name('pix2pix') is Pix2PixModel; "
            "assert sys.modules['models.pix2pix_model'].Pix2PixModel is Pix2PixModel; print('OK')")
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.join(ROOT, "dropin"), ROOT]), CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "OK" in r.stdout, r.stderr[-3000:]


@pytest.mark.skipif(not RH.available(), reason="reference tree not mounted")
@pytest.mark.parametrize("model,extra", [("pix2pix", ["--dataset", "texture_b200"]),
                                         ("pix2pix", ["--dataset", "texture"]),
                                         ("texture", ["--netG", "unet_128", "--dataset", "texture_b200"])])
def test_launcher_parses_and_reaches_the_plugin(tmp_path, model, extra):
    """The unmodified reference train.py through `python -m swapnet_b200.run`: options parsed through the plugin's
    modifier, the reference's dataset registry, the plugin's constructor (which, without a GPU, refuses to run)."""
    import test_dropin_launcher as TL

    data = tmp_path / "data"
    TL.make_dataset(str(data), size=128)
    r = TL.run([sys.executable, "-m", "swapnet_b200.run", "train.py", "--name", "t", "--model", model, "--dataroot",
                str(data), "--checkpoints_dir", str(tmp_path / "ck"), "--display_id", "0", "--batch_size", "1",
                "--load_size", "128", "--crop_size", "128", "--num_workers", "0", "--no_confirm", "--gpu_id", "0",
                "--n_epochs", "1", *extra], cwd=TL.REF)
    out = r.stdout + r.stderr
    assert "b200_precision" in out and "The number of training images = 2" in out, out[-3000:]
    if model == "pix2pix":
        assert "lambda_l1" in out and "beta1" in out, out[-3000:]
    assert r.returncode != 0 and "swapnet_b200 models run on a CUDA device only" in out, out[-3000:]
