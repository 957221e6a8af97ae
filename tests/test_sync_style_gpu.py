"""The style term over row blocks of a Gram matrix of any size (`gram_rows`, `gram_rows_mse`, `gram_rows_bwd` in
csrc/perceptual.cu) and `--b200_sync_style` on the GPU.

Kernels: against fp64 with the bounds of tests/test_perceptual_logits_gpu.py (k u per entry, u = 2^-24, normalised by
sqrt(G_ii G_jj) for the Gram matrices and by the sum of the absolute terms for the gradient), from 3 x 3 to 48 x 384
row blocks and from 1 pixel to 512^2, NHWC and NCHW sources, pitched dx with and without accumulate, default and
deterministic mode.  Emulated ranks on one GPU: the assembled partials and gradient rows equal the single-process fp64
full-batch style loss and gradient.  Plugin: a one-GPU texture step at batch 40 (R = 120 rows) against the fp64
oracle, graph replay against eager, flag 0 against flag 1; and tests/tools/sync_style_equiv.py, 2 ranks x B/2 against
1 x B over NCCL on two GPUs and over gloo with both ranks on one GPU."""
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from swapnet_b200 import _lib, ops
from test_engine_gpu import _opt, _texture_step_vs_oracle, record, synth_texture_batch
from test_perceptual_logits_gpu import GRAM_K, NAN, U, bounded, gen, gram_scale, gram_source, refused

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def dev():
    return torch.device("cuda:0")


def _stream():
    return torch.cuda.current_stream().cuda_stream


def local(x, r0, n):
    """Samples [r0, r0 + n) of a gram_source tensor, contiguous (a rank's own shard)."""
    return x[r0:r0 + n].contiguous()


# (R_l, R): square blocks of one GPU's samples, rectangular blocks of 2, 4 and 8 ranks
ROW_CASES = [(3, 3), (48, 48), (24, 96), (97, 97), (48, 192), (144, 144), (48, 384)]


def rows_of(rl, r):
    """(channels, local samples, all samples) for an (R_l, R) case: 97 rows are 97 one-channel samples."""
    c = 1 if rl % 3 else 3
    return c, rl // c, r // c


def run_gram_rows(rl, r, npix, src_nhwc, seed):
    c, na, nb = rows_of(rl, r)
    g = gen(seed)
    x, rows = gram_source(nb, c, npix, src_nhwc, g)
    r0 = (nb - na) // 2                     # a middle rank's rows
    a = local(x, r0, na)
    ref = rows[r0 * c:r0 * c + rl] @ rows.T
    dg = rows.pow(2).sum(1)                 # G_jj of every row
    scale = torch.sqrt(dg[r0 * c:r0 * c + rl, None] * dg[None, :])
    ws = ops.DetWorkspace(dev())
    outs = []
    tag = f"R_l={rl},R={r},npix={npix},{'nhwc' if src_nhwc else 'nchw'}"
    for det in (False, True, True):
        out = torch.full((rl, r), NAN, dtype=torch.float64, device=dev())
        ops.gram_rows(a, x, src_nhwc, out, ws=ws if det else None)
        torch.cuda.synchronize()
        bounded(f"gram_rows[{tag},{'det' if det else 'atomic'}]", out, ref, scale, GRAM_K)
        outs.append(out)
    assert torch.equal(outs[1], outs[2]), "gram_rows_det did not repeat bit for bit"


GRAM_ROWS_NPIX = [1, 127, 129, 128 * 296 + 1]


@pytest.mark.parametrize("src_nhwc", [True, False])
@pytest.mark.parametrize("npix", GRAM_ROWS_NPIX)
@pytest.mark.parametrize("rl,r", ROW_CASES)
def test_gram_rows(rl, r, npix, src_nhwc):
    run_gram_rows(rl, r, npix, src_nhwc, seed=rl * 7 + r + npix)


@pytest.mark.parametrize("src_nhwc", [True, False])
@pytest.mark.parametrize("rl,r", [(48, 48), (48, 192), (144, 144)])
def test_gram_rows_512(rl, r, src_nhwc):
    """The style term at 512 x 512: 16 images per rank on 1 and 4 ranks, and 48 images on one GPU."""
    run_gram_rows(rl, r, 512 * 512, src_nhwc, seed=rl + r)


@pytest.mark.parametrize("rl,r", [(3, 3), (48, 48), (24, 96), (48, 384), (144, 144)])
def test_gram_rows_mse(rl, r):
    """loss += w sum((Go - Gt)^2) / R^2 over the block; m = fp32(4 w gscale (Go - Gt) / R^2), restated in the kernel's
    order, for gscale 1 and a rank count."""
    g = gen(rl + r)
    go = torch.randn(rl, r, generator=g, device=dev(), dtype=torch.float64) * 1e4
    gt = torch.randn(rl, r, generator=g, device=dev(), dtype=torch.float64) * 1e4
    w, acc0 = 5.0 * 3e-8, 0.625
    d = go - gt
    inv = 1.0 / (r * r)
    for gscale in (1.0, float(r // rl), 3.0):
        acc = torch.full((1,), acc0, dtype=torch.float64, device=dev())
        m = torch.full((rl, r), NAN, device=dev())
        ops.gram_rows_mse(go, gt, w, acc, m, gscale=gscale)
        torch.cuda.synchronize()
        assert torch.equal(m, ((4.0 * w * gscale) * d * inv).float()), f"m differs (gscale {gscale})"
        loss = w * (d * d).sum().item() * inv
        err = abs(acc.item() - acc0 - loss) / (acc0 + loss)
        record(f"gram_rows_mse[R_l={rl},R={r},gscale={gscale}]", f"{err:.2e}")
        assert err < 1e-14, err


GRAM_ROWS_BWD_NPIX = [1, 129, 128 * 592 + 1]


@pytest.mark.parametrize("src_nhwc", [True, False])
@pytest.mark.parametrize("npix", GRAM_ROWS_BWD_NPIX)
@pytest.mark.parametrize("rl,r", ROW_CASES)
def test_gram_rows_bwd(rl, r, npix, src_nhwc):
    """dx[b, p, ch] (+)= sum_j m[b*c + ch][j] X_j[p] into a dx whose pitch has one spare channel holding a sentinel."""
    c, na, nb = rows_of(rl, r)
    g = gen(rl + r + npix)
    x, rows = gram_source(nb, c, npix, src_nhwc, g)
    m = torch.randn(rl, r, generator=g, device=dev()) * 1e-3
    prod = m.double() @ rows
    mag = m.double().abs() @ rows.abs()

    def as_dx(t):            # [R_l, npix] -> NHWC [na, 1, npix, c]
        return t.view(na, c, npix).permute(0, 2, 1).reshape(na, 1, npix, c)

    base = torch.randn(na, 1, npix, c, generator=g, device=dev()) * prod.abs().max().float()
    for accumulate in (False, True):
        dx = torch.full((na, 1, npix, c + 1), NAN, device=dev())
        if accumulate:
            dx[..., :c] = base
        ops.gram_rows_bwd(m, x, src_nhwc, dx[..., :c], accumulate=accumulate)
        torch.cuda.synchronize()
        want = as_dx(prod) + (base.double() if accumulate else 0.0)
        scale = as_dx(mag) + (base.double().abs() if accumulate else 0.0)
        bounded(f"gram_rows_bwd[R_l={rl},R={r},npix={npix},{'nhwc' if src_nhwc else 'nchw'},acc={accumulate}]",
                dx[..., :c], want, scale, r + 2)
        assert bool(torch.isnan(dx[..., c]).all()), "wrote the spare channel"


def test_gram_rows_refusals():
    x = torch.rand(4, 3, 1, 100, device=dev())
    a = x[:2].contiguous()
    out = torch.zeros(6, 12, dtype=torch.float64, device=dev())
    lib = _lib.load()
    refused(lambda: _lib.check(lib.sn_gram_rows(0, 300, 100, 1, 2, x.data_ptr(), 300, 100, 1, 4, 3, 100,
                                                out.data_ptr(), _stream())))
    refused(lambda: _lib.check(lib.sn_gram_rows(x.data_ptr(), 300, 100, 1, 4, a.data_ptr(), 300, 100, 1, 2, 3, 100,
                                                out.data_ptr(), _stream())))          # R_l > R
    refused(lambda: _lib.check(lib.sn_gram_rows(a.data_ptr(), 300, 100, 0, 2, x.data_ptr(), 300, 100, 1, 4, 3, 100,
                                                out.data_ptr(), _stream())))          # zero pixel stride
    refused(lambda: _lib.check(lib.sn_gram_rows_det(a.data_ptr(), 300, 100, 1, 2, x.data_ptr(), 300, 100, 1, 4, 3,
                                                    100, out.data_ptr(), 0, 1 << 20, _stream())))   # null slots
    need = 1 * 6 * 12                                    # 100 pixels are one chunk: one pixel split
    assert lib.sn_gram_rows_det_slots(6, 12) >= need
    slots = torch.zeros(need, dtype=torch.float64, device=dev())

    def call(cap):
        _lib.check(lib.sn_gram_rows_det(a.data_ptr(), 300, 100, 1, 2, x.data_ptr(), 300, 100, 1, 4, 3, 100,
                                        out.data_ptr(), slots.data_ptr(), cap, _stream()))
    refused(lambda: call(need - 1))
    call(need)
    torch.cuda.synchronize()
    rows = x.reshape(12, 100).double()
    ref = rows[:6] @ rows.T
    dg = rows.pow(2).sum(1)
    bounded("gram_rows_det[exact slot capacity]", out, ref, torch.sqrt(dg[:6, None] * dg[None, :]), GRAM_K)

    go = torch.zeros(6, 12, dtype=torch.float64, device=dev())
    m = torch.zeros(6, 12, device=dev())
    acc = torch.zeros(1, dtype=torch.float64, device=dev())
    refused(lambda: _lib.check(lib.sn_gram_rows_mse(go.data_ptr(), 0, 6, 12, 1.0, 1.0, acc.data_ptr(), m.data_ptr(),
                                                    _stream())))
    refused(lambda: _lib.check(lib.sn_gram_rows_mse(go.data_ptr(), go.data_ptr(), 13, 12, 1.0, 1.0, acc.data_ptr(),
                                                    m.data_ptr(), _stream())))
    dx = torch.zeros(2, 1, 100, 3, device=dev())
    refused(lambda: _lib.check(lib.sn_gram_rows_bwd(0, 6, x.data_ptr(), 300, 100, 1, 4, 3, 100, dx.data_ptr(), 3, 0,
                                                    _stream())))
    refused(lambda: _lib.check(lib.sn_gram_rows_bwd(m.data_ptr(), 15, x.data_ptr(), 300, 100, 1, 4, 3, 100,
                                                    dx.data_ptr(), 3, 0, _stream())))    # R_l > R
    refused(lambda: _lib.check(lib.sn_gram_rows_bwd(m.data_ptr(), 5, x.data_ptr(), 300, 100, 1, 4, 3, 100,
                                                    dx.data_ptr(), 3, 0, _stream())))    # not whole samples
    refused(lambda: _lib.check(lib.sn_gram_rows_bwd(m.data_ptr(), 6, x.data_ptr(), 300, 100, 1, 4, 3, 100,
                                                    dx.data_ptr(), 2, 0, _stream())))    # pitch < c


# ---------------------------------------------------------------------------------------------
# emulated ranks on one GPU
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("world,per,S", [(2, 4, 64), (4, 2, 64), (4, 16, 96)])
def test_emulated_ranks_assemble_the_full_batch_style_term(world, per, S, det):
    """Each emulated rank runs PerceptualEngine.style's launches on its shard against the gathered batch:
    gram_rows, gram_rows_mse with gscale = world into a partial, gram_rows_bwd.  The partials added in rank order and the
    gradient rows x 1/world against fp64 autograd of 5 lam MSE(gram(fakes), gram(targets)) over the whole batch."""
    B, lam = per * world, 1e-6
    g = gen(world * 1000 + per * 10 + S + det)
    fakes = torch.rand(B, S, S, 3, generator=g, device=dev()) * 2 - 1
    targets = torch.rand(B, 3, S, S, generator=g, device=dev()) * 4.5 - 2
    r, rl, npix = 3 * B, 3 * per, S * S
    xo = fakes.permute(0, 3, 1, 2).reshape(r, npix).double().requires_grad_()
    xt = targets.reshape(r, npix).double()
    go_ref, gt_ref = xo @ xo.T, xt @ xt.T
    loss = 5 * F.mse_loss(go_ref, gt_ref) * lam
    (gx,) = torch.autograd.grad(loss, xo)
    ws = ops.DetWorkspace(dev()) if det else None
    parts = torch.zeros(world, dtype=torch.float64, device=dev())
    dx = torch.zeros(B, S, S, 3, device=dev())
    for rank in range(world):
        mine = slice(rank * per, (rank + 1) * per)
        go = torch.full((rl, r), NAN, dtype=torch.float64, device=dev())
        gt = torch.full_like(go, NAN)
        m = torch.full((rl, r), NAN, device=dev())
        ops.gram_rows(fakes[mine].contiguous(), fakes, True, go, ws=ws)
        ops.gram_rows(targets[mine].contiguous(), targets, False, gt, ws=ws)
        ops.gram_rows_mse(go, gt, 5.0 * lam, parts[rank:rank + 1], m, gscale=float(world))
        ops.gram_rows_bwd(m, fakes, True, dx[mine], accumulate=True)
    acc = torch.zeros(1, dtype=torch.float64, device=dev())
    for rank in range(world):
        acc.add_(parts[rank:rank + 1])
    torch.cuda.synchronize()
    grad = (dx.double() / world).permute(0, 3, 1, 2).reshape(r, npix)
    with torch.no_grad():
        dg = GRAM_K * U * (gram_scale(go_ref) + gram_scale(gt_ref))
        d = (go_ref - gt_ref).abs()
        loss_bound = 5 * lam / r ** 2 * (2 * d * dg + dg * dg).sum().item()
        m_ref = 4 * 5 * lam * (go_ref - gt_ref) / r ** 2
        dm = 4 * 5 * lam / r ** 2 * dg + U * m_ref.abs()
        xabs = xo.detach().abs()
        g_scale = dm @ xabs + (r + 2) * U * (m_ref.abs() @ xabs)
    tag = f"emulated_ranks[w={world},per={per},S={S},{'det' if det else 'atomic'}]"
    lerr = abs(acc.item() - loss.item())
    record(tag + " loss", f"{lerr:.3e} (bound {loss_bound:.3e}, loss {loss.item():.3e})")
    assert lerr <= loss_bound + 1e-15 * loss.item(), (lerr, loss_bound)
    ratio = ((grad - gx).abs() / g_scale).max().item()
    record(tag + " grad", f"{ratio:.3e} of the bound")
    assert ratio <= 1.0, ratio


# ---------------------------------------------------------------------------------------------
# one GPU, the texture plugin
# ---------------------------------------------------------------------------------------------
def test_texture_step_batch40_matches_oracle():
    """Batch 40 (120 Gram rows) at 64 x 64 with the default content and style terms, seeded-random
    VGG16: no longer refused; losses and every G gradient against the fp64 oracle (test_engine_gpu's protocol)."""
    _texture_step_vs_oracle(40, 64, True, tag="_b40")


def _texture_runs(B, S, configs, steps=3):
    from swapnet_b200.models import create_model

    tex, rois, cloth, tgt = synth_texture_batch(B, S)
    batch = dict(input_textures=tex, rois=rois, cloths=cloth, target_textures=tgt, cloth_paths=["c"] * B,
                 texture_paths=["t"] * B)
    runs = {}
    for graph, flag in configs:
        torch.manual_seed(0)
        model = create_model(_opt(B, S, model="texture", name="texture", netG="swapnet", lambda_l1=10,
                                  lambda_content=20, lambda_style=1e-8, b200_vgg="random", b200_deterministic=1,
                                  b200_graph=graph, b200_sync_style=flag))
        model.setup(model.opt)
        torch.manual_seed(99)
        hist = []
        for _ in range(steps):
            model.set_input(batch)
            model.optimize_parameters()
            hist.append(dict(model.get_current_losses()))
        assert model._eng_P.style_exchange is None
        assert len(model._graphs) == graph
        state = {p + k: v.detach().cpu().clone() for p, net in (("G.", model.net_generator),
                                                                ("D.", model.net_discriminator))
                 for k, v in net.state_dict().items()}
        runs[(graph, flag)] = (hist, state)
        del model
    return runs


def test_batch40_replay_equals_eager_and_sync_style_flag_is_a_noop():
    """--b200_deterministic 1, batch 40 at 64 x 64, content and style on: three eager steps, three steps whose third is
    a graph replay (the row kernels are captured with the rest of the step), and the same with --b200_sync_style 1 —
    all bit-identical: losses, parameters, buffers."""
    runs = _texture_runs(40, 64, [(0, 0), (1, 0), (1, 1)])
    ref_hist, ref_state = runs[(0, 0)]
    assert all(v["G_style"] > 0 for v in ref_hist)
    for key in ((1, 0), (1, 1)):
        hist, state = runs[key]
        assert hist == ref_hist, key
        for k, v in ref_state.items():
            assert torch.equal(v, state[k]), (key, k)


# ---------------------------------------------------------------------------------------------
# two ranks
# ---------------------------------------------------------------------------------------------
def _run_equiv(backend, nproc):
    env = dict(os.environ, SN_SSTYLE_BACKEND=backend)
    port = 29700 + os.getpid() % 200 + (0 if backend == "nccl" else 1)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc),
           "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(ROOT, "tests", "tools", "sync_style_equiv.py")]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("SYNC_STYLE_EQUIV")]
    for ln in lines:
        record(f"sync_style_equivalence[{backend}]", ln)
    ok = r.returncode == 0 and len(lines) == 2 and all(" OK " in ln for ln in lines)
    assert ok, "\n".join(lines) + "\n--- stderr ---\n" + r.stderr[-8000:]


def test_two_rank_nccl_sync_style_equals_full_batch():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _run_equiv("nccl", 2)


def test_two_rank_gloo_sync_style_on_one_gpu_equals_full_batch():
    _run_equiv("gloo", 2)
