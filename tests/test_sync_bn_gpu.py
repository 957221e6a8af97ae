"""Cross-rank batch statistics (`--b200_sync_bn 1`) on the GPU.

Kernels: ranks emulated in one process, their partials stacked in rank order as the gather leaves them, against fp64
F.batch_norm over the whole group; with one rank, bit-identical to the single-process kernels.  Plugin: the flag is a
no-op on one GPU, and 2 ranks x B/2 samples reproduce one process with B samples (tests/tools/sync_bn_equiv.py) over
NCCL on two GPUs and over gloo with both ranks on one GPU."""
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

from test_engine_gpu import _opt, record, relmax, synth_texture_batch  # noqa: E402


def dev():
    return torch.device("cuda:0")


def _bn(c, g):
    bn = torch.nn.BatchNorm2d(c).to(dev())
    with torch.no_grad():
        bn.weight.copy_(1.0 + 0.3 * torch.randn(c, generator=g))
        bn.bias.copy_(0.2 * torch.randn(c, generator=g))
        bn.running_mean.copy_(0.1 * torch.randn(c, generator=g))
        bn.running_var.copy_(1.0 + 0.5 * torch.rand(c, generator=g))
    return bn


def _clone_bn(bn):
    b = torch.nn.BatchNorm2d(bn.num_features).to(dev())
    b.load_state_dict(bn.state_dict())
    return b


# ---------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shards,h,c,groups", [((2,), 8, 64, 1), ((2, 2), 63, 64, 2), ((1, 3), 7, 256, 1),
                                               ((2, 4, 2), 5, 512, 2), ((1, 1, 1), 63, 256, 1), ((4, 2), 4, 512, 2),
                                               ((3, 1), 63, 512, 1)])
def test_gathered_bn_kernels_match_batch_norm_over_all_ranks(shards, h, c, groups):
    """Per emulated rank: plane_sums -> bn_group_sums; the partials stacked in rank order; per rank
    bn_finalize_gathered, the affine forward and the split backward (reduce, group sums, gather, group + apply).
    Against fp64 F.batch_norm over each group's samples of all ranks: outputs, dL/dy, d gamma / d beta summed over
    the shards, running buffers (the same bits on every rank) and the batch counter."""
    from swapnet_b200 import ops

    shards = [n * groups for n in shards]          # samples per rank: n_r / groups of each group
    g = torch.Generator().manual_seed(sum(shards) * 1000 + h * 10 + c + groups)
    ys = [(torch.randn(n, h, h, c, generator=g) * 1.7 + 0.3).to(dev()) for n in shards]
    ups = [torch.randn(n, h, h, c, generator=g).to(dev()) for n in shards]
    bn0 = _bn(c, g)
    rm0, rv0 = bn0.running_mean.double().cpu(), bn0.running_var.double().cpu()
    hw = h * h
    bns = [_clone_bn(bn0) for _ in shards]         # every rank holds its own copy of the module
    stats, parts = [], []
    for y, n in zip(ys, shards):
        st = torch.zeros(n, c, 2, dtype=torch.float64, device=dev())
        ops.plane_sums(y, c, st)
        part = torch.zeros(groups, c, 3, dtype=torch.float64, device=dev())
        ops.bn_group_sums(st, n, c, groups, hw, part)
        stats.append(st)
        parts.append(part)
    gathered = torch.stack(parts)
    outs, dys, gsts, gparts = [], [], [], []
    dgam, dbet = torch.zeros(c, device=dev()), torch.zeros(c, device=dev())
    for y, up, n, st, bn in zip(ys, ups, shards, stats, bns):
        ops.bn_finalize_gathered(st, n, c, groups, gathered, bn)
        out = torch.zeros(n, h, h, c, device=dev())
        ops.norm_act_fwd(y, c, st, ops.ACT_LRELU, 0.2, out_f32=out, gamma=bn.weight.data, beta=bn.bias.data)
        dy = ops.Planes(n, h, h, c, dev(), fmt=ops.FMT_BF16)
        gst = torch.zeros(n, c, 2, dtype=torch.float64, device=dev())
        ops.norm_act_bwd([ops.GradSrc(up)], y, c, st, ops.ACT_LRELU, dy, gst, 0.2, bn=(bn.weight.data, bn.bias.data),
                         bn_groups=groups, bn_phase=1)
        gp = torch.zeros(groups, c, 3, dtype=torch.float64, device=dev())
        ops.bn_group_sums(gst, n, c, groups, hw, gp)
        outs.append(out)
        dys.append(dy)
        gsts.append(gst)
        gparts.append(gp)
    ggathered = torch.stack(gparts)
    for r, (y, up, n, st, bn) in enumerate(zip(ys, ups, shards, stats, bns)):
        ops.norm_act_bwd([ops.GradSrc(up)], y, c, st, ops.ACT_LRELU, dys[r], gsts[r], 0.2,
                         bn=(bn.weight.data, bn.bias.data), bn_groups=groups, bn_grads=(dgam, dbet), bn_phase=2,
                         bn_gathered=ggathered, bn_rank=r)
    torch.cuda.synchronize()

    y64 = [y.cpu().double().permute(0, 3, 1, 2).requires_grad_() for y in ys]
    w64 = bn0.weight.detach().cpu().double().requires_grad_()
    b64 = bn0.bias.detach().cpu().double().requires_grad_()
    rm, rv = rm0.clone(), rv0.clone()
    z = [[None] * groups for _ in shards]
    for gi in range(groups):
        parts_g = [y[gi * (n // groups):(gi + 1) * (n // groups)] for y, n in zip(y64, shards)]
        zg = F.batch_norm(torch.cat(parts_g), rm, rv, w64, b64, True, 0.1, 1e-5)
        z_split = zg.split([n // groups for n in shards])
        for r in range(len(shards)):
            z[r][gi] = z_split[r]
    z = [torch.cat(zr) for zr in z]
    loss, flips, total = 0.0, 0, 0
    refs = []
    for r, out in enumerate(outs):
        gate = (out > 0).cpu().permute(0, 3, 1, 2)
        ref = torch.where(gate, z[r], 0.2 * z[r])
        refs.append(ref)
        loss = loss + (ref * ups[r].cpu().double().permute(0, 3, 1, 2)).sum()
        flips += int((gate != (z[r] > 0)).sum())
        total += z[r].numel()
    loss.backward()
    assert flips <= max(2, 1e-4 * total), flips
    assert relmax(torch.cat([o.cpu().permute(0, 3, 1, 2) for o in outs]), torch.cat(refs).detach()) < 1e-5
    dyd = torch.cat([dy.dense()[..., :c].cpu().permute(0, 3, 1, 2) for dy in dys])
    assert relmax(dyd, torch.cat([y.grad for y in y64])) < 1e-3
    assert relmax(dgam.cpu(), w64.grad) < 1e-4
    assert relmax(dbet.cpu(), b64.grad) < 1e-4
    for bn in bns:
        assert torch.equal(bn.running_mean, bns[0].running_mean) and torch.equal(bn.running_var, bns[0].running_var)
        assert int(bn.num_batches_tracked) == groups
    assert relmax(bns[0].running_mean.cpu(), rm) < 1e-5 and relmax(bns[0].running_var.cpu(), rv) < 1e-5


@pytest.mark.parametrize("n,h,c,groups", [(2, 8, 64, 1), (4, 63, 64, 2), (4, 4, 512, 2), (2, 63, 256, 2)])
def test_world_one_is_bit_identical_to_single_process_kernels(n, h, c, groups):
    """One rank: bn_group_sums + bn_finalize_gathered give bn_finalize's stats and running buffers bit for bit, and
    the split backward gives the unsplit norm_act_bwd's dL/dy, d gamma and d beta bit for bit.  Both paths start from
    the same plane sums, and the backward's gradient sums use the fixed-order reduction (the default one adds with
    atomics, whose order varies from launch to launch)."""
    from swapnet_b200 import ops

    g = torch.Generator().manual_seed(n * 100 + h + c + groups)
    y = (torch.randn(n, h, h, c, generator=g) * 1.7 + 0.3).to(dev())
    up = torch.randn(n, h, h, c, generator=g).to(dev())
    bn_a = _bn(c, g)
    bn_b = _clone_bn(bn_a)
    ws = ops.DetWorkspace(dev())
    hw = h * h
    sums = torch.zeros(n, c, 2, dtype=torch.float64, device=dev())
    ops.plane_sums(y, c, sums)
    res = {}
    for name, bn in (("single", bn_a), ("gathered", bn_b)):
        st = sums.clone()
        if name == "single":
            ops.bn_finalize(st, n, c, groups, hw, bn)
        else:
            part = torch.zeros(groups, c, 3, dtype=torch.float64, device=dev())
            ops.bn_group_sums(st, n, c, groups, hw, part)
            ops.bn_finalize_gathered(st, n, c, groups, part[None].contiguous(), bn)
        out = torch.zeros(n, h, h, c, device=dev())
        ops.norm_act_fwd(y, c, st, ops.ACT_LRELU, 0.2, out_f32=out, gamma=bn.weight.data, beta=bn.bias.data)
        dy = ops.Planes(n, h, h, c, dev(), fmt=ops.FMT_BF16)
        gst = torch.zeros(n, c, 2, dtype=torch.float64, device=dev())
        dgam, dbet = torch.zeros(c, device=dev()), torch.zeros(c, device=dev())
        args = ([ops.GradSrc(up)], y, c, st, ops.ACT_LRELU, dy, gst, 0.2)
        kw = dict(bn=(bn.weight.data, bn.bias.data), bn_groups=groups, bn_grads=(dgam, dbet), ws=ws)
        if name == "single":
            ops.norm_act_bwd(*args, **kw)
        else:
            ops.norm_act_bwd(*args, **kw, bn_phase=1)
            gp = torch.zeros(groups, c, 3, dtype=torch.float64, device=dev())
            ops.bn_group_sums(gst, n, c, groups, hw, gp)
            ops.norm_act_bwd(*args, **kw, bn_phase=2, bn_gathered=gp[None].contiguous(), bn_rank=0)
        torch.cuda.synchronize()
        res[name] = dict(stats=st, out=out, dy=dy.dense(), gstats=gst, dgamma=dgam, dbeta=dbet,
                         **{k: v.clone() for k, v in bn.state_dict().items()})
    for k, v in res["single"].items():
        assert torch.equal(v, res["gathered"][k]), k


# ---------------------------------------------------------------------------------------------
# plugin
# ---------------------------------------------------------------------------------------------
def test_refusal_without_the_flag_names_it(monkeypatch):
    from swapnet_b200 import parallel
    from swapnet_b200.models import create_model

    monkeypatch.setattr(parallel, "world_size", lambda: 2)
    with pytest.raises(NotImplementedError, match="cross-rank batch statistics.*--b200_sync_bn 1"):
        create_model(_opt(2, 64, model="texture", name="texture", netG="swapnet", lambda_l1=10, lambda_content=0,
                          lambda_style=0, norm="batch", b200_sync_bn=0))


def test_flag_is_a_noop_on_one_gpu():
    """--b200_sync_bn 1 on one GPU: three deterministic texture steps with --norm batch (the third a graph replay) are
    bit-identical to three without the flag: losses, parameters, running buffers."""
    from swapnet_b200.models import create_model

    B, S = 2, 64
    tex, rois, cloth, tgt = synth_texture_batch(B, S)
    batch = dict(input_textures=tex, rois=rois, cloths=cloth, target_textures=tgt, cloth_paths=["c"] * B,
                 texture_paths=["t"] * B)
    runs = {}
    for flag in (0, 1):
        torch.manual_seed(0)
        model = create_model(_opt(B, S, model="texture", name="texture", netG="swapnet", lambda_l1=10,
                                  lambda_content=0, lambda_style=0, norm="batch", b200_deterministic=1,
                                  b200_sync_bn=flag))
        model.setup(model.opt)
        assert model._bn_sync is None
        torch.manual_seed(99)
        hist = []
        for _ in range(3):
            model.set_input(batch)
            model.optimize_parameters()
            hist.append(dict(model.get_current_losses()))
        assert len(model._graphs) == 1
        state = {p + k: v.detach().cpu().clone() for p, net in (("G.", model.net_generator),
                                                                ("D.", model.net_discriminator))
                 for k, v in net.state_dict().items()}
        runs[flag] = (hist, state)
    assert runs[0][0] == runs[1][0]
    for k, v in runs[0][1].items():
        assert torch.equal(v, runs[1][1][k]), k


def _run_equiv(backend, nproc):
    env = dict(os.environ, SN_SBN_BACKEND=backend)
    port = 29300 + os.getpid() % 300 + (0 if backend == "nccl" else 1)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc),
           "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(ROOT, "tests", "tools", "sync_bn_equiv.py")]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("SYNC_BN_EQUIV")]
    for ln in lines:
        record(f"sync_bn_equivalence[{backend}]", ln)
    ok = r.returncode == 0 and len(lines) == 2 and all(" OK " in ln for ln in lines)
    assert ok, "\n".join(lines) + "\n--- stderr ---\n" + r.stderr[-8000:]


def test_two_rank_nccl_sync_bn_equals_full_batch():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _run_equiv("nccl", 2)


def test_two_rank_gloo_sync_bn_on_one_gpu_equals_full_batch():
    _run_equiv("gloo", 2)
