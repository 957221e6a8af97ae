"""CPU tests of host-side invariants the CUDA kernels rely on (no GPU, no library calls)."""
import builtins
import io

import torch

import bench
from swapnet_b200 import lowering as L
from swapnet_b200 import ops


def test_planes_views_keep_the_plane_stride():
    """The GEMM kernels fetch the hi and lo planes of a tile with ONE TMA box whose outermost dimension is the
    plane (csrc/gemm_tc.cu sn_make_act_map(plane_stride)): hi and lo must live a fixed stride apart, also for
    channel slices and batch slices of a buffer."""
    p = ops.Planes(4, 6, 8, 64, "cpu", dual=True)
    stride = p.lo.data_ptr() - p.hi.data_ptr()
    assert stride == 2 * 4 * 6 * 8 * 64 and stride % 16 == 0
    for v in (p.slice(16, 32), p.batch_slice(1, 2), p.slice(8, 8).batch_slice(2, 2), p.twin, p.twin.batch_slice(3, 1)):
        assert v.lo_ptr - v.hi_ptr == stride
        assert v.lo.data_ptr() - v.hi.data_ptr() == stride
    w = ops.PackedWeights(48, 128, "cpu")
    assert w.lo.data_ptr() - w.hi.data_ptr() == 2 * 48 * 128


def test_pack_table_refuses_a_misaligned_weight():
    """The scale kernel reads weights as float4 (csrc/elementwise.cu weight_scale_multi_kernel): a weight that does not
    start on a 16-byte boundary is refused when it is registered, not read misaligned on the device."""
    import pytest

    table = ops.PackTable("cpu")
    flat = torch.zeros(20)
    table.add_scale(flat[4:13], torch.ones(2))        # 16-byte aligned, 9 floats: the tail is the kernel's business
    with pytest.raises(AssertionError, match="16-byte aligned"):
        table.add_scale(flat[1:9], torch.ones(2))


def test_reflect_pad_fanout_matches_torch(tmp_path):
    """csrc/reflect_pad.h compiled for the host: the padded positions of every interior index are exactly the
    positions torch's ReflectionPad2d(1) fills from it, for axes of 2..9 elements (3 is the axis whose middle
    index owns both mirrors, three positions)."""
    import os
    import sys

    import pytest
    import torch.nn.functional as F

    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "tools"))
    import kernel_host_shim

    lib = kernel_host_shim.build_reflect(str(tmp_path))
    if lib is None:
        pytest.skip("no g++")
    for n in range(2, 10):
        src = F.pad(torch.arange(n, dtype=torch.float64).view(1, 1, n), (1, 1), mode="reflect").view(-1).long()
        for i in range(n):
            pos = [lib.position(i, n, k) for k in range(lib.count(i, n))]
            assert pos[0] == i + 1 and sorted(pos) == (src == i).nonzero().view(-1).tolist(), (n, i, pos)


def test_phase_merge_only_for_the_four_parity_phases():
    specs = L.forward_specs("convT4s2", 8, 8)
    m = ops.merge_phase_specs(specs)
    assert m is not None and len(m.taps) == 16 and m.out_mul == (2, 2)
    assert [t.kb for t in m.taps] == list(range(16))          # phase-major packed slots: phase z owns taps 4z..4z+3
    assert ops.merge_phase_specs(L.forward_specs("head", 8, 8)) is None      # unequal tap counts / per-phase weights
    assert ops.merge_phase_specs(L.forward_specs("conv3r", 8, 8)) is None


def test_block_n_and_channel_padding_rules():
    assert [L.padc(c) for c in (1, 3, 16, 19, 22, 36, 64, 65)] == [16, 16, 16, 32, 32, 64, 64, 128]
    assert [L.pick_block_n(n) for n in (1, 16, 19, 36, 64, 100, 128, 1024)] == [16, 16, 32, 64, 64, 128, 128, 128]


def test_host_cores_respects_the_cgroup_quota(monkeypatch):
    """bench.host_cores(): the GPU boxes show 128 logical CPUs under a 16-CPU cgroup quota."""
    real_open = builtins.open

    def fake_open(path, *a, **k):
        if path == "/sys/fs/cgroup/cpu.max":
            return io.StringIO("1600000 100000\n")
        return real_open(path, *a, **k)

    monkeypatch.setattr(bench.os, "sched_getaffinity", lambda pid: set(range(128)), raising=False)
    monkeypatch.setattr(builtins, "open", fake_open)
    assert bench.host_cores() == 16

    def fake_open_max(path, *a, **k):
        if path == "/sys/fs/cgroup/cpu.max":
            return io.StringIO("max 100000\n")
        if path.startswith("/sys/fs/cgroup/cpu/"):
            raise OSError(path)
        return real_open(path, *a, **k)

    monkeypatch.setattr(builtins, "open", fake_open_max)
    assert bench.host_cores() == 128


def test_segmap_roundtrip_and_format_choice():
    """ops.SegMap: the compact wire format of the 0/1 cloth tensors (uint8 label map when one-hot with an empty channel
    0 — datasets/data_utils.py:330-343 —, else an int32 bit mask); dense() restores the tensor exactly."""
    import torch

    from swapnet_b200.ops import SegMap

    g = torch.Generator().manual_seed(0)
    lab = torch.randint(0, 19, (2, 8, 8), generator=g)
    onehot = torch.zeros(2, 19, 8, 8)
    for c in range(1, 19):
        onehot[:, c] = (lab == c).float()
    s = SegMap.from_dense(onehot)
    assert s.data.dtype == torch.uint8 and torch.equal(s.data, lab.to(torch.uint8)) and s.shape == (2, 19, 8, 8)
    assert torch.equal(s.dense(), onehot)
    multi = onehot.clone()
    multi[:, 5] = torch.roll(multi[:, 5], 1, 1)
    multi[:, 0, 0, 0] = 1.0                      # something in channel 0: not representable as a label map
    m = SegMap.from_dense(multi)
    assert m.data.dtype == torch.int32 and torch.equal(m.dense(), multi)
    import pytest

    with pytest.raises(ValueError):
        SegMap.from_dense(onehot * 0.5)


def test_grad_buckets_tile_the_flat_gradient_buffer():
    """WarpEngine.grad_buckets(): the seven all-reduce buckets are disjoint contiguous slices that cover the flat
    gradient buffer exactly, in the order backward() retires them (decoder + head first, the small down-path layers last)."""
    from swapnet_b200 import modules as M
    from swapnet_b200.engine import WarpEngine

    G = M.WarpModule()

    class Stub:          # grad_buckets only reads the parameter names and sizes
        net = G

    b = WarpEngine.grad_buckets(Stub())
    total = sum(p.numel() for p in G.parameters())
    assert len(b) == 7
    cov = sorted(b)
    assert cov[0][0] == 0 and cov[-1][1] == total and all(cov[i][1] == cov[i + 1][0] for i in range(len(cov) - 1))
    names = [n for n, _ in G.named_parameters()]
    offs, o = {}, 0
    for n, p in G.named_parameters():
        offs[n] = o
        o += p.numel()
    lo, hi = b[0]
    assert lo <= offs["upsample_and_pad.2.weight"] < hi and lo <= offs["dual_up1.model.0.weight"] < hi
    assert b[1][0] <= offs["resblocks.3.conv_block.1.weight"] < b[1][1]          # the last resblock retires first
    assert b[4][0] <= offs["resblocks.0.conv_block.6.weight"] < b[4][1]
    assert b[5][0] <= offs["cloth_up2.model.0.weight"] < b[5][1] and b[5][0] <= offs["cloth_down5.model.0.weight"] < b[5][1]
    assert b[6][0] == 0 and b[6][0] <= offs["cloth_down4.model.0.weight"] < b[6][1]
    assert names[0].startswith("body_down1")


def test_adamw_hyper_matches_torch_formula():
    """sn_adamw_hyper (host side of the device-parameterised AdamW): the eight fp32 scalars of step t are the ones
    torch.optim.AdamW forms from its Python-float hyper-parameters (bias corrections in double, rounded once)."""
    import math

    from swapnet_b200 import ops

    lr, b1, b2, eps, wd = 4e-4, 0.9, 0.999, 1e-8, 0.01
    for step in (1, 2, 17, 1000):
        h = ops.adamw_hyper(lr, b1, b2, eps, wd, step, 0.125)
        bc1, bc2 = 1.0 - b1 ** step, 1.0 - b2 ** step
        want = [1.0 - lr * wd, 1.0 - b1, b2, 1.0 - b2, lr / bc1, 1.0 / math.sqrt(bc2), eps, 0.125]
        import numpy as np

        assert np.array_equal(np.float32(want), np.float32(h)), (step, want, h)


def test_launcher_path_order(tmp_path, monkeypatch):
    """swapnet_b200.run puts <repo>/dropin ahead of the script's directory (where the reference's own `models`
    package lives) and runs the script as __main__ with its argv."""
    import os
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    ck = tmp_path / "checkout"
    (ck / "models").mkdir(parents=True)
    (ck / "models" / "__init__.py").write_text("WHO = 'reference'\n")
    (ck / "probe.py").write_text("import sys, models\nprint('PROBE', models.__name__, models.__file__, sys.argv[1:], __name__)\n")
    r = subprocess.run([sys.executable, "-m", "swapnet_b200.run", "probe.py", "--model", "warp"], cwd=str(ck),
                       env=dict(os.environ, PYTHONPATH=root), capture_output=True, text=True, timeout=300)
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("PROBE")]
    assert r.returncode == 0 and line, (r.stdout, r.stderr[-1500:])
    assert os.path.join(root, "dropin", "models") in line[0] and "['--model', 'warp']" in line[0] and line[0].endswith("__main__")
