"""Host logic of --b200_deterministic (no GPU): how the mode is selected, the shape-only split-K rule of the
deterministic weight-gradient plans, and the sizing of the slot workspaces."""
import argparse

import pytest
import torch

from swapnet_b200 import _lib
from swapnet_b200 import lowering as L
from swapnet_b200 import ops
from swapnet_b200.models.base_gan import BaseGAN, deterministic_mode


@pytest.fixture
def torch_flag():
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    yield lambda on: torch.use_deterministic_algorithms(on, warn_only=True)
    torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def test_option_defaults_to_torch_flag_and_overrides_it(torch_flag):
    p = argparse.ArgumentParser()
    BaseGAN.modify_commandline_options(p, False)          # registered outside is_train: inference uses it too
    assert p.parse_args([]).b200_deterministic is None
    assert p.parse_args(["--b200_deterministic", "1"]).b200_deterministic == 1
    torch_flag(True)
    assert deterministic_mode(argparse.Namespace())      # options built by hand (no attribute): torch's flag
    assert deterministic_mode(p.parse_args([]))
    assert not deterministic_mode(p.parse_args(["--b200_deterministic", "0"]))
    torch_flag(False)
    assert not deterministic_mode(argparse.Namespace())
    assert deterministic_mode(argparse.Namespace(b200_deterministic=1))


def _wgrad_desc(kind, cin, cout, hw, n, deterministic):
    (ws,) = L.wgrad_specs(kind, hw, hw)
    in_h = hw + 2 if kind == "conv3r" else hw
    x = ops.Planes(n, in_h, in_h, L.padc(cin), "cpu", fmt=ops.FMT_BF16)
    oh, ow = L.out_hw(kind, hw, hw)
    dy = ops.Planes(n, oh, ow, max(L.padc(cout), 64), "cpu", fmt=ops.FMT_BF16)
    xs, ys = (dy, x) if ws.x_is == "dy" else (x, dy)
    cx, cy = (cout, cin) if ws.x_is == "dy" else (cin, cout)
    s_row, s_col = L.wgrad_out_strides(kind, cin, cout, ws.x_is == "dy")
    out = torch.zeros(1)
    swap = xs.c < 64 or (ys.c >= 64 and cy > cx)
    return ops.wgrad_desc(xs, ys, ws, out, s_row, s_col, list(ws.tap_ids), cx, cy, swap=swap,
                          deterministic=deterministic)


@pytest.mark.parametrize("kind,cin,cout,hw,n", [("conv4s2", 64, 64, 128, 4), ("conv4s2", 3, 64, 512, 16),
                                                ("conv3r", 1024, 1024, 32, 16), ("convT4s2", 128, 64, 64, 16)])
def test_deterministic_split_count_depends_on_shapes_only(kind, cin, cout, hw, n):
    _lib.load(build_if_missing=True)
    det = _wgrad_desc(kind, cin, cout, hw, n, True)
    ks = {ops.wgrad_ksplit(det, sms) for sms in (1, 78, 114, 132, 148, 1000)}
    assert len(ks) == 1, ks
    assert ks == {ops.wgrad_ksplit(_wgrad_desc(kind, cin, cout, hw, n, False), 132)}   # = the default rule on 132 SMs


def test_default_split_count_follows_the_device():
    _lib.load(build_if_missing=True)
    d = _wgrad_desc("conv4s2", 64, 64, 128, 4, False)
    assert ops.wgrad_ksplit(d, 16) < ops.wgrad_ksplit(d, 132)


def test_slot_workspace_sizing():
    lib = _lib.load(build_if_missing=True)
    num_sms = 132
    for n, c in ((1, 1), (16, 64), (32, 1024)):
        need = lib.sn_det_slots(n, c)
        assert need >= 2 * n * c + 2 * 6 * num_sms * 256
    assert lib.sn_to_one_wgrad_det_slots(512) == 4 * num_sms * 512 * 16
    ws = ops.DetWorkspace("cpu")
    assert ws.nbytes == 0
    a = ws.get(100)
    assert a.dtype == torch.float64 and a.numel() >= 100 and ws.nbytes == 800
    f = ws.get(150, torch.float32)              # fits: the buffer is reused, viewed as float32
    assert f.dtype == torch.float32 and f.numel() >= 150 and ws.nbytes == 800
    ws.get(1000)
    assert ws.nbytes == 8000
