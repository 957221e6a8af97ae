"""Model lifecycle shared by the plugins — same public protocol as
/root/reference/models/base_model.py:20-246 (setup / set_input / optimize_parameters / test /
get_current_losses / get_current_visuals / save_checkpoint / load_checkpoint_dir / ...), so that
train.py:38-116 and inference.py drive it unchanged.
"""
from __future__ import annotations

import os
from abc import ABC, abstractmethod
from collections import OrderedDict

import torch


class LazyLoss:
    """A loss that lives on the device until somebody asks for a float (train.py:74 does, every
    iteration — the only host sync of a step: BaseGAN.loss_values() fetches all terms of the step with ONE
    64-byte device-to-host copy)."""

    def __init__(self, fn):
        self._fn = fn

    def __float__(self):
        return float(self._fn())

    def item(self):
        return float(self)

    def __repr__(self):
        return f"{float(self):.6f}"


class BaseModel(ABC):
    def __init__(self, opt):
        self.opt = opt
        self.gpu_id = opt.gpu_id
        self.is_train = opt.is_train
        if self.gpu_id is None or not torch.cuda.is_available():
            raise RuntimeError(
                "swapnet_b200 models run on a CUDA device only (--gpu_id >= 0 on a B200); there is no "
                "CPU / eager fallback of the hot path")
        # data parallel without touching train.py: under `torchrun ... train.py` (WORLD_SIZE > 1 in the environment)
        # every rank drives the GPU of its LOCAL_RANK (train.py's --gpu_id default of 0 would put all ranks on one
        # device) and the NCCL process group is created here, before the parameters are broadcast (base_gan.py)
        from .. import parallel

        if parallel.launched_distributed():
            self.gpu_id = parallel.init_from_env()
        self.device = torch.device(f"cuda:{self.gpu_id}")
        torch.cuda.set_device(self.device)
        self.save_dir = os.path.join(opt.checkpoints_dir, opt.name)
        if self.is_train:
            try:        # base_model.py:43-44: ask before re-using a non-empty experiment directory (--no_confirm skips)
                from util.util import PromptOnce
            except ImportError:                # standalone use (bench, tests): no reference tree on the path
                os.makedirs(self.save_dir, exist_ok=True)
            else:
                PromptOnce.makedirs(self.save_dir, not getattr(opt, "no_confirm", True))
        self.loss_names = []
        self.model_names = []
        self.visual_names = []
        self.optimizer_names = []
        self.image_paths = []
        self.metric = 0
        self.training = True

    # ---- late H2D copies: tensors that the step needs only after its first phase ----
    def copy_late(self, t, key: str = None, seg_channels: int = 0):
        """H2D copy on a side stream (pinned host tensors; plain conversion for device tensors).  The step
        waits for it where the tensor is first needed: `wait_copy(key)` or, for everything still pending,
        `wait_late_copies()`.  Copies run in issue order, so the tensors a step needs first go first.

        seg_channels > 0: the entry may also arrive in compact form — a uint8 label map or an int32 bit mask [B,H,W]
        (ops.SegMap; SURVEY §8f rank 4) — which travels as 1-4 bytes per pixel instead of 4*channels and is expanded
        by the consuming kernels; fp32 [B,C,H,W] tensors are handled as before."""
        from ..ops import SegMap

        if isinstance(t, SegMap):
            seg_channels, t = t.channels, t.data
        compact = seg_channels > 0 and t.dim() == 3 and t.dtype in (torch.uint8, torch.int32)
        dtype = t.dtype if compact else torch.float32
        if t.is_cuda:
            out = t.to(device=self.device, dtype=dtype).contiguous()
            return SegMap(out, seg_channels) if compact else out
        if not hasattr(self, "_copy_stream"):
            self._copy_stream = torch.cuda.Stream(device=self.device)
            self._late_events = []
            self._copy_events = {}
        cur = torch.cuda.current_stream(self.device)
        # no wait on `cur`: the destination is a fresh allocation of the copy stream's pool (the caching allocator
        # only recycles a block once the streams recorded on it — record_stream below — have passed its last use),
        # so the copy of step N+1's inputs overlaps the compute of step N
        with torch.cuda.stream(self._copy_stream):
            out = t.to(device=self.device, dtype=dtype, non_blocking=True).contiguous()
            ev = torch.cuda.Event()
            ev.record(self._copy_stream)
        out.record_stream(cur)
        self._late_events.append(ev)
        if key is not None:
            self._copy_events[key] = ev
        return SegMap(out, seg_channels) if compact else out

    @staticmethod
    def dense(t):
        """fp32 [B,C,H,W] view of an input that may have arrived in compact form (visuals, off the hot path)."""
        return t.dense() if hasattr(t, "dense") else t

    def wait_copy(self, key: str) -> None:
        ev = getattr(self, "_copy_events", {}).pop(key, None)
        if ev is not None:
            torch.cuda.current_stream(self.device).wait_event(ev)
            if ev in self._late_events:
                self._late_events.remove(ev)

    def wait_late_copies(self) -> None:
        for ev in getattr(self, "_late_events", []):
            torch.cuda.current_stream(self.device).wait_event(ev)
        if hasattr(self, "_late_events"):
            self._late_events.clear()
            self._copy_events.clear()

    @staticmethod
    def modify_commandline_options(parser, is_train):
        return parser

    @abstractmethod
    def set_input(self, input):
        ...

    @abstractmethod
    def forward(self):
        ...

    @abstractmethod
    def optimize_parameters(self):
        ...

    def setup(self, opt):
        if not self.is_train or opt.continue_train:
            self.load_checkpoint_dir(opt.load_epoch)
        self.print_networks(opt.verbose)
        return self

    def eval(self):
        """Dropout off (SURVEY App. B #3); with --norm batch the engines use the running statistics."""
        self.training = False
        for name in self.model_names:
            getattr(self, "net_" + name).eval()
        return self

    def train(self):
        self.training = True
        for name in self.model_names:
            getattr(self, "net_" + name).train()
        return self

    def test(self):
        with torch.no_grad():
            self.forward()
            self.compute_visuals()

    def compute_visuals(self):
        pass

    def get_image_paths(self):
        return self.image_paths

    def update_learning_rate(self):
        lr = getattr(self, "optimizer_" + self.optimizer_names[0]).param_groups[0]["lr"]
        print("learning rate = %.7f" % lr)

    def get_current_visuals(self):
        return OrderedDict((n, getattr(self, n)) for n in self.visual_names if isinstance(n, str))

    def get_current_losses(self):
        return OrderedDict((n, float(getattr(self, "loss_" + n))) for n in self.loss_names if isinstance(n, str))

    # ---- checkpoints: same file names and state_dict keys as the reference ----
    def save_checkpoint(self, epoch):
        from .. import parallel

        if parallel.rank() != 0:      # replicas are identical: one writer (all ranks share checkpoints_dir/name)
            return
        for name in self.model_names:
            net = getattr(self, f"net_{name}")
            # parameters stay where they are (the engines hold their addresses); save a CPU copy
            sd = OrderedDict((k, v.detach().cpu()) for k, v in net.state_dict().items())
            torch.save(sd, os.path.join(self.save_dir, f"{epoch}_net_{name}.pth"))
        for name in self.optimizer_names:
            torch.save(getattr(self, f"optimizer_{name}").state_dict(),
                       os.path.join(self.save_dir, f"{epoch}_optim_{name}.pth"))

    def load_model_weights(self, model_name, weights_file):
        net = getattr(self, f"net_{model_name}")
        print(f"loading the model {model_name} from {weights_file}")
        state_dict = torch.load(weights_file, map_location=self.device)
        if hasattr(state_dict, "_metadata"):
            del state_dict._metadata
        net.load_state_dict(state_dict)  # in place: engine plans keep pointing at the same storage
        return self

    def load_checkpoint_dir(self, epoch):
        for name in self.model_names:
            self.load_model_weights(name, os.path.join(self.save_dir, f"{epoch}_net_{name}.pth"))
        if self.is_train:
            for name in self.optimizer_names:
                path = os.path.join(self.save_dir, f"{epoch}_optim_{name}.pth")
                print(f"loading the optimizer {name} from {path}")
                getattr(self, f"optimizer_{name}").load_state_dict(torch.load(path))
        return self

    def print_networks(self, verbose):
        print("---------- Networks initialized -------------")
        for name in self.model_names:
            net = getattr(self, "net_" + name)
            if verbose:
                print(net)
            print("[Network %s] Total number of parameters : %.3f M"
                  % (name, sum(p.numel() for p in net.parameters()) / 1e6))
        print("-----------------------------------------------")

    def set_requires_grad(self, nets, requires_grad=False):
        for net in nets if isinstance(nets, list) else [nets]:
            if net is not None:
                for p in net.parameters():
                    p.requires_grad = requires_grad
