"""Fused AdamW and AdaBound over flat parameter / gradient / moment buffers (SURVEY §8f rank 1).

Same update rule and hyper-parameters as the `torch.optim.AdamW(params, lr, weight_decay, betas)` the
reference builds (optimizers/__init__.py:48-59), one kernel launch per network instead of torch's
foreach pass (7 reads/writes of 140 M parameters).  `state_dict()` / `load_state_dict()` keep
torch.optim.AdamW's layout ('step', 'exp_avg', 'exp_avg_sq' per parameter), so `{epoch}_optim_{G,D}.pth`
files are interchangeable with the reference's (base_model.py:168-173,203-212).

`FusedAdaBound` is the reference's other choice (`adabound.AdaBound`, optimizers/__init__.py:55-56) built the same way,
with that package's `state_dict()` layout: a Python int 'step', and `final_lr`, `gamma`, `amsbound` in the group.
"""
from __future__ import annotations

from typing import List

import torch

from . import ops


def flatten_parameters(params: List[torch.nn.Parameter]) -> torch.Tensor:
    """Move the parameters into ONE contiguous fp32 buffer; each p.data becomes a view of it (values,
    state_dict keys and in-place load_state_dict are unaffected)."""
    total = sum(p.numel() for p in params)
    flat = torch.empty(total, dtype=torch.float32, device=params[0].device)
    off = 0
    for p in params:
        n = p.numel()
        flat[off:off + n].copy_(p.data.reshape(-1))
        p.data = flat[off:off + n].view_as(p)
        off += n
    return flat


class _FlatOptimizer(torch.optim.Optimizer):
    """What the fused optimizers share: the parameters as consecutive views of one flat buffer, flat first and second
    moments exposed per parameter in the layout of the optimizer they stand in for, and a step counter."""
    TENSOR_STEP = True      # per-parameter 'step' entry: a float tensor (torch.optim) or a Python int (adabound)

    def __init__(self, params, flat_param: torch.Tensor, defaults: dict):
        params = list(params)
        super().__init__(params, defaults)
        assert flat_param.numel() == sum(p.numel() for p in params)
        off = 0
        for p in params:   # the parameters must be consecutive views of flat_param
            assert p.data_ptr() == flat_param.data_ptr() + 4 * off, "parameters are not views of the flat buffer"
            off += p.numel()
        self.flat_param = flat_param
        self.flat_grad = None                      # attached by the engine (Engine.alloc_grads)
        self.exp_avg = torch.zeros_like(flat_param)
        self.exp_avg_sq = torch.zeros_like(flat_param)
        self._step = 0
        self._expose_state()

    def _expose_state(self) -> None:
        off = 0
        for p in self.param_groups[0]["params"]:
            n = p.numel()
            self.state[p] = {"step": torch.tensor(float(self._step)) if self.TENSOR_STEP else self._step,
                             "exp_avg": self.exp_avg[off:off + n].view_as(p),
                             "exp_avg_sq": self.exp_avg_sq[off:off + n].view_as(p)}
            off += n

    def _count_step(self) -> None:
        self._step += 1
        for st in self.state.values():
            if self.TENSOR_STEP:
                st["step"].fill_(float(self._step))
            else:
                st["step"] = self._step

    def load_state_dict(self, state_dict):
        super().load_state_dict(state_dict)
        # torch replaced the per-parameter tensors: copy them back into the flat buffers
        off = 0
        step = 0
        for p in self.param_groups[0]["params"]:
            n = p.numel()
            st = self.state.get(p, {})
            if "exp_avg" in st:
                self.exp_avg[off:off + n].copy_(st["exp_avg"].reshape(-1))
                self.exp_avg_sq[off:off + n].copy_(st["exp_avg_sq"].reshape(-1))
                step = int(float(st["step"]))
            off += n
        self._step = step
        self._expose_state()


class FusedAdamW(_FlatOptimizer):
    def __init__(self, params, flat_param: torch.Tensor, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2):
        super().__init__(params, flat_param, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))

    @torch.no_grad()
    def step(self, closure=None):
        assert closure is None and self.flat_grad is not None, "FusedAdamW needs the engine's flat gradient buffer"
        g = self.param_groups[0]
        self._count_step()
        ops.adamw_step(self.flat_param, self.flat_grad, self.exp_avg, self.exp_avg_sq, g["lr"], g["betas"][0],
                       g["betas"][1], g["eps"], g["weight_decay"], self._step)

    def advance(self, gscale: float = 1.0):
        """Host half of a step whose kernel reads its scalars from device memory (BaseGAN's step-parameter buffer):
        bump the step counter and return the 8 scalars of ops.adamw_step_dev for it."""
        g = self.param_groups[0]
        self._count_step()
        return ops.adamw_hyper(g["lr"], g["betas"][0], g["betas"][1], g["eps"], g["weight_decay"], self._step, gscale)

    @torch.no_grad()
    def launch(self, hyper_dev: torch.Tensor) -> None:
        """Device half: one fused kernel over the flat buffers (capturable: no host state is touched)."""
        assert self.flat_grad is not None, "FusedAdamW needs the engine's flat gradient buffer"
        ops.adamw_step_dev(self.flat_param, self.flat_grad, self.exp_avg, self.exp_avg_sq, hyper_dev)


class FusedAdaBound(_FlatOptimizer):
    """AdaBound (Luo et al., ICLR 2019) as `adabound.AdaBound(params, lr, betas, final_lr, weight_decay=...)` of
    adabound 0.0.5 runs it, AMSBound excluded: Adam with L2 decay whose per-element step size is clipped into
    [lower, upper], two bounds that close in on `final_lr * lr / base_lr` as the step count grows."""
    TENSOR_STEP = False

    def __init__(self, params, flat_param: torch.Tensor, lr=1e-3, betas=(0.9, 0.999), final_lr=0.1, gamma=1e-3,
                 eps=1e-8, weight_decay=0):
        if not (lr > 0 and final_lr >= 0 and gamma > 0):
            raise ValueError(f"AdaBound needs lr > 0 (final_lr is scaled by lr / base_lr), final_lr >= 0, gamma > 0; "
                             f"got lr={lr}, final_lr={final_lr}, gamma={gamma}")
        super().__init__(params, flat_param, dict(lr=lr, betas=betas, final_lr=final_lr, gamma=gamma, eps=eps,
                                                  weight_decay=weight_decay, amsbound=False))
        self.base_lrs = [g["lr"] for g in self.param_groups]

    def _hyper(self):
        g = self.param_groups[0]
        return (g["lr"], self.base_lrs[0], g["betas"][0], g["betas"][1], g["eps"], g["weight_decay"], g["final_lr"],
                g["gamma"])

    @torch.no_grad()
    def step(self, closure=None):
        assert closure is None and self.flat_grad is not None, "FusedAdaBound needs the engine's flat gradient buffer"
        self._count_step()
        ops.adabound_step(self.flat_param, self.flat_grad, self.exp_avg, self.exp_avg_sq, *self._hyper(), self._step)

    def advance(self, gscale: float = 1.0):
        """Host half of a step (see FusedAdamW.advance): the 8 scalars of ops.adabound_step_dev for the next step."""
        self._count_step()
        return ops.adabound_hyper(*self._hyper(), self._step, gscale)

    @torch.no_grad()
    def launch(self, hyper_dev: torch.Tensor) -> None:
        """Device half: one fused kernel over the flat buffers (capturable: no host state is touched)."""
        assert self.flat_grad is not None, "FusedAdaBound needs the engine's flat gradient buffer"
        ops.adabound_step_dev(self.flat_param, self.flat_grad, self.exp_avg, self.exp_avg_sq, hyper_dev)

    def load_state_dict(self, state_dict):
        if any(g.get("amsbound") for g in state_dict["param_groups"]):
            raise NotImplementedError("AdaBound state saved with amsbound=True: the AMSBound variant is not provided")
        super().load_state_dict(state_dict)
