"""AdaBound in plain torch, one tensor at a time, in the dtype of the tensors it is given (tests only).

The update of Luo et al., "Adaptive Gradient Methods with Dynamic Bound of Learning Rate" (ICLR 2019), as the
`adabound` package (0.0.5, the version the reference pins) applies it with `amsbound=False`: Adam moments over a gradient
that includes the L2 decay term, and a per-element step size clipped into bounds that close in on
`final_lr * lr / base_lr`.  Restated from the published algorithm: the package itself is not a dependency of this
repository.
"""
import math

import torch

GAMMA, EPS = 1e-3, 1e-8          # the package's defaults; the reference sets neither


def scalars(t, lr, base_lr, betas, final_lr, gamma=GAMMA):
    """(step_size, lower, upper) of optimizer step t >= 1 as Python floats (double)."""
    b1, b2 = betas
    step_size = lr * math.sqrt(1 - b2 ** t) / (1 - b1 ** t)
    final = final_lr * lr / base_lr
    return step_size, final * (1 - 1 / (gamma * t + 1)), final * (1 + 1 / (gamma * t))


def step(p, g, m, v, t, lr, betas=(0.9, 0.999), final_lr=0.1, gamma=GAMMA, eps=EPS, weight_decay=0.0, base_lr=None,
         gscale=1.0):
    """Step t (1-based) on p, m, v in place; g is left alone.  Returns the clipped per-element step size."""
    b1, b2 = betas
    step_size, lower, upper = scalars(t, lr, lr if base_lr is None else base_lr, betas, final_lr, gamma)
    g = g * gscale
    if weight_decay != 0:
        g = g + weight_decay * p
    m.mul_(b1).add_(g, alpha=1 - b1)
    v.mul_(b2).addcmul_(g, g, value=1 - b2)
    eta = (step_size / (v.sqrt() + eps)).clamp_(lower, upper)
    p.sub_(eta * m)
    return eta
