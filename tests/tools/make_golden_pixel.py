"""Generate tests/golden/pixel_disc_64.pt from the UNMODIFIED reference (needs the reference tree, see
oracle/ref_harness.py).
  * For --norm instance and none: the state dict of define_D(22, 64, 'pixel', norm=...) built after
    torch.manual_seed(SEED) and initialised by modules.init_weights ('kaiming'), and its fp32 output on the seeded
    2 x 22 x 64 x 64 input x_input().
  * ONE full reference WarpModel and ONE TextureModel optimize_parameters() with --discriminator pixel (--gan_mode
    vanilla, --norm instance), recorded as tests/tools/make_golden_gan_modes.py records its steps: losses, checksums of
    every state_dict entry before and after the step, and the CPU generator's state around it.

    python tests/tools/make_golden_pixel.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_harness as RH  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "pixel_disc_64.pt")
CIN, SEED, X_SEED = 22, 0, 4


def x_input():
    return torch.rand(2, CIN, 64, 64, generator=torch.Generator().manual_seed(X_SEED)) * 2 - 1


def reference_net(norm):
    from modules import init_weights
    from modules.discriminators import define_D

    torch.manual_seed(SEED)
    net = define_D(CIN, 64, "pixel", norm=norm)
    init_weights(net, "kaiming", 0.02)
    return net


def reference_step(kind):
    """make_golden_gan_modes.reference_step with --discriminator pixel (same seeds, batch, size, dropout in eval)."""
    import make_golden_gan_modes as MGM

    over = dict(discriminator="pixel")
    warp_opt, texture_opt = RH.warp_opt, RH.texture_opt
    RH.warp_opt = lambda *a, **k: warp_opt(*a, **{**k, **over})
    RH.texture_opt = lambda *a, **k: texture_opt(*a, **{**k, **over})
    try:
        return MGM.reference_step(kind, "vanilla")
    finally:
        RH.warp_opt, RH.texture_opt = warp_opt, texture_opt


def main():
    RH.import_reference()
    x, out = x_input(), {}
    for kind in ("warp", "texture"):
        out[f"{kind}_step"] = reference_step(kind)
    for norm in ("instance", "none"):
        net = reference_net(norm)
        with torch.no_grad():
            out[norm] = {"state_dict": {k: v.clone() for k, v in net.state_dict().items()},
                         "pred": net(x).clone()}
    torch.save(out, OUT)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
