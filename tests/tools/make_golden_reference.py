"""Generate tests/golden/reference_modules.pt and tests/golden/augment_reference_96.npz from the UNMODIFIED reference
(imported through oracle/ref_harness.py): what test_oracle_is_bit_identical_to_reference_modules,
test_perceptual_oracle_is_bit_identical_to_reference and test_matches_the_reference_function compare with, so that the
same comparisons run where the reference is absent.

    python tests/tools/make_golden_reference.py
"""
import os
import random
import sys
from argparse import Namespace

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torchvision  # noqa: E402

from oracle import augment as A  # noqa: E402
from oracle import ref_harness as RH  # noqa: E402
from test_augment_cpu import label_map, rng_digest  # noqa: E402
from test_engine_gpu import synth_texture_batch, synth_warp_batch  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def sums(t):
    return (float(t.double().sum()), float(t.double().abs().sum()))


RH.import_reference()
from datasets import get_transforms  # noqa: E402
from datasets.data_utils import per_channel_transform  # noqa: E402
from modules import init_weights  # noqa: E402
from modules.discriminators import define_D  # noqa: E402
from modules.swapnet_modules import TextureModule, WarpModule  # noqa: E402
import modules.losses.perceptual as P  # noqa: E402

gold = {}
torch.manual_seed(0)
G = WarpModule(); init_weights(G, "kaiming")
D = define_D(22, 64, "basic", 3, "instance"); init_weights(D, "kaiming")
G.eval(); D.eval()
body, inp, _ = synth_warp_batch(2, 64)
with torch.no_grad():
    fakes = G(body, inp)
    pred = D(torch.cat((body, fakes), 1))
gold["warp_fakes_sub"], gold["warp_fakes_sums"] = fakes[:, :, ::4, ::4].clone(), sums(fakes)
gold["patchgan_pred"] = pred.clone()
torch.manual_seed(0)
T = TextureModule(3, 19, 12, "instance", 0.5, "pix2pix", 128); init_weights(T, "kaiming"); T.eval()
tex, rois, cloth, _ = synth_texture_batch(2, 128)
with torch.no_grad():
    tout = T(tex, rois, cloth.clone())
gold["texture_fakes_sub"], gold["texture_fakes_sums"] = tout[:, :, ::4, ::4].clone(), sums(tout)
torch.manual_seed(3)
W = WarpModule(); init_weights(W, "kaiming")
gold["warp_state_keys"] = list(W.state_dict())
gold["warp_seed3_sums"] = {k: sums(v) for k, v in W.state_dict().items()}


def seeded(pretrained=False, **kw):
    with torch.random.fork_rng():
        torch.manual_seed(1234)
        return torchvision.models.vgg16(weights=None)


orig = P.vgg16
P.vgg16 = seeded
try:
    crit = P.PerceptualLoss(use_style=True)
finally:
    P.vgg16 = orig
g = torch.Generator().manual_seed(5)
out = torch.rand(2, 3, 64, 64, generator=g).requires_grad_()
tgt = torch.rand(2, 3, 64, 64, generator=g)
c, s = crit(out, tgt)
(c * 20 + s * 1e-8).backward()
gold["perceptual"] = dict(content=float(c.detach()), style=float(s.detach()), grad_sub=out.grad[:, :, ::4, ::4].clone(),
                          grad_sums=sums(out.grad))
torch.save(gold, os.path.join(GOLD, "reference_modules.pt"))

tf = get_transforms(Namespace(input_transforms=("hflip", "vflip", "affine", "perspective")))
cloth = torch.from_numpy(A.onehot(label_map(96, 96, 7), 19))
aug = {}
for seed in (0, 1, 2):
    random.seed(seed); torch.manual_seed(seed)
    aug[f"out_{seed}"] = per_channel_transform(cloth, tf).numpy()
    aug[f"rng_{seed}"] = np.array(rng_digest())
np.savez_compressed(os.path.join(GOLD, "augment_reference_96.npz"), **aug)
print("warp", gold["warp_fakes_sums"], "texture", gold["texture_fakes_sums"], "perceptual", gold["perceptual"]["content"])
