"""Top-level `models` package for the reference's train.py / options code.

Put this directory AHEAD of the reference checkout on PYTHONPATH (INTEGRATION.md): `from models import
create_model`, `models.get_options_modifier(...)` and `import models.warp_model` then resolve to the
B200 plugins in swapnet_b200.models, everything else (options/, datasets/, util/, optimizers/) still
comes from the reference tree.
"""
import sys as _sys

from swapnet_b200 import models as _impl
from swapnet_b200.models import BaseModel, create_model  # noqa: F401
from swapnet_b200.models import base_gan, base_model, pix2pix_model, texture_model, warp_model  # noqa: F401

for _name in ("base_model", "base_gan", "warp_model", "texture_model", "pix2pix_model"):
    _sys.modules[f"{__name__}.{_name}"] = getattr(_impl, _name)


def find_model_using_name(model_name):
    return _impl.find_model_using_name(model_name)


def get_options_modifier(model_name):
    return _impl.get_options_modifier(model_name)
