"""Parameter containers for the B200 engines.

These nn.Modules hold ONLY the trainable tensors, under exactly the state_dict keys (and in the
construction / nn.Module.apply order, so that a seeded init matches) of the reference networks:
  WarpModule           /root/reference/modules/swapnet_modules.py:22-90
  NLayerDiscriminator  /root/reference/modules/discriminators.py:91-132
  PixelDiscriminator   /root/reference/modules/discriminators.py:138-168
  TextureModule        /root/reference/modules/swapnet_modules.py:154-207
  UnetGenerator        /root/reference/modules/pix2pix_modules.py:113-262
Checkpoints are therefore interchangeable with the reference (`base_model.py:156-213`).  The
modules have no eager forward: compute runs in swapnet_b200.engine through the CUDA library and
calling them raises.
"""
from __future__ import annotations

import math

import torch
from torch import nn
from torch.nn import init


class _NoEager(nn.Module):
    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError(
            f"{type(self).__name__} is a parameter container; the forward/backward of this network "
            "runs in swapnet_b200.engine (CUDA, sm_90a) — there is no eager fallback")


def _slots(conv: nn.Module, index: int, total: int) -> nn.Sequential:
    """Sequential with `conv` at position `index` and parameter-free placeholders elsewhere, so that
    the state_dict key is '<...>.{index}.weight' like the reference Sequential."""
    return nn.Sequential(*[conv if i == index else nn.Identity() for i in range(total)])


class _Holder(_NoEager):
    def __init__(self, attr: str, seq: nn.Sequential):
        super().__init__()
        setattr(self, attr, seq)


def _down(cin, cout, norm=True, drop=0.0):   # layers.py:12-24: conv is model.0
    n = 2 + int(norm) + int(bool(drop))
    return _Holder("model", _slots(nn.Conv2d(cin, cout, 4, 2, 1, bias=False), 0, n))


def _up(cin, cout, drop=0.0):                # layers.py:27-44: convT is model.0
    return _Holder("model", _slots(nn.ConvTranspose2d(cin, cout, 4, 2, 1, bias=False), 0, 3 + int(bool(drop))))


class _ResBlock(_NoEager):                   # layers.py:126-144: convs are conv_block.1 / .6
    def __init__(self, c):
        super().__init__()
        seq = [nn.Identity() for _ in range(8)]
        seq[1] = nn.Conv2d(c, c, 3)
        seq[6] = nn.Conv2d(c, c, 3)
        self.conv_block = nn.Sequential(*seq)


class WarpModule(_NoEager):
    def __init__(self, body_channels=3, cloth_channels=19, dropout=0.5):
        super().__init__()
        self.body_channels, self.cloth_channels, self.dropout = body_channels, cloth_channels, dropout
        self.body_down1 = _down(body_channels, 64, norm=False)
        self.body_down2 = _down(64, 128)
        self.body_down3 = _down(128, 256)
        self.body_down4 = _down(256, 512, drop=dropout)
        self.cloth_down1 = _down(cloth_channels, 64, norm=False)
        self.cloth_down2 = _down(64, 128)
        self.cloth_down3 = _down(128, 256)
        self.cloth_down4 = _down(256, 512)
        self.cloth_down5 = _down(512, 1024, drop=dropout)
        self.cloth_down6 = _down(1024, 1024, norm=False, drop=dropout)
        self.cloth_up1 = _up(1024, 1024)
        self.cloth_up2 = _up(1024, 512)
        self.resblocks = nn.Sequential(*[_ResBlock(1024) for _ in range(4)])
        self.dual_up1 = _up(1024, 256)
        self.dual_up2 = _up(3 * 256, 128)
        self.dual_up3 = _up(3 * 128, 64)
        self.upsample_and_pad = _slots(nn.Conv2d(3 * 64, cloth_channels, 4, padding=1), 2, 4)


NORMS = ("instance", "batch", "none")


def check_norm(norm: str) -> str:
    """modules/__init__.py:53-74 get_norm_layer's choices."""
    if norm not in NORMS:
        raise NotImplementedError(f"normalization layer [{norm}] is not found")
    return norm


def _norm_slot(norm: str, c: int) -> nn.Module:
    """The module get_norm_layer(norm)(c) puts in a norm slot: a real BatchNorm2d (weight, bias and running buffers
    under the reference's keys; initialised by init_weights in the same apply order), else a parameter-free
    placeholder (InstanceNorm2d(affine=False) and Identity hold no state)."""
    return nn.BatchNorm2d(c) if norm == "batch" else nn.Identity()


class NLayerDiscriminator(_NoEager):
    """PatchGAN 'basic' (n_layers=3).  norm: 'instance' (bias on every conv), 'batch' (BatchNorm2d at model.3/6/9,
    no bias on the convs it follows), 'none'."""

    def __init__(self, input_nc, ndf=64, n_layers=3, norm="instance"):
        super().__init__()
        self.norm, self.input_nc, self.ndf, self.n_layers = check_norm(norm), input_nc, ndf, n_layers
        use_bias = norm == "instance"    # discriminators.py:104-107
        seq = [nn.Conv2d(input_nc, ndf, 4, 2, 1), nn.Identity()]
        self.conv_index = [0]
        mult = 1
        for n in range(1, n_layers):
            prev, mult = mult, min(2 ** n, 8)
            self.conv_index.append(len(seq))
            seq += [nn.Conv2d(ndf * prev, ndf * mult, 4, 2, 1, bias=use_bias), _norm_slot(norm, ndf * mult), nn.Identity()]
        prev, mult = mult, min(2 ** n_layers, 8)
        self.conv_index.append(len(seq))
        seq += [nn.Conv2d(ndf * prev, ndf * mult, 4, 1, 1, bias=use_bias), _norm_slot(norm, ndf * mult), nn.Identity()]
        self.conv_index.append(len(seq))
        seq += [nn.Conv2d(ndf * mult, 1, 4, 1, 1)]
        self.model = nn.Sequential(*seq)

    def convs(self):
        return [self.model[i] for i in self.conv_index]

    def bns(self):
        """The BatchNorm2d after each conv (None where there is none), aligned with convs()."""
        return [self.model[i + 1] if isinstance(self.model[i + 1], nn.BatchNorm2d) else None
                for i in self.conv_index[:-1]] + [None]


PIXEL_MAX_INPUT_NC = 32   # the widest operand the fused passes of csrc/pixel_disc.cu read (KX)


class PixelDiscriminator(_NoEager):
    """The 1x1 PatchGAN ('pixel', discriminators.py:138-168): net.0 Conv 1x1 input_nc -> ndf (bias), net.1 LeakyReLU,
    net.2 Conv ndf -> 2 ndf, net.3 the norm slot, net.4 LeakyReLU, net.5 Conv 2 ndf -> 1.  As in the reference, net.2 and
    net.5 have a bias only with InstanceNorm2d.  ndf = 64 and input_nc <= PIXEL_MAX_INPUT_NC only (csrc/pixel_disc.cu's
    widths)."""

    def __init__(self, input_nc, ndf=64, norm="instance"):
        super().__init__()
        self.norm, self.input_nc, self.ndf = check_norm(norm), input_nc, ndf
        use_bias = norm == "instance"    # discriminators.py:150-153
        self.net = nn.Sequential(nn.Conv2d(input_nc, ndf, 1), nn.Identity(),
                                 nn.Conv2d(ndf, ndf * 2, 1, bias=use_bias), _norm_slot(norm, ndf * 2), nn.Identity(),
                                 nn.Conv2d(ndf * 2, 1, 1, bias=use_bias))


class _SkipBlock(_NoEager):
    """pix2pix_modules.py:180-262 — Sequential positions of down conv / submodule / up conv differ per
    block type; reproduce the indices so the keys match (model.{i}.weight)."""

    def __init__(self, outer_nc, inner_nc, input_nc=None, submodule=None, outermost=False, innermost=False,
                 use_dropout=False, norm="instance"):
        super().__init__()
        self.outermost, self.innermost, self.use_dropout = outermost, innermost, use_dropout
        use_bias = norm == "instance"    # pix2pix_modules.py:214-217
        input_nc = outer_nc if input_nc is None else input_nc
        down = nn.Conv2d(input_nc, inner_nc, 4, 2, 1, bias=use_bias)
        self.down_bn_i = self.up_bn_i = None
        if outermost:      # [downconv, sub, uprelu, upconv, tanh]
            up = nn.ConvTranspose2d(inner_nc * 2, outer_nc, 4, 2, 1)
            seq = [down, submodule, nn.Identity(), up, nn.Identity()]
            self.down_i, self.sub_i, self.up_i = 0, 1, 3
        elif innermost:    # [downrelu, downconv, uprelu, upconv, upnorm]
            up = nn.ConvTranspose2d(inner_nc, outer_nc, 4, 2, 1, bias=use_bias)
            seq = [nn.Identity(), down, nn.Identity(), up, _norm_slot(norm, outer_nc)]
            self.down_i, self.sub_i, self.up_i = 1, None, 3
            self.up_bn_i = 4
        else:              # [downrelu, downconv, downnorm, sub, uprelu, upconv, upnorm, (dropout)]
            up = nn.ConvTranspose2d(inner_nc * 2, outer_nc, 4, 2, 1, bias=use_bias)
            seq = [nn.Identity(), down, _norm_slot(norm, inner_nc), submodule, nn.Identity(), up,
                   _norm_slot(norm, outer_nc)]
            if use_dropout:
                seq.append(nn.Identity())
            self.down_i, self.sub_i, self.up_i = 1, 3, 5
            self.down_bn_i, self.up_bn_i = 2, 6
        self.model = nn.Sequential(*seq)

    def _bn(self, i):
        return self.model[i] if i is not None and isinstance(self.model[i], nn.BatchNorm2d) else None

    @property
    def down_bn(self):
        """BatchNorm2d after the down conv (norm 'batch', middle blocks), else None."""
        return self._bn(self.down_bn_i)

    @property
    def up_bn(self):
        """BatchNorm2d after the up conv (norm 'batch', all but the outermost block), else None."""
        return self._bn(self.up_bn_i)

    @property
    def down(self):
        return self.model[self.down_i]

    @property
    def up(self):
        return self.model[self.up_i]

    @property
    def sub(self):
        return None if self.sub_i is None else self.model[self.sub_i]


class UnetGenerator(_NoEager):
    def __init__(self, input_nc, output_nc, num_downs, ngf=64, use_dropout=False, norm="instance"):
        super().__init__()
        self.norm = check_norm(norm)
        blk = _SkipBlock(ngf * 8, ngf * 8, innermost=True, norm=norm)
        for _ in range(num_downs - 5):
            blk = _SkipBlock(ngf * 8, ngf * 8, submodule=blk, use_dropout=use_dropout, norm=norm)
        blk = _SkipBlock(ngf * 4, ngf * 8, submodule=blk, norm=norm)
        blk = _SkipBlock(ngf * 2, ngf * 4, submodule=blk, norm=norm)
        blk = _SkipBlock(ngf, ngf * 2, submodule=blk, norm=norm)
        self.model = _SkipBlock(output_nc, ngf, input_nc=input_nc, submodule=blk, outermost=True, norm=norm)
        self.num_downs = num_downs

    def blocks(self):
        """outermost -> innermost"""
        out, b = [], self.model
        while b is not None:
            out.append(b)
            b = b.sub
        return out


class TextureModule(_NoEager):
    def __init__(self, texture_channels=3, cloth_channels=19, num_roi=12, norm_type="instance", dropout=0.5,
                 img_size=128):
        super().__init__()
        self.norm = check_norm(norm_type)     # the U-Net's norm; `encode` (a UNetDown) always uses InstanceNorm
        self.texture_channels, self.cloth_channels, self.num_roi = texture_channels, cloth_channels, num_roi
        self.img_size = img_size
        ch = texture_channels * num_roi
        self.encode = _down(ch, ch)
        num_downs = math.frexp(img_size)[1] - 1
        self.unet = UnetGenerator(ch + cloth_channels, texture_channels, num_downs,
                                  use_dropout=dropout is not None, norm=norm_type)


def init_weights(net: nn.Module, init_type: str = "normal", init_gain: float = 0.02) -> None:
    """modules/__init__.py:7-45 — same traversal (nn.Module.apply) and same torch initialisers, so a
    given torch.manual_seed yields the reference's weights bit for bit."""

    def fn(m):
        name = m.__class__.__name__
        if hasattr(m, "weight") and (name.find("Conv") != -1 or name.find("Linear") != -1):
            if init_type == "normal":
                init.normal_(m.weight.data, 0.0, init_gain)
            elif init_type == "xavier":
                init.xavier_normal_(m.weight.data, gain=init_gain)
            elif init_type == "kaiming":
                init.kaiming_normal_(m.weight.data, a=0, mode="fan_in")
            elif init_type == "orthogonal":
                init.orthogonal_(m.weight.data, gain=init_gain)
            else:
                raise NotImplementedError(f"initialization method [{init_type}] is not implemented")
            if getattr(m, "bias", None) is not None:
                init.constant_(m.bias.data, 0.0)
        elif name.find("BatchNorm2d") != -1:
            init.normal_(m.weight.data, 1.0, init_gain)
            init.constant_(m.bias.data, 0.0)

    print("initialize network with %s" % init_type)
    net.apply(fn)


# ---------------------------------------------------------------------------------------------
# frozen VGG16 feature extractor of the perceptual loss (modules/losses/perceptual.py:26-46)
# ---------------------------------------------------------------------------------------------
VGG16_CFG = (64, 64, "M", 128, 128, "M", 256, 256, 256, "M", 512, 512, 512, "M", 512, 512, 512)
VGG16_CONVS = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)     # indices inside vgg16().features
VGG16_TAP_CONVS = (2, 7, 14, 21, 28)     # convs whose ReLU output ends a slice [0:4],[4:9],[9:16],[16:23],[23:30]
VGG16_POOLED_CONVS = (2, 7, 14, 21)      # convs followed by ReLU + MaxPool2d(2)


class VGG16Features(nn.Sequential):
    """Parameter container for torchvision `vgg16().features[0:30]`; state_dict keys '0.weight', '0.bias',
    '2.weight', ... as in torchvision.  No eager forward: swapnet_b200.engine.PerceptualEngine runs it."""

    def __init__(self):
        layers, cin = [], 3
        for v in VGG16_CFG:
            if v == "M":
                layers.append(nn.Identity())            # MaxPool2d(2, 2): no parameters
            else:
                layers += [nn.Conv2d(cin, v, 3, padding=1), nn.Identity()]   # conv, ReLU
                cin = v
        super().__init__(*layers)
        assert len(self) == 30 and all(isinstance(self[i], nn.Conv2d) for i in VGG16_CONVS)
        for p in self.parameters():
            p.requires_grad = False                     # perceptual.py:44-45

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("VGG16Features is a parameter container; there is no eager fallback")


def load_vgg16_features(spec: str = "pretrained") -> VGG16Features:
    """spec: 'pretrained' — torchvision's ImageNet weights exactly as perceptual.py:26 requests them
             (needs the torch hub cache or network; raises otherwise — there is no silent substitute);
             'random' / 'random:<seed>' — torchvision's own constructor init under a fixed seed (default 1234):
             the stand-in used by the tests and bench.py, where the weights cannot be downloaded;
             any other string — path of a torch-saved vgg16 (or vgg16.features) state_dict."""
    import torchvision

    net = VGG16Features()
    if spec == "pretrained":
        try:
            tv = torchvision.models.vgg16(weights=torchvision.models.VGG16_Weights.IMAGENET1K_V1)
        except Exception as e:  # offline: URLError etc.
            raise RuntimeError(
                "vgg16(pretrained=True) (modules/losses/perceptual.py:26) could not be loaded: "
                f"{type(e).__name__}: {e}.  Put vgg16-397923af.pth in the torch hub cache, pass "
                "--b200_vgg /path/to/vgg16.pth, or --b200_vgg random for seeded random weights") from e
        sd = tv.features.state_dict()
    elif spec.startswith("random"):
        seed = int(spec.split(":", 1)[1]) if ":" in spec else 1234
        with torch.random.fork_rng():
            torch.manual_seed(seed)
            sd = torchvision.models.vgg16(weights=None).features.state_dict()
    else:
        sd = torch.load(spec, map_location="cpu")
        if any(k.startswith("features.") for k in sd):
            sd = {k[len("features."):]: v for k, v in sd.items() if k.startswith("features.")}
    net.load_state_dict({k: v for k, v in sd.items() if int(k.split(".")[0]) < 30})
    return net
