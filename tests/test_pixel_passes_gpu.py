"""The four fused PixelGAN passes of csrc/pixel_disc.cu (`fwd_stats`, `fwd`, `bwd_reduce`, `bwd_apply`) driven through
`ops.pixel_desc` / `ops.pixel_pass`, against the fp64 oracle of tests/tools/pixel_oracle.py with the device's LeakyReLU
gates imposed.

Every checked entry has its own bound, built from |.| of every term that feeds it (terms that cancel included):
  z1     |W1||x| + |b1|                               B_a1 = |gate1| B_z1
  z2     |W2| B_a1 + |b2|                             y2: rstd (B_z2 + mean_px B_z2) with instance norm, else B_z2
  stats  mean: mean_px B_z2; rstd: rstd^3 mean_px(|z2 - mean| B_z2)
  pred   |w3| |gate2| B_y2 + |b3|
  g2 = dpred w3 gate2;  B_dz2 = |g2| (none) or rstd (|g2| + |mean g2| + |y2| |mean(g2 y2)|) (instance)
  B_g1 = (|W2|^T B_dz2) |gate1|;  dx: |W1|^T B_g1
  dW2, db2: sum_px B_dz2 [|a1|; 1];  dW1, db1: sum_px B_g1 [|x|; 1];  dW3, db3: sum_px |dpred| [|a2|; 1]
The forward bounds chain through the layers because every pass recomputes a1 and a2 from its own z1 and y2.  The
default (three-product) passes are held to max(|err| / bound) <= 1.5e-5 forward and 1e-4 backward, the bars of the
conv GEMMs, and to max|err| / max|ref| (relmax) below the same bars; the deterministic passes to the same bars, and a
second launch of them to identical bits.  A per-entry bound sums |.| over the pixels a weight gradient reduces, so
rounding errors of random sign shrink against it by sqrt(pixels); relmax is what sees a dropped lo product there.  It
is not asserted on db2 under instance norm, which is zero in exact arithmetic.  At the D step's training shape each
block sums 497 tiles of weight-gradient partials; the kernel promotes every tile's partial with round-to-nearest adds,
and without that promotion relmax reached 1.1e-4 there.  Every device output must be finite, and a NaN counts as an
infinite error.

Each case also runs at nsplit = 1 (hi x hi products only).  Its forward is held to the operand model of
test_kernels_gpu.check_single_pass (z1 from the fp16 hi words of x and of W1 s, divided by s; z2 from the fp16 hi words
of lrelu(z1 as the device computed it) and of W2 s), and every gradient that split products compute must miss the
backward bar by 10x, measured as relmax for the reason above.  dW3 and db3 are fp64 sums of fp32 products on
the CUDA cores and take no part in it.

The operand x is quantised to multiples of 2^-14, so that its fp16 and bf16 splits both hold it exactly: the fp64
oracle then reads the same x as the kernels.  Planes outside the operand (other channels of the pitch, other images of
a batch slice) hold finite garbage.  Every case asserts its geometry: tiles of 64 pixels, the fixed grid of 264 blocks
and the contiguous range of tiles each block takes."""
import math
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "tools"))

import pixel_oracle as PO  # noqa: E402

FWD_TOL, BWD_TOL = 1.5e-5, 1e-4
SEP = 10.0                        # nsplit = 1 misses the backward bar by at least this factor
SP_SEP_FP16 = 4.0                 # test_kernels_gpu.SP_SEP_FP16: the fp16 operand model's distance from exact
KTILE, KBLOCKS = 64, 264          # pixels per tile; the grid of every pass (2 x 132 SMs)
SLOPE = PO.SLOPE
NAN = float("nan")
DX_SENTINEL = 7.0
CHUNK_PIXELS = 1 << 18            # the oracle runs over whole images, at most this many pixels at a time (or one image)


def record(name, value):
    from conftest import record as _r

    _r(name, value)


def lib():
    from swapnet_b200 import _lib

    return _lib.load()


def geometry(n, hw):
    """(tiles per image, total tiles, tiles per block) of the passes' fixed grid"""
    tpi = -(-hw // KTILE)
    total = n * tpi
    return tpi, total, -(-total // KBLOCKS)


def test_grid_is_264_blocks():
    """The grid the case geometries below are written against, read from the library's slot count: the statistics
    take [blocks][n][128][2] doubles."""
    per_image = int(lib().sn_pixel_det_slots(2, 1)) - int(lib().sn_pixel_det_slots(1, 1))
    assert per_image == KBLOCKS * 128 * 2


# ---------------------------------------------------------------------------------------------
# operands, networks and one run of the passes
# ---------------------------------------------------------------------------------------------
class Operand:
    """x [n, h, w, cin] (fp32 on the device, multiples of 2^-14) as fp16-split planes with a bf16-split twin, at channel
    offset c_off of a `pitch`-channel buffer, images n0 .. n0 + n - 1 of a larger batch."""

    def __init__(self, n, h, w, cin, x_c, pitch=None, c_off=0, n0=0, dx_pitch=None, seed=0):
        from swapnet_b200 import ops

        pitch = pitch or x_c
        assert c_off % 2 == 0 and c_off + x_c <= pitch
        g = torch.Generator().manual_seed(seed)
        x = torch.round((torch.rand(n, h, w, cin, generator=g) * 2 - 1) * 2.0 ** 14) / 2.0 ** 14
        self.x = x.cuda()
        full = ops.Planes(n0 + n + (1 if n0 else 0), h, w, pitch, "cuda", c=x_c, c_off=c_off, dual=True)
        for p in (full, full.twin):   # finite garbage wherever the passes must not read
            p.hi.fill_(0.75)
            p.lo.fill_(-0.375)
            p.hi[n0:n0 + n, ..., c_off:c_off + x_c] = 0
            p.lo[n0:n0 + n, ..., c_off:c_off + x_c] = 0
        hi16 = self.x.half()
        hb = self.x.bfloat16()
        s = slice(c_off, c_off + cin)
        full.hi[n0:n0 + n, ..., s] = hi16.view(torch.bfloat16)
        full.lo[n0:n0 + n, ..., s] = (self.x - hi16.float()).half().view(torch.bfloat16)
        full.twin.hi[n0:n0 + n, ..., s] = hb
        full.twin.lo[n0:n0 + n, ..., s] = (self.x - hb.float()).bfloat16()
        self.planes = full if (n0 == 0 and full.n == n) else full.batch_slice(n0, n)
        for p in (self.planes, self.planes.twin):   # both splits hold x exactly
            assert torch.equal(p.dense()[..., :cin], self.x) and not p.dense()[..., cin:].any()
        self.n, self.h, self.w, self.hw, self.cin, self.x_c = n, h, w, h * w, cin, x_c
        self.dx_pitch = dx_pitch or cin

    def nchw(self, n0, n1):
        return self.x[n0:n1].permute(0, 3, 1, 2).double()


def make_net(cin, norm, seed=0, init="kaiming", w0_exp=0):
    """PixelDiscriminator with seeded weights; kaiming also draws non-zero biases so that every bias path runs.
    w0_exp: net.0's weight and bias scaled by 2^w0_exp (moves a1 through the fp16-split window)."""
    from swapnet_b200 import modules as M

    torch.manual_seed(seed)
    net = M.PixelDiscriminator(cin, 64, norm)
    M.init_weights(net, init, 0.02)
    with torch.no_grad():
        if init == "kaiming":
            for m in net.modules():
                if isinstance(m, torch.nn.Conv2d) and m.bias is not None:
                    m.bias.normal_(0.0, 0.1)
        net.net[0].weight.mul_(2.0 ** w0_exp)
        net.net[0].bias.mul_(2.0 ** w0_exp)
    return net.cuda()


def weight_scales(net):
    """(s, 1/s) of net.0 and net.2 weights, as the engine's pack() sets them"""
    from swapnet_b200 import ops

    scales = torch.zeros(2, 2, device="cuda")
    pt = ops.PackTable("cuda")
    pt.add_scale(net.net[0].weight.data, scales[0])
    pt.add_scale(net.net[2].weight.data, scales[1])
    pt.run()
    return scales


def run_passes(op, net, scales, nsplit, det, wg, want_dx, dpred, w3_only=False):
    """The passes of one forward + backward, as PixelGANEngine calls them; returns every output (fresh buffers)."""
    from swapnet_b200 import ops

    N, hw, cin = op.n, op.hw, op.cin
    norm = net.norm == "instance"
    z = lambda *s: torch.zeros(*s, device="cuda")  # noqa: E731
    o = dict(stats=torch.zeros(N, 128, 2, dtype=torch.float64, device="cuda") if norm else None,
             pred=torch.full((N * hw,), NAN, device="cuda"), debug=torch.full((N * hw, 192), NAN, device="cuda"))
    gstats = torch.zeros_like(o["stats"]) if norm else None
    grads = {}
    if wg:
        grads = dict(dw1=z(64, cin), db1=z(64), dw2=z(128, 64), dw3=z(128))
        if norm:
            grads.update(db2=z(128), db3=z(1))
    elif w3_only:
        grads = dict(dw3=z(128), **({"db3": z(1)} if norm else {}))
    dxkw = {}
    if want_dx:
        o["dx"] = torch.full((N * hw, op.dx_pitch), DX_SENTINEL, device="cuda")
        dxkw = dict(dx=o["dx"], dx_pitch=op.dx_pitch)
    ws = ops.DetWorkspace("cuda") if det else None
    desc = lambda **kw: ops.pixel_desc(op.planes, net, scales, nsplit, stats=o["stats"], gstats=gstats, **kw)  # noqa
    if norm:
        ops.pixel_pass("fwd_stats", desc(), ws=ws)
    ops.pixel_pass("fwd", desc(pred=o["pred"], debug=o["debug"]))
    if norm:
        o["stats_fwd"] = o["stats"].clone()
        ops.pixel_pass("bwd_reduce", desc(dpred=dpred, **grads), ws=ws)
    ops.pixel_pass("bwd_apply", desc(dpred=dpred, **grads, **dxkw), ws=ws)
    torch.cuda.synchronize()
    o.update(grads)
    return o


# ---------------------------------------------------------------------------------------------
# measuring
# ---------------------------------------------------------------------------------------------
def worst(t):
    """max of t with NaN counted as +inf (Python's max() would drop a NaN against the running maximum)"""
    return torch.nan_to_num(t, nan=math.inf).max().item()


class Meter:
    """Per checked tensor: the worst |err| / bound, and max|err|, max|ref| (relmax = their ratio)."""

    def __init__(self):
        self.ratio, self.err, self.ref = {}, {}, {}

    def add(self, key, dev, ref, bound):
        assert torch.isfinite(dev).all(), f"{key}: non-finite device output"
        err = (dev.double() - ref).abs()
        r = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
        self.ratio[key] = max(self.ratio.get(key, 0.0), worst(r))
        self.err[key] = max(self.err.get(key, 0.0), worst(err))
        self.ref[key] = max(self.ref.get(key, 0.0), worst(ref.abs()))

    def relmax(self, key):
        return self.err[key] / max(self.ref[key], 1e-300)


class ModelMeter:
    """check_single_pass over chunks: got vs the operand model, and the model vs the exact result"""

    def __init__(self):
        self.v = {}

    def add(self, key, got, model, exact):
        assert torch.isfinite(got).all(), f"{key}: non-finite device output"
        a = self.v.setdefault(key, [0.0, 0.0, 0.0, 0.0])
        a[0] = max(a[0], worst((got.double() - model).abs()))
        a[1] = max(a[1], worst(model.abs()))
        a[2] = max(a[2], worst((model - exact).abs()))
        a[3] = max(a[3], worst(exact.abs()))

    def result(self, key):
        a = self.v[key]
        return a[0] / max(a[1], 1e-300), a[2] / max(a[3], 1e-300)


def _gate(g):
    return torch.where(g, 1.0, SLOPE).double()


GRAD_KEYS = {"dw1": "net.0.weight", "db1": "net.0.bias", "dw2": "net.2.weight", "db2": "net.2.bias",
             "dw3": "net.5.weight", "db3": "net.5.bias"}


def check_passes(tag, op, net, dpred, *, wg, want_dx, modes=("default", "det", "nsplit1"), w3_only=False,
                 fwd_asserted=True, bwd_asserted=True):
    """Run the passes in every mode, compare them with the fp64 oracle image chunk by image chunk, record and assert.
    Returns {mode: {tensor: worst ratio}}."""
    norm = net.norm == "instance"
    N, h, w, cin = op.n, op.h, op.w, op.cin
    scales = weight_scales(net)
    cfg = {"default": (3, False), "det": (3, True), "nsplit1": (1, False)}
    outs = {m: run_passes(op, net, scales, cfg[m][0], cfg[m][1], wg, want_dx, dpred, w3_only) for m in modes}
    if "det" in modes:   # a second deterministic launch gives the same bits
        again = run_passes(op, net, scales, 3, True, wg, want_dx, dpred, w3_only)
        for k, v in outs["det"].items():
            if v is not None:
                assert torch.equal(v, again[k]), f"{tag}: det {k} differs"
        del again
    # outside the operand's cin channels dx keeps what the buffer held
    for m in modes:
        if want_dx and op.dx_pitch > cin:
            assert torch.all(outs[m]["dx"][:, cin:] == DX_SENTINEL), f"{tag} {m}: dx written past cin"
    sd = {k: v.detach().double() for k, v in net.state_dict().items()}
    aW1, ab1 = sd["net.0.weight"].view(64, cin).abs(), sd["net.0.bias"].abs().view(1, 64, 1, 1)
    W2 = sd["net.2.weight"].view(128, 64)
    aW2 = W2.abs()
    ab2 = sd["net.2.bias"].abs().view(1, 128, 1, 1) if "net.2.bias" in sd else 0.0
    w3 = sd["net.5.weight"].view(128)
    ab3 = sd["net.5.bias"].abs().view(1, 1, 1) if "net.5.bias" in sd else 0.0
    s1, s2 = scales[0, 0].item(), scales[1, 0].item()
    # fp16 hi words of the pre-scaled weights (the nsplit = 1 operand model)
    W1h = (net.net[0].weight.detach().view(64, cin) * s1).half().double() / s1
    W2h = (net.net[2].weight.detach().view(128, 64) * s2).half().double() / s2
    b1 = sd["net.0.bias"].view(1, 64, 1, 1)
    b2 = sd["net.2.bias"].view(1, 128, 1, 1) if "net.2.bias" in sd else 0.0
    meters = {m: Meter() for m in modes}
    model = ModelMeter()
    pref, pbound = {}, {}
    step = max(1, CHUNK_PIXELS // op.hw)
    for n0 in range(0, N, step):
        n1 = min(N, n0 + step)
        x = op.nchw(n0, n1)
        view = lambda t, c: t.view(N, h, w, c)[n0:n1].permute(0, 3, 1, 2)  # noqa: E731
        dbg = view(outs[modes[0]]["debug"], 192)
        z1g, y2g = dbg[:, :64] > 0, dbg[:, 64:] > 0
        dp = dpred[n0:n1].double().unsqueeze(1)
        r = PO.pixel_grads(sd, x, net.norm, dp, z1g, y2g)
        f1, f2 = _gate(z1g), _gate(y2g)
        # ---- bounds ----
        Bz1 = torch.einsum("kc,nchw->nkhw", aW1, x.abs()) + ab1
        Bz2 = torch.einsum("jk,nkhw->njhw", aW2, f1 * Bz1) + ab2
        if norm:
            z2 = r["z2"]
            mean = z2.mean((2, 3), keepdim=True)
            rstd = (z2.var((2, 3), unbiased=False, keepdim=True) + 1e-5).rsqrt()
            mBz2 = Bz2.mean((2, 3), keepdim=True)
            By2 = rstd * (Bz2 + mBz2)
            b_mean, b_rstd = mBz2[..., 0, 0], (rstd ** 3 * ((z2 - mean).abs() * Bz2).mean((2, 3), keepdim=True))[..., 0, 0]
        else:
            By2 = Bz2
        Bpred = torch.einsum("j,njhw->nhw", w3.abs(), f2 * By2) + ab3
        g2 = dp * w3.view(1, 128, 1, 1) * f2
        if norm:
            y2 = r["y2"]
            Bdz2 = rstd * (g2.abs() + g2.mean((2, 3), keepdim=True).abs() +
                           y2.abs() * (g2 * y2).mean((2, 3), keepdim=True).abs())
        else:
            Bdz2 = g2.abs()
        Bg1 = torch.einsum("jk,njhw->nkhw", aW2, Bdz2) * f1
        pb = {"dw2": torch.einsum("njhw,nkhw->jk", Bdz2, r["a1"].abs()), "db2": Bdz2.sum((0, 2, 3)),
              "dw1": torch.einsum("nkhw,nchw->kc", Bg1, x.abs()), "db1": Bg1.sum((0, 2, 3)),
              "dw3": torch.einsum("nhw,njhw->j", dp[:, 0].abs(), r["a2"].abs()), "db3": dp.abs().sum().view(1)}
        for k, key in GRAD_KEYS.items():
            if key in r:
                ref = r[key].reshape(pb[k].shape)
                pref[k] = ref if k not in pref else pref[k] + ref
                pbound[k] = pb[k] if k not in pbound else pbound[k] + pb[k]
        Bdx = torch.einsum("kc,nkhw->nchw", aW1, Bg1) if want_dx else None
        # ---- every mode's per-pixel outputs ----
        for m in modes:
            o, M_ = outs[m], meters[m]
            d = view(o["debug"], 192)
            pred = o["pred"].view(N, h, w)[n0:n1]
            if m == "nsplit1":   # the operand model of the single-pass forward
                z1d = d[:, :64]
                z1m = torch.einsum("kc,nchw->nkhw", W1h, x.half().double()) + b1
                a1f = torch.where(z1d > 0, z1d, z1d * SLOPE)          # fp32, as the kernel computes it
                z2m = torch.einsum("jk,nkhw->njhw", W2h, a1f.half().double()) + b2
                if norm:
                    st = o["stats_fwd"][n0:n1].float().double()
                    z2m = (z2m - st[..., 0, None, None]) * st[..., 1, None, None]
                model.add("z1", z1d, z1m, r["z1"])
                model.add("y2", d[:, 64:], z2m, r["y2"])
            else:
                M_.add("z1", d[:, :64], r["z1"], Bz1)
                M_.add("y2", d[:, 64:], r["y2"], By2)
                M_.add("pred", pred, r["pred"][:, 0], Bpred)
                if norm:
                    st = o["stats_fwd"][n0:n1]
                    M_.add("mean", st[..., 0], mean[..., 0, 0], b_mean)
                    M_.add("rstd", st[..., 1], rstd[..., 0, 0], b_rstd)
            if want_dx:
                M_.add("dx", view(o["dx"], op.dx_pitch)[:, :cin], r["x"], Bdx)
        del r, Bz1, Bz2, By2, Bdz2, Bg1, Bdx, g2, dbg
    for m in modes:
        for k in GRAD_KEYS:
            if outs[m].get(k) is not None:
                meters[m].add(k, outs[m][k].view(pref[k].shape), pref[k], pbound[k])
    # ---- record, then assert ----
    result = {}
    for m in modes:
        M_ = meters[m]
        result[m] = {k: M_.ratio[k] for k in M_.ratio}
        record(f"pixel_passes[{tag}][{m}]", " ".join(f"{k} {M_.ratio[k]:.3e}/{M_.relmax(k):.3e}" for k in M_.ratio) +
               "  (worst |err|/bound / max|err|/max|ref|)")
    if "nsplit1" in modes:
        record(f"pixel_passes[{tag}][nsplit1-model]",
               " ".join(f"{k} {e:.3e} (model vs exact {s:.3e})" for k, (e, s) in
                        ((k, model.result(k)) for k in model.v)))
    for m in modes:
        if m == "nsplit1":
            continue
        for k, v in result[m].items():
            fwd = k in ("z1", "y2", "pred", "mean", "rstd")
            if (fwd and fwd_asserted) or (not fwd and bwd_asserted):
                tol = FWD_TOL if fwd else BWD_TOL
                assert v <= tol, f"{tag} {m}: {k} at {v:.3e} of its bound (tol {tol:.1e})"
                if not (k == "db2" and norm):   # zero in exact arithmetic: the per-entry bound alone
                    rm = meters[m].relmax(k)
                    assert rm <= tol, f"{tag} {m}: {k} relmax {rm:.3e} (tol {tol:.1e})"
    if "nsplit1" in modes:
        for k in ("z1", "y2"):
            err, sep = model.result(k)
            assert err < FWD_TOL, f"{tag} nsplit1: {k} relmax {err:.3e} vs the operand model"
            assert sep >= SP_SEP_FP16 * FWD_TOL and sep >= 20 * err, f"{tag} nsplit1: {k} model vs exact {sep:.3e}"
        M_ = meters["nsplit1"]
        split_keys = [k for k in ("dx", "dw1", "db1", "dw2") if k in M_.err]
        if not norm:
            split_keys += [k for k in ("db2",) if k in M_.err]
        for k in split_keys:
            assert M_.relmax(k) >= SEP * BWD_TOL, \
                f"{tag} nsplit1: {k} relmax {M_.relmax(k):.3e} does not miss the bar {BWD_TOL:.0e} by {SEP:.0f}x"
    return result


def dpred_noise(n, h, w, seed=1):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(n, h, w, generator=g) / (n * h * w) ** 0.5).cuda()


# ---------------------------------------------------------------------------------------------
# the case matrix
# ---------------------------------------------------------------------------------------------
# (id, cin, x_c, n, h, w, norm, wg, dx, total-tiles relation to the grid, tiles per block, operand extras)
CASES = [
    ("c1-x16-hw1-n263", 1, 16, 263, 1, 1, "none", True, True, "<", 1, {}),
    ("c3-x16-hw63-n264", 3, 16, 264, 7, 9, "instance", True, False, "=", 1, {}),
    ("c15-x16-hw64-n265", 15, 16, 265, 8, 8, "none", False, True, "+1", 2, {}),
    ("c16-x16-hw65-n132", 16, 16, 132, 5, 13, "instance", True, True, "=", 1, {}),
    ("c17-x32-hw63-n529", 17, 32, 529, 7, 9, "instance", True, True, "2x+1", 3, {}),
    ("c22-x32-hw1-n529", 22, 32, 529, 1, 1, "none", True, False, "2x+1", 3, {}),
    ("c31-x32-hw65-n4", 31, 32, 4, 5, 13, "instance", False, True, "<", 1, {}),
    ("c32-x32-hw64-n265", 32, 32, 265, 8, 8, "instance", True, True, "+1", 2, {}),
    ("c22-x32-hw65-n265", 22, 32, 265, 5, 13, "none", True, True, ">", 3, {}),
    # pitched, offset and batch-sliced operands; dx at a pitch above cin
    ("c19-x32-pitch48-coff6-slice3", 19, 32, 6, 8, 8, "instance", True, True, "<", 1,
     dict(pitch=48, c_off=6, n0=3, dx_pitch=24)),
    ("c9-x16-pitch24-coff2-slice1", 9, 16, 5, 5, 13, "none", True, True, "<", 1,
     dict(pitch=24, c_off=2, n0=1, dx_pitch=12)),
]


def _assert_geometry(n, hw, x_c, rel, tpb):
    tpi, total, got_tpb = geometry(n, hw)
    assert tpi == -(-hw // 64) and got_tpb == tpb, (n, hw, tpi, total, got_tpb)
    assert {"<": total < KBLOCKS, "=": total == KBLOCKS, "+1": total == KBLOCKS + 1,
            "2x+1": total == 2 * KBLOCKS + 1, ">": total > 2 * KBLOCKS + 1}[rel], (rel, total)
    assert x_c in (16, 32)


@pytest.mark.parametrize("cid,cin,x_c,n,h,w,norm,wg,dx,rel,tpb,extra", CASES, ids=[c[0] for c in CASES])
def test_passes_match_fp64(cid, cin, x_c, n, h, w, norm, wg, dx, rel, tpb, extra):
    _assert_geometry(n, h * w, x_c, rel, tpb)
    op = Operand(n, h, w, cin, x_c, seed=cin + n, **extra)
    assert op.planes.c == x_c and op.planes.pitch == extra.get("pitch", x_c)
    net = make_net(cin, norm, seed=cin)
    check_passes(cid, op, net, dpred_noise(n, h, w, seed=n), wg=wg, want_dx=dx)


def test_dw3_without_the_other_weight_gradients():
    """bwd_apply with dx and dW3 only (no instance norm, so dW3 comes from this pass): the deterministic mode sums
    its dW3 slots too."""
    op = Operand(4, 8, 8, 22, 32, seed=5)
    net = make_net(22, "none", seed=5)
    check_passes("c22-x32-dx-dw3-only", op, net, dpred_noise(4, 8, 8), wg=False, want_dx=True, w3_only=True)


# ---------------------------------------------------------------------------------------------
# the training shapes: 512^2, the D step (32 images: fakes and reals) and the G step (16 images, dx only)
# ---------------------------------------------------------------------------------------------
def test_d_step_training_shape():
    n, s = 32, 512
    tpi, total, tpb = geometry(n, s * s)
    assert (tpi, total, tpb) == (4096, 131072, 497)
    op = Operand(n, s, s, 22, 32, seed=11)
    net = make_net(22, "instance", seed=11)
    check_passes("train-D-32x512^2-instance", op, net, dpred_noise(n, s, s, seed=12), wg=True, want_dx=False)


def test_d_step_training_shape_same_sign_dpred():
    """A D step's dpred has one sign over each image (fakes one way, reals the other); here all 32 images take the
    same sign.  Without a norm, dz2 then keeps its sign over every pixel, so every tile's dW2 partial adds to the
    block's sums in the same direction: the regime where truncating accumulation would grow with the number of tiles
    a block sums (497 here), and where no cancellation hides it from max|err| / max|ref|."""
    n, s = 32, 512
    op = Operand(n, s, s, 22, 32, seed=13)
    net = make_net(22, "none", seed=13)
    g = torch.Generator().manual_seed(14)
    dpred = ((0.2 + torch.rand(n, s, s, generator=g)) / (n * s * s)).cuda()
    check_passes("train-D-32x512^2-none-same-sign", op, net, dpred, wg=True, want_dx=False, modes=("default", "det"))


def test_g_step_training_shape():
    n, s = 16, 512
    tpi, total, tpb = geometry(n, s * s)
    assert (tpi, total, tpb) == (4096, 65536, 249)
    op = Operand(n, s, s, 22, 32, dx_pitch=24, seed=15)
    net = make_net(22, "instance", seed=15)
    check_passes("train-G-16x512^2-instance", op, net, dpred_noise(n, s, s, seed=16), wg=False, want_dx=True)


# ---------------------------------------------------------------------------------------------
# the fp16-split window of a1: net.0 scaled by 2^k, and the reference's `--init_type normal` (gain 0.02)
# ---------------------------------------------------------------------------------------------
A1_SCALES = [-10, -6, -3, 0, 4, 8]
A1_ASSERTED = (-6, -3, 0, 4, 8)


@pytest.mark.parametrize("k", A1_SCALES)
def test_a1_scale_window(k):
    op = Operand(16, 8, 8, 22, 32, seed=21)
    net = make_net(22, "instance", seed=21, w0_exp=k)
    asserted = k in A1_ASSERTED
    check_passes(f"a1-scale-2^{k}", op, net, dpred_noise(16, 8, 8, seed=22), wg=True, want_dx=True,
                 modes=("default",), fwd_asserted=asserted, bwd_asserted=asserted)


@pytest.mark.parametrize("norm", ["instance", "none"])
def test_normal_init(norm):
    op = Operand(16, 8, 8, 22, 32, seed=23)
    net = make_net(22, norm, seed=23, init="normal")
    check_passes(f"init-normal-0.02-{norm}", op, net, dpred_noise(16, 8, 8, seed=24), wg=True, want_dx=True,
                 modes=("default", "det"))


# ---------------------------------------------------------------------------------------------
# refusals: each returns an error before anything is launched
# ---------------------------------------------------------------------------------------------
def _refusal_descs():
    from swapnet_b200 import ops

    op = Operand(2, 8, 8, 22, 32, pitch=40, c_off=8, seed=31)
    net = make_net(22, "instance", seed=31)
    scales = weight_scales(net)
    stats = torch.zeros(2, 128, 2, dtype=torch.float64, device="cuda")
    pred = torch.zeros(2 * 64, device="cuda")
    keep = [op, net, scales, stats, pred]

    def base():
        return ops.pixel_desc(op.planes, net, scales, 3, stats=stats, pred=pred)

    def with_(**kw):
        d = base()
        for k, v in kw.items():
            setattr(d, k, v)
        return d

    slots = torch.zeros(int(lib().sn_pixel_det_slots(2, 22)), dtype=torch.float64, device="cuda")
    keep.append(slots)
    odd = op.planes.slice(1, 31)   # channel offset 9: the passes' 32-bit loads would be misaligned
    cases = {
        "cin above x_c": (with_(cin=33), "cin 33, x_c 32"),
        "x_c 64": (with_(x_c=64, x_pitch=64), "x_c 64"),
        "odd pitch": (with_(x_pitch=41), "pitch 41"),
        "too few slots": (with_(slots=slots.data_ptr(), slots_cap=slots.numel() - 1), "slots given"),
        "nsplit 2": (with_(nsplit=2), "nsplit must be 1 or 3"),
        "instance norm without stats": (with_(stats=None), "needs the statistics buffer"),
        "misaligned x": (with_(x_hi=odd.hi_ptr, x_lo=odd.lo_ptr), "4-byte aligned"),
        "misaligned twin": (with_(xb_hi=odd.twin.hi_ptr, xb_lo=odd.twin.lo_ptr), "4-byte aligned"),
    }
    assert base().x_hi % 4 == 0 and odd.hi_ptr % 4 == 2 and odd.twin.lo_ptr % 4 == 2
    return cases, base, keep


def test_check_desc_refusals_launch_nothing():
    from swapnet_b200 import ops

    cases, base, keep = _refusal_descs()
    torch.cuda.synchronize()
    stream = torch.cuda.current_stream().cuda_stream
    import ctypes as C

    for entry in ("fwd_stats", "fwd", "bwd_reduce", "bwd_apply"):
        for what, (d, msg) in cases.items():
            before = ops.launch_count()
            rc = getattr(lib(), "sn_pixel_" + entry)(C.byref(d), stream)
            assert rc != 0, f"{entry}: {what} accepted"
            err = lib().sn_last_error().decode()
            assert msg in err, (entry, what, err)
            assert ops.launch_count() == before, f"{entry}: {what} launched"
    torch.cuda.synchronize()
    del keep


def test_pix2pix_with_pixel_discriminator_is_refused_with_its_reason():
    """pix2pix's discriminator reads 19 + 36 + 3 = 58 channels; the fused passes take at most 32."""
    from test_unet_gpu import pix2pix_opt

    from swapnet_b200.models import create_model

    with pytest.raises(NotImplementedError, match="at most 32 input channels.*reads 58"):
        create_model(pix2pix_opt(2, 128, norm="instance", discriminator="pixel"))


def test_engine_refuses_a_wide_input():
    from swapnet_b200 import engine as E
    from swapnet_b200 import modules as M

    with pytest.raises(ValueError, match="58 input channels"):
        E.PixelGANEngine(M.PixelDiscriminator(58, 64, "instance").cuda(), 2, 8, "cuda")
