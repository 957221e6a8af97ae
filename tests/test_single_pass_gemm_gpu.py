"""The single-pass GEMMs of `--b200_precision bf16` (nsplit = 1) at the positions of their shared-memory ring.

At nsplit = 1 both kernels of csrc/gemm_tc.cu run a 6-stage ring (Cfg<1>; nsplit = 3 runs 3).  The stage index and
the mbarrier phase are `it % kStages` and `(it / kStages) & 1`, and in the persistent tap GEMM `it` carries over from
one tile to the next: when the K iterations per tile are not a multiple of 6, each new tile starts partway around the
ring.  The weight-gradient GEMM restarts its ring per CTA, and the number of 64-pixel tiles in its K split decides
where the ring stands when the split ends.  The cases are chosen by those counts, not by layer:

- tap GEMM: K iterations per tile in {1, 3, 4, 6, 7, 9, 16, 18}, fp16 (forward) and bf16 (input-gradient) operands,
  with at least 3x as many tiles as the device has SMs, so that every persistent CTA takes tiles at several ring
  positions;
- weight gradient: explicit split-K with 1, 5, 6, 7, 12 and 13 pixel tiles per split, the wide and the grouped
  narrow-Y layouts, atomic and deterministic plans.

The operands are written straight into the hi planes (nsplit = 1 reads nothing else), and the reference is the fp64
contraction of those 16-bit values (oracle/emulate.py over the same spec), with the bound and the sensitivity check of
test_kernels_gpu's operand model.
"""
import pytest
import torch

from oracle import emulate as E
from swapnet_b200 import lowering as L
from test_gemm_edges_gpu import geometry, sm_count
from test_kernels_gpu import SP_SEP_BF16, SP_SEP_FP16, check_single_pass, dev, record

pytestmark = pytest.mark.gpu

TOL = 1.5e-5
RING = 6          # Cfg<1>::kStages


def hi_store(vals, fmt):
    """16-bit hi words of fp32 values as the planes store them (bfloat16 storage), and their fp64 values."""
    from swapnet_b200 import ops

    if fmt == ops.FMT_F16:
        h = vals.half()
        return h.view(torch.bfloat16), h.double()
    h = vals.bfloat16()
    return h, h.double()


def hi_planes(vals, fmt):
    """Planes [n, h, w, c] whose hi plane holds the 16-bit rounding of vals (NHWC fp32 on the device); lo is NaN, which
    a single-pass GEMM must not read."""
    from swapnet_b200 import ops

    n, h, w, c = vals.shape
    p = ops.Planes(n, h, w, c, dev(), fmt=fmt)
    words, v64 = hi_store(vals, fmt)
    p.hi.copy_(words)
    p.lo.fill_(float("nan"))
    return p, v64


# ---------------------------------------------------------------------------------------------
# tap GEMM
# ---------------------------------------------------------------------------------------------
def _spec(name, h, w):
    """(spec of the launch, nphase, the specs the reference contracts) of a tap-GEMM launch over an h x w input."""
    from swapnet_b200 import ops

    if name == "convT4s2":          # the 4 output-parity phases merged into one launch (grid.z = 4)
        phases = L.forward_specs("convT4s2", h, w)
        return ops.merge_phase_specs(phases), 4, phases
    if name == "head_phase1":       # the unstacked head's (py, px) = (0, 1) phase: 6 effective taps
        spec = L.forward_specs("head", h, w)[1]
    elif name == "1x1":
        spec = L.GemmSpec(False, h, w, [L.Tap(0, 0, 0, 0)], a_hw=(h, w))
    else:
        spec = L.forward_specs(name, h, w)[0]
    return spec, 1, [spec]


# (spec, input channels, channels per tap (the plane width), outputs, K iterations per tile)
TAP_RING_CASES = [
    ("convT4s2", 16, 16, 16, 1),        # 4 taps per phase on 16-channel rows: one stage per tile
    ("conv3z", 3, 16, 32, 3),           # vgg16.features.0: 9 taps padded to 12, 4 per stage
    ("convT4s2", 64, 64, 64, 4),
    ("head_phase1", 64, 64, 27, 6),     # exactly one turn of the ring per tile
    ("1x1", 448, 448, 96, 7),           # one tap, 7 channel chunks
    ("conv3z", 64, 64, 64, 9),
    ("conv4s2", 64, 64, 128, 16),       # stride 2: the parity view
    ("conv3r", 128, 128, 128, 18),      # the resblock conv
]


def tap_k_iters(spec, nphase, k_per_tap, geo):
    """K iterations per tile of a tap-GEMM plan (tap_gemm_kernel's k_iters) from the spec and sn_plan_geometry."""
    chunk, phases = geo[5], geo[3]
    assert phases == nphase
    ntaps = len(spec.taps)
    if chunk < 64 and nphase == 1:      # narrow rows: padded with zero-weight taps to whole stages
        ntaps = -(-ntaps // (64 // chunk)) * (64 // chunk)
    tpp = ntaps // phases
    return tpp * (k_per_tap // 64) if chunk == 64 else tpp // (64 // chunk)


@pytest.mark.parametrize("fmt", ["f16", "bf16"])
@pytest.mark.parametrize("name,cin,k,cout,k_iters", TAP_RING_CASES)
def test_tap_gemm_ring_positions(name, cin, k, cout, k_iters, fmt):
    from swapnet_b200 import ops

    f = ops.FMT_F16 if fmt == "f16" else ops.FMT_BF16
    d = dev()
    h = w = 16
    spec, nphase, ref_specs = _spec(name, h, w)
    ah, aw = spec.a_hw
    mh, mw = spec.out_mul
    oh, ow = spec.m_h * mh, spec.m_w * mw
    # packed weights [cout][taps * k]: the taps' own columns random, the zero-weight padding taps' columns zero
    kb_end = max(t.kb for t in spec.taps) + 1
    tps = 64 // k if k < 64 else 1
    n_pad = 0 if nphase == 4 else (-len(spec.taps)) % tps
    g = torch.Generator().manual_seed(k_iters * 10 + (fmt == "bf16"))
    wv = torch.zeros(cout, kb_end + n_pad, k)
    wv[:, :kb_end, :cin] = torch.randn(cout, kb_end, cin, generator=g) / (cin * len(spec.taps)) ** 0.5
    wv = wv.reshape(cout, -1).to(d)
    wp = ops.PackedWeights(cout, wv.shape[1], d, fmt=f)
    words, w64 = hi_store(wv, f)
    wp.hi.copy_(words)
    wp.lo.fill_(float("nan"))
    bias = torch.randn(cout, generator=g).to(d)

    def plan_for(x, y):
        desc = ops.tap_gemm_desc(x, spec, wp, k, y, cout, bias=bias, nsplit=1, nphase=nphase)
        return ops.tap_gemm_plan(desc, keep=(x.hi, wp.hi, y))

    def operands(n):
        xv = torch.zeros(n, ah, aw, k)
        xv[..., :cin] = torch.randn(n, ah, aw, cin, generator=g)
        x, x64 = hi_planes(xv.to(d), f)
        return xv.to(d), x, x64, torch.zeros(n, oh, ow, cout, device=d)

    # images: enough for >= 3 tiles per SM (small planes share a tile between images: probe with 8), plus one
    _, x8, _, y8 = operands(8)
    probe = geometry(plan_for(x8, y8))
    n = -(-3 * sm_count() * 8 // (probe[1] * probe[2] * probe[3])) + 1
    xv, x, x64, y = operands(n)
    plan = plan_for(x, y)
    geo = geometry(plan)
    assert tap_k_iters(spec, nphase, k, geo) == k_iters
    tiles = geo[1] * geo[2] * geo[3]
    assert tiles >= 3 * sm_count(), tiles
    plan.run()
    torch.cuda.synchronize()
    model = torch.zeros(n, oh, ow, cout, dtype=torch.float64, device=d)
    exact = torch.zeros_like(model)
    for rs in ref_specs:
        E.emul_tap_gemm(x64, rs, w64, k, cout, model, bias=bias.double())
        E.emul_tap_gemm(xv.double(), rs, wv.double(), k, cout, exact, bias=bias.double())
    err, sep = check_single_pass(f"tap ring {name} {fmt}", y, model, exact, TOL,
                                 SP_SEP_FP16 if fmt == "f16" else SP_SEP_BF16)
    record(f"single_pass_tap_ring[{name},{cin}->{cout},k_iters={k_iters},mod6={k_iters % RING},{fmt},tiles={tiles},"
           f"block_n={geo[4]},chunk={geo[5]},nsplit=1]", f"{err:.3e} (model vs exact {sep:.3e})")


# ---------------------------------------------------------------------------------------------
# weight-gradient GEMM
# ---------------------------------------------------------------------------------------------
# conv3z's weight gradient over an 8 x 8 output plane: one 64-pixel tile per image, so n = tiles per split x K splits.
# X = dy (64 or 128 channels), Y = the layer input: 64 channels (wide: one tap per CTA) or 16 (narrow: the 9 taps in
# column groups of one accumulator)
WGRAD_TILES_PER_SPLIT = [1, 5, 6, 7, 12, 13]
KSPLIT = 3


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("layout", ["wide", "narrow"])
@pytest.mark.parametrize("per_split", WGRAD_TILES_PER_SPLIT)
def test_wgrad_ring_positions(per_split, layout, det):
    from swapnet_b200 import ops

    d = dev()
    hw = 8
    n = per_split * KSPLIT
    cin, cx = (64, 128) if layout == "wide" else (16, 64)
    g = torch.Generator().manual_seed(per_split * 4 + (layout == "wide") * 2 + det)
    dyv = torch.randn(n, hw, hw, cx, generator=g).to(d)
    xv = torch.randn(n, hw, hw, cin, generator=g).to(d)
    dy, dy64 = hi_planes(dyv, ops.FMT_BF16)
    x, x64 = hi_planes(xv, ops.FMT_BF16)
    (ws,) = L.wgrad_specs("conv3z", hw, hw)
    assert ws.x_is == "dy"
    ntap = len(ws.tap_ids)
    # output [tap][row = dy channel][col = input channel]
    taps_off = [t * cx * cin for t in range(ntap)]

    def plan_for(out, ksplit):
        desc = ops.wgrad_desc(dy, x, ws, out, cin, 1, taps_off, cx, cin, nsplit=1, ksplit=ksplit, deterministic=det)
        assert (desc.ngroups > 0) == (layout == "narrow")
        return ops.wgrad_plan(desc, keep=(dy.hi, x.hi, out))

    out = torch.zeros(ntap, cx, cin, device=d)
    total = geometry(plan_for(torch.zeros_like(out), 1 << 20))[3]     # an over-large split is clamped to the tiles
    assert total == n
    plan = plan_for(out, KSPLIT)
    geo = geometry(plan)
    assert geo[3] == KSPLIT and total // KSPLIT == per_split and total % KSPLIT == 0
    assert (plan.workspace_bytes > 0) == det
    plan.run()
    torch.cuda.synchronize()
    model = E.emul_wgrad(dy64, x64, ws, cx, cin)
    exact = E.emul_wgrad(dyv.double(), xv.double(), ws, cx, cin)
    err, sep = check_single_pass(f"wgrad ring {per_split} {layout} det={det}", out, model, exact, TOL, SP_SEP_BF16)
    if det:   # the fixed-order sum: the same bits again
        again = torch.zeros_like(out)
        p2 = plan_for(again, KSPLIT)
        p2.run()
        p2.run()
        torch.cuda.synchronize()
        assert torch.equal(again, 2 * out), "deterministic plan: a repeated launch added different bits"
    record(f"single_pass_wgrad_ring[tiles_per_split={per_split},mod6={per_split % RING},ksplit={KSPLIT},{layout},"
           f"det={det},block_n={geo[4]},y_chunk={geo[5]},nsplit=1]", f"{err:.3e} (model vs exact {sep:.3e})")
