"""Edges of the two implicit-GEMM kernels of csrc/gemm_tc.cu that the CONV_CASES parity tests do not reach.

- the vectorised (float2) epilogue, taken only when the output pixels are 16-byte aligned;
- the tanh epilogue (phase-stacked head store, vectorised and scalar plain stores);
- tap-GEMM tile totals around the SM count (persistent CTAs drawing tiles from a per-plan counter);
- one plan launched repeatedly, replayed from a CUDA graph, and run beside a weight-gradient plan on a second stream:
  the output must be bit-identical from launch to launch (same MMAs in the same order, plain stores);
- explicit weight-gradient split-K, accumulating (+=) into a non-zero gradient;
- the input-magnitude window of the fp16-split operands.

References are fp64 torch on the GPU.  Bounds as in test_kernels_gpu: forward (fp16-split x3) 1.5e-5, backward
(bf16-split x3) 1e-4, as max|err| / max|ref|.  The schedule, repeat, split-K and fused-statistics tests also run every
case single-pass (nsplit = 1, `--b200_precision bf16`: a 6-stage ring in place of 3), held to 1.5e-5 of the fp64
product of the 16-bit operands the plan reads (test_kernels_gpu's operand model).
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from swapnet_b200 import lowering as L
from test_kernels_gpu import (SP_SEP_BF16, SP_SEP_FP16, at_both_nsplits, check_single_pass, dev, make_layer,
                              model_forward, model_wgrad, nhwc, record, ref_forward, ref_fwd_bwd, relmax)

pytestmark = pytest.mark.gpu

FWD_TOL = 1.5e-5
BWD_TOL = 1e-4
# Split-K changes only how the fp32 partial sums over pixel tiles are grouped and in which order the fp32 atomics land
# on the prefilled gradient.  max|out_k - out_1| / max|ref| over the sweep of test_wgrad_split_k_accumulates measured
# 1.0e-6 .. 1.8e-6 on an H100 80GB HBM3 (400 W limit); most of it is the rounding of the adds onto the prefill G0,
# which is several times larger than the gradient.  One pixel tile lost per split moves it to 0.2 and more.
SPLIT_SPREAD = 4e-6
NAN = float("nan")


def sm_count():
    return torch.cuda.get_device_properties(dev()).multi_processor_count


def geometry(plan):
    """sn_plan_geometry: [kind, grid.x, grid.y, grid.z, block_n, chunk].  Tap GEMM: grid = (M tiles, N tiles,
    phases); weight gradient: (M x N tiles, taps or tap groups, K splits)."""
    from swapnet_b200 import _lib

    g = (ctypes.c_int * 6)()
    _lib.check(_lib.load().sn_plan_geometry(plan.handle, g))
    return list(g)


def total_tiles(plan):
    g = geometry(plan)
    assert g[0] == 0, "not a tap-GEMM plan"
    return g[1] * g[2] * g[3]


def vec4_epilogue(out, c_off, bias):
    """Whether a tap-GEMM plan writing `out` from channel c_off takes the float2 store (the condition of
    sn_tap_gemm_plan_init): 16-byte aligned output base and bias, pixel strides that are multiples of 4 floats."""
    return ((out.data_ptr() + 4 * c_off) % 16 == 0 and all(s % 4 == 0 for s in out.stride()[:3])
            and (bias is None or bias.data_ptr() % 16 == 0))


def pitch4(c):
    """A channel pitch that keeps every pixel 16-byte aligned and leaves at least one pad channel."""
    return (c + 3) // 4 * 4 + 4


def repack(layer, x):
    """Write new NCHW input values into the layer's operand planes in place (as make_layer packed them)."""
    from swapnet_b200 import ops

    xp = F.pad(x, (1, 1, 1, 1), mode="reflect") if layer.kind == "conv3r" else x
    assert x.shape[1] * 33 * 4 <= 48 * 1024
    ops.pack_planes(xp.contiguous().to(dev()), layer.x)


def ref_gpu(kind, x, wt, bias):
    d = dev()
    return ref_forward(kind, x.to(d).double(), wt.to(d).double(), None if bias is None else bias.to(d).double())


def grad_planes(gy, c):
    """bf16-split planes of an NCHW gradient on the device, c channels (>= gy's)."""
    from swapnet_b200 import ops

    n, cg, h, w = gy.shape
    dy = ops.Planes(n, h, w, c, dev(), fmt=ops.FMT_BF16)
    if cg * 33 * 4 > 48 * 1024:   # too wide for the NCHW packer's shared-memory stage: pack from NHWC
        assert c == cg
        ops.pack_planes(nhwc(gy), dy, nhwc=True)
    else:
        ops.pack_planes(gy.contiguous(), dy)
    return dy


def dy_channels(layer, cout):
    return L.padc(cout) if layer.x.c >= 64 else L.pad64(cout)   # as test_conv_backward


# ---------------------------------------------------------------------------------------------
# 1. the vectorised epilogue
# ---------------------------------------------------------------------------------------------
# one CONV_CASES row per kind (the head with more outputs than a stacked slot, so it takes the plain store) plus the
# texture-stage widths; outputs at channel 0 of a pitch that is a multiple of 4
ALIGNED_CASES = [
    ("conv4s2", 2, 64, 128, 32, 64),
    ("convT4s2", 2, 128, 64, 8, 8),
    ("conv3r", 2, 128, 128, 32, 32),
    ("conv4s1", 2, 256, 512, 24, 24),
    ("conv3z", 2, 64, 64, 32, 48),
    ("head", 2, 192, 27, 16, 16),
    ("conv4s2", 2, 36, 36, 64, 64),
    ("conv4s2", 2, 55, 64, 64, 64),
    ("convT4s2", 2, 128, 36, 16, 16),
]


@pytest.mark.parametrize("kind,n,cin,cout,h,w", ALIGNED_CASES)
def test_aligned_epilogue(kind, n, cin, cout, h, w):
    d = dev()
    layer, x, wt, bias = make_layer(kind, n, cin, cout, h, w, 3)
    assert not layer.stacked
    oh, ow = L.out_hw(kind, h, w)
    gy = torch.randn((n, cout, oh, ow), generator=torch.Generator().manual_seed(99)).to(d)
    yr, gx, _, _ = ref_fwd_bwd(kind, x, wt, bias, gy)

    y = torch.full((n, oh, ow, pitch4(cout)), NAN, device=d)
    assert vec4_epilogue(y, 0, layer.bias)
    layer.bind_forward(y)
    ih, iw = (h + 2, w + 2) if kind == "conv3r" else (h, w)
    dx = torch.full((n, ih, iw, pitch4(cin)), NAN, device=d)
    assert vec4_epilogue(dx, 0, None)
    layer.bind_backward(grad_planes(gy, dy_channels(layer, cout)), dx, None)
    layer.pack()
    layer.forward()
    layer.backward()
    torch.cuda.synchronize()
    e_y = relmax(y[..., :cout], nhwc(yr))
    e_dx = relmax(dx[..., :cin], nhwc(gx))
    record(f"aligned_epilogue[{kind},{n},{cin},{cout},{h}x{w}]", f"fwd {e_y:.3e} dx {e_dx:.3e}")
    assert e_y < FWD_TOL and e_dx < BWD_TOL, (e_y, e_dx)
    # exactly the valid channels were written: no NaN left inside, every pad channel untouched
    assert not torch.isnan(y[..., :cout]).any() and torch.isnan(y[..., cout:]).all()
    assert not torch.isnan(dx[..., :cin]).any() and torch.isnan(dx[..., cin:]).all()


# ---------------------------------------------------------------------------------------------
# 2. the tanh epilogue
# ---------------------------------------------------------------------------------------------
# (kind, n, cin, cout, h, w, output pitch): the phase-stacked head, the unstacked head through the float2 store
# (pitch 28) and a 3-channel ConvTranspose2d output through the scalar store (pitch 3)
TANH_CASES = [
    ("head", 2, 192, 19, 32, 32, 19),
    ("head", 2, 192, 27, 16, 16, 28),
    ("convT4s2", 2, 128, 3, 16, 16, 3),
]


@pytest.mark.parametrize("kind,n,cin,cout,h,w,pitch", TANH_CASES)
def test_tanh_epilogue(kind, n, cin, cout, h, w, pitch):
    from swapnet_b200 import ops
    from swapnet_b200.layers import ConvLayer

    d = dev()
    base, x, wt, bias = make_layer(kind, n, cin, cout, h, w, 3)
    layer = ConvLayer(kind, base.weight, base.bias, base.x, nsplit=3, act=ops.ACT_TANH, name=f"{kind}-tanh")
    assert layer.stacked == (cout <= L.HEAD_SLOT and kind == "head")
    oh, ow = L.out_hw(kind, h, w)
    y = torch.full((n, oh, ow, pitch), NAN, device=d)
    assert vec4_epilogue(y, 0, layer.bias) == (pitch % 4 == 0)
    layer.bind_forward(y)
    layer.pack()
    layer.forward()
    torch.cuda.synchronize()
    z = nhwc(ref_gpu(kind, x, wt, bias))
    got = y[..., :cout].double()
    # tanh is 1-Lipschitz: the forward bound on the pre-activation, max|err| / max|z|, bounds the output's error too
    err = ((got - torch.tanh(z)).abs().max() / z.abs().max()).item()
    record(f"tanh_epilogue[{kind},{n},{cin},{cout},{h}x{w},pitch={pitch}]",
           f"{err:.3e} (relmax vs tanh {relmax(got, torch.tanh(z)):.3e})")
    assert err < FWD_TOL, err
    assert not torch.isnan(got).any() and torch.isnan(y[..., cout:]).all()


# ---------------------------------------------------------------------------------------------
# 3. tile totals around the SM count
# ---------------------------------------------------------------------------------------------
# 8 x 16 planes: one 128-row M tile per image, so the image count sets the M tiles.  (kind, cout, target total):
# the total is a function of the SM count s; cout 64 is one N tile, cout 640 five; convT4s2 launches 4 phases
SCHEDULE_CASES = [
    ("conv3z", 64, "1"),
    ("conv3z", 64, "s-1"),
    ("conv3z", 64, "s"),
    ("conv3z", 64, "s+1"),
    ("conv3z", 64, "2s+1"),
    ("convT4s2", 64, "s"),
    ("conv3z", 640, "2s+1"),
]


@pytest.mark.parametrize("kind,cout,target,nsplit", at_both_nsplits(SCHEDULE_CASES))
def test_tile_totals_around_sm_count(kind, cout, target, nsplit):
    s = sm_count()
    want = {"1": 1, "s-1": s - 1, "s": s, "s+1": s + 1, "2s+1": 2 * s + 1}[target]
    per_image = (4 if kind == "convT4s2" else 1) * -(-cout // L.pick_block_n(cout))   # phases x N tiles
    n = -(-want // per_image)
    cin, h, w = 64, 8, 16
    layer, x, wt, bias = make_layer(kind, n, cin, cout, h, w, nsplit)
    oh, ow = L.out_hw(kind, h, w)
    y = torch.full((n, oh, ow, cout), NAN, device=dev())
    layer.bind_forward(y)
    assert len(layer.fwd_plans) == 1
    tiles = total_tiles(layer.fwd_plans[0])
    assert tiles == n * per_image and tiles - want < per_image, (tiles, want)
    layer.pack()
    layer.forward()
    torch.cuda.synchronize()
    exact = nhwc(ref_gpu(kind, x, wt, bias))
    tag = f"tile_totals[{kind},{cin},{cout},n={n},tiles={tiles},sms={s}" + ("]" if nsplit == 3 else ",nsplit=1]")
    if nsplit == 3:
        err = relmax(y, exact)
        record(tag, f"{err:.3e}")
        assert err < FWD_TOL, err
    else:
        err, sep = check_single_pass(tag, y, model_forward(layer), exact, FWD_TOL, SP_SEP_FP16)
        record(tag, f"{err:.3e} (model vs exact {sep:.3e})")
    assert not torch.isnan(y).any()


# ---------------------------------------------------------------------------------------------
# 4. repeated, graph-replayed and concurrent launches of one plan
# ---------------------------------------------------------------------------------------------
# a 1-phase plan with fused InstanceNorm statistics, a 4-phase plan and the phase-stacked head; each has more tiles
# than an H100 has SMs, so the persistent CTAs draw tickets from the plan's tile counter
REPEAT_CASES = [
    ("conv3r", 24, 64, 128, 32, 32),
    ("convT4s2", 24, 128, 64, 16, 16),
    ("head", 24, 64, 19, 32, 32),
]


@pytest.mark.parametrize("kind,n,cin,cout,h,w,nsplit", at_both_nsplits(REPEAT_CASES))
def test_repeated_launches_bit_identical(kind, n, cin, cout, h, w, nsplit):
    from swapnet_b200 import ops

    d = dev()
    layer, x, wt, bias = make_layer(kind, n, cin, cout, h, w, nsplit)
    oh, ow = L.out_hw(kind, h, w)
    y = torch.empty(n, oh, ow, cout, device=d)
    stats = torch.empty(n, cout, 2, dtype=torch.float64, device=d) if kind == "conv3r" else None
    layer.bind_forward(y, stats=stats)
    assert len(layer.fwd_plans) == 1 and layer.fused_stats == (stats is not None)
    assert layer.stacked == (kind == "head")
    plan = layer.fwd_plans[0]
    assert geometry(plan)[3] == (4 if kind == "convT4s2" else 1)
    assert total_tiles(plan) > sm_count(), "the plan must outrun one tile per SM"
    layer.pack()

    def clear():   # every launch must write every output (the statistics launch zeroes its own sums)
        y.fill_(NAN)
        if stats is not None:
            stats.fill_(NAN)

    def check_ref(xv, tag):
        ref = nhwc(ref_gpu(kind, xv, wt, bias))
        sep = ""
        if nsplit == 1:   # against the operand model (the planes hold xv's 16-bit words)
            model = model_forward(layer)
            err, s_ = check_single_pass(f"repeat {tag}", y, model, ref, FWD_TOL, SP_SEP_FP16)
            ref, sep = model, f" (model vs exact {s_:.3e})"
        err = relmax(y, ref)
        e_s = 0.0
        if stats is not None:
            e_s = max(relmax(stats[..., 0], ref.sum((1, 2))), relmax(stats[..., 1], (ref * ref).sum((1, 2))))
        record(f"repeat[{kind},{n},{cin},{cout},{h}x{w},{tag},nsplit={nsplit}]", f"fwd {err:.3e} stats {e_s:.3e}{sep}")
        assert err < FWD_TOL and e_s < 1e-5, (tag, err, e_s)

    def check_same(tag):
        assert torch.equal(y, y0), f"{tag}: output differs from the first launch"
        if stats is not None:   # fp64 atomics: the order of the adds varies, the sums agree to rounding
            assert relmax(stats, s0) < 1e-12, tag

    # first eager launch: the bit pattern every later launch on the same inputs must reproduce
    clear()
    layer.forward()
    torch.cuda.synchronize()
    y0 = y.clone()
    s0 = None if stats is None else stats.clone()
    check_ref(x, "eager")
    for i in range(2):
        clear()
        layer.forward()
        torch.cuda.synchronize()
        check_same(f"eager launch {i + 2}")

    # CUDA graph: one captured launch, replayed with the original inputs, two new inputs, and the original again
    g = torch.cuda.CUDAGraph()
    clear()
    with torch.cuda.graph(g):
        layer.forward()
    gen = torch.Generator().manual_seed(7)
    for i, xv in enumerate([x, torch.randn(x.shape, generator=gen), torch.randn(x.shape, generator=gen), x]):
        repack(layer, xv)
        clear()
        g.replay()
        torch.cuda.synchronize()
        if xv is x:
            check_same(f"graph replay {i}")
        else:
            check_ref(xv, f"graph replay {i}")
    del g

    # beside a weight-gradient plan of another layer on a second stream (fork and join through events)
    other, ox, owt, ob = make_layer("conv3r", 4, 128, 128, 32, 32, nsplit)
    ogy = torch.randn((4, 128, 32, 32), generator=torch.Generator().manual_seed(3)).to(d)
    _, _, ogw, _ = ref_fwd_bwd("conv3r", ox, owt, ob, ogy)
    owg = torch.zeros_like(other.weight)
    other.bind_backward(grad_planes(ogy, 128), None, owg)
    other.pack()
    side = torch.cuda.Stream()
    main = torch.cuda.current_stream()
    clear()
    fork = torch.cuda.Event()
    fork.record(main)
    side.wait_event(fork)
    with torch.cuda.stream(side):
        other.backward(dgrad=False, bias=False)
    layer.forward()
    join = torch.cuda.Event()
    join.record(side)
    main.wait_event(join)
    torch.cuda.synchronize()
    check_same("beside a weight-gradient launch")
    if nsplit == 3:
        e_w = relmax(owg, ogw)
        assert e_w < BWD_TOL, e_w
    else:
        e_w, _ = check_single_pass("concurrent wgrad", owg, model_wgrad(other), ogw, FWD_TOL, SP_SEP_BF16)
    record(f"repeat[{kind},{n},{cin},{cout},{h}x{w},concurrent wgrad,nsplit={nsplit}]", f"wgrad {e_w:.3e}")


# ---------------------------------------------------------------------------------------------
# 5. weight-gradient split-K and += accumulation
# ---------------------------------------------------------------------------------------------
# (kind, n, cin, cout, h, w, swap, rows_valid, cols_valid)
WGRAD_CASES = [
    # wide Y: X = dy, 96 rows (a partial 128-row M tile), Y = the padded input, 80 columns (a partial 128-column N tile)
    ("conv3r", 2, 80, 96, 32, 32, False, 96, 80),
    # X = the 55-channel input through the merged parity map (h parity folded into the channel coordinate)
    ("conv4s2", 2, 55, 64, 64, 64, True, 55, 64),
    # the 19-channel first conv: 32-channel Y rows, the 16 taps share one X tap and form groups of 4
    ("conv4s2", 2, 19, 64, 64, 64, False, 64, 19),
    # a 3x3 pixel plane (S = 192): 4x4 patches of 4 images, pixels past the plane masked by dy's extents
    ("conv4s2", 40, 128, 256, 6, 6, False, 256, 128),
]


@pytest.mark.parametrize("kind,n,cin,cout,h,w,swap,rows,cols,nsplit", at_both_nsplits(WGRAD_CASES))
def test_wgrad_split_k_accumulates(kind, n, cin, cout, h, w, swap, rows, cols, nsplit):
    from swapnet_b200 import ops

    d = dev()
    layer, x, wt, bias = make_layer(kind, n, cin, cout, h, w, nsplit)
    oh, ow = L.out_hw(kind, h, w)
    gen = torch.Generator().manual_seed(99)
    gy = torch.randn((n, cout, oh, ow), generator=gen).to(d)
    _, _, gw, _ = ref_fwd_bwd(kind, x, wt, bias, gy)
    dy = grad_planes(gy, dy_channels(layer, cout))
    (ws,) = L.wgrad_specs(kind, h, w)
    x_is_dy = ws.x_is == "dy"
    xs, ys = (dy, layer.x.twin) if x_is_dy else (layer.x.twin, dy)
    cx, cy = (cout, cin) if x_is_dy else (cin, cout)
    s_row, s_col = L.wgrad_out_strides(kind, cin, cout, x_is_dy)

    def plan_for(out, ksplit):
        desc = ops.wgrad_desc(xs, ys, ws, out, s_row, s_col, list(ws.tap_ids), cx, cy, swap=swap, nsplit=nsplit,
                              ksplit=ksplit)
        assert (desc.rows_valid, desc.cols_valid) == (rows, cols)
        assert (desc.ngroups > 0) == (min(xs.c, ys.c) < 64)
        return ops.wgrad_plan(desc, keep=(xs.hi, xs.lo, ys.hi, ys.lo, out)), desc

    # the number of pixel tiles: an over-large split is clamped to it
    probe = torch.zeros_like(layer.weight)
    total = geometry(plan_for(probe, 1 << 20)[0])[3]
    g0 = (torch.randn(wt.shape, generator=gen) * gw.abs().max().item()).float().to(d)
    ref, tol, sep = gw, BWD_TOL, ""
    if nsplit == 1:   # single pass: against the operand model, at the forward bound
        ref, tol = model_wgrad(layer, dy), FWD_TOL
        sep = f" model vs exact {relmax(ref, gw):.3e}"
        assert relmax(ref, gw) >= SP_SEP_BF16 * tol
    outs, errs = {}, {}
    for ks in (1, 2, 3, 7, total, total + 5):
        out = g0.clone()
        plan, desc = plan_for(out, ks)
        assert geometry(plan)[3] == min(ks, total)
        plan.run()
        torch.cuda.synchronize()
        outs[ks] = out
        errs[ks] = relmax(out.double() - g0.double(), ref)    # += into the torch-layout gradient
    scale = gw.abs().max().item()
    spread = max((outs[k].double() - outs[1].double()).abs().max().item() / scale for k in outs)
    groups = [desc.group_size[i] for i in range(desc.ngroups)]
    record(f"wgrad_split_k[{kind},{n},{cin},{cout},{h}x{w},swap={swap},tiles={total},groups={groups},nsplit={nsplit}]",
           " ".join(f"k{k} {e:.3e}" for k, e in errs.items()) + f" spread {spread:.3e}" + sep)
    assert max(errs.values()) < tol, errs
    assert spread < SPLIT_SPREAD, spread


# ---------------------------------------------------------------------------------------------
# 6. input-magnitude window of the fp16-split operands
# ---------------------------------------------------------------------------------------------
# hi = fp16(v), lo = fp16(v - hi) carries 22 bits only while lo stays a normal fp16 number (|lo| >= 2^-14, i.e.
# |v| >~ 2^-3) and hi does not saturate (|v| <= 65504).  Below the window lo loses bits to the subnormals; the error
# of the smallest scale is recorded, not asserted.
FP16_SCALES = [-10, -6, -3, 0, 4, 8, 10]
FP16_ASSERTED = (-6, -3, 0, 4, 8, 10)


@pytest.mark.parametrize("k", FP16_SCALES)
def test_fp16_split_input_range(k):
    layer, x, wt, _ = make_layer("conv3r", 2, 128, 128, 32, 32, 3, with_bias=False)
    xs = x * 2.0 ** k
    repack(layer, xs)
    y = torch.full((2, 32, 32, 128), NAN, device=dev())
    layer.bind_forward(y)
    layer.pack()
    layer.forward()
    torch.cuda.synchronize()
    err = relmax(y, nhwc(ref_gpu("conv3r", xs, wt, None)))
    record(f"fp16_split_range[conv3r,128,128,x*2^{k}]", f"{err:.3e}")
    if k in FP16_ASSERTED:
        assert err < FWD_TOL, (k, err)
