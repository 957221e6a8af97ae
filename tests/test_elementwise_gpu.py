"""The element-wise kernels of csrc/elementwise.cu against plain fp64 torch of the same operation.

- norm_act_fwd: InstanceNorm or none, each activation, dropout with a global-sample offset, the residual, and the four
  kinds of output (fp16-split planes with their bf16 twin, bf16-split planes, the fp32 copy, reflect-padded planes);
- the dropout mask: the counter hash, the sample offset under data parallelism, the seed a replayed graph reads from
  the step-parameter buffer;
- norm_act_bwd, sum_grads and tanh_bwd over 1..SN_MAX_SRC gradient sources (channel offsets, reflect-padded, nearest
  upsampled, a ReLU consumer of a LeakyReLU stage) and the fused bias gradient;
- ce_tanh_bwd, the warp stage's loss kernel: cross entropy on the tanh outputs, the extra gradient sources and the tanh
  backward in one pass;
- the input packers pack_concat (direct and shared-memory kernels) and pack_planes from compact segmentation maps;
- the texture stage fed its cloth as a uint8 label map.

Each norm/activation kernel has one body templated on the channels a thread handles: V = 4 (a channel quad) where the
host's alignment predicates hold, else V = 1.  `fwd_vec`, `bwd_vec` and `sum_vec` restate those predicates; every case
asserts which instantiation it meant to reach, and the option cases run on both.  Beyond 4096 channels forward (3072
with the BatchNorm affine) and 2048 in the backward apply pass a block stages one slice of the channels.

Split planes: where the kernel's fp32 value is known (the packers' inputs, norm_act_fwd's fp32 copy) the hi and lo words
must be the split of common.cuh's split16 bit for bit: hi = r16(clamp(v, +-65504)) for fp16, r16(v) for bf16, and
lo = r16(v - hi).  Values are compared with fp64 references as max|err| / max|ref|: 1e-5 for fp32 and fp16-split
forward outputs, 2e-5 for bf16-split ones, 1e-4 for bf16-split gradients, 1e-6 for sum_grads' fp32 output.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle.dropout import keep_mask
from swapnet_b200 import _lib
from swapnet_b200 import ops
from swapnet_b200.engine import _mix_seed
from test_kernels_gpu import dev, nhwc, record, relmax

pytestmark = pytest.mark.gpu

IN, NONE = True, False
A_NONE, A_RELU, A_LRELU = ops.ACT_NONE, ops.ACT_RELU, ops.ACT_LRELU
SLOPE = 0.2
P_DROP = 0.5
SEED = 0x5EED1234ABC
SENT16 = 0x1357           # sentinel word in every plane channel a kernel must not write
SENT32 = 7.25             # sentinel in fp32 buffers


# ---------------------------------------------------------------------------------------------
# path predicates (the host conditions of sn_norm_act_fwd, sn_norm_act_bwd and sn_sum_grads)
# ---------------------------------------------------------------------------------------------
def _al(t, k):
    return t.data_ptr() % k == 0


def fwd_vec(y, c, residual=None, out_f32=None, out=None):
    ok = c % 4 == 0 and _al(y, 16) and ops._pitch(y) % 4 == 0
    if residual is not None:
        ok = ok and _al(residual, 16) and ops._pitch(residual) % 4 == 0
    if out_f32 is not None:
        ok = ok and _al(out_f32, 16) and ops._pitch(out_f32) % 4 == 0
    if out is not None:
        planes = [out.hi, out.lo] + ([] if out.twin is None else [out.twin.hi, out.twin.lo])
        ok = ok and out.pitch % 4 == 0 and out.c_off % 4 == 0 and all(_al(p, 8) for p in planes)
    return ok


def srcs_vec(srcs):
    return all(_al(s.t, 16) and ops._pitch(s.t) % 4 == 0 and s.c_off % 4 == 0 for s in srcs)


def bwd_vec(srcs, y, c, dy):
    return (c % 4 == 0 and _al(y, 16) and ops._pitch(y) % 4 == 0 and srcs_vec(srcs) and dy.pitch % 4 == 0
            and dy.c_off % 4 == 0 and _al(dy.hi, 8) and _al(dy.lo, 8))


def sum_vec(srcs, c, dst):
    return c % 4 == 0 and srcs_vec(srcs) and _al(dst, 16) and ops._pitch(dst) % 4 == 0


# ---------------------------------------------------------------------------------------------
# references
# ---------------------------------------------------------------------------------------------
def split_ref(v, fmt):
    """(hi, lo) int16 words of common.cuh's split16 of the fp32 tensor v."""
    v = v.float()
    if fmt == ops.FMT_F16:
        v = torch.where(v.abs() <= 3.4028234663852886e38, v.clamp(-65504.0, 65504.0), v)
        hi = v.to(torch.float16)
        lo = (v - hi.float()).to(torch.float16)
    else:
        hi = v.to(torch.bfloat16)
        lo = (v - hi.float()).to(torch.bfloat16)
    return hi.view(torch.int16), lo.view(torch.int16)


def words(t):
    return t.view(torch.int16)


def planes_of(p):
    """[(hi, lo, fmt)] of a Planes and of its twin."""
    out = [(p.hi, p.lo, p.fmt)]
    if p.twin is not None:
        out.append((p.twin.hi, p.twin.lo, p.twin.fmt))
    return out


def fill_sentinel(p):
    for hi, lo, _ in planes_of(p):
        words(hi).fill_(SENT16)
        words(lo).fill_(SENT16)


def assert_outside_untouched(p, c0, c1):
    """channels [0, c0) and [c1, pitch) of every plane of p still hold the sentinel."""
    for hi, lo, _ in planes_of(p):
        for t in (hi, lo):
            assert bool((words(t[..., :c0]) == SENT16).all()) and bool((words(t[..., c1:]) == SENT16).all()), \
                "wrote outside its channel slice"


def assert_split_exact(p, c0, c1, v):
    """hi and lo words of channels [c0, c1) of every plane of p are the split of the fp32 values v, bit for bit."""
    for hi, lo, fmt in planes_of(p):
        rh, rl = split_ref(v, fmt)
        assert torch.equal(words(hi[..., c0:c1]), rh.to(hi.device)), f"hi words (fmt {fmt})"
        assert torch.equal(words(lo[..., c0:c1]), rl.to(lo.device)), f"lo words (fmt {fmt})"


def dense_of(hi, lo, fmt, c0, c1):
    dt = torch.float16 if fmt == ops.FMT_F16 else torch.bfloat16
    return hi[..., c0:c1].view(dt).double() + lo[..., c0:c1].view(dt).double()


def inorm(y):
    """InstanceNorm2d (eps 1e-5, biased variance, no affine) of NCHW fp64.  F.instance_norm refuses a 1x1 plane, whose
    normalised value is 0: the same formula written out."""
    if y.shape[2] * y.shape[3] > 1:
        return F.instance_norm(y, eps=ops.IN_EPS)
    m = y.mean((2, 3), keepdim=True)
    return (y - m) / torch.sqrt(y.var((2, 3), unbiased=False, keepdim=True) + ops.IN_EPS)


def act_ref(x, act):
    if act == A_LRELU:
        return F.leaky_relu(x, SLOPE)
    if act == A_RELU:
        return F.relu(x)
    return x


def drop_mask(n, h, w, c, offset, seed=SEED):
    """keep mask * 1/(1-p) of the library's dropout, NCHW fp64 on the device (index: NHWC order + offset)."""
    m = keep_mask(seed, P_DROP, n * h * w * c, offset).reshape(n, h, w, c)
    return torch.from_numpy(m).to(dev()).permute(0, 3, 1, 2).double() * (1.0 / (1.0 - P_DROP))


def gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def randn(shape, g, scale=1.0, shift=0.0):
    return (torch.randn(*shape, generator=g) * scale + shift).to(dev())


# ---------------------------------------------------------------------------------------------
# norm_act_fwd
# ---------------------------------------------------------------------------------------------
# (c, h, w, stats, act, dropout, residual, output): output "twin" = fp16-split planes + bf16 twin, "bf16" = bf16-split
# planes, "f32" = the fp32 copy alone, "reflect" = reflect-padded fp16 planes + twin.  Every plane output also writes the
# fp32 copy, which gives the exact fp32 values the split words must hold.
FWD_CASES = [
    (3, 4, 4, IN, A_LRELU, 0, 0, "twin"),
    (3, 3, 3, IN, A_RELU, 1, 0, "reflect"),
    (3, 63, 63, NONE, A_NONE, 1, 0, "f32"),            # dropout without InstanceNorm
    (4, 1, 1, IN, A_LRELU, 0, 1, "twin"),
    (4, 3, 5, NONE, A_NONE, 1, 0, "reflect"),
    (4, 63, 63, IN, A_RELU, 1, 1, "bf16"),
    (19, 5, 3, IN, A_LRELU, 1, 0, "reflect"),
    (19, 63, 63, NONE, A_LRELU, 0, 0, "bf16"),
    (19, 1, 1, NONE, A_RELU, 1, 1, "f32"),
    (19, 3, 3, IN, A_NONE, 0, 1, "reflect"),
    (36, 3, 3, IN, A_RELU, 0, 1, "reflect"),
    (36, 63, 63, IN, A_LRELU, 1, 0, "twin"),
    (36, 4, 4, NONE, A_RELU, 1, 1, "f32"),
    (36, 5, 3, NONE, A_LRELU, 0, 0, "reflect"),
    (36, 1, 1, IN, A_NONE, 1, 1, "f32"),
    (64, 63, 63, IN, A_NONE, 0, 1, "reflect"),         # the residual block's tail
    (64, 1, 1, NONE, A_LRELU, 1, 0, "bf16"),
    (64, 5, 3, IN, A_NONE, 1, 1, "reflect"),
    (64, 3, 5, IN, A_RELU, 0, 0, "twin"),
    (64, 4, 4, IN, A_LRELU, 1, 1, "bf16"),
    (1024, 4, 4, IN, A_LRELU, 1, 0, "twin"),
    (1024, 3, 3, IN, A_NONE, 0, 1, "reflect"),
    (1024, 1, 1, IN, A_RELU, 1, 0, "bf16"),
    (1024, 63, 63, IN, A_RELU, 1, 0, "twin"),
    (4096, 4, 4, IN, A_LRELU, 0, 0, "twin"),           # the widest single slice
    (4096, 3, 5, NONE, A_NONE, 1, 1, "reflect"),
    (4096, 63, 63, IN, A_LRELU, 1, 0, "bf16"),
    (4100, 4, 4, IN, A_LRELU, 1, 0, "twin"),           # beyond it: two slices
    (4100, 3, 3, IN, A_RELU, 0, 1, "f32"),
    (4100, 5, 3, NONE, A_LRELU, 1, 0, "reflect"),
]


def _fwd_inputs(c, h, w, stats_on, res_on, seed):
    n = 1 if c * h * w >= 4096 * 63 * 63 else 2
    g = gen(seed)
    y = randn((n, h, w, c), g, 2.0, 0.5)
    res = randn((n, h, w, c), g) if res_on else None
    return n, y, res


def _run_fwd(y, c, stats, act, drop, res, output, n, h, w, aligned):
    """one norm_act_fwd call; -> (taken vector path?, fp32 copy [n,h,w,c], planes or None)"""
    d = dev()
    if aligned:
        yv = y
    else:                                             # pitch c + 1: not a multiple of 4 floats
        yv = torch.full((n, h, w, c + 1), SENT32, device=d)[..., :c]
        yv.copy_(y)
    f32_buf = torch.full((n, h, w, c + 4), SENT32, device=d)
    f32 = f32_buf[..., :c]
    out = None
    if output != "f32":
        oh, ow = (h + 2, w + 2) if output == "reflect" else (h, w)
        coff = 4
        pitch = (coff + c + 4 + 7) // 8 * 8
        fmt = ops.FMT_BF16 if output == "bf16" else ops.FMT_F16
        out = ops.Planes(n, oh, ow, pitch, d, c=c, c_off=coff, fmt=fmt, dual=output in ("twin", "reflect"))
        fill_sentinel(out)
    vec = fwd_vec(yv, c, res, f32, out)
    ops.norm_act_fwd(yv, c, stats, act, SLOPE, P_DROP if drop else 0.0, SEED, residual=res, out=out,
                     reflect_pad=output == "reflect", out_f32=f32, drop_offset=5 * h * w * c if drop else 0)
    torch.cuda.synchronize()
    assert bool((f32_buf[..., c:] == SENT32).all()), "fp32 copy: wrote past its channels"
    return vec, f32, out


@pytest.mark.parametrize("c,h,w,stats_on,act,drop,res_on,output", FWD_CASES)
def test_norm_act_fwd(c, h, w, stats_on, act, drop, res_on, output):
    n, y, res = _fwd_inputs(c, h, w, stats_on, res_on, c + 7 * h + w)
    stats = None
    if stats_on:
        stats = torch.zeros(n, c, 2, dtype=torch.float64, device=dev())
        ops.plane_stats(y, c, stats)
    yr = y.permute(0, 3, 1, 2).double()
    ref = act_ref(inorm(yr) if stats_on else yr, act)
    if drop:
        ref = ref * drop_mask(n, h, w, c, 5 * h * w * c)
    if res_on:
        ref = ref + res.permute(0, 3, 1, 2).double()
    ref_nhwc = nhwc(ref)
    runs = {}
    for aligned in (True, False):
        vec, f32, out = _run_fwd(y, c, stats, act, drop, res, output, n, h, w, aligned)
        assert vec == (aligned and c % 4 == 0), "took the other instantiation"
        e = relmax(f32, ref_nhwc)
        assert e < 1e-5, f"fp32 copy relmax {e:.3e} (V = 4: {vec})"
        if out is not None:
            co = out.c_off
            assert_outside_untouched(out, co, co + c)
            assert_split_exact(out, co, co + c, F.pad(f32.permute(0, 3, 1, 2), (1, 1, 1, 1), mode="reflect")
                               .permute(0, 2, 3, 1) if output == "reflect" else f32)
            want = nhwc(F.pad(ref, (1, 1, 1, 1), mode="reflect")) if output == "reflect" else ref_nhwc
            for hi, lo, fmt in planes_of(out):
                ep = relmax(dense_of(hi, lo, fmt, co, co + c), want)
                assert ep < (1e-5 if fmt == ops.FMT_F16 else 2e-5), f"planes (fmt {fmt}) relmax {ep:.3e}"
        runs[vec] = (f32.clone(), None if out is None else [(hi.clone(), lo.clone()) for hi, lo, _ in planes_of(out)])
        record(f"norm_act_fwd[{c},{h}x{w},{output},vec={vec}]", f"{e:.3e}")
    if len(runs) == 2:   # both instantiations do the same fp32 operations per element: bit-identical results
        (fa, pa), (fb, pb) = runs[True], runs[False]
        assert torch.equal(fa, fb), "the V = 4 and V = 1 forwards differ"
        if pa is not None:
            assert all(torch.equal(words(a), words(b)) for x, y_ in zip(pa, pb) for a, b in zip(x, y_))


# ---------------------------------------------------------------------------------------------
# dropout addressing
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed,p,count", [(0, 0.5, 4097), (SEED, 0.5, 100003), (0xFFFFFFFFFFFF, 0.1, 77777),
                                          (12345, 0.9, 65536)])
def test_dropout_mask_equals_host_hash(seed, p, count):
    got = ops.dropout_mask(seed, p, count, dev()).cpu().numpy().astype(bool)
    want = keep_mask(seed, p, count)
    assert np.array_equal(got, want)
    assert abs(want.mean() - (1 - p)) < 0.02


def _aligned_or_pitched(t, aligned):
    if aligned:
        return t
    v = torch.zeros(*t.shape[:3], t.shape[3] + 1, device=t.device)[..., :t.shape[3]]
    v.copy_(t)
    return v


@pytest.mark.parametrize("aligned", [True, False])
def test_dropout_offset_splits_the_batch(aligned):
    """One call over B samples equals two calls over B/2 samples with drop_offset = b0*h*w*c (the global sample index
    of the first local sample under data parallelism), forward and backward, bit for bit."""
    d = dev()
    B, h, w, c = 4, 6, 7, 36
    g = gen(11)
    y = _aligned_or_pitched(randn((B, h, w, c), g, 2.0, 0.5), aligned)
    ga = randn((B, h, w, c), g)
    stats = torch.zeros(B, c, 2, dtype=torch.float64, device=d)
    ops.plane_stats(y, c, stats)
    hw = h * w * c

    def fwd(n0, n1):
        o = torch.zeros(n1 - n0, h, w, c, device=d)
        ops.norm_act_fwd(y[n0:n1], c, stats[n0:n1], A_LRELU, SLOPE, P_DROP, SEED, out_f32=o, drop_offset=n0 * hw)
        return o

    def bwd(n0, n1):
        dy = ops.Planes(n1 - n0, h, w, 40, d, c=c, fmt=ops.FMT_BF16)
        srcs = [ops.GradSrc(ga[n0:n1])]
        assert bwd_vec(srcs, y[n0:n1], c, dy) == aligned
        ops.norm_act_bwd(srcs, y[n0:n1], c, None, A_LRELU, dy, None, SLOPE, P_DROP, SEED, drop_offset=n0 * hw)
        return torch.cat([dy.hi, dy.lo], -1)

    assert fwd_vec(y, c, out_f32=torch.zeros(1, 1, 1, 4, device=d)) == aligned
    whole_f, whole_b = fwd(0, B), bwd(0, B)
    half_f = torch.cat([fwd(0, B // 2), fwd(B // 2, B)])
    half_b = torch.cat([bwd(0, B // 2), bwd(B // 2, B)])
    torch.cuda.synchronize()
    assert torch.equal(whole_f, half_f) and torch.equal(words(whole_b), words(half_b))
    # and the offset matters: the second half without it gets the first half's masks
    wrong = torch.zeros(B // 2, h, w, c, device=d)
    ops.norm_act_fwd(y[B // 2:], c, stats[B // 2:], A_LRELU, SLOPE, P_DROP, SEED, out_f32=wrong)
    assert not torch.equal(wrong, whole_f[B // 2:])


@pytest.mark.parametrize("aligned", [True, False])
def test_dropout_seed_from_step_parameters(aligned):
    """The seed a replayed graph reads from device memory: the 32-bit step seed written through set_step_params as
    its (lo16, hi16) halves plus a stage id gives the masks of the host seed engine._mix_seed(step_seed, stage_id)."""
    d = dev()
    n, h, w, c = 2, 5, 9, 64
    g = gen(12)
    y = _aligned_or_pitched(randn((n, h, w, c), g, 2.0, 0.5), aligned)
    ga = randn((n, h, w, c), g)
    stats = torch.zeros(n, c, 2, dtype=torch.float64, device=d)
    ops.plane_stats(y, c, stats)
    sp = torch.zeros(22, device=d)
    results = {}
    for step_seed in (0xDEADBEEF, 7):
        vals = [0.0] * 22
        vals[20], vals[21] = float(step_seed & 0xFFFF), float(step_seed >> 16)
        ops.set_step_params(sp, vals)
        for stage in (3, 17):
            outs = []
            for dev_seed in (True, False):
                o = torch.zeros(n, h, w, c, device=d)
                dy = ops.Planes(n, h, w, 64, d, fmt=ops.FMT_BF16)
                assert fwd_vec(y, c, out_f32=o) == aligned and bwd_vec([ops.GradSrc(ga)], y, c, dy) == aligned
                kw = dict(seed_dev=sp[20:22], stage_id=stage) if dev_seed else {}
                host_seed = 999 if dev_seed else _mix_seed(step_seed, stage)   # ignored when seed_dev is given
                ops.norm_act_fwd(y, c, stats, A_LRELU, SLOPE, P_DROP, host_seed, out_f32=o, **kw)
                ops.norm_act_bwd([ops.GradSrc(ga)], y, c, None, A_LRELU, dy, None, SLOPE, P_DROP, host_seed, **kw)
                outs.append((o, torch.cat([dy.hi, dy.lo], -1)))
            torch.cuda.synchronize()
            (fa, ba), (fb, bb) = outs
            assert torch.equal(fa, fb) and torch.equal(words(ba), words(bb)), (hex(step_seed), stage)
            results[(step_seed, stage)] = fa
    keys = list(results)
    assert all(not torch.equal(results[a], results[b]) for i, a in enumerate(keys) for b in keys[i + 1:])


# ---------------------------------------------------------------------------------------------
# gradient sources: norm_act_bwd, sum_grads, tanh_bwd
# ---------------------------------------------------------------------------------------------
# a source spec: "plain" (at a channel offset of a wider tensor), "reflect" (reflect-padded plane), "upK" (nearest
# upsampled by K), "relu" (plain, read by a ReLU consumer of the stage's LeakyReLU output)
def make_src(kind, n, h, w, c, g, aligned):
    """-> (GradSrc, fp64 NCHW adjoint of the source onto the [n,c,h,w] plane, act override or None)"""
    if kind in ("plain", "relu"):
        off = 4 if aligned else 3
        t = randn((n, h, w, c + 8), g)
        src = ops.GradSrc(t, off, act=A_RELU if kind == "relu" else -1)
        return src, t[..., off:off + c].permute(0, 3, 1, 2).double(), A_RELU if kind == "relu" else None
    if kind == "reflect":
        t = randn((n, h + 2, w + 2, c + 4), g)
        xin = torch.zeros(n, c, h, w, dtype=torch.float64, device=dev(), requires_grad=True)
        (adj,) = torch.autograd.grad(F.pad(xin, (1, 1, 1, 1), mode="reflect"), xin, t[..., :c].permute(0, 3, 1, 2).double())
        return ops.GradSrc(t, 0, True), adj, None
    assert kind.startswith("up")
    u = int(kind[2:])
    t = randn((n, h * u, w * u, c + 8), g)
    xin = torch.zeros(n, c, h, w, dtype=torch.float64, device=dev(), requires_grad=True)
    (adj,) = torch.autograd.grad(F.interpolate(xin, scale_factor=u, mode="nearest"), xin,
                                 t[..., 8:8 + c].permute(0, 3, 1, 2).double())
    return ops.GradSrc(t, 8, up=u), adj, None


# (c, h, w, stats, stage act, dropout, sources)
BWD_CASES = [
    (64, 3, 3, IN, A_LRELU, 0, ("reflect",)),
    (64, 3, 5, IN, A_LRELU, 1, ("reflect", "plain")),
    (64, 5, 3, NONE, A_RELU, 1, ("reflect",)),
    (36, 4, 4, IN, A_LRELU, 0, ("up8",)),                   # the encode backward of the texture stage at 512x512
    (36, 6, 5, IN, A_LRELU, 1, ("up2", "plain")),
    (128, 8, 8, IN, A_LRELU, 1, ("plain", "relu")),         # the pix2pix skip: LeakyReLU to D_{j+1}, ReLU to the concat
    (256, 4, 4, IN, A_LRELU, 0, ("relu", "plain", "reflect")),
    (19, 7, 9, IN, A_NONE, 1, ("plain", "plain")),
    (4, 1, 1, NONE, A_LRELU, 1, ("plain", "relu")),
    (1024, 4, 4, IN, A_RELU, 1, ("plain", "up2")),
    (2048, 3, 3, IN, A_LRELU, 0, ("reflect", "relu")),      # the widest single slice of the apply pass
    (2052, 4, 4, IN, A_LRELU, 1, ("plain",)),               # beyond it: two slices
    (64, 63, 63, IN, A_LRELU, 1, ("plain", "relu", "reflect")),
]


def _bwd_reference(y, srcs_ref, stats_on, act, drop, n, h, w, c):
    """d/dy of sum_s <adj_s, drop(act_s(IN(y)))>, the composed forward in fp64 autograd"""
    yr = y.permute(0, 3, 1, 2).double().requires_grad_()
    x = inorm(yr) if stats_on else yr
    mask = drop_mask(n, h, w, c, 3 * h * w * c) if drop else None
    total = 0.0
    for adj, a in srcs_ref:
        o = act_ref(x, act if a is None else a)
        if mask is not None:
            o = o * mask
        total = total + (o * adj).sum()
    (gy,) = torch.autograd.grad(total, yr)
    return nhwc(gy)


@pytest.mark.parametrize("c,h,w,stats_on,act,drop,kinds", BWD_CASES)
def test_norm_act_bwd(c, h, w, stats_on, act, drop, kinds):
    d = dev()
    n = 2
    for aligned in (True, False):
        g = gen(c + h + 3 * w)
        y = randn((n, h, w, c), g, 2.0, 0.5)
        made = [make_src(k, n, h, w, c, g, aligned) for k in kinds]
        srcs = [m[0] for m in made]
        stats = gst = None
        if stats_on:
            stats = torch.zeros(n, c, 2, dtype=torch.float64, device=d)
            gst = torch.zeros_like(stats)
            ops.plane_stats(y, c, stats)
        coff = 4 if aligned else 1
        dy = ops.Planes(n, h, w, (coff + c + 4 + 7) // 8 * 8, d, c=c, c_off=coff, fmt=ops.FMT_BF16)
        fill_sentinel(dy)
        vec = bwd_vec(srcs, y, c, dy)
        assert vec == (aligned and c % 4 == 0), "took the other instantiation"
        ops.norm_act_bwd(srcs, y, c, stats, act, dy, gst, SLOPE, P_DROP if drop else 0.0, SEED,
                         drop_offset=3 * h * w * c if drop else 0)
        torch.cuda.synchronize()
        ref = _bwd_reference(y, [(m[1], m[2]) for m in made], stats_on, act, drop, n, h, w, c)
        assert_outside_untouched(dy, coff, coff + c)
        e = relmax(dense_of(dy.hi, dy.lo, dy.fmt, coff, coff + c), ref)
        record(f"norm_act_bwd[{c},{h}x{w},{'+'.join(kinds)},vec={vec}]", f"{e:.3e}")
        assert e < 1e-4, f"dy relmax {e:.3e} (V = 4: {vec})"


@pytest.mark.parametrize("c", [64, 256, 512, 1024])
def test_fused_bias_grad_accumulates(c):
    """norm_act_bwd(bias_grad=b): b += per-channel sums of the dy written, from a non-zero start.  The V = 4 apply pass
    takes c in {256, 512, 1024}, the V = 1 one (unaligned sources) c in {64, 128, 256}: at c = 64 four threads of a
    block share each channel."""
    d = dev()
    n, h, w = 2, 5, 6
    for aligned in {64: (False,), 256: (True, False)}.get(c, (True,)):
        g = gen(c)
        y = randn((n, h, w, c), g, 2.0, 0.5)
        made = [make_src(k, n, h, w, c, g, aligned) for k in ("plain", "relu", "reflect")]
        srcs = [m[0] for m in made]
        dy = ops.Planes(n, h, w, c, d, fmt=ops.FMT_BF16)
        start = randn((c,), g, 3.0)
        bg = start.clone()
        assert bwd_vec(srcs, y, c, dy) == aligned and (ops.fused_bias_grad_ok(c) or not aligned)
        ops.norm_act_bwd(srcs, y, c, None, A_LRELU, dy, None, SLOPE, P_DROP, SEED, drop_offset=3 * h * w * c,
                         bias_grad=bg)
        torch.cuda.synchronize()
        ref = _bwd_reference(y, [(m[1], m[2]) for m in made], False, A_LRELU, True, n, h, w, c)
        assert relmax(dy.dense(), ref) < 1e-4
        e = relmax(bg.double() - start.double(), ref.sum((0, 1, 2)))
        record(f"fused_bias_grad[{c},vec={aligned}]", f"{e:.3e}")
        assert e < 1e-5, e


# (c, h, w, sources) — sum_grads ignores the consumer's activation
SUM_CASES = [
    (64, 3, 3, ("reflect",)),
    (64, 3, 5, ("reflect", "plain")),
    (32, 5, 3, ("reflect", "up2")),
    (36, 4, 4, ("up8",)),
    (36, 6, 6, ("up4", "plain", "reflect")),
    (19, 7, 5, ("plain", "reflect")),
    (1024, 3, 4, ("plain", "plain", "plain")),
]


@pytest.mark.parametrize("c,h,w,kinds", SUM_CASES)
def test_sum_grads(c, h, w, kinds):
    d = dev()
    n = 2
    for aligned in (True, False):
        g = gen(c + 5 * h + w)
        made = [make_src(k, n, h, w, c, g, aligned) for k in kinds]
        srcs = [m[0] for m in made]
        dst_off = 0 if aligned else 1
        base = torch.full((n, h, w, c + 4), SENT32, device=d)
        dst = base[..., dst_off:dst_off + c]
        vec = sum_vec(srcs, c, dst)
        assert vec == (aligned and c % 4 == 0), "took the other instantiation"
        ops.sum_grads(srcs, n, h, w, c, dst)
        torch.cuda.synchronize()
        ref = nhwc(sum(m[1] for m in made))
        e = relmax(dst, ref)
        record(f"sum_grads[{c},{h}x{w},{'+'.join(kinds)},vec={vec}]", f"{e:.3e}")
        # an up = 8 block adds 64 fp32 terms per value; measured 2.1e-7 on an H100 80GB HBM3 (700 W limit)
        assert e < 1e-6, f"relmax {e:.3e} (V = 4: {vec})"
        assert bool((base[..., :dst_off] == SENT32).all()) and bool((base[..., dst_off + c:] == SENT32).all())


@pytest.mark.parametrize("c,h,w,kinds", [(19, 16, 16, ("plain", "plain")), (3, 5, 3, ("reflect", "up2")),
                                         (12, 3, 3, ("reflect", "plain", "up4"))])
def test_tanh_bwd(c, h, w, kinds):
    d = dev()
    n = 2
    g = gen(c * 3 + h)
    z = randn((n, h, w, c), g)
    o = torch.tanh(z)
    made = [make_src(k, n, h, w, c, g, False) for k in kinds]
    dy = ops.Planes(n, h, w, (c + 4 + 7) // 8 * 8 + 8, d, c=c, c_off=4, fmt=ops.FMT_BF16)
    fill_sentinel(dy)
    ops.tanh_bwd([m[0] for m in made], o, c, dy)
    torch.cuda.synchronize()
    ref = nhwc(sum(m[1] for m in made)) * (1 - o.double() ** 2)
    assert_outside_untouched(dy, 4, 4 + c)
    e = relmax(dense_of(dy.hi, dy.lo, dy.fmt, 4, 4 + c), ref)
    record(f"tanh_bwd[{c},{h}x{w},{'+'.join(kinds)}]", f"{e:.3e}")
    assert e < 1e-4, e


# ---------------------------------------------------------------------------------------------
# ce_tanh_bwd
# ---------------------------------------------------------------------------------------------
def _ce_target(kind, n, c, h, w, g):
    """-> (target passed to the kernel, argmax index [n,h,w] on the device)"""
    if kind == "label":
        lab = torch.randint(0, c + 6, (n, h, w), generator=g, dtype=torch.int64)   # 0, in range, and >= C
        lab[0, 0, :3] = torch.tensor([0, c, 255])
        arg = torch.where(lab >= c, torch.zeros_like(lab), lab)
        return ops.SegMap(lab.to(torch.uint8).to(dev()), c), arg.to(dev())
    t = torch.rand(n, c, h, w, generator=g)                      # non-one-hot values
    t[:, :, 0, :] = 0.0                                          # all-zero vectors: index 0
    t[:, :, 1, :] = 0.0
    t[:, c - 1, 1, :] = 1.0
    t[:, c // 2, 1, 1::2] = 1.0                                  # ties between c/2 and c-1: the first maximum wins
    t[:, :, 2, 0] = 0.5                                          # every channel tied
    onehot = torch.randint(0, c, (n, h, w), generator=g)
    t[:, :, 3:5, :] = F.one_hot(onehot, c).permute(0, 3, 1, 2).float()[:, :, 3:5, :]
    return t.to(dev()), t.argmax(1).to(dev())


@pytest.mark.parametrize("fmt", [ops.FMT_BF16, ops.FMT_F16])
@pytest.mark.parametrize("c,target_kind,extra", [(3, "dense", 0), (8, "label", 1), (19, "dense", 2), (19, "label", 1),
                                                 (32, "dense", 1), (32, "label", 2), (8, "dense", 2), (3, "label", 0)])
def test_ce_tanh_bwd(c, target_kind, extra, fmt):
    d = dev()
    n, h, w = 2, 9, 13
    weight = 100.0
    g = gen(c * 10 + extra)
    cp = c + 3
    o_buf = torch.tanh(randn((n, h, w, cp), g))                  # the head's outputs in a wider pitch
    target, arg = _ce_target(target_kind, n, c, h, w, g)
    made = []
    if extra >= 1:                                               # the GAN term: body channels first (warp_model.py)
        gan = randn((n, h, w, 3 + c), g, 0.1)
        made.append((ops.GradSrc(gan, 3), gan[..., 3:].permute(0, 3, 1, 2).double()))
    if extra >= 2:
        s, adj, _ = make_src("reflect", n, h, w, c, g, True)
        made.append((s, adj))
    c8 = (c + 7) // 8 * 8
    runs = []
    for ws in (None, ops.DetWorkspace(d)):
        acc = torch.zeros(1, dtype=torch.float64, device=d)
        dy = ops.Planes(n, h, w, 8 + c8 + 8, d, c=c8, c_off=8, fmt=fmt)
        fill_sentinel(dy)
        ops.ce_tanh_bwd(o_buf, c, target, weight, acc, [m[0] for m in made], dy, ws=ws)
        torch.cuda.synchronize()
        runs.append((acc.item(), dy))
    od = o_buf[..., :c].permute(0, 3, 1, 2).double().requires_grad_()
    loss = weight * F.cross_entropy(od, arg)
    (gce,) = torch.autograd.grad(loss, od)
    gsum = gce + sum((m[1] for m in made), torch.zeros_like(gce))
    ref = nhwc(gsum * (1 - od.detach() ** 2))
    (l0, dy0), (l1, dy1) = runs
    e_l = abs(l0 - loss.item()) / abs(loss.item())
    e = relmax(dense_of(dy0.hi, dy0.lo, fmt, 8, 8 + c), ref)
    record(f"ce_tanh_bwd[{c},{target_kind},extra={extra},fmt={fmt}]", f"loss {e_l:.3e} dy {e:.3e}")
    assert e_l < 1e-6, e_l
    assert e < 1e-4, e
    for t in (dy0.hi, dy0.lo):
        assert bool((words(t[..., 8 + c:8 + c8]) == 0).all()), "channels C..C8 not zero-filled"
    assert_outside_untouched(dy0, 8, 8 + c8)
    assert torch.equal(words(dy0.hi), words(dy1.hi)) and torch.equal(words(dy0.lo), words(dy1.lo)), "_det dy differs"
    assert abs(l1 - l0) <= 1e-12 * abs(l0)


def test_ce_tanh_bwd_refusals():
    d = dev()
    n, h, w = 1, 4, 4
    acc = torch.zeros(1, dtype=torch.float64, device=d)
    o = torch.zeros(n, h, w, 33, device=d)
    t = torch.zeros(n, 33, h, w, device=d)
    dy = ops.Planes(n, h, w, 48, d, c=40, fmt=ops.FMT_BF16)
    with pytest.raises(_lib.SwapnetB200Error, match="at most 32 classes"):
        ops.ce_tanh_bwd(o, 33, t, 1.0, acc, [], dy)
    o = torch.zeros(n, h, w, 19, device=d)
    t = torch.zeros(n, 19, h, w, device=d)
    dy = ops.Planes(n, h, w, 48, d, c=24, c_off=4, fmt=ops.FMT_BF16)
    with pytest.raises(_lib.SwapnetB200Error, match="8-channel aligned slices"):
        ops.ce_tanh_bwd(o, 19, t, 1.0, acc, [], dy)


# ---------------------------------------------------------------------------------------------
# input packers
# ---------------------------------------------------------------------------------------------
def make_pack_src(kind, n, c, h, w, g):
    """-> ((tensor or SegMap, nhwc flag), fp32 NCHW values on the CPU)"""
    if kind == "nchw":
        t = torch.randn(n, c, h, w, generator=g)
        t[0, 0, 0, :2] = torch.tensor([1e5, -7e4])                # beyond the fp16 range: hi saturates at 65504
        return (t.to(dev()), False), t
    if kind == "nhwc":
        buf = torch.randn(n, h, w, c + 3, generator=g)
        return (buf.to(dev())[..., :c], True), buf[..., :c].permute(0, 3, 1, 2).contiguous()
    if kind == "label":
        lab = torch.randint(0, c + 4, (n, h, w), generator=g)       # labels >= C expand to the all-zero vector
        lab[0, 0, :3] = torch.tensor([0, c - 1, c])
        ch = torch.arange(c).view(1, -1, 1, 1)
        return (ops.SegMap(lab.to(torch.uint8).to(dev()), c), False), ((lab.unsqueeze(1) == ch) & (ch > 0)).float()
    assert kind == "mask"
    m = torch.randint(0, 2 ** 31, (n, h, w), generator=g, dtype=torch.int64) | (1 << 31)   # bit 31 set everywhere
    m[0, 0, 0] = 0
    bits = ((m.unsqueeze(1) >> torch.arange(c).view(1, -1, 1, 1)) & 1).float()
    as_i32 = torch.where(m >= 1 << 31, m - (1 << 32), m).to(torch.int32)      # same 32 bits, two's complement
    return (ops.SegMap(as_i32.to(dev()), c), False), bits


# (c_fill, [(kind, channels)], w): c_fill 16 / 32 take the thread-per-pixel kernel, others the shared-memory one
PACK_CASES = [
    (16, [("nchw", 3), ("label", 9)], 37),
    (16, [("mask", 12), ("nhwc", 4)], 19),
    (32, [("nhwc", 3), ("label", 19)], 45),           # the warp stage's D input: body + cloth
    (32, [("mask", 32)], 33),                        # bit 31 is channel 31
    (32, [("nchw", 19), ("nchw", 3)], 7),
    (24, [("label", 19), ("nchw", 3)], 70),          # 64-pixel runs: a partial run
    (24, [("mask", 20), ("nhwc", 4)], 129),
    (64, [("nchw", 36), ("label", 19)], 40),         # 32-pixel runs
    (64, [("nhwc", 60), ("mask", 4)], 31),
]


@pytest.mark.parametrize("c_fill,specs,w", PACK_CASES)
def test_pack_concat(c_fill, specs, w):
    n, h = 2, 3
    g = gen(c_fill * 100 + w)
    srcs, vals = [], []
    for kind, c in specs:
        s, v = make_pack_src(kind, n, c, h, w, g)
        srcs.append(s)
        vals.append(v)
    coff = 16
    dst = ops.Planes(n, h, w, coff + c_fill + 8, dev(), c=c_fill, c_off=coff, dual=True)
    fill_sentinel(dst)
    ops.pack_concat(srcs, dst)
    torch.cuda.synchronize()
    v = torch.cat(vals, 1)
    v = torch.cat([v, torch.zeros(n, c_fill - v.shape[1], h, w)], 1)    # pad channels up to c_fill are zero
    assert_split_exact(dst, coff, coff + c_fill, nhwc(v))
    assert_outside_untouched(dst, coff, coff + c_fill)


@pytest.mark.parametrize("kind", ["label", "mask"])
def test_pack_planes_segmap_into_texture_slice(kind):
    """The texture U-Net's input: the cloth expanded from a compact map into channels 36..54 of the 64-channel planes
    and their bf16 twin (engine.TextureEngine.forward)."""
    n, h, w, c = 2, 5, 40, 19
    g = gen(36)
    (sm, _), v = make_pack_src(kind, n, c, h, w, g)
    dst = ops.Planes(n, h, w, 64, dev(), dual=True)
    fill_sentinel(dst)
    ops.pack_planes(sm, dst.slice(36, c))
    torch.cuda.synchronize()
    assert_split_exact(dst, 36, 36 + c, nhwc(v))
    assert_outside_untouched(dst, 36, 36 + c)


# ---------------------------------------------------------------------------------------------
# the texture stage with its cloth as a uint8 label map
# ---------------------------------------------------------------------------------------------
def test_texture_compact_cloths_equal_dense_cloths():
    """TextureModel fed `cloths` as a uint8 label map (what --dataset texture_b200 yields) gives the step the dense
    one-hot fp32 cloths give: the expanded planes are identical, so the fakes are bit for bit and only the atomics'
    summation order may move the gradients."""
    from swapnet_b200.models import create_model
    from test_engine_gpu import _opt, _run_phases, synth_texture_batch

    B, S = 2, 128
    torch.manual_seed(0)
    opt = _opt(B, S, model="texture", name="texture", netG="swapnet", lambda_l1=10, lambda_content=0.0,
               lambda_style=0.0, b200_vgg="random")
    model = create_model(opt)
    model.setup(opt)
    model.is_train = True
    tex, rois, cloth, tgt = synth_texture_batch(B, S)
    dense = dict(input_textures=tex, rois=rois, cloths=cloth, target_textures=tgt, cloth_paths=["c"] * B,
                 texture_paths=["t"] * B)
    sm = ops.SegMap.from_dense(cloth)
    assert sm.data.dtype == torch.uint8 and torch.equal(sm.dense(), cloth)
    compact = dict(dense, cloths=sm.data)
    l0, gD0, gG0 = _run_phases(model, dense, 5)
    f0 = model.fakes.clone()
    l1, gD1, gG1 = _run_phases(model, compact, 5)
    assert isinstance(model.cloths, ops.SegMap)
    assert torch.equal(f0, model.fakes), "forward differs between dense and compact cloths"
    assert relmax(gD1, gD0) < 1e-5 and relmax(gG1, gG0) < 1e-5
    assert all(abs(l0[k] - l1[k]) <= 1e-6 * abs(l0[k]) for k in l0), (l0, l1)
