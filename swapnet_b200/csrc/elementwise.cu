// swapnet_b200 — HBM-bound kernels of the SwapNet hot path (sm_90a).
//
// Operand packing (fp32 -> split-bf16 NHWC planes), InstanceNorm statistics, the fused
// InstanceNorm-apply + activation + dropout (+ residual, + reflect padding) forward and
// backward blocks, gradient merges and the loss kernels.  Reference semantics:
//   modules/layers.py:12-63,126-144 (UNetDown/UNetUp/ResidualBlock element ops),
//   modules/__init__.py:67-69 (InstanceNorm2d: eps 1e-5, biased variance, no affine),
//   models/warp_model.py:147-150 (CE on argmax targets), modules/loss.py:58,110-122 (BCE),
//   models/texture_model.py:168-170 (L1).
// All tensors are NHWC fp32 with an explicit pixel pitch; threads map to channels fastest
// so that every warp touches contiguous 128-B lines.
#include "common.cuh"
#include "reflect_pad.h"
#include "../../include/swapnet_b200.h"

void sn_count_launch(int n);

namespace {

constexpr int kEwThreads = 256;

// ---------------------------------------------------------------------------------
// dropout: counter-based keep mask.  keep(seed, idx) must be reproducible on the host
// (oracle/dropout.py restates it) so that parity tests can share masks.
// ---------------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint32_t sn_hash32(unsigned long long seed, unsigned long long idx) {
  unsigned long long z = idx + seed * 0x9E3779B97F4A7C15ull + 0x632BE59BD9B4E019ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z = z ^ (z >> 31);
  return (uint32_t)(z >> 32);
}
__host__ __device__ __forceinline__ bool sn_keep(unsigned long long seed, unsigned long long idx,
                                                 uint32_t thresh) {
  return sn_hash32(seed, idx) >= thresh;  // P(drop) = thresh / 2^32
}
__host__ __device__ __forceinline__ uint32_t drop_thresh(float p) {
  double t = (double)p * 4294967296.0;
  if (t < 0) t = 0;
  if (t > 4294967295.0) t = 4294967295.0;
  return (uint32_t)t;
}

// per-stage dropout seed from the step seed (host twin: engine._mix_seed).  With `seed_dev` the step seed lives in
// device memory (updated once per step), so that a captured CUDA graph of the step replays with fresh masks.
__host__ __device__ __forceinline__ unsigned long long sn_mix_seed(unsigned long long step_seed, unsigned int stage_id) {
  return (step_seed * 0x9E3779B1ull + (unsigned long long)stage_id * 0x85EBCA77ull + 0x165667B1ull) & 0xFFFFFFFFFFFFull;
}
template <class Args>
__device__ __forceinline__ unsigned long long drop_seed_of(const Args& a) {
  if (!a.seed_dev) return a.seed;
  // the 32-bit step seed travels in the float step-parameter buffer as two exact 16-bit halves (lo, hi)
  const unsigned long long step_seed =
      ((unsigned long long)(unsigned int)a.seed_dev[1] << 16) | (unsigned long long)(unsigned int)a.seed_dev[0];
  return sn_mix_seed(step_seed, a.stage_id);
}

// V consecutive channels moved as one load or store: V fp32 values (V = 1, 4) or V 16-bit words (V = 1, 4, 8).  The
// caller guarantees the alignment of the V-wide access.
template <int V>
__device__ __forceinline__ void load_f32(const float* p, float v[V]) {
  static_assert(V == 1 || V == 4, "fp32 vectors are 1 or 4 wide");
  if constexpr (V == 1) {
    v[0] = *p;
  } else {
    const float4 t = *reinterpret_cast<const float4*>(p);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  }
}
// acc[0..V) += the V fp32 values at p, written out rather than as a loop: the gathers that call it sit inside
// `unroll 1` loops, where an inner loop costs the backward reduce kernels registers
template <int V>
__device__ __forceinline__ void add_f32(const float* p, float acc[V]) {
  static_assert(V == 1 || V == 4, "fp32 vectors are 1 or 4 wide");
  if constexpr (V == 1) {
    acc[0] += *p;
  } else {
    const float4 t = *reinterpret_cast<const float4*>(p);
    acc[0] += t.x; acc[1] += t.y; acc[2] += t.z; acc[3] += t.w;
  }
}
template <int V>
__device__ __forceinline__ void store_f32(float* p, const float v[V]) {
  static_assert(V == 1 || V == 4, "fp32 vectors are 1 or 4 wide");
  if constexpr (V == 1) *p = v[0];
  else *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
}
// V 16-bit words travel packed, two per 32-bit word: word j sits in bits 16 (j & 1) of u[j / 2]
template <int V>
__device__ __forceinline__ void load_w16(const uint16_t* p, uint32_t u[(V + 1) / 2]) {
  static_assert(V == 1 || V == 4 || V == 8, "16-bit vectors are 1, 4 or 8 wide");
  if constexpr (V == 1) {
    u[0] = *p;
  } else if constexpr (V == 4) {
    const uint2 t = *reinterpret_cast<const uint2*>(p);
    u[0] = t.x; u[1] = t.y;
  } else {
    const uint4 t = *reinterpret_cast<const uint4*>(p);
    u[0] = t.x; u[1] = t.y; u[2] = t.z; u[3] = t.w;
  }
}
template <int V>
__device__ __forceinline__ void store_w16(uint16_t* p, const uint32_t u[(V + 1) / 2]) {
  static_assert(V == 1 || V == 4 || V == 8, "16-bit vectors are 1, 4 or 8 wide");
  if constexpr (V == 1) *p = (uint16_t)u[0];
  else if constexpr (V == 4) *reinterpret_cast<uint2*>(p) = make_uint2(u[0], u[1]);
  else *reinterpret_cast<uint4*>(p) = make_uint4(u[0], u[1], u[2], u[3]);
}
__device__ __forceinline__ uint16_t word16(const uint32_t* u, int j) {
  return (uint16_t)(u[j >> 1] >> (16 * (j & 1)));
}

// channel counts are signed ints: C >> log2(V) is one shift where C / V would round towards zero
__host__ __device__ constexpr int log2_of(int v) { return v > 1 ? 1 + log2_of(v >> 1) : 0; }

// V fp32 values -> split16 words at hi[off..off+V) (and lo, when given)
template <int V>
__device__ __forceinline__ void store_split(uint16_t* hi, uint16_t* lo, long long off, const float v[V], int fmt) {
  uint16_t h[V], l[V];
#pragma unroll
  for (int j = 0; j < V; ++j) split16(v[j], fmt, h[j], l[j]);
  uint32_t ph[(V + 1) / 2], pl[(V + 1) / 2];
#pragma unroll
  for (int j = 0; j < (V + 1) / 2; ++j) {
    ph[j] = (uint32_t)h[2 * j] | (2 * j + 1 < V ? (uint32_t)h[2 * j + 1] << 16 : 0u);
    pl[j] = (uint32_t)l[2 * j] | (2 * j + 1 < V ? (uint32_t)l[2 * j + 1] << 16 : 0u);
  }
  store_w16<V>(hi + off, ph);
  if (lo) store_w16<V>(lo + off, pl);
}

// ---------------------------------------------------------------------------------
// pack_planes
// ---------------------------------------------------------------------------------
// NCHW source: one block per (n, h, 32-pixel run); smem transposes [c][w] -> [w][c].
// value of channel c at a pixel of a compact segmentation map (see SN_LAYOUT_LABEL_U8 / SN_LAYOUT_MASK_I32)
__device__ __forceinline__ float seg_value(const void* src, int layout, long long pix, int c) {
  if (layout == SN_LAYOUT_LABEL_U8) {
    const int lab = reinterpret_cast<const uint8_t*>(src)[pix];
    return (c > 0 && lab == c) ? 1.f : 0.f;          // label 0 = background = the all-zero vector
  }
  return (float)((reinterpret_cast<const uint32_t*>(src)[pix] >> c) & 1u);
}

__global__ void pack_planes_nchw_kernel(const float* __restrict__ src, int layout, int N, int C, int H, int W,
                                        uint16_t* __restrict__ hi, uint16_t* __restrict__ lo,
                                        int pitch, int coff, int fmt) {
  extern __shared__ float tile[];  // [C][33]
  const int w0 = blockIdx.x * 32;
  const int h = blockIdx.y;
  const int n = blockIdx.z;
  for (int i = threadIdx.x; i < C * 32; i += blockDim.x) {
    const int c = i / 32, w = i % 32;
    float v = 0.f;
    if (w0 + w < W) {
      if (layout == SN_LAYOUT_NCHW) v = src[(((long long)n * C + c) * H + h) * W + w0 + w];
      else v = seg_value(src, layout, ((long long)n * H + h) * W + w0 + w, c);
    }
    tile[c * 33 + w] = v;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < C * 32; i += blockDim.x) {
    const int w = i / C, c = i % C;
    if (w0 + w < W) {
      const long long off = (((long long)n * H + h) * W + w0 + w) * pitch + coff + c;
      store_split<1>(hi, lo, off, &tile[c * 33 + w], fmt);
    }
  }
}
__global__ void pack_planes_nhwc_kernel(const float* __restrict__ src, int src_pitch, long long npix,
                                        int C, uint16_t* __restrict__ hi,
                                        uint16_t* __restrict__ lo, int pitch, int coff, int fmt) {
  const long long total = npix * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long pix = i / C;
    const int c = (int)(i - pix * C);
    store_split<1>(hi, lo, pix * pitch + coff + c, &src[pix * src_pitch + c], fmt);
  }
}

// pack_concat: `lead` zero channels, then up to two fp32 sources (NCHW or NHWC) concatenated along channels,
// zero-filled up to c_fill channels, written as full 16-byte groups of 8 channels into the fp16 planes AND their
// bf16 twin in one pass.  One block = one (n, h, 32-pixel run).
struct PackSrc { const float* p; int layout, pitch, c; };
struct PackConcatArgs {
  PackSrc s[2]; int nsrc;
  int N, H, W, c_fill;
  uint16_t *hi, *lo, *hi2, *lo2; int pitch, coff, fmt, fmt2;
  int lead;                 // zero channels in front of the sources
};
__global__ void __launch_bounds__(256) pack_concat_kernel(const PackConcatArgs a) {
  // one block = one (n, h, PW-pixel run), PW = 32 * (64 / c_fill) so that narrow outputs keep all
  // 256 threads busy (c_fill = 16 -> 128 pixels); smem tile [c_fill][PW + 1]
  extern __shared__ float tile[];
  const int PW = 32 * (64 / (a.c_fill < 64 ? a.c_fill : 64));
  const int TP = PW + 1;
  const int w0 = blockIdx.x * PW, h = blockIdx.y, n = blockIdx.z;
  int cbase = a.lead;
  for (int si = 0; si < a.nsrc; ++si) {
    const PackSrc s = a.s[si];
    if (s.layout == SN_LAYOUT_NCHW) {
      for (int i = threadIdx.x; i < s.c * PW; i += blockDim.x) {
        const int c = i / PW, w = i - c * PW;
        tile[(cbase + c) * TP + w] = (w0 + w < a.W) ? s.p[(((long long)n * s.c + c) * a.H + h) * a.W + w0 + w] : 0.f;
      }
    } else if (s.layout == SN_LAYOUT_NHWC) {
      for (int i = threadIdx.x; i < s.c * PW; i += blockDim.x) {
        const int w = i / s.c, c = i - w * s.c;
        tile[(cbase + c) * TP + w] = (w0 + w < a.W) ? s.p[(((long long)n * a.H + h) * a.W + w0 + w) * s.pitch + c] : 0.f;
      }
    } else {   // compact segmentation map (uint8 labels / int32 bit mask) expanded to s.c 0/1 channels
      for (int i = threadIdx.x; i < s.c * PW; i += blockDim.x) {
        const int c = i / PW, w = i - c * PW;
        tile[(cbase + c) * TP + w] = (w0 + w < a.W) ? seg_value(s.p, s.layout, ((long long)n * a.H + h) * a.W + w0 + w, c) : 0.f;
      }
    }
    cbase += s.c;
  }
  // zero channels: the lead [0, lead) and the fill [cbase, c_fill)
  for (int i = threadIdx.x; i < (a.lead + a.c_fill - cbase) * PW; i += blockDim.x) {
    const int z = i / PW;
    tile[(z < a.lead ? z : cbase + z - a.lead) * TP + (i % PW)] = 0.f;
  }
  __syncthreads();
  const int G = a.c_fill >> 3;
  for (int i = threadIdx.x; i < PW * G; i += blockDim.x) {
    const int w = i / G, g = i - w * G;
    if (w0 + w >= a.W) continue;
    uint16_t h1[8], l1[8], h2[8], l2[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float v = tile[(g * 8 + j) * TP + w];
      split16(v, a.fmt, h1[j], l1[j]);
      if (a.hi2) split16(v, a.fmt2, h2[j], l2[j]);
    }
    const long long off = (((long long)n * a.H + h) * a.W + w0 + w) * a.pitch + a.coff + g * 8;
    auto pk = [](const uint16_t* x) {
      uint4 r;
      r.x = x[0] | ((uint32_t)x[1] << 16); r.y = x[2] | ((uint32_t)x[3] << 16);
      r.z = x[4] | ((uint32_t)x[5] << 16); r.w = x[6] | ((uint32_t)x[7] << 16);
      return r;
    };
    *reinterpret_cast<uint4*>(a.hi + off) = pk(h1);
    if (a.lo) *reinterpret_cast<uint4*>(a.lo + off) = pk(l1);
    if (a.hi2) {
      *reinterpret_cast<uint4*>(a.hi2 + off) = pk(h2);
      if (a.lo2) *reinterpret_cast<uint4*>(a.lo2 + off) = pk(l2);
    }
  }
}

// pack_concat, narrow outputs (c_fill <= 32: the 3/19/22-channel network inputs): one thread = one pixel, no shared
// memory.  NCHW sources are read one channel at a time (coalesced across the warp's 32 pixels), NHWC sources as the
// pixel's own run of channels, compact maps as ONE byte / word; the pixel's 16 or 32 channels are written as 16-byte
// stores (a warp writes 1-2 KB contiguous per plane).  The streams are write-bound: 2 planes (+ 2 twin planes).
template <int CF>
__global__ void __launch_bounds__(256) pack_concat_direct_kernel(const PackConcatArgs a) {
  const long long npix = (long long)a.N * a.H * a.W;
  const long long HW = (long long)a.H * a.W;
  for (long long pix = blockIdx.x * (long long)blockDim.x + threadIdx.x; pix < npix;
       pix += (long long)gridDim.x * blockDim.x) {
    const long long n = pix / HW, p = pix - n * HW;
    float v[CF];
#pragma unroll
    for (int c = 0; c < CF; ++c) v[c] = 0.f;
    int cbase = a.lead;
    for (int si = 0; si < a.nsrc; ++si) {
      const PackSrc s = a.s[si];
      if (s.layout == SN_LAYOUT_NCHW) {
#pragma unroll
        for (int c = 0; c < CF; ++c)
          if (c >= cbase && c < cbase + s.c) v[c] = s.p[(n * s.c + (c - cbase)) * HW + p];
      } else if (s.layout == SN_LAYOUT_NHWC) {
#pragma unroll
        for (int c = 0; c < CF; ++c)
          if (c >= cbase && c < cbase + s.c) v[c] = s.p[pix * s.pitch + (c - cbase)];
      } else if (s.layout == SN_LAYOUT_LABEL_U8) {
        const int lab = reinterpret_cast<const uint8_t*>(s.p)[pix];
#pragma unroll
        for (int c = 0; c < CF; ++c)
          if (c >= cbase && c < cbase + s.c) v[c] = (c - cbase > 0 && lab == c - cbase) ? 1.f : 0.f;
      } else {
        const uint32_t m = reinterpret_cast<const uint32_t*>(s.p)[pix];
#pragma unroll
        for (int c = 0; c < CF; ++c)
          if (c >= cbase && c < cbase + s.c) v[c] = (float)((m >> (c - cbase)) & 1u);
      }
      cbase += s.c;
    }
    const long long off = pix * a.pitch + a.coff;
#pragma unroll
    for (int g8 = 0; g8 < CF / 8; ++g8) {
      uint16_t h1[8], l1[8], h2[8], l2[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        split16(v[g8 * 8 + j], a.fmt, h1[j], l1[j]);
        if (a.hi2) split16(v[g8 * 8 + j], a.fmt2, h2[j], l2[j]);
      }
      auto pk = [](const uint16_t* x) {
        uint4 r;
        r.x = x[0] | ((uint32_t)x[1] << 16); r.y = x[2] | ((uint32_t)x[3] << 16);
        r.z = x[4] | ((uint32_t)x[5] << 16); r.w = x[6] | ((uint32_t)x[7] << 16);
        return r;
      };
      *reinterpret_cast<uint4*>(a.hi + off + g8 * 8) = pk(h1);
      if (a.lo) *reinterpret_cast<uint4*>(a.lo + off + g8 * 8) = pk(l1);
      if (a.hi2) {
        *reinterpret_cast<uint4*>(a.hi2 + off + g8 * 8) = pk(h2);
        if (a.lo2) *reinterpret_cast<uint4*>(a.lo2 + off + g8 * 8) = pk(l2);
      }
    }
  }
}

// ---------------------------------------------------------------------------------
// head weights: nearest-x2 upsample + ZeroPad2d((1,0,1,0)) + Conv2d(k=4, p=1) seen from an
// output pixel o = 2m + par reads up-sampled u = o + k - 2, k = 0..3, i.e. source s = u >> 1:
//   par 0: k=0,1 -> m-1 ; k=2,3 -> m          (2 effective taps: d = -1, 0)
//   par 1: k=0 -> m-1 ; k=1,2 -> m ; k=3 -> m+1 (3 effective taps: d = -1, 0, +1)
// effective tap index e = d + 1.  Phase p = 2*py + px owns neff(py) x neff(px) taps, laid out
// contiguously: phase offsets {0, 4, 10, 16}, 25 taps in total, order (ey, ex) row-major.
// ---------------------------------------------------------------------------------
__host__ __device__ __forceinline__ int head_neff(int par) { return par ? 3 : 2; }
__host__ __device__ __forceinline__ int head_phase_off(int p) {
  const int o[4] = {0, 4, 10, 16};
  return o[p];
}
// which original taps k map onto effective tap e for parity par: returns count, fills ks[]
__host__ __device__ __forceinline__ int head_taps_of(int par, int e, int ks[2]) {
  if (par == 0) {
    ks[0] = 2 * e; ks[1] = 2 * e + 1;
    return 2;
  }
  if (e == 0) { ks[0] = 0; return 1; }
  if (e == 1) { ks[0] = 1; ks[1] = 2; return 2; }
  ks[0] = 3;
  return 1;
}
__global__ void pack_head_weights_kernel(const float* __restrict__ w, int cout, int cin, int rows_pad,
                                         int k_pad, int dgrad, int taps_pitch, uint16_t* __restrict__ hi,
                                         uint16_t* __restrict__ lo, int fmt,
                                         const float* __restrict__ scale2) {
  // one thread per (co, te, ci) with te the global effective tap 0..24
  const float sc = scale2 ? scale2[0] : 1.f;
  const long long total = (long long)cout * 25 * cin;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int ci = (int)(i % cin);
    const int te = (int)((i / cin) % 25);
    const int co = (int)(i / ((long long)cin * 25));
    int p = 3;
    while (te < head_phase_off(p)) --p;
    const int py = p >> 1, px = p & 1;
    const int local = te - head_phase_off(p);
    const int ey = local / head_neff(px), ex = local % head_neff(px);
    int kys[2], kxs[2];
    const int ny = head_taps_of(py, ey, kys), nx = head_taps_of(px, ex, kxs);
    float acc = 0.f;
    for (int a = 0; a < ny; ++a)
      for (int b = 0; b < nx; ++b) acc += w[(((long long)co * cin + ci) * 4 + kys[a]) * 4 + kxs[b]];
    long long off;
    if (!dgrad) {
      // [phase][rows_pad][neff taps][k_pad] with per-phase base = rows_pad * k_pad * phase_off
      off = (long long)rows_pad * k_pad * head_phase_off(p) +
            ((long long)co * (head_neff(py) * head_neff(px)) + local) * k_pad + ci;
    } else {
      off = ((long long)ci * taps_pitch + te) * k_pad + co;  // [ci][taps_pitch >= 25][k_pad]
    }
    acc *= sc;
    store_split<1>(hi, lo, off, &acc, fmt);
  }
}
// stacked-phase layout of the same effective taps: dst[row = phase*slot + co][tap9 = (sy+1)*3 + (sx+1)][ci]
__global__ void pack_head_stacked_kernel(const float* __restrict__ w, int cout, int cin, int slot, int k_pad,
                                         uint16_t* __restrict__ hi, uint16_t* __restrict__ lo, int fmt,
                                         const float* __restrict__ scale2) {
  const float sc = scale2 ? scale2[0] : 1.f;
  const long long total = (long long)4 * slot * 9 * k_pad;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int ci = (int)(i % k_pad);
    const int t9 = (int)((i / k_pad) % 9);
    const int row = (int)(i / ((long long)k_pad * 9));
    const int p = row / slot, co = row - p * slot;
    const int py = p >> 1, px = p & 1;
    const int ey = t9 / 3, ex = t9 % 3;          // effective tap index = shift + 1
    float acc = 0.f;
    if (co < cout && ci < cin && ey < head_neff(py) && ex < head_neff(px)) {
      int kys[2], kxs[2];
      const int ny = head_taps_of(py, ey, kys), nx = head_taps_of(px, ex, kxs);
      for (int a = 0; a < ny; ++a)
        for (int b = 0; b < nx; ++b) acc += w[(((long long)co * cin + ci) * 4 + kys[a]) * 4 + kxs[b]];
    }
    acc *= sc;
    store_split<1>(hi, lo, i, &acc, fmt);
  }
}
__global__ void fold_head_wgrad_kernel(const float* __restrict__ geff, int cout, int cin,
                                       float* __restrict__ dw) {
  const long long total = (long long)cout * cin * 16;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int kx = (int)(i & 3), ky = (int)((i >> 2) & 3);
    const int ci = (int)((i >> 4) % cin);
    const int co = (int)((i >> 4) / cin);
    float acc = 0.f;
    for (int p = 0; p < 4; ++p) {
      const int py = p >> 1, px = p & 1;
      const int ey = py == 0 ? (ky >> 1) : (ky == 0 ? 0 : (ky == 3 ? 2 : 1));
      const int ex = px == 0 ? (kx >> 1) : (kx == 0 ? 0 : (kx == 3 ? 2 : 1));
      const int te = head_phase_off(p) + ey * head_neff(px) + ex;
      acc += geff[((long long)co * 25 + te) * cin + ci];
    }
    dw[i] += acc;
  }
}

// ---------------------------------------------------------------------------------
// weight packing: ONE launch computes the power-of-two scales of every weight tensor of a network (fp16-split
// operands: s = 2^k with max|w|*s in [2^13, 2^14)), ONE launch writes every packed copy (forward and input-gradient
// layouts: dst[r][slot[t]][k] <- src[r*s_row + k*s_k + t] * s).
// ---------------------------------------------------------------------------------
// grid (blocks per tensor, tensors).  scratch[2t] = max |w| bits, scratch[2t+1] = blocks done; the last block of a
// tensor finalises its scale and resets both words (the buffer is zero again when the launch retires).
__global__ void __launch_bounds__(256) weight_scale_multi_kernel(const sn_scale_item* __restrict__ items,
                                                                 unsigned int* __restrict__ scratch) {
  const sn_scale_item it = items[blockIdx.y];
  float m = 0.f;
  const long long n4 = it.count >> 2;
  const float4* w4 = reinterpret_cast<const float4*>(it.w);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = w4[i];
    m = fmaxf(fmaxf(m, fabsf(v.x)), fmaxf(fabsf(v.y), fmaxf(fabsf(v.z), fabsf(v.w))));
  }
  if (blockIdx.x == 0)
    for (long long i = (n4 << 2) + threadIdx.x; i < it.count; i += blockDim.x) m = fmaxf(m, fabsf(it.w[i]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  __shared__ float wm[8];
  if ((threadIdx.x & 31) == 0) wm[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < (int)(blockDim.x >> 5); ++i) m = fmaxf(m, wm[i]);
    unsigned int* sc = scratch + 2 * blockIdx.y;
    atomicMax(sc, __float_as_uint(m));
    __threadfence();
    if (atomicAdd(sc + 1, 1u) == gridDim.x - 1) {
      const float mx = __uint_as_float(atomicExch(sc, 0u));
      sc[1] = 0u;
      float sv = 1.f;
      if (mx > 0.f && isfinite(mx)) {
        int e;
        frexpf(mx, &e);
        sv = ldexpf(1.f, 14 - e);
      }
      it.scale2[0] = sv;
      it.scale2[1] = 1.f / sv;
    }
  }
}

// one block = 8 rows x 64 K x all taps of one pack item; items are found by binary search over block_begin
constexpr int kPkRows = 8, kPkK = 64;
__global__ void __launch_bounds__(256) pack_weights_multi_kernel(const sn_pack_item* __restrict__ items, int nitems) {
  extern __shared__ float tile[];   // [rows][k][taps + 1]
  int lo = 0, hi = nitems - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (items[mid].block_begin <= (int)blockIdx.x) lo = mid; else hi = mid - 1;
  }
  const sn_pack_item it = items[lo];
  const int local = blockIdx.x - it.block_begin;
  const int gx = (it.k_pad + kPkK - 1) / kPkK;
  const int k0 = (local % gx) * kPkK, r0 = (local / gx) * kPkRows;
  const int taps = it.taps, T1 = taps + 1;
  const float sc = it.scale2 ? it.scale2[0] : 1.f;
  const int nr = min(kPkRows, it.rows - r0);
  // gather: element (r, k, t) at src[r*s_row + k*s_k + t]; walk t fastest, then the dimension with the smaller stride
  const bool k_minor = it.s_k <= it.s_row;
  const int total = nr * kPkK * taps;
  for (int i = threadIdx.x; i < total; i += blockDim.x) {
    const int t = i % taps, j = i / taps;
    int r, kk;
    if (k_minor) { kk = j % kPkK; r = j / kPkK; } else { r = j % nr; kk = j / nr; }
    float v = 0.f;
    if (k0 + kk < it.k_real) v = it.src[(long long)(r0 + r) * it.s_row + (long long)(k0 + kk) * it.s_k + t];
    tile[(r * kPkK + kk) * T1 + t] = v;
  }
  __syncthreads();
  uint16_t* hi16 = (uint16_t*)it.hi;
  uint16_t* lo16 = (uint16_t*)it.lo;
  // scatter: one thread = 8 consecutive k of one (row, tap): a 16-byte store per plane (k_pad % 8 == 0)
  constexpr int G = kPkK / 8;
  const int groups = nr * taps * G;
  for (int i = threadIdx.x; i < groups; i += blockDim.x) {
    const int kg = i % G, j = i / G, t = j % taps, r = j / taps;
    const int kk = kg * 8;
    if (k0 + kk >= it.k_pad) continue;
    uint16_t hh[8], ll[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) split16(tile[(r * kPkK + kk + q) * T1 + t] * sc, it.fmt, hh[q], ll[q]);
    const long long off = ((long long)(r0 + r) * it.taps_pitch + it.slot[t]) * it.k_pad + k0 + kk;
    uint4 a, b;
    a.x = hh[0] | ((uint32_t)hh[1] << 16); a.y = hh[2] | ((uint32_t)hh[3] << 16);
    a.z = hh[4] | ((uint32_t)hh[5] << 16); a.w = hh[6] | ((uint32_t)hh[7] << 16);
    b.x = ll[0] | ((uint32_t)ll[1] << 16); b.y = ll[2] | ((uint32_t)ll[3] << 16);
    b.z = ll[4] | ((uint32_t)ll[5] << 16); b.w = ll[6] | ((uint32_t)ll[7] << 16);
    *reinterpret_cast<uint4*>(hi16 + off) = a;
    *reinterpret_cast<uint4*>(lo16 + off) = b;
  }
}

// ---------------------------------------------------------------------------------
// plane statistics
// ---------------------------------------------------------------------------------
__device__ __forceinline__ double atomic_add_f64(double* a, double v) { return atomicAdd(a, v); }

// grid (ceil(C/32), slabs, N), block (32, 8).  DET: the slab's partials go to slot blockIdx.y (det_sum_slots)
template <bool DET>
__global__ void plane_stats_kernel(const float* __restrict__ y, int pitch, int hw, int C,
                                   double* __restrict__ stats, double* __restrict__ slots) {
  __shared__ float s1s[8][33], s2s[8][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  const int n = blockIdx.z;
  const int per = (hw + gridDim.y - 1) / gridDim.y;
  const int p0 = blockIdx.y * per;
  const int p1 = min(hw, p0 + per);
  float s1 = 0.f, s2 = 0.f;
  if (c < C) {
    const float* base = y + (long long)n * hw * pitch + c;
    for (int p = p0 + threadIdx.y; p < p1; p += 8) {
      const float v = base[(long long)p * pitch];
      s1 += v;
      s2 += v * v;
    }
  }
  s1s[threadIdx.y][threadIdx.x] = s1;
  s2s[threadIdx.y][threadIdx.x] = s2;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    double a = 0.0, b = 0.0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      a += (double)s1s[j][threadIdx.x];
      b += (double)s2s[j][threadIdx.x];
    }
    const long long i = ((long long)n * C + c) * 2;
    if constexpr (DET) {
      double* sl = slots + (long long)blockIdx.y * (2LL * gridDim.z * C);
      sl[i] = a;
      sl[i + 1] = b;
    } else {
      atomic_add_f64(&stats[i + 0], a);
      atomic_add_f64(&stats[i + 1], b);
    }
  }
}
// (sum, sumsq) -> (mean, rstd), biased variance (torch instance_norm)
__global__ void stats_finalize_kernel(double* stats, int count, int hw, double eps) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < count) {
    const double mean = stats[2 * i] / hw;
    double var = stats[2 * i + 1] / hw - mean * mean;
    if (var < 0) var = 0;
    stats[2 * i] = mean;
    stats[2 * i + 1] = rsqrt(var + eps);
  }
}
// (sum g, sum g*xhat) -> means
__global__ void gstats_finalize_kernel(double* g, int count, int hw) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < count) {
    g[2 * i] /= hw;
    g[2 * i + 1] /= hw;
  }
}

// ---------------------------------------------------------------------------------
// BatchNorm2d (affine, tracked running statistics) on top of the per-(n, c) sums.  The N samples form `groups`
// consecutive groups of N/groups samples, each normalised with its own statistics as if it were a call of its own
// (the discriminator's fake and real halves).  One thread per channel sums the samples in index order: no atomics,
// the same result on every run.
// ---------------------------------------------------------------------------------
// One group's statistics from its element count and sums, shared by the single-process and the cross-rank kernels so
// that the two cannot drift: (mean, 1/sqrt(var_biased + eps)) for the normalisation, and the running-buffer update
__device__ __forceinline__ void bn_group_stat(double s1, double s2, double cnt, double eps, float momentum,
                                              double& mean, double& rstd, float& rm, float& rv) {
  mean = s1 / cnt;
  double var = s2 / cnt - mean * mean;
  if (var < 0) var = 0;
  rstd = rsqrt(var + eps);
  // torch: running <- (1 - momentum) * running + momentum * stat, the variance stat unbiased (n / (n - 1))
  rm = (float)((1.0 - momentum) * rm + momentum * mean);
  rv = (float)((1.0 - momentum) * rv + momentum * (cnt > 1 ? var * cnt / (cnt - 1) : var));
}
// stats[n][c] = (sum y, sum y^2) -> (mean_G, rstd_G) of the sample's group; running buffers updated group by group
__global__ void bn_finalize_kernel(double* stats, int N, int C, int groups, int hw, double eps, float momentum,
                                   float* run_mean, float* run_var, long long* num_batches) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c == 0 && num_batches) *num_batches += groups;
  if (c >= C) return;
  const int per = N / groups;
  const double cnt = (double)per * hw;
  float rm = run_mean ? run_mean[c] : 0.f, rv = run_var ? run_var[c] : 0.f;
  for (int gi = 0; gi < groups; ++gi) {
    double s1 = 0.0, s2 = 0.0;
    for (int n = gi * per; n < (gi + 1) * per; ++n) {
      s1 += stats[((long long)n * C + c) * 2];
      s2 += stats[((long long)n * C + c) * 2 + 1];
    }
    double mean, rstd;
    bn_group_stat(s1, s2, cnt, eps, momentum, mean, rstd, rm, rv);
    for (int n = gi * per; n < (gi + 1) * per; ++n) {
      stats[((long long)n * C + c) * 2] = mean;
      stats[((long long)n * C + c) * 2 + 1] = rstd;
    }
  }
  if (run_mean) run_mean[c] = rm;
  if (run_var) run_var[c] = rv;
}
// Cross-rank batch statistics.  A rank's partials are part[g][c] = (element count, sum, sum of squares) of its samples
// of group g; the ranks' slices are gathered in rank order into [world][groups][C][3] and summed in that order, so
// every rank gets the same bits whatever the transport.  With one rank the sums are those of the kernels above.
// part[g][c] = (per * hw, sum over the group's samples in sample order of stats[n][c]): the forward's (sum y, sum y^2)
// or the backward's (sum g, sum g*xhat)
__global__ void bn_group_sums_kernel(const double* stats, int N, int C, int groups, int hw, double* part) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const int per = N / groups;
  for (int gi = 0; gi < groups; ++gi) {
    double s1 = 0.0, s2 = 0.0;
    for (int n = gi * per; n < (gi + 1) * per; ++n) {
      s1 += stats[((long long)n * C + c) * 2];
      s2 += stats[((long long)n * C + c) * 2 + 1];
    }
    double* p = part + ((long long)gi * C + c) * 3;
    p[0] = (double)per * hw;
    p[1] = s1;
    p[2] = s2;
  }
}
// sum of the gathered slices of group gi, channel c, in rank order
__device__ __forceinline__ void bn_gathered_sums(const double* gathered, int world, int groups, int C, int gi, int c,
                                                 double& cnt, double& s1, double& s2) {
  cnt = 0.0, s1 = 0.0, s2 = 0.0;
  for (int r = 0; r < world; ++r) {
    const double* p = gathered + (((long long)r * groups + gi) * C + c) * 3;
    cnt += p[0];
    s1 += p[1];
    s2 += p[2];
  }
}
// stats[n][c] <- (mean, rstd) of the sample's group over all ranks; running buffers updated group by group from the
// global statistics (the same bits on every rank)
__global__ void bn_finalize_gathered_kernel(double* stats, int N, int C, int groups, const double* gathered, int world,
                                            double eps, float momentum, float* run_mean, float* run_var,
                                            long long* num_batches) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c == 0 && num_batches) *num_batches += groups;
  if (c >= C) return;
  const int per = N / groups;
  float rm = run_mean ? run_mean[c] : 0.f, rv = run_var ? run_var[c] : 0.f;
  for (int gi = 0; gi < groups; ++gi) {
    double cnt, s1, s2, mean, rstd;
    bn_gathered_sums(gathered, world, groups, C, gi, c, cnt, s1, s2);
    bn_group_stat(s1, s2, cnt, eps, momentum, mean, rstd, rm, rv);
    for (int n = gi * per; n < (gi + 1) * per; ++n) {
      stats[((long long)n * C + c) * 2] = mean;
      stats[((long long)n * C + c) * 2 + 1] = rstd;
    }
  }
  if (run_mean) run_mean[c] = rm;
  if (run_var) run_var[c] = rv;
}
// eval mode: stats[n][c] = (running_mean, 1/sqrt(running_var + eps))
__global__ void bn_eval_stats_kernel(double* stats, int N, int C, const float* run_mean, const float* run_var,
                                     double eps) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N * C) {
    const int c = i % C;
    stats[2 * i] = run_mean[c];
    stats[2 * i + 1] = rsqrt((double)run_var[c] + eps);
  }
}
// g[n][c] = (sum g, sum g*xhat) -> the group means the apply pass subtracts (train) or zeros (eval: the statistics are
// constants); d(gamma) += sum g*xhat, d(beta) += sum g over every sample
__global__ void bn_bwd_group_kernel(double* g, int N, int C, int groups, int hw, int train, float* dgamma,
                                    float* dbeta) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const int per = N / groups;
  const double cnt = (double)per * hw;
  double tb = 0.0, tg = 0.0;
  for (int gi = 0; gi < groups; ++gi) {
    double s1 = 0.0, s2 = 0.0;
    for (int n = gi * per; n < (gi + 1) * per; ++n) {
      s1 += g[((long long)n * C + c) * 2];
      s2 += g[((long long)n * C + c) * 2 + 1];
    }
    tb += s1;
    tg += s2;
    for (int n = gi * per; n < (gi + 1) * per; ++n) {
      g[((long long)n * C + c) * 2] = train ? s1 / cnt : 0.0;
      g[((long long)n * C + c) * 2 + 1] = train ? s2 / cnt : 0.0;
    }
  }
  if (dbeta) dbeta[c] += (float)tb;
  if (dgamma) dgamma[c] += (float)tg;
}
// train mode across ranks: g[n][c] <- the global group means of (g, g*xhat) for the apply pass.  d(gamma), d(beta) add
// this rank's sums only (its slice of `gathered`): the gradient all-reduce that follows sums them over the ranks
__global__ void bn_bwd_group_gathered_kernel(double* g, int N, int C, int groups, const double* gathered, int world,
                                             int rank, float* dgamma, float* dbeta) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const int per = N / groups;
  double tb = 0.0, tg = 0.0;
  for (int gi = 0; gi < groups; ++gi) {
    double cnt, s1, s2;
    bn_gathered_sums(gathered, world, groups, C, gi, c, cnt, s1, s2);
    const double* mine = gathered + (((long long)rank * groups + gi) * C + c) * 3;
    tb += mine[1];
    tg += mine[2];
    for (int n = gi * per; n < (gi + 1) * per; ++n) {
      g[((long long)n * C + c) * 2] = s1 / cnt;
      g[((long long)n * C + c) * 2 + 1] = s2 / cnt;
    }
  }
  if (dbeta) dbeta[c] += (float)tb;
  if (dgamma) dgamma[c] += (float)tg;
}


// bias gradient: db[c] = sum over pixels of dy (dy carried as split planes).  V channels per thread (one V-word load
// per plane); block (bx = min(32, pow2 >= G), 256/bx pixel rows) over the G = ceil(C/V) channel groups
template <int V, bool DET>
__global__ void bias_grad_kernel(const uint16_t* __restrict__ hi, const uint16_t* __restrict__ lo, int pitch, int fmt,
                                 long long npix, int C, double* __restrict__ acc, double* __restrict__ slots) {
  __shared__ float red[256][V];
  const int gch = blockIdx.x * blockDim.x + threadIdx.x;   // channel group
  const int c = gch * V;
  const long long per = (npix + gridDim.y - 1) / gridDim.y;
  const long long p0 = blockIdx.y * per;
  const long long p1 = p0 + per < npix ? p0 + per : npix;
  float s[V];
  double d[V];
#pragma unroll
  for (int j = 0; j < V; ++j) {
    s[j] = 0.f;
    d[j] = 0.0;
  }
  if (c < C) {
    int cnt = 0;
    for (long long p = p0 + threadIdx.y; p < p1; p += blockDim.y) {
      uint32_t wh[(V + 1) / 2], wl[(V + 1) / 2];
      load_w16<V>(hi + p * pitch + c, wh);
      if (lo) load_w16<V>(lo + p * pitch + c, wl);
#pragma unroll
      for (int j = 0; j < V; ++j) s[j] += decode16(word16(wh, j), fmt) + (lo ? decode16(word16(wl, j), fmt) : 0.f);
      if (++cnt == 64) {
#pragma unroll
        for (int j = 0; j < V; ++j) { d[j] += (double)s[j]; s[j] = 0.f; }
        cnt = 0;
      }
    }
#pragma unroll
    for (int j = 0; j < V; ++j) d[j] += (double)s[j];
  }
  const int slot = threadIdx.y * blockDim.x + threadIdx.x;
#pragma unroll
  for (int j = 0; j < V; ++j) red[slot][j] = (float)d[j];
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
#pragma unroll
    for (int j = 0; j < V; ++j) {
      if (c + j >= C) break;
      double u = 0.0;
      for (int r = 0; r < (int)blockDim.y; ++r) u += (double)red[r * blockDim.x + threadIdx.x][j];
      if constexpr (DET) slots[(long long)blockIdx.y * C + c + j] = u;
      else atomic_add_f64(&acc[c + j], u);
    }
  }
}
__global__ void bias_grad_finalize_kernel(const double* acc, int C, float* db) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < C) db[i] = (float)acc[i];
}

// ---------------------------------------------------------------------------------
// InstanceNorm-apply + activation + dropout (+ residual) forward and its backward.
// V = 4 channels per thread where C % 4 == 0 and the rows are 16-B (fp32) / 8-B (planes) aligned, else V = 1; the host
// picks the instantiation, the arithmetic per element is the same.  One block = one image n, one slab of pixels and
// one slice of channels; the slice's per-channel statistics sit in shared memory; threads walk the flattened (pixel,
// channel group) index so that a warp touches 128 V contiguous bytes.  The kernels are compiled for 4 resident blocks
// per SM (at most 64 registers): one group in flight per thread, latency hidden by occupancy.
// ---------------------------------------------------------------------------------
struct NormActFwdArgs {
  const float* y; int y_pitch;
  int H, W, C;
  const double* stats;
  int act; float slope;
  uint32_t drop_thresh; float drop_scale; unsigned long long seed;
  unsigned long long drop_off; const float* seed_dev; unsigned int stage_id;
  const float* residual; int res_pitch;
  uint16_t* hi; uint16_t* lo; int out_pitch, out_coff, reflect, fmt;
  uint16_t* hi2; uint16_t* lo2; int fmt2;
  float* f32; int f32_pitch;
  const float* gamma; const float* beta;   // BatchNorm affine (the AFF kernel instantiations): out = gamma*xhat + beta
};

// channels of one block's slice: its shared-memory arrays (2 x S floats forward, 4 x S backward apply, two more with
// the BatchNorm affine) stay within the 48 KB a launch gets without opting in; wider tensors take ceil(C / S) slices
__host__ __device__ constexpr int fwd_slice(bool aff) { return aff ? 3072 : 4096; }
constexpr int kApplySlice = 2048;

__device__ __forceinline__ float act_fwd(float v, int act, float slope) {
  if (act == SN_ACT_LRELU) return v > 0.f ? v : v * slope;
  if (act == SN_ACT_RELU) return v > 0.f ? v : 0.f;
  return v;
}
__device__ __forceinline__ float act_grad(float xhat, int act, float slope) {
  if (act == SN_ACT_LRELU) return xhat > 0.f ? 1.f : slope;
  if (act == SN_ACT_RELU) return xhat > 0.f ? 1.f : 0.f;
  return 1.f;
}

// grid (slabs, N, slices), block 256
template <int V, bool AFF>
__global__ void __launch_bounds__(256, 4) norm_act_fwd_kernel(const NormActFwdArgs a) {
  extern __shared__ float sm[];  // mean[cs], rstd[cs] (+ gamma[cs], beta[cs] when AFF)
  constexpr int S = fwd_slice(AFF);
  const int c0 = blockIdx.z * S, cs = min(S, a.C - c0);
  float* s_mean = sm;
  float* s_rstd = sm + cs;
  float* s_gam = sm + 2 * cs;
  float* s_bet = sm + 3 * cs;
  const unsigned long long seed = a.drop_thresh ? drop_seed_of(a) : 0ull;
  const int n = blockIdx.y;
  for (int c = threadIdx.x; c < cs; c += blockDim.x) {
    s_mean[c] = a.stats ? (float)a.stats[((long long)n * a.C + c0 + c) * 2] : 0.f;
    s_rstd[c] = a.stats ? (float)a.stats[((long long)n * a.C + c0 + c) * 2 + 1] : 1.f;
    if constexpr (AFF) {
      s_gam[c] = a.gamma[c0 + c];
      s_bet[c] = a.beta[c0 + c];
    }
  }
  __syncthreads();
  const int HW = a.H * a.W, Q = cs >> log2_of(V);
  const int per = (HW + gridDim.x - 1) / gridDim.x;
  const int p0 = blockIdx.x * per, p1 = min(HW, p0 + per);
  const int i1 = (p1 - p0) * Q;   // slab-relative 32-bit index
  for (int i = threadIdx.x; i < i1; i += blockDim.x) {
    const int pl = i / Q;
    const int p = p0 + pl;
    const int cl = (i - pl * Q) * V;   // channel within the slice
    const int c = c0 + cl;
    const long long pix = (long long)n * HW + p;
    float v[V];
    load_f32<V>(a.y + pix * a.y_pitch + c, v);
#pragma unroll
    for (int j = 0; j < V; ++j) {
      float t = (v[j] - s_mean[cl + j]) * s_rstd[cl + j];
      if constexpr (AFF) t = t * s_gam[cl + j] + s_bet[cl + j];
      t = act_fwd(t, a.act, a.slope);
      if (a.drop_thresh) {
        const bool keep = sn_keep(seed, a.drop_off + (unsigned long long)pix * a.C + c + j, a.drop_thresh);
        t = keep ? t * a.drop_scale : 0.f;
      }
      v[j] = t;
    }
    if (a.residual) {
      float r[V];
      load_f32<V>(a.residual + pix * a.res_pitch + c, r);
#pragma unroll
      for (int j = 0; j < V; ++j) v[j] += r[j];
    }
    if (a.f32) store_f32<V>(a.f32 + pix * a.f32_pitch + c, v);
    if (a.hi) {
      if (!a.reflect) {
        const long long off = pix * a.out_pitch + a.out_coff + c;
        store_split<V>(a.hi, a.lo, off, v, a.fmt);
        if (a.hi2) store_split<V>(a.hi2, a.lo2, off, v, a.fmt2);
      } else {
        const int hh = p / a.W, ww = p - hh * a.W;
        const int Hp = a.H + 2, Wp = a.W + 2;
        const int nr = reflect_pad1_count(hh, a.H), nc = reflect_pad1_count(ww, a.W);
        for (int ii = 0; ii < nr; ++ii)
          for (int jj = 0; jj < nc; ++jj) {
            const long long off = (((long long)n * Hp + reflect_pad1_position(hh, a.H, ii)) * Wp +
                                   reflect_pad1_position(ww, a.W, jj)) * a.out_pitch + a.out_coff + c;
            store_split<V>(a.hi, a.lo, off, v, a.fmt);
            if (a.hi2) store_split<V>(a.hi2, a.lo2, off, v, a.fmt2);
          }
      }
    }
  }
}

struct GradSrcs {
  sn_grad_src s[SN_MAX_SRC];
  int n;
};
// upstream gradient at (n, h, w, c..c+V): sum of sources; a reflect-padded source folds its
// mirrored border rows/cols back onto the interior pixel (adjoint of ReflectionPad2d(1)).
template <int V>
__device__ __forceinline__ void gather_one(const sn_grad_src& s, int n, int h, int w, int H, int W, int c, float acc[V]) {
#pragma unroll
  for (int j = 0; j < V; ++j) acc[j] = 0.f;
  if (s.up > 1) {
    const int u = s.up;
    for (int a = 0; a < u; ++a)
      for (int b = 0; b < u; ++b)
        add_f32<V>(s.ptr + (((long long)n * H * u + h * u + a) * W * u + w * u + b) * s.pitch + s.c_off + c, acc);
  } else if (!s.reflect_padded) {
    add_f32<V>(s.ptr + (((long long)n * H + h) * W + w) * s.pitch + s.c_off + c, acc);
  } else {
    const int Hp = H + 2, Wp = W + 2;
    const int nr = reflect_pad1_count(h, H), nc = reflect_pad1_count(w, W);
    // kept as loops: the gathers are inlined once per source, and unrolled blocks of up to 3x3 loads raise the
    // register count of ce_tanh_bwd and of the backward kernels
#pragma unroll 1
    for (int a = 0; a < nr; ++a)
#pragma unroll 1
      for (int b = 0; b < nc; ++b)
        add_f32<V>(s.ptr + (((long long)n * Hp + reflect_pad1_position(h, H, a)) * Wp + reflect_pad1_position(w, W, b)) *
                               s.pitch + s.c_off + c, acc);
  }
}
template <int V>
__device__ __forceinline__ void gather_grad(const GradSrcs& g, int n, int h, int w, int H, int W, int c, float acc[V]) {
  float v[V];
#pragma unroll
  for (int j = 0; j < V; ++j) acc[j] = 0.f;
#pragma unroll
  for (int i = 0; i < SN_MAX_SRC; ++i) {
    if (i >= g.n) break;
    gather_one<V>(g.s[i], n, h, w, H, W, c, v);
#pragma unroll
    for (int j = 0; j < V; ++j) acc[j] += v[j];
  }
}

struct NormActBwdArgs {
  GradSrcs g;
  const float* y; int y_pitch;
  int H, W, C;
  const double* stats;
  int act; float slope;
  uint32_t drop_thresh; float drop_scale; unsigned long long seed;
  unsigned long long drop_off; const float* seed_dev; unsigned int stage_id;
  double* gstats;
  uint16_t* hi; uint16_t* lo; int dy_pitch, dy_coff, fmt;
  float* bias_grad;   // optional [C]: += per-channel sums of the dy written (the conv's bias gradient)
  const float* gamma; const float* beta;   // BatchNorm affine (AFF instantiations): the gate is on gamma*xhat + beta
  double* slots;      // DET reduce instantiations: per-slab partials of gstats (det_sum_slots)
};

// g (w.r.t. the normalised value, gamma*xhat + beta when AFF) and xhat for channels c..c+V
template <int V, bool AFF>
__device__ __forceinline__ void grad_xhat(const NormActBwdArgs& a, unsigned long long seed, int n, int p, int c,
                                          const float* mean, const float* rstd, float g[V], float xh[V],
                                          const float* gam, const float* bet) {
  const int HW = a.H * a.W;
  const long long pix = (long long)n * HW + p;
  const int h = p / a.W, w = p - h * a.W;
  float yy[V];
  load_f32<V>(a.y + pix * a.y_pitch + c, yy);
#pragma unroll
  for (int j = 0; j < V; ++j) {
    xh[j] = (yy[j] - mean[j]) * rstd[j];
    g[j] = 0.f;
  }
#pragma unroll
  for (int i = 0; i < SN_MAX_SRC; ++i) {
    if (i >= a.g.n) break;
    const sn_grad_src& s = a.g.s[i];
    float gg[V];
    gather_one<V>(s, n, h, w, a.H, a.W, c, gg);
    const int act = s.act >= 0 ? s.act : a.act;
#pragma unroll
    for (int j = 0; j < V; ++j) {
      if constexpr (AFF) g[j] += gg[j] * act_grad(xh[j] * gam[j] + bet[j], act, a.slope);
      else g[j] += gg[j] * act_grad(xh[j], act, a.slope);
    }
  }
  if (a.drop_thresh) {
#pragma unroll
    for (int j = 0; j < V; ++j) {
      const bool keep = sn_keep(seed, a.drop_off + (unsigned long long)pix * a.C + c + j, a.drop_thresh);
      g[j] = keep ? g[j] * a.drop_scale : 0.f;
    }
  }
}

// grid (ceil(Q/bx), slabs, N), block (bx, 256/bx) with Q = C/V channel groups and bx = min(32, pow2 >= Q): thread =
// channel group, strided over pixels (C = 64 layers, the largest tensors, use bx = 16 and 16 pixel rows at V = 4)
template <int V, bool AFF, bool DET>
__global__ void __launch_bounds__(256, 4) norm_act_bwd_reduce_kernel(const NormActBwdArgs a) {
  __shared__ float red[256][2 * V];
  const unsigned long long seed = a.drop_thresh ? drop_seed_of(a) : 0ull;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  const int c = q * V;
  const int n = blockIdx.z;
  const int HW = a.H * a.W;
  const int per = (HW + gridDim.y - 1) / gridDim.y;
  const int p0 = blockIdx.y * per, p1 = min(HW, p0 + per);
  float s1[V], s2[V];
#pragma unroll
  for (int j = 0; j < V; ++j) s1[j] = 0.f;
#pragma unroll
  for (int j = 0; j < V; ++j) s2[j] = 0.f;
  if (c < a.C) {
    float mean[V], rstd[V], gam[V], bet[V];
#pragma unroll
    for (int j = 0; j < V; ++j) {
      mean[j] = (float)a.stats[((long long)n * a.C + c + j) * 2];
      rstd[j] = (float)a.stats[((long long)n * a.C + c + j) * 2 + 1];
      if constexpr (AFF) {
        gam[j] = a.gamma[c + j];
        bet[j] = a.beta[c + j];
      }
    }
    for (int p = p0 + threadIdx.y; p < p1; p += blockDim.y) {
      float g[V], xh[V];
      grad_xhat<V, AFF>(a, seed, n, p, c, mean, rstd, g, xh, gam, bet);
#pragma unroll
      for (int j = 0; j < V; ++j) {
        s1[j] += g[j];
        s2[j] += g[j] * xh[j];
      }
    }
  }
  const int slot = threadIdx.y * blockDim.x + threadIdx.x;
#pragma unroll
  for (int j = 0; j < V; ++j) {
    red[slot][j] = s1[j];
    red[slot][V + j] = s2[j];
  }
  __syncthreads();
  if (threadIdx.y == 0 && c < a.C) {
#pragma unroll
    for (int j = 0; j < V; ++j) {
      double u = 0.0, v = 0.0;
      for (int r = 0; r < (int)blockDim.y; ++r) {
        u += (double)red[r * blockDim.x + threadIdx.x][j];
        v += (double)red[r * blockDim.x + threadIdx.x][V + j];
      }
      const long long i = ((long long)n * a.C + c + j) * 2;
      if constexpr (DET) {
        double* sl = a.slots + (long long)blockIdx.y * (2LL * gridDim.z * a.C);
        sl[i] = u;
        sl[i + 1] = v;
      } else {
        atomic_add_f64(&a.gstats[i + 0], u);
        atomic_add_f64(&a.gstats[i + 1], v);
      }
    }
  }
}

// grid (slabs, N, slices), block 256
template <int V, bool AFF>
__global__ void __launch_bounds__(256, 4) norm_act_bwd_apply_kernel(const NormActBwdArgs a) {
  extern __shared__ float sm[];  // mean, rstd, m1, m2 : 4 x cs (+ gamma, beta when AFF)
  const int c0 = blockIdx.z * kApplySlice, cs = min(kApplySlice, a.C - c0);
  float* s_mean = sm;
  float* s_rstd = sm + cs;
  float* s_m1 = sm + 2 * cs;
  float* s_m2 = sm + 3 * cs;
  float* s_gam = sm + 4 * cs;
  float* s_bet = sm + 5 * cs;
  const unsigned long long seed = a.drop_thresh ? drop_seed_of(a) : 0ull;
  const int n = blockIdx.y;
  for (int c = threadIdx.x; c < cs; c += blockDim.x) {
    const long long k = ((long long)n * a.C + c0 + c) * 2;
    s_mean[c] = a.stats ? (float)a.stats[k] : 0.f;
    s_rstd[c] = a.stats ? (float)a.stats[k + 1] : 1.f;
    s_m1[c] = a.stats ? (float)a.gstats[k] : 0.f;
    s_m2[c] = a.stats ? (float)a.gstats[k + 1] : 0.f;
    if constexpr (AFF) {
      s_gam[c] = a.gamma[c0 + c];
      s_bet[c] = a.beta[c0 + c];
    }
  }
  __syncthreads();
  const int HW = a.H * a.W, Q = cs / V;   // a division here: the shift costs the AFF instantiation spills
  const int per = (HW + gridDim.x - 1) / gridDim.x;
  const int p0 = blockIdx.x * per, p1 = min(HW, p0 + per);
  const int i1 = (p1 - p0) * Q;   // slab-relative 32-bit index
  float bsum[V];   // fused bias gradient: the thread's channel group is fixed when blockDim % Q == 0
#pragma unroll
  for (int j = 0; j < V; ++j) bsum[j] = 0.f;
  for (int i = threadIdx.x; i < i1; i += blockDim.x) {
    const int pl = i / Q;
    const int p = p0 + pl;
    const int cl = (i - pl * Q) * V;   // channel within the slice
    const int c = c0 + cl;
    float g[V], xh[V];
    grad_xhat<V, AFF>(a, seed, n, p, c, s_mean + cl, s_rstd + cl, g, xh, s_gam + cl, s_bet + cl);
    if constexpr (AFF) {
#pragma unroll
      for (int j = 0; j < V; ++j) g[j] = s_gam[cl + j] * s_rstd[cl + j] * (g[j] - s_m1[cl + j] - xh[j] * s_m2[cl + j]);
    } else if (a.stats) {
      const float *rstd = s_rstd + cl, *m1 = s_m1 + cl, *m2 = s_m2 + cl;
#pragma unroll
      for (int j = 0; j < V; ++j) g[j] = rstd[j] * (g[j] - m1[j] - xh[j] * m2[j]);
    }
    store_split<V>(a.hi, a.lo, ((long long)n * HW + p) * a.dy_pitch + a.dy_coff + c, g, a.fmt);
#pragma unroll
    for (int j = 0; j < V; ++j) bsum[j] += g[j];
  }
  if (a.bias_grad) {   // host guarantees one slice, blockDim.x % Q == 0 and 4*C >= 256*V floats of scratch
    __syncthreads();
    store_f32<V>(sm + threadIdx.x * V, bsum);
    __syncthreads();
    if ((int)threadIdx.x < Q) {
      float t[V], v[V];
#pragma unroll
      for (int j = 0; j < V; ++j) t[j] = 0.f;
      for (int r = threadIdx.x; r < (int)blockDim.x; r += Q) {
        load_f32<V>(sm + r * V, v);
#pragma unroll
        for (int j = 0; j < V; ++j) t[j] += v[j];
      }
#pragma unroll
      for (int j = 0; j < V; ++j) atomicAdd(a.bias_grad + threadIdx.x * V + j, t[j]);
    }
  }
}

// grid (slabs, N), block 256
template <int V>
__global__ void sum_grads_kernel(const GradSrcs g, int H, int W, int C, float* dst, int dst_pitch) {
  const int n = blockIdx.y;
  const int HW = H * W, Q = C >> log2_of(V);
  const int per = (HW + gridDim.x - 1) / gridDim.x;
  const int p0 = blockIdx.x * per, p1 = min(HW, p0 + per);
  const int i1 = (p1 - p0) * Q;   // slab-relative 32-bit index
  for (int i = threadIdx.x; i < i1; i += blockDim.x) {
    const int pl = i / Q;
    const int p = p0 + pl;
    const int c = (i - pl * Q) * V;
    const int h = p / W, w = p - h * W;
    float v[V];
    gather_grad<V>(g, n, h, w, H, W, c, v);
    store_f32<V>(dst + ((long long)n * HW + p) * dst_pitch + c, v);
  }
}

// flat (pixel, channel) index: consecutive threads walk consecutive channels then pixels, so the 19-channel
// head rows (76 B) are read fully coalesced
__global__ void tanh_bwd_kernel(const GradSrcs g, const float* __restrict__ out, int out_pitch, int N, int H,
                                int W, int C, uint16_t* hi, uint16_t* lo, int dy_pitch,
                                int dy_coff, int fmt) {
  const int HW = H * W;
  const long long total = (long long)N * HW * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long pix = i / C;
    const int c = (int)(i - pix * C);
    const int n = (int)(pix / HW);
    const int p = (int)(pix - (long long)n * HW);
    const int h = p / W, w = p - h * W;
    const float o = out[pix * out_pitch + c];
    float v;
    gather_grad<1>(g, n, h, w, H, W, c, &v);
    v *= 1.f - o * o;
    store_split<1>(hi, lo, pix * dy_pitch + dy_coff + c, &v, fmt);
  }
}

// V channels (V 16-bit words) per thread
template <int V>
__global__ void upsample_planes_kernel(const uint16_t* __restrict__ shi, const uint16_t* __restrict__ slo, int spitch,
                                       int H, int W, int CV, int f, uint16_t* __restrict__ dhi,
                                       uint16_t* __restrict__ dlo, int dpitch, long long total) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % CV) * V;
    const long long pix = i / CV;
    const int w = (int)(pix % W), h = (int)((pix / W) % H);
    const long long n = pix / ((long long)W * H);
    const long long sp = (n * (H / f) + h / f) * (W / f) + w / f;
    uint32_t t[(V + 1) / 2];
    load_w16<V>(shi + sp * spitch + c, t);
    store_w16<V>(dhi + pix * dpitch + c, t);
    if (dlo) {
      load_w16<V>(slo + sp * spitch + c, t);
      store_w16<V>(dlo + pix * dpitch + c, t);
    }
  }
}

// ---------------------------------------------------------------------------------
// fused AdamW over flat fp32 buffers (torch.optim.AdamW semantics, optimizers/__init__.py:48-59):
//   p *= 1 - lr*wd;  m += (g - m)(1 - b1);  v = v*b2 + (1 - b2) g*g;
//   p -= (lr / (1 - b1^t)) * m / (sqrt(v) / sqrt(1 - b2^t) + eps)
// ---------------------------------------------------------------------------------
struct AdamHyper { float decay, omb1, b2, omb2, step_size, inv_bc2_sqrt, eps, gscale; };
__global__ void __launch_bounds__(256) adamw_kernel(float* __restrict__ p, const float* __restrict__ g,
                                                    float* __restrict__ m, float* __restrict__ v, long long n,
                                                    const AdamHyper hv, const float* __restrict__ hyper_dev) {
  AdamHyper h = hv;
  if (hyper_dev) {
    h.decay = hyper_dev[0]; h.omb1 = hyper_dev[1]; h.b2 = hyper_dev[2]; h.omb2 = hyper_dev[3];
    h.step_size = hyper_dev[4]; h.inv_bc2_sqrt = hyper_dev[5]; h.eps = hyper_dev[6]; h.gscale = hyper_dev[7];
  }
  const float decay = h.decay, omb1 = h.omb1, b2 = h.b2, omb2 = h.omb2, step_size = h.step_size,
              inv_bc2_sqrt = h.inv_bc2_sqrt, eps = h.eps, gscale = h.gscale;
  const long long n4 = n >> 2;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    float4 P = reinterpret_cast<float4*>(p)[i];
    float4 G = reinterpret_cast<const float4*>(g)[i];
    float4 M = reinterpret_cast<float4*>(m)[i];
    float4 V = reinterpret_cast<float4*>(v)[i];
    float* pp = &P.x; float* gg = &G.x; float* mm = &M.x; float* vv = &V.x;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      gg[j] *= gscale;                 // exact for the power-of-two 1/world of 2, 4, 8 ranks
      pp[j] *= decay;
      mm[j] = mm[j] + (gg[j] - mm[j]) * omb1;
      vv[j] = vv[j] * b2 + omb2 * gg[j] * gg[j];
      pp[j] -= step_size * (mm[j] / (sqrtf(vv[j]) * inv_bc2_sqrt + eps));
    }
    reinterpret_cast<float4*>(p)[i] = P;
    reinterpret_cast<float4*>(m)[i] = M;
    reinterpret_cast<float4*>(v)[i] = V;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {   // tail
    const long long i = (n4 << 2) + threadIdx.x;
    float P = p[i] * decay;
    const float G = g[i] * gscale;
    const float M = m[i] + (G - m[i]) * omb1;
    const float V = v[i] * b2 + omb2 * G * G;
    P -= step_size * (M / (sqrtf(V) * inv_bc2_sqrt + eps));
    p[i] = P; m[i] = M; v[i] = V;
  }
}

// ---------------------------------------------------------------------------------
// fused AdaBound over flat fp32 buffers (Luo et al., ICLR 2019; the rule of adabound.AdaBound.step as
// optimizers/__init__.py:55-59 builds it, amsbound off), with g' = gscale * g:
//   g' += wd * p  (L2 decay, part of the gradient; skipped when wd == 0)
//   m += (g' - m)(1 - b1);  v += (g'*g' - v)(1 - b2)
//   p -= clamp(step_size / (sqrt(v) + eps), lower, upper) * m
// 1 - b1 and 1 - b2 are passed as rounded on the host: 1.f - (float)0.999 is 1.3e-5 away from 0.001.
// ---------------------------------------------------------------------------------
struct AdaBoundHyper { float omb1, omb2, eps, wd, step_size, lower, upper, gscale; };
__device__ __forceinline__ void adabound_update(float& p, float g, float& m, float& v, const AdaBoundHyper& h) {
  g *= h.gscale;                     // exact for the power-of-two 1/world of 2, 4, 8 ranks
  if (h.wd != 0.f) g += h.wd * p;    // after the scaling: 2 ranks of B/2 then decay like 1 rank of B
  m = m + (g - m) * h.omb1;
  v = v + (g * g - v) * h.omb2;
  const float eta = fminf(fmaxf(h.step_size / (sqrtf(v) + h.eps), h.lower), h.upper);
  p -= eta * m;
}
__global__ void __launch_bounds__(256) adabound_kernel(float* __restrict__ p, const float* __restrict__ g,
                                                       float* __restrict__ m, float* __restrict__ v, long long n,
                                                       const AdaBoundHyper hv, const float* __restrict__ hyper_dev) {
  AdaBoundHyper h = hv;
  if (hyper_dev) {
    h.omb1 = hyper_dev[0]; h.omb2 = hyper_dev[1]; h.eps = hyper_dev[2]; h.wd = hyper_dev[3];
    h.step_size = hyper_dev[4]; h.lower = hyper_dev[5]; h.upper = hyper_dev[6]; h.gscale = hyper_dev[7];
  }
  const long long n4 = n >> 2;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    float4 P = reinterpret_cast<float4*>(p)[i];
    const float4 G = reinterpret_cast<const float4*>(g)[i];
    float4 M = reinterpret_cast<float4*>(m)[i];
    float4 V = reinterpret_cast<float4*>(v)[i];
    adabound_update(P.x, G.x, M.x, V.x, h);
    adabound_update(P.y, G.y, M.y, V.y, h);
    adabound_update(P.z, G.z, M.z, V.z, h);
    adabound_update(P.w, G.w, M.w, V.w, h);
    reinterpret_cast<float4*>(p)[i] = P;
    reinterpret_cast<float4*>(m)[i] = M;
    reinterpret_cast<float4*>(v)[i] = V;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {   // tail
    const long long i = (n4 << 2) + threadIdx.x;
    float P = p[i], M = m[i], V = v[i];
    adabound_update(P, g[i], M, V, h);
    p[i] = P; m[i] = M; v[i] = V;
  }
}

__global__ void dropout_mask_kernel(unsigned long long seed, uint32_t thresh, long long count,
                                    uint8_t* out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < count;
       i += (long long)gridDim.x * blockDim.x)
    out[i] = sn_keep(seed, (unsigned long long)i, thresh) ? 1 : 0;
}

// ---------------------------------------------------------------------------------
// losses
// ---------------------------------------------------------------------------------
// DET: the block's sum goes to slots[blockIdx.x * gridDim.y + blockIdx.y] (det_sum_slots over gridDim.x slots)
template <bool DET>
__device__ __forceinline__ void block_add_double(double v, double* dst, double* slots) {
  __shared__ double red[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (lane == 0) red[warp] = v;
  __syncthreads();
  if (warp == 0) {
    v = lane < (blockDim.x >> 5) ? red[lane] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) {
      if constexpr (DET) slots[(long long)blockIdx.x * gridDim.y + blockIdx.y] = v;
      else atomicAdd(dst, v);
    }
  }
}

constexpr int kMaxCE = 32;
__global__ void ce_loss_kernel(const float* __restrict__ logits, int pitch,
                               const float* __restrict__ target, const uint8_t* __restrict__ label, int N, int H, int W,
                               int C, float weight, double* loss_acc, float* __restrict__ grad, int gpitch) {
  const long long npix = (long long)N * H * W;
  const long long HW = (long long)H * W;
  double local = 0.0;
  const float scale = weight / (float)npix;
  for (long long pix = blockIdx.x * (long long)blockDim.x + threadIdx.x; pix < npix;
       pix += (long long)gridDim.x * blockDim.x) {
    const long long n = pix / HW, p = pix - n * HW;
    float x[kMaxCE];
    int arg = 0;
    float best = 0.f, mx = -INFINITY;
    for (int c = 0; c < C; ++c) {
      x[c] = logits[pix * pitch + c];
      mx = fmaxf(mx, x[c]);
      if (label) continue;
      const float t = target[(n * C + c) * HW + p];
      if (c == 0 || t > best) {  // first maximum wins (torch.argmax tie-break)
        best = t;
        arg = c;
      }
    }
    if (label) {   // argmax of the one-hot expansion of a label map: the label (0 = all-zero vector -> index 0)
      arg = label[pix];
      if (arg >= C) arg = 0;
    }
    float se = 0.f;
    for (int c = 0; c < C; ++c) se += expf(x[c] - mx);
    const float lse = mx + logf(se);
    local += (double)(lse - x[arg]);
    const float inv = 1.f / se;
    for (int c = 0; c < C; ++c) {
      float sm = expf(x[c] - mx) * inv;
      grad[pix * gpitch + c] = scale * (sm - (c == arg ? 1.f : 0.f));
    }
  }
  block_add_double<false>(local * (double)weight / (double)npix, loss_acc, nullptr);
}

// CE on the tanh head fused with the head's own backward (warp_model.py:147-150 + swapnet_modules.py:85-90): per pixel
//   g_c  = weight/npix * (softmax(o)_c - [c == argmax target])  +  sum of the extra gradient sources (the GAN term),
//   dy_c = g_c * (1 - o_c^2)          written as split planes (channels c..pad8 zero-filled, 16-byte stores)
// replaces ce_loss + tanh_bwd: the 19-channel logits are read once and the fp32 CE gradient never touches HBM.
template <bool DET>
__global__ void __launch_bounds__(128) ce_tanh_bwd_kernel(const float* __restrict__ logits, int pitch,
                                                          const float* __restrict__ target,
                                                          const uint8_t* __restrict__ label, const GradSrcs g, int N,
                                                          int H, int W, int C, float weight, double* loss_acc,
                                                          uint16_t* __restrict__ hi, uint16_t* __restrict__ lo,
                                                          int dy_pitch, int dy_coff, int fmt, double* slots) {
  const long long npix = (long long)N * H * W;
  const long long HW = (long long)H * W;
  double local = 0.0;
  const float scale = weight / (float)npix;
  const int C8 = (C + 7) & ~7;
  for (long long pix = blockIdx.x * (long long)blockDim.x + threadIdx.x; pix < npix;
       pix += (long long)gridDim.x * blockDim.x) {
    const long long n = pix / HW, p = pix - n * HW;
    const int h = (int)(p / W), w = (int)(p - (long long)h * W);
    float x[kMaxCE];
    int arg = 0;
    float best = 0.f, mx = -INFINITY;
    for (int c = 0; c < C; ++c) {
      x[c] = logits[pix * pitch + c];
      mx = fmaxf(mx, x[c]);
      if (label) continue;
      const float t = target[(n * C + c) * HW + p];
      if (c == 0 || t > best) {  // first maximum wins (torch.argmax tie-break)
        best = t;
        arg = c;
      }
    }
    if (label) {
      arg = label[pix];
      if (arg >= C) arg = 0;
    }
    float se = 0.f;
    for (int c = 0; c < C; ++c) se += expf(x[c] - mx);
    const float lse = mx + logf(se);
    local += (double)(lse - x[arg]);
    const float inv = 1.f / se;
    for (int c0 = 0; c0 < C8; c0 += 8) {
      uint16_t hh[8], ll[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = c0 + j;
        float v = 0.f;
        if (c < C) {
          float gsum = scale * (expf(x[c] - mx) * inv - (c == arg ? 1.f : 0.f));
          float ge;
          gather_grad<1>(g, (int)n, h, w, H, W, c, &ge);
          gsum += ge;
          v = gsum * (1.f - x[c] * x[c]);
        }
        split16(v, fmt, hh[j], ll[j]);
      }
      const long long off = pix * dy_pitch + dy_coff + c0;
      uint4 a, b;
      a.x = hh[0] | ((uint32_t)hh[1] << 16); a.y = hh[2] | ((uint32_t)hh[3] << 16);
      a.z = hh[4] | ((uint32_t)hh[5] << 16); a.w = hh[6] | ((uint32_t)hh[7] << 16);
      b.x = ll[0] | ((uint32_t)ll[1] << 16); b.y = ll[2] | ((uint32_t)ll[3] << 16);
      b.z = ll[4] | ((uint32_t)ll[5] << 16); b.w = ll[6] | ((uint32_t)ll[7] << 16);
      *reinterpret_cast<uint4*>(hi + off) = a;
      if (lo) *reinterpret_cast<uint4*>(lo + off) = b;
    }
  }
  block_add_double<DET>(local * (double)weight / (double)npix, loss_acc, slots);
}

// GANLoss (loss.py:110-130) over `halves` consecutive blocks of `count` predictions, one per blockIdx.y, each with its own
// scalar t (t_dev[half] when t_dev is set, else t0 / t1): loss_acc[half] += the objective's batch mean, and
// dpred = gscale * d(mean)/dx in the same pass.
//   SN_GAN_BCE   BCEWithLogitsLoss(x, t)      dL/dx = (sigmoid(x) - t) / count
//   SN_GAN_MSE   MSELoss(x, t)                dL/dx = 2 (x - t) / count
//   SN_GAN_WGAN  t * mean(x), t = +1 / -1     dL/dx = t / count            (t is a sign, not a label)
template <int OBJ, bool DET>
__global__ void gan_loss_kernel(const float* __restrict__ pred, long long count, int halves, float t0, float t1,
                                const float* __restrict__ t_dev, float gscale, double* loss_acc,
                                float* __restrict__ dpred, double* slots) {
  const int half = blockIdx.y;
  const float t = t_dev ? t_dev[half] : (half == 0 ? t0 : t1);
  double local = 0.0;
  const float gs = gscale / (float)count;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < count;
       i += (long long)gridDim.x * blockDim.x) {
    const float x = pred[half * count + i];
    if constexpr (OBJ == SN_GAN_BCE) {
      // max(x,0) - x*t + log1p(exp(-|x|))   (ATen binary_cross_entropy_with_logits)
      const float l = (1.f - t) * x + (fmaxf(-x, 0.f) + log1pf(expf(-fabsf(x))));
      local += (double)l;
      const float sg = 1.f / (1.f + expf(-x));
      if (dpred) dpred[half * count + i] = gs * (sg - t);
    } else if constexpr (OBJ == SN_GAN_MSE) {
      const float d = x - t;
      local += (double)(d * d);
      if (dpred) dpred[half * count + i] = gs * (2.f * d);
    } else {
      local += (double)x;
      if (dpred) dpred[half * count + i] = gs * t;
    }
  }
  (void)halves;
  if constexpr (OBJ == SN_GAN_WGAN) local *= (double)t;
  block_add_double<DET>(local / (double)count, loss_acc + half, slots);
}

template <bool DET>
__global__ void l1_loss_kernel(const float* __restrict__ a, int pitch, const float* __restrict__ b,
                               int N, int H, int W, int C, float weight, double* loss_acc,
                               float* __restrict__ grad, int gpitch, double* slots) {
  const long long HW = (long long)H * W;
  const long long total = (long long)N * HW * C;
  double local = 0.0;
  const float gs = weight / (float)total;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long pix = i / C;
    const int c = (int)(i - pix * C);
    const long long n = pix / HW, p = pix - n * HW;
    const float d = a[pix * pitch + c] - b[(n * C + c) * HW + p];
    local += (double)fabsf(d);
    grad[pix * gpitch + c] = d > 0.f ? gs : (d < 0.f ? -gs : 0.f);
  }
  block_add_double<DET>(local * (double)weight / (double)total, loss_acc, slots);
}

// ---------------------------------------------------------------------------------
// SIMT fp32 tap GEMM (test cross-check only)
// ---------------------------------------------------------------------------------
struct SimtArgs {
  const uint16_t *a_hi, *a_lo, *b_hi, *b_lo;
  int a_fmt, b_fmt;
  const float* b_scale;
  int a_n, a_h, a_w, a_c, a_pitch, parity;
  long long b_k;
  int b_rows;
  int m_n, m_h, m_w, ntaps, k_per_tap;
  sn_tap taps[SN_MAX_TAPS];
  float* out;
  long long out_sn, out_sh, out_sw;
  int omh, ooh, omw, oow, n_valid;
  const float* bias;
  int act, nsplit;
};
__global__ void tap_gemm_simt_kernel(const SimtArgs a) {
  const long long rows = (long long)a.m_n * a.m_h * a.m_w;
  const long long total = rows * a.n_valid;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int col = (int)(i % a.n_valid);
    const long long row = i / a.n_valid;
    const int w = (int)(row % a.m_w), h = (int)((row / a.m_w) % a.m_h), n = (int)(row / ((long long)a.m_w * a.m_h));
    float acc = 0.f;
    for (int t = 0; t < a.ntaps; ++t) {
      const sn_tap tp = a.taps[t];
      int sh, sw, cbase;
      bool inb;
      if (!a.parity) {
        sh = h + tp.dh; sw = w + tp.dw; cbase = tp.c_off;
        inb = sh >= 0 && sh < a.a_h && sw >= 0 && sw < a.a_w;
      } else {
        const int h2 = h + tp.dh, w2 = w + tp.dw;
        const int pw = tp.c_off / a.a_pitch;
        cbase = tp.c_off - pw * a.a_pitch;
        inb = h2 >= 0 && h2 < a.a_h / 2 && w2 >= 0 && w2 < a.a_w / 2;
        sh = 2 * h2 + tp.hp; sw = 2 * w2 + pw;
      }
      if (!inb) continue;
      const long long abase = (((long long)n * a.a_h + sh) * a.a_w + sw) * a.a_pitch + cbase;
      const long long bbase = (long long)col * a.b_k + tp.kb_off;
      for (int k = 0; k < a.k_per_tap; ++k) {
        float av = decode16(a.a_hi[abase + k], a.a_fmt);
        float bv = col < a.b_rows ? decode16(a.b_hi[bbase + k], a.b_fmt) : 0.f;
        if (a.nsplit == 3) {
          av += decode16(a.a_lo[abase + k], a.a_fmt);
          if (col < a.b_rows) bv += decode16(a.b_lo[bbase + k], a.b_fmt);
        }
        acc = fmaf(av, bv, acc);
      }
    }
    if (a.b_scale) acc *= a.b_scale[1];
    if (a.bias) acc += a.bias[col];
    if (a.act == SN_ACT_TANH) acc = tanhf(acc);
    a.out[(long long)n * a.out_sn + (long long)(h * a.omh + a.ooh) * a.out_sh +
          (long long)(w * a.omw + a.oow) * a.out_sw + col] = acc;
  }
}


inline bool al16(const void* p) { return ((uintptr_t)p & 15) == 0; }
inline bool srcs_vec_ok(const GradSrcs& g) {
  for (int i = 0; i < g.n; ++i)
    if (!al16(g.s[i].ptr) || (g.s[i].pitch & 3) || (g.s[i].c_off & 3)) return false;
  return true;
}
inline int vslabs(int hw, int n) {  // ~6 waves of 256-thread blocks, at least 32 pixels per block
  int want = (SN_NUM_SMS * 6 + n - 1) / n;
  int maxs = (hw + 31) / 32;
  if (want > maxs) want = maxs;
  return want < 1 ? 1 : want;
}

inline int grid_for(long long total, int threads = kEwThreads) {
  long long g = (total + threads - 1) / threads;
  if (g > SN_NUM_SMS * 16) g = SN_NUM_SMS * 16;
  if (g < 1) g = 1;
  return (int)g;
}

}  // namespace

#define LAUNCH_CHECK()                         \
  do {                                         \
    sn_count_launch(1);                        \
    SN_CHECK_CUDA(cudaGetLastError());         \
  } while (0)

// Launchers of the V-templated kernels.  Each entry point computes its vector predicate once and launches the V = 4
// (bias gradient: 8) or the V = 1 instantiation; both take the same geometry formulas over the C / V channel groups.
template <int V>
static int launch_norm_act_fwd(const NormActFwdArgs& a, int n, cudaStream_t st) {
  const bool aff = a.gamma != nullptr;
  const int S = fwd_slice(aff), cs = a.C < S ? a.C : S;
  const dim3 grid(vslabs(a.H * a.W, n), n, (a.C + S - 1) / S);
  if (aff) norm_act_fwd_kernel<V, true><<<grid, 256, 4 * cs * sizeof(float), st>>>(a);
  else norm_act_fwd_kernel<V, false><<<grid, 256, 2 * cs * sizeof(float), st>>>(a);
  LAUNCH_CHECK();
  return SN_OK;
}

// ~6 waves of blocks, at least 128 pixels per slab; *nslabs: the slabs (slots per output in deterministic mode)
template <int V>
static int launch_norm_act_bwd_reduce(const NormActBwdArgs& a, int n, long long slots_cap, cudaStream_t st,
                                      int* nslabs) {
  const int q = a.C / V, hw = a.H * a.W;
  int bx = 1;
  while (bx < q && bx < 32) bx <<= 1;
  const int qg = (q + bx - 1) / bx;
  int slabs = (SN_NUM_SMS * 6 + n * qg - 1) / (n * qg);
  if (slabs > (hw + 127) / 128) slabs = (hw + 127) / 128;
  if (slabs < 1) slabs = 1;
  *nslabs = slabs;
  const dim3 grid(qg, slabs, n), blk(bx, 256 / bx);
  const bool aff = a.gamma != nullptr, det = a.slots != nullptr;
  if (det) SN_REQUIRE((long long)slabs * 2 * n * a.C <= slots_cap, "norm_act_bwd: det_slots too small");
  if (aff && det) norm_act_bwd_reduce_kernel<V, true, true><<<grid, blk, 0, st>>>(a);
  else if (aff) norm_act_bwd_reduce_kernel<V, true, false><<<grid, blk, 0, st>>>(a);
  else if (det) norm_act_bwd_reduce_kernel<V, false, true><<<grid, blk, 0, st>>>(a);
  else norm_act_bwd_reduce_kernel<V, false, false><<<grid, blk, 0, st>>>(a);
  LAUNCH_CHECK();
  return SN_OK;
}

template <int V>
static int launch_norm_act_bwd_apply(const NormActBwdArgs& a, int n, cudaStream_t st) {
  // the fused bias gradient needs a fixed channel group per thread (256 % (c/V) == 0) and 256 V floats of scratch
  // (4 c >= 256 V), hence one slice
  SN_REQUIRE(!a.bias_grad || (256 % (a.C / V) == 0 && 4 * a.C >= 256 * V),
             "norm_act_bwd: fused bias gradient needs c in {%d, %d, %d} (c=%d)", 64 * V, 128 * V, 256 * V, a.C);
  const int cs = a.C < kApplySlice ? a.C : kApplySlice;
  const dim3 grid(vslabs(a.H * a.W, n), n, (a.C + kApplySlice - 1) / kApplySlice);
  if (a.gamma) norm_act_bwd_apply_kernel<V, true><<<grid, 256, 6 * cs * sizeof(float), st>>>(a);
  else norm_act_bwd_apply_kernel<V, false><<<grid, 256, 4 * cs * sizeof(float), st>>>(a);
  LAUNCH_CHECK();
  return SN_OK;
}

// block (bx, 256/bx) with bx = min(32, pow2 >= ceil(c/V)); ~6 waves of pixel slabs, at least 256 pixels each
template <int V>
static int launch_bias_grad(const uint16_t* hi, const uint16_t* lo, int pitch, int fmt, long long npix, int c,
                            double* scratch, double* slots, long long slots_cap, cudaStream_t st, int* nslabs) {
  const int groups = (c + V - 1) / V;
  int bx = 1;
  while (bx < groups && bx < 32) bx <<= 1;
  const int gx = (groups + bx - 1) / bx;
  long long sl = (SN_NUM_SMS * 6 + gx - 1) / gx;
  if (sl > (npix + 255) / 256) sl = (npix + 255) / 256;
  if (sl < 1) sl = 1;
  *nslabs = (int)sl;
  SN_REQUIRE(!slots || sl * c <= slots_cap, "bias_grad_det: %lld slots needed, %lld given", sl * c, slots_cap);
  const dim3 grid(gx, (int)sl), blk(bx, 256 / bx);
  if (slots) bias_grad_kernel<V, true><<<grid, blk, 0, st>>>(hi, lo, pitch, fmt, npix, c, scratch, slots);
  else bias_grad_kernel<V, false><<<grid, blk, 0, st>>>(hi, lo, pitch, fmt, npix, c, scratch, nullptr);
  LAUNCH_CHECK();
  return SN_OK;
}

extern "C" {

int sn_pack_planes(const float* src, int src_layout, int src_pitch, int n, int c, int h, int w,
                   void* dst_hi, void* dst_lo, int dst_pitch, int dst_coff, int fmt, void* stream) {
  SN_REQUIRE(src && dst_hi, "null pointer");
  SN_REQUIRE(dst_coff + c <= dst_pitch, "channel slice exceeds pitch");
  cudaStream_t st = (cudaStream_t)stream;
  if (src_layout != SN_LAYOUT_NHWC) {
    SN_REQUIRE(src_layout != SN_LAYOUT_MASK_I32 || c <= 32, "pack_planes: a bit mask holds at most 32 channels");
    SN_REQUIRE(src_layout != SN_LAYOUT_LABEL_U8 || c <= 256, "pack_planes: a uint8 label map holds at most 256 classes");
    dim3 grid((w + 31) / 32, h, n);
    size_t smem = (size_t)c * 33 * sizeof(float);
    SN_REQUIRE(smem <= 48 * 1024, "pack_planes: too many channels for NCHW path (%d)", c);
    pack_planes_nchw_kernel<<<grid, 256, smem, st>>>(src, src_layout, n, c, h, w, (uint16_t*)dst_hi,
                                                     (uint16_t*)dst_lo, dst_pitch, dst_coff, fmt);
  } else {
    const long long npix = (long long)n * h * w;
    pack_planes_nhwc_kernel<<<grid_for(npix * c), kEwThreads, 0, st>>>(
        src, src_pitch, npix, c, (uint16_t*)dst_hi, (uint16_t*)dst_lo, dst_pitch, dst_coff, fmt);
  }
  LAUNCH_CHECK();
  return SN_OK;
}

int sn_pack_concat(int lead, const float* src0, int layout0, int pitch0, int c0, const float* src1, int layout1,
                   int pitch1, int c1, int n, int h, int w, int c_fill, void* dst_hi, void* dst_lo, void* dst2_hi,
                   void* dst2_lo, int dst_pitch, int dst_coff, int fmt, int fmt2, void* stream) {
  SN_REQUIRE(src0 && dst_hi, "null pointer");
  SN_REQUIRE(lead >= 0, "pack_concat: negative zero lead (%d)", lead);
  SN_REQUIRE(c_fill % 8 == 0 && dst_coff % 8 == 0 && dst_pitch % 8 == 0 && lead + c0 + (src1 ? c1 : 0) <= c_fill &&
                 dst_coff + c_fill <= dst_pitch,
             "pack_concat: channel slice must be 8-aligned and fit (coff=%d fill=%d pitch=%d)", dst_coff, c_fill,
             dst_pitch);
  SN_REQUIRE((((uintptr_t)dst_hi | (uintptr_t)dst_lo | (uintptr_t)dst2_hi | (uintptr_t)dst2_lo) & 15) == 0,
             "pack_concat: planes must be 16-byte aligned");
  PackConcatArgs a;
  a.s[0] = PackSrc{src0, layout0, pitch0, c0};
  a.s[1] = PackSrc{src1, layout1, pitch1, src1 ? c1 : 0};
  a.nsrc = src1 ? 2 : 1;
  a.lead = lead;
  a.N = n; a.H = h; a.W = w; a.c_fill = c_fill;
  a.hi = (uint16_t*)dst_hi; a.lo = (uint16_t*)dst_lo; a.hi2 = (uint16_t*)dst2_hi; a.lo2 = (uint16_t*)dst2_lo;
  a.pitch = dst_pitch; a.coff = dst_coff; a.fmt = fmt; a.fmt2 = fmt2;
  if (c_fill == 16 || c_fill == 32) {   // narrow outputs: thread-per-pixel, no shared memory
    const long long npix = (long long)n * h * w;
    const int blocks = grid_for(npix);
    if (c_fill == 16) pack_concat_direct_kernel<16><<<blocks, 256, 0, (cudaStream_t)stream>>>(a);
    else pack_concat_direct_kernel<32><<<blocks, 256, 0, (cudaStream_t)stream>>>(a);
    LAUNCH_CHECK();
    return SN_OK;
  }
  const int pw = 32 * (64 / (c_fill < 64 ? c_fill : 64));
  const size_t smem = (size_t)c_fill * (pw + 1) * sizeof(float);
  SN_REQUIRE(smem <= 48 * 1024, "pack_concat: c_fill too large (%d)", c_fill);
  pack_concat_kernel<<<dim3((w + pw - 1) / pw, h, n), 256, smem, (cudaStream_t)stream>>>(a);
  LAUNCH_CHECK();
  return SN_OK;
}

int sn_pack_head_weights(const float* src, int cout, int cin, int rows_pad, int k_pad, int dgrad, int taps_pitch,
                         void* dst_hi, void* dst_lo, int fmt, const float* scale2, void* stream) {
  SN_REQUIRE(src && dst_hi, "null pointer");
  SN_REQUIRE(taps_pitch >= 25, "head pack: taps_pitch must be >= 25");
  SN_REQUIRE(dgrad ? (k_pad >= cout) : (k_pad >= cin && rows_pad >= cout), "bad head pack shape");
  pack_head_weights_kernel<<<grid_for((long long)cout * 25 * cin), kEwThreads, 0, (cudaStream_t)stream>>>(
      src, cout, cin, rows_pad, k_pad, dgrad, taps_pitch, (uint16_t*)dst_hi, (uint16_t*)dst_lo, fmt, scale2);
  LAUNCH_CHECK();
  return SN_OK;
}

int sn_pack_head_stacked(const float* src, int cout, int cin, int slot, int k_pad, void* dst_hi, void* dst_lo, int fmt,
                         const float* scale2, void* stream) {
  SN_REQUIRE(src && dst_hi && slot >= cout && k_pad >= cin, "bad stacked head pack shape");
  pack_head_stacked_kernel<<<grid_for((long long)4 * slot * 9 * k_pad), kEwThreads, 0, (cudaStream_t)stream>>>(
      src, cout, cin, slot, k_pad, (uint16_t*)dst_hi, (uint16_t*)dst_lo, fmt, scale2);
  LAUNCH_CHECK();
  return SN_OK;
}

int sn_weight_scale_multi(const sn_scale_item* items_dev, int nitems, unsigned int* scratch_dev, void* stream) {
  SN_REQUIRE(items_dev && scratch_dev && nitems >= 1, "weight_scale_multi: bad arguments");
  weight_scale_multi_kernel<<<dim3(32, nitems), 256, 0, (cudaStream_t)stream>>>(items_dev, scratch_dev);
  LAUNCH_CHECK();
  return SN_OK;
}

int sn_pack_weights_multi(const sn_pack_item* items_dev, int nitems, int total_blocks, int max_taps, void* stream) {
  SN_REQUIRE(items_dev && nitems >= 1 && total_blocks >= 1 && max_taps >= 1 && max_taps <= 16,
             "pack_weights_multi: bad arguments (k_pad of every item must be a multiple of 8, planes 16-byte aligned)");
  const size_t smem = (size_t)kPkRows * kPkK * (max_taps + 1) * sizeof(float);
  static bool attr = false;
  if (!attr) {
    SN_CHECK_CUDA(cudaFuncSetAttribute(pack_weights_multi_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    attr = true;
  }
  SN_REQUIRE(smem <= 64 * 1024, "pack_weights_multi: tile too large");
  pack_weights_multi_kernel<<<total_blocks, 256, smem, (cudaStream_t)stream>>>(items_dev, nitems);
  LAUNCH_CHECK();
  return SN_OK;
}
int sn_pack_rows_per_block(void) { return kPkRows; }
int sn_pack_k_per_block(void) { return kPkK; }

int sn_fold_head_wgrad(const float* geff, int cout, int cin, float* dw, void* stream) {
  fold_head_wgrad_kernel<<<grid_for((long long)cout * cin * 16), kEwThreads, 0, (cudaStream_t)stream>>>(
      geff, cout, cin, dw);
  LAUNCH_CHECK();
  return SN_OK;
}

int sn_plane_stats(const float* y, int pitch, int n, int hw, int c, float eps, double* stats,
                   void* stream) {
  const int rc = sn_plane_sums(y, pitch, n, hw, c, stats, stream);
  if (rc) return rc;
  return sn_stats_finalize(stats, n * c, hw, eps, stream);
}

int sn_plane_stats_det(const float* y, int pitch, int n, int hw, int c, float eps, double* stats, double* slots,
                       long long slots_cap, void* stream) {
  const int rc = sn_plane_sums_det(y, pitch, n, hw, c, stats, slots, slots_cap, stream);
  if (rc) return rc;
  return sn_stats_finalize(stats, n * c, hw, eps, stream);
}

static int plane_sums_impl(const float* y, int pitch, int n, int hw, int c, double* stats, double* slots,
                           long long slots_cap, cudaStream_t st) {
  SN_REQUIRE(y && stats, "null pointer");
  SN_CHECK_CUDA(cudaMemsetAsync(stats, 0, sizeof(double) * 2 * n * c, st));
  const int cg = (c + 31) / 32;
  int slabs = (SN_NUM_SMS * 4 + n * cg - 1) / (n * cg);
  if (slabs > (hw + 63) / 64) slabs = (hw + 63) / 64;
  if (slabs < 1) slabs = 1;
  if (!slots) {
    plane_stats_kernel<false><<<dim3(cg, slabs, n), dim3(32, 8), 0, st>>>(y, pitch, hw, c, stats, nullptr);
    LAUNCH_CHECK();
    return SN_OK;
  }
  SN_REQUIRE((long long)slabs * 2 * n * c <= slots_cap, "plane_sums_det: %lld slots needed, %lld given",
             (long long)slabs * 2 * n * c, slots_cap);
  plane_stats_kernel<true><<<dim3(cg, slabs, n), dim3(32, 8), 0, st>>>(y, pitch, hw, c, stats, slots);
  LAUNCH_CHECK();
  SN_CHECK_CUDA(det_sum_slots(slots, slabs, 2LL * n * c, stats, st));
  LAUNCH_CHECK();
  return SN_OK;
}

int sn_plane_sums(const float* y, int pitch, int n, int hw, int c, double* stats, void* stream) {
  return plane_sums_impl(y, pitch, n, hw, c, stats, nullptr, 0, (cudaStream_t)stream);
}

int sn_plane_sums_det(const float* y, int pitch, int n, int hw, int c, double* stats, double* slots,
                      long long slots_cap, void* stream) {
  SN_REQUIRE(slots, "plane_sums_det: null slots");
  return plane_sums_impl(y, pitch, n, hw, c, stats, slots, slots_cap, (cudaStream_t)stream);
}

long long sn_det_slots(int n, int c) {
  // every *_det reduction but the weight gradients' runs slabs * g <= 6 * SN_NUM_SMS + g blocks per sample, where one
  // block covers at most 256 channels of the output
  return 2LL * 6 * SN_NUM_SMS * 256 + 2LL * n * c + 2LL * SN_NUM_SMS * 16;
}

int sn_bn_finalize(double* stats, int n, int c, int groups, int hw, float eps, float momentum, float* running_mean,
                   float* running_var, long long* num_batches_tracked, void* stream) {
  SN_REQUIRE(stats && n >= 1 && c >= 1 && hw >= 1, "bn_finalize: bad arguments");
  SN_REQUIRE(groups >= 1 && n % groups == 0, "bn_finalize: %d samples do not split into %d groups", n, groups);
  SN_REQUIRE((running_mean == nullptr) == (running_var == nullptr), "bn_finalize: running mean and variance go together");
  bn_finalize_kernel<<<(c + 127) / 128, 128, 0, (cudaStream_t)stream>>>(stats, n, c, groups, hw, (double)eps, momentum,
                                                                       running_mean, running_var, num_batches_tracked);
  LAUNCH_CHECK();
  return SN_OK;
}

int sn_bn_group_sums(const double* stats, int n, int c, int groups, int hw, double* part, void* stream) {
  SN_REQUIRE(stats && part && n >= 1 && c >= 1 && hw >= 1, "bn_group_sums: bad arguments");
  SN_REQUIRE(groups >= 1 && n % groups == 0, "bn_group_sums: %d samples do not split into %d groups", n, groups);
  bn_group_sums_kernel<<<(c + 127) / 128, 128, 0, (cudaStream_t)stream>>>(stats, n, c, groups, hw, part);
  LAUNCH_CHECK();
  return SN_OK;
}

int sn_bn_finalize_gathered(double* stats, int n, int c, int groups, const double* gathered, int world, float eps,
                            float momentum, float* running_mean, float* running_var, long long* num_batches_tracked,
                            void* stream) {
  SN_REQUIRE(stats && gathered && n >= 1 && c >= 1 && world >= 1, "bn_finalize_gathered: bad arguments");
  SN_REQUIRE(groups >= 1 && n % groups == 0, "bn_finalize_gathered: %d samples do not split into %d groups", n, groups);
  SN_REQUIRE((running_mean == nullptr) == (running_var == nullptr),
             "bn_finalize_gathered: running mean and variance go together");
  bn_finalize_gathered_kernel<<<(c + 127) / 128, 128, 0, (cudaStream_t)stream>>>(
      stats, n, c, groups, gathered, world, (double)eps, momentum, running_mean, running_var, num_batches_tracked);
  LAUNCH_CHECK();
  return SN_OK;
}

int sn_bn_eval_stats(double* stats, int n, int c, const float* running_mean, const float* running_var, float eps,
                     void* stream) {
  SN_REQUIRE(stats && running_mean && running_var && n >= 1 && c >= 1, "bn_eval_stats: bad arguments");
  bn_eval_stats_kernel<<<(n * c + 255) / 256, 256, 0, (cudaStream_t)stream>>>(stats, n, c, running_mean, running_var,
                                                                              (double)eps);
  LAUNCH_CHECK();
  return SN_OK;
}

int sn_stats_finalize(double* stats, int count, int hw, float eps, void* stream) {
  SN_REQUIRE(stats && count >= 1 && hw >= 1, "stats_finalize: bad arguments");
  stats_finalize_kernel<<<(count + 255) / 256, 256, 0, (cudaStream_t)stream>>>(stats, count, hw, (double)eps);
  LAUNCH_CHECK();
  return SN_OK;
}

int sn_norm_act_fwd(const sn_norm_act_desc* d, void* stream) {
  SN_REQUIRE(d && d->y, "null pointer");
  SN_REQUIRE(!d->out_reflect_pad || (d->h >= 3 && d->w >= 3), "reflect pad needs h, w >= 3");
  NormActFwdArgs a;
  a.y = d->y; a.y_pitch = d->y_pitch;
  a.H = d->h; a.W = d->w; a.C = d->c;
  a.stats = d->stats;
  a.act = d->act; a.slope = d->slope;
  a.drop_thresh = d->drop_p > 0.f ? drop_thresh(d->drop_p) : 0u;
  a.drop_scale = d->drop_p > 0.f ? 1.f / (1.f - d->drop_p) : 1.f;
  a.seed = d->drop_seed;
  a.drop_off = d->drop_offset; a.seed_dev = d->drop_step_seed_dev; a.stage_id = d->drop_stage_id;
  a.residual = d->residual; a.res_pitch = d->res_pitch;
  a.hi = (uint16_t*)d->out_hi; a.lo = (uint16_t*)d->out_lo;
  a.out_pitch = d->out_pitch; a.out_coff = d->out_coff; a.reflect = d->out_reflect_pad;
  a.fmt = d->out_fmt;
  a.hi2 = (uint16_t*)d->out2_hi; a.lo2 = (uint16_t*)d->out2_lo; a.fmt2 = d->out2_fmt;
  a.f32 = d->out_f32; a.f32_pitch = d->f32_pitch;
  a.gamma = d->gamma; a.beta = d->beta;
  SN_REQUIRE((d->gamma == nullptr) == (d->beta == nullptr), "norm_act_fwd: gamma and beta go together");
  SN_REQUIRE(!d->gamma || d->stats, "norm_act_fwd: the affine (BatchNorm) variant needs stats");
  const bool vec = (d->c % 4 == 0) && al16(d->y) && (d->y_pitch % 4 == 0) &&
                   (!d->residual || (al16(d->residual) && d->res_pitch % 4 == 0)) &&
                   (!d->out_f32 || (al16(d->out_f32) && d->f32_pitch % 4 == 0)) &&
                   (!d->out_hi || (d->out_pitch % 4 == 0 && d->out_coff % 4 == 0 && ((uintptr_t)d->out_hi & 7) == 0 &&
                                   ((uintptr_t)d->out_lo & 7) == 0 && ((uintptr_t)d->out2_hi & 7) == 0 &&
                                   ((uintptr_t)d->out2_lo & 7) == 0));
  return vec ? launch_norm_act_fwd<4>(a, d->n, (cudaStream_t)stream) : launch_norm_act_fwd<1>(a, d->n, (cudaStream_t)stream);
}

static int fill_srcs(GradSrcs* g, const sn_grad_src* src, int nsrc) {
  SN_REQUIRE(nsrc >= 1 && nsrc <= SN_MAX_SRC, "nsrc out of range: %d", nsrc);
  g->n = nsrc;
  for (int i = 0; i < nsrc; ++i) {
    SN_REQUIRE(src[i].ptr, "null gradient source %d", i);
    SN_REQUIRE(!(src[i].up > 1 && src[i].reflect_padded), "gradient source %d: up and reflect_padded are exclusive", i);
    g->s[i] = src[i];
  }
  return SN_OK;
}

int sn_norm_act_bwd(const sn_norm_act_bwd_desc* d, void* stream) {
  SN_REQUIRE(d && d->y && d->dy_hi, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  NormActBwdArgs a;
  int rc = fill_srcs(&a.g, d->src, d->nsrc);
  if (rc) return rc;
  a.y = d->y; a.y_pitch = d->y_pitch;
  a.H = d->h; a.W = d->w; a.C = d->c;
  a.stats = d->stats;
  a.act = d->act; a.slope = d->slope;
  a.drop_thresh = d->drop_p > 0.f ? drop_thresh(d->drop_p) : 0u;
  a.drop_scale = d->drop_p > 0.f ? 1.f / (1.f - d->drop_p) : 1.f;
  a.seed = d->drop_seed;
  a.drop_off = d->drop_offset; a.seed_dev = d->drop_step_seed_dev; a.stage_id = d->drop_stage_id;
  a.gstats = d->gstats;
  a.hi = (uint16_t*)d->dy_hi; a.lo = (uint16_t*)d->dy_lo;
  a.dy_pitch = d->dy_pitch; a.dy_coff = d->dy_coff; a.fmt = d->dy_fmt;
  a.bias_grad = d->bias_grad;
  a.gamma = d->gamma; a.beta = d->beta;
  a.slots = d->det_slots;
  const bool aff = d->gamma != nullptr;
  const bool det = d->det_slots != nullptr;
  SN_REQUIRE(!det || !d->bias_grad, "norm_act_bwd: the deterministic reduction has no fused bias gradient");
  SN_REQUIRE((d->gamma == nullptr) == (d->beta == nullptr), "norm_act_bwd: gamma and beta go together");
  SN_REQUIRE(!aff || (d->stats && d->bn_groups >= 1 && d->n % d->bn_groups == 0 && !d->bias_grad),
             "norm_act_bwd: the BatchNorm variant needs stats, bn_groups dividing n, and no fused bias gradient");
  const int hw = d->h * d->w;
  const bool vec = (d->c % 4 == 0) && al16(d->y) && (d->y_pitch % 4 == 0) && srcs_vec_ok(a.g) &&
                   (d->dy_pitch % 4 == 0) && (d->dy_coff % 4 == 0) && ((uintptr_t)d->dy_hi & 7) == 0 &&
                   ((uintptr_t)d->dy_lo & 7) == 0;
  SN_REQUIRE(d->bn_phase >= 0 && d->bn_phase <= 2, "norm_act_bwd: bn_phase %d", d->bn_phase);
  SN_REQUIRE(d->bn_phase == 0 || (aff && d->bn_train), "norm_act_bwd: bn_phase needs the BatchNorm variant in train mode");
  SN_REQUIRE(d->bn_phase != 2 || (d->gstats && d->bn_gathered && d->bn_world >= 1 && d->bn_rank >= 0 && d->bn_rank < d->bn_world),
             "norm_act_bwd: bn_phase 2 needs bn_gathered and 0 <= bn_rank < bn_world (%d, %d)", d->bn_rank, d->bn_world);
  if (d->bn_phase == 2) {
    bn_bwd_group_gathered_kernel<<<(d->c + 127) / 128, 128, 0, st>>>(d->gstats, d->n, d->c, d->bn_groups, d->bn_gathered,
                                                                     d->bn_world, d->bn_rank, d->gamma_grad, d->beta_grad);
    LAUNCH_CHECK();
  } else if (d->stats) {
    SN_REQUIRE(d->gstats, "InstanceNorm backward needs gstats scratch");
    SN_CHECK_CUDA(cudaMemsetAsync(d->gstats, 0, sizeof(double) * 2 * d->n * d->c, st));
    int nslabs = 1;
    rc = vec ? launch_norm_act_bwd_reduce<4>(a, d->n, d->det_slots_cap, st, &nslabs)
             : launch_norm_act_bwd_reduce<1>(a, d->n, d->det_slots_cap, st, &nslabs);
    if (rc) return rc;
    if (det) {
      SN_CHECK_CUDA(det_sum_slots(d->det_slots, nslabs, 2LL * d->n * d->c, d->gstats, st));
      LAUNCH_CHECK();
    }
    if (d->bn_phase == 1) return SN_OK;
    if (aff)
      bn_bwd_group_kernel<<<(d->c + 127) / 128, 128, 0, st>>>(d->gstats, d->n, d->c, d->bn_groups, hw, d->bn_train,
                                                              d->gamma_grad, d->beta_grad);
    else
      gstats_finalize_kernel<<<(d->n * d->c + 255) / 256, 256, 0, st>>>(d->gstats, d->n * d->c, hw);
    LAUNCH_CHECK();
  }
  return vec ? launch_norm_act_bwd_apply<4>(a, d->n, st) : launch_norm_act_bwd_apply<1>(a, d->n, st);
}


static int bias_grad_impl(const void* dy_hi, const void* dy_lo, int pitch, int coff, int fmt, long long npix, int c,
                          double* scratch, float* db, double* slots, long long slots_cap, cudaStream_t st) {
  SN_REQUIRE(dy_hi && scratch && db, "null pointer");
  SN_CHECK_CUDA(cudaMemsetAsync(scratch, 0, sizeof(double) * c, st));
  const uint16_t* hi = (const uint16_t*)dy_hi + coff;
  const uint16_t* lo = dy_lo ? (const uint16_t*)dy_lo + coff : nullptr;
  const bool v8 = (pitch % 8 == 0) && (coff % 8 == 0) && (((uintptr_t)dy_hi | (uintptr_t)dy_lo) & 15) == 0 &&
                  ((c + 7) / 8 * 8 + coff <= pitch);
  int slabs = 1;
  const int rc = v8 ? launch_bias_grad<8>(hi, lo, pitch, fmt, npix, c, scratch, slots, slots_cap, st, &slabs)
                    : launch_bias_grad<1>(hi, lo, pitch, fmt, npix, c, scratch, slots, slots_cap, st, &slabs);
  if (rc) return rc;
  if (slots) {
    SN_CHECK_CUDA(det_sum_slots(slots, slabs, (long long)c, scratch, st));
    LAUNCH_CHECK();
  }
  bias_grad_finalize_kernel<<<(c + 255) / 256, 256, 0, st>>>(scratch, c, db);
  LAUNCH_CHECK();
  return SN_OK;
}

int sn_bias_grad(const void* dy_hi, const void* dy_lo, int pitch, int coff, int fmt, long long npix, int c,
                 double* scratch, float* db, void* stream) {
  return bias_grad_impl(dy_hi, dy_lo, pitch, coff, fmt, npix, c, scratch, db, nullptr, 0, (cudaStream_t)stream);
}

int sn_bias_grad_det(const void* dy_hi, const void* dy_lo, int pitch, int coff, int fmt, long long npix, int c,
                     double* scratch, float* db, double* slots, long long slots_cap, void* stream) {
  SN_REQUIRE(slots, "bias_grad_det: null slots");
  return bias_grad_impl(dy_hi, dy_lo, pitch, coff, fmt, npix, c, scratch, db, slots, slots_cap, (cudaStream_t)stream);
}

int sn_sum_grads(const sn_grad_src* src, int nsrc, int n, int h, int w, int c, float* dst,
                 int dst_pitch, void* stream) {
  GradSrcs g;
  int rc = fill_srcs(&g, src, nsrc);
  if (rc) return rc;
  const dim3 grid(vslabs(h * w, n), n);
  if ((c % 4 == 0) && srcs_vec_ok(g) && al16(dst) && (dst_pitch % 4 == 0))
    sum_grads_kernel<4><<<grid, 256, 0, (cudaStream_t)stream>>>(g, h, w, c, dst, dst_pitch);
  else
    sum_grads_kernel<1><<<grid, 256, 0, (cudaStream_t)stream>>>(g, h, w, c, dst, dst_pitch);
  LAUNCH_CHECK();
  return SN_OK;
}

int sn_tanh_bwd(const sn_grad_src* src, int nsrc, const float* out, int out_pitch, int n, int h,
                int w, int c, void* dy_hi, void* dy_lo, int dy_pitch, int dy_coff, int dy_fmt, void* stream) {
  GradSrcs g;
  int rc = fill_srcs(&g, src, nsrc);
  if (rc) return rc;
  tanh_bwd_kernel<<<grid_for((long long)n * h * w * c), kEwThreads, 0, (cudaStream_t)stream>>>(g, out, out_pitch, n, h, w, c,
                                                          (uint16_t*)dy_hi, (uint16_t*)dy_lo,
                                                          dy_pitch, dy_coff, dy_fmt);
  LAUNCH_CHECK();
  return SN_OK;
}

int sn_upsample_planes(const void* src_hi, const void* src_lo, int src_pitch, int src_coff, int n, int h, int w,
                       int c, int factor, void* dst_hi, void* dst_lo, int dst_pitch, int dst_coff, void* stream) {
  SN_REQUIRE(src_hi && dst_hi && factor >= 1 && h % factor == 0 && w % factor == 0, "bad upsample arguments");
  const long long total = (long long)n * h * w * c;
  const uint16_t* shi = (const uint16_t*)src_hi + src_coff;
  const uint16_t* slo = src_lo ? (const uint16_t*)src_lo + src_coff : nullptr;
  uint16_t* dhi = (uint16_t*)dst_hi + dst_coff;
  uint16_t* dlo = dst_lo ? (uint16_t*)dst_lo + dst_coff : nullptr;
  const cudaStream_t st = (cudaStream_t)stream;
  if (c % 4 == 0 && src_pitch % 4 == 0 && dst_pitch % 4 == 0 && src_coff % 4 == 0 && dst_coff % 4 == 0 &&
      ((uintptr_t)src_hi % 8) == 0 && ((uintptr_t)dst_hi % 8) == 0 && (!src_lo || ((uintptr_t)src_lo % 8) == 0) &&
      (!dst_lo || ((uintptr_t)dst_lo % 8) == 0))
    upsample_planes_kernel<4><<<grid_for(total / 4), kEwThreads, 0, st>>>(shi, slo, src_pitch, h, w, c / 4, factor, dhi,
                                                                        dlo, dst_pitch, total / 4);
  else
    upsample_planes_kernel<1><<<grid_for(total), kEwThreads, 0, st>>>(shi, slo, src_pitch, h, w, c, factor, dhi, dlo,
                                                                    dst_pitch, total);
  LAUNCH_CHECK();
  return SN_OK;
}

void sn_adamw_hyper(double lr, double beta1, double beta2, double eps, double weight_decay, int step, double gscale,
                    float out[8]) {
  // scalars are formed in double and rounded once, as torch does with its Python-float hyper-parameters
  const double bc1 = 1.0 - pow(beta1, (double)step);
  const double bc2 = 1.0 - pow(beta2, (double)step);
  out[0] = (float)(1.0 - lr * weight_decay); out[1] = (float)(1.0 - beta1); out[2] = (float)beta2;
  out[3] = (float)(1.0 - beta2); out[4] = (float)(lr / bc1); out[5] = (float)(1.0 / sqrt(bc2)); out[6] = (float)eps;
  out[7] = (float)gscale;
}

int sn_adamw_step(float* p, const float* g, float* m, float* v, long long n, double lr, double beta1, double beta2,
                  double eps, double weight_decay, int step, void* stream) {
  SN_REQUIRE(p && g && m && v && n > 0 && step >= 1, "bad adamw arguments");
  SN_REQUIRE((((uintptr_t)p | (uintptr_t)g | (uintptr_t)m | (uintptr_t)v) & 15) == 0, "adamw buffers must be 16-B aligned");
  float hp[8];
  sn_adamw_hyper(lr, beta1, beta2, eps, weight_decay, step, 1.0, hp);
  const AdamHyper h{hp[0], hp[1], hp[2], hp[3], hp[4], hp[5], hp[6], hp[7]};
  adamw_kernel<<<grid_for(n / 4 + 1), kEwThreads, 0, (cudaStream_t)stream>>>(p, g, m, v, n, h, nullptr);
  LAUNCH_CHECK();
  return SN_OK;
}

int sn_adamw_step_dev(float* p, const float* g, float* m, float* v, long long n, const float* hyper_dev, void* stream) {
  SN_REQUIRE(p && g && m && v && n > 0 && hyper_dev, "bad adamw arguments");
  SN_REQUIRE((((uintptr_t)p | (uintptr_t)g | (uintptr_t)m | (uintptr_t)v) & 15) == 0, "adamw buffers must be 16-B aligned");
  adamw_kernel<<<grid_for(n / 4 + 1), kEwThreads, 0, (cudaStream_t)stream>>>(p, g, m, v, n, AdamHyper{}, hyper_dev);
  LAUNCH_CHECK();
  return SN_OK;
}

void sn_adabound_hyper(double lr, double base_lr, double beta1, double beta2, double eps, double weight_decay,
                       double final_lr, double gamma, int step, double gscale, float out[8]) {
  const double bc1 = 1.0 - pow(beta1, (double)step);
  const double bc2 = 1.0 - pow(beta2, (double)step);
  const double fin = final_lr * lr / base_lr;   // the bounds follow a scheduler's lr
  out[0] = (float)(1.0 - beta1); out[1] = (float)(1.0 - beta2); out[2] = (float)eps; out[3] = (float)weight_decay;
  out[4] = (float)(lr * sqrt(bc2) / bc1);
  out[5] = (float)(fin * (1.0 - 1.0 / (gamma * step + 1.0)));
  out[6] = (float)(fin * (1.0 + 1.0 / (gamma * step)));
  out[7] = (float)gscale;
}

int sn_adabound_step(float* p, const float* g, float* m, float* v, long long n, double lr, double base_lr, double beta1,
                     double beta2, double eps, double weight_decay, double final_lr, double gamma, int step,
                     void* stream) {
  SN_REQUIRE(p && g && m && v && n > 0 && step >= 1, "bad adabound arguments");
  SN_REQUIRE(base_lr > 0.0 && gamma > 0.0 && final_lr >= 0.0, "adabound needs base_lr > 0, gamma > 0, final_lr >= 0");
  SN_REQUIRE((((uintptr_t)p | (uintptr_t)g | (uintptr_t)m | (uintptr_t)v) & 15) == 0, "adabound buffers must be 16-B aligned");
  float hp[8];
  sn_adabound_hyper(lr, base_lr, beta1, beta2, eps, weight_decay, final_lr, gamma, step, 1.0, hp);
  const AdaBoundHyper h{hp[0], hp[1], hp[2], hp[3], hp[4], hp[5], hp[6], hp[7]};
  adabound_kernel<<<grid_for(n / 4 + 1), kEwThreads, 0, (cudaStream_t)stream>>>(p, g, m, v, n, h, nullptr);
  LAUNCH_CHECK();
  return SN_OK;
}

int sn_adabound_step_dev(float* p, const float* g, float* m, float* v, long long n, const float* hyper_dev,
                         void* stream) {
  SN_REQUIRE(p && g && m && v && n > 0 && hyper_dev, "bad adabound arguments");
  SN_REQUIRE((((uintptr_t)p | (uintptr_t)g | (uintptr_t)m | (uintptr_t)v) & 15) == 0, "adabound buffers must be 16-B aligned");
  adabound_kernel<<<grid_for(n / 4 + 1), kEwThreads, 0, (cudaStream_t)stream>>>(p, g, m, v, n, AdaBoundHyper{}, hyper_dev);
  LAUNCH_CHECK();
  return SN_OK;
}

struct StepParams { float v[64]; };
__global__ void set_step_params_kernel(float* dst, const StepParams sp, int n) {
  if (threadIdx.x < n) dst[threadIdx.x] = sp.v[threadIdx.x];
}
int sn_set_step_params(float* dst, const float* vals, int n, void* stream) {
  SN_REQUIRE(dst && vals && n >= 1 && n <= 64, "set_step_params: 1..64 floats");
  StepParams sp;
  for (int i = 0; i < 64; ++i) sp.v[i] = i < n ? vals[i] : 0.f;
  set_step_params_kernel<<<1, 64, 0, (cudaStream_t)stream>>>(dst, sp, n);
  LAUNCH_CHECK();
  return SN_OK;
}

int sn_dropout_mask(unsigned long long seed, float p, long long count, uint8_t* out, void* stream) {
  dropout_mask_kernel<<<grid_for(count), kEwThreads, 0, (cudaStream_t)stream>>>(seed, drop_thresh(p),
                                                                               count, out);
  LAUNCH_CHECK();
  return SN_OK;
}

int sn_ce_loss_fwd_bwd(const float* logits, int pitch, const void* target, int target_layout, int n, int h, int w,
                       int c, float weight, double* loss_acc, float* grad, int grad_pitch, void* stream) {
  SN_REQUIRE(c <= kMaxCE, "ce loss supports at most %d classes", kMaxCE);
  SN_REQUIRE(target_layout == SN_LAYOUT_NCHW || target_layout == SN_LAYOUT_LABEL_U8,
             "ce loss: target must be NCHW fp32 or a uint8 label map");
  const bool lab = target_layout == SN_LAYOUT_LABEL_U8;
  ce_loss_kernel<<<grid_for((long long)n * h * w, 128), 128, 0, (cudaStream_t)stream>>>(
      logits, pitch, lab ? nullptr : (const float*)target, lab ? (const uint8_t*)target : nullptr, n, h, w, c, weight,
      loss_acc, grad, grad_pitch);
  LAUNCH_CHECK();
  return SN_OK;
}

static int ce_tanh_bwd_impl(const float* logits, int pitch, const void* target, int target_layout,
                            const sn_grad_src* src, int nsrc, int n, int h, int w, int c, float weight, double* loss_acc,
                            void* dy_hi, void* dy_lo, int dy_pitch, int dy_coff, int dy_fmt, double* slots,
                            long long slots_cap, cudaStream_t st) {
  SN_REQUIRE(c <= kMaxCE && logits && dy_hi && loss_acc, "ce_tanh_bwd: bad arguments (at most %d classes)", kMaxCE);
  SN_REQUIRE(target_layout == SN_LAYOUT_NCHW || target_layout == SN_LAYOUT_LABEL_U8,
             "ce_tanh_bwd: target must be NCHW fp32 or a uint8 label map");
  SN_REQUIRE(dy_pitch % 8 == 0 && dy_coff % 8 == 0 && ((c + 7) & ~7) + dy_coff <= dy_pitch &&
                 (((uintptr_t)dy_hi | (uintptr_t)dy_lo) & 15) == 0,
             "ce_tanh_bwd: dy planes need 8-channel aligned slices and 16-byte aligned bases");
  GradSrcs g;
  g.n = 0;
  if (nsrc > 0) {
    int rc = fill_srcs(&g, src, nsrc);
    if (rc) return rc;
  }
  const bool lab = target_layout == SN_LAYOUT_LABEL_U8;
  const int blocks = grid_for((long long)n * h * w, 128);
  const float* tf = lab ? nullptr : (const float*)target;
  const uint8_t* tl = lab ? (const uint8_t*)target : nullptr;
  if (!slots) {
    ce_tanh_bwd_kernel<false><<<blocks, 128, 0, st>>>(logits, pitch, tf, tl, g, n, h, w, c, weight, loss_acc,
                                                      (uint16_t*)dy_hi, (uint16_t*)dy_lo, dy_pitch, dy_coff, dy_fmt,
                                                      nullptr);
    LAUNCH_CHECK();
    return SN_OK;
  }
  SN_REQUIRE(blocks <= slots_cap, "ce_tanh_bwd_det: %d slots needed, %lld given", blocks, slots_cap);
  ce_tanh_bwd_kernel<true><<<blocks, 128, 0, st>>>(logits, pitch, tf, tl, g, n, h, w, c, weight, loss_acc,
                                                   (uint16_t*)dy_hi, (uint16_t*)dy_lo, dy_pitch, dy_coff, dy_fmt, slots);
  LAUNCH_CHECK();
  SN_CHECK_CUDA(det_sum_slots(slots, blocks, 1, loss_acc, st));
  LAUNCH_CHECK();
  return SN_OK;
}

int sn_ce_tanh_bwd(const float* logits, int pitch, const void* target, int target_layout, const sn_grad_src* src,
                   int nsrc, int n, int h, int w, int c, float weight, double* loss_acc, void* dy_hi, void* dy_lo,
                   int dy_pitch, int dy_coff, int dy_fmt, void* stream) {
  return ce_tanh_bwd_impl(logits, pitch, target, target_layout, src, nsrc, n, h, w, c, weight, loss_acc, dy_hi, dy_lo,
                          dy_pitch, dy_coff, dy_fmt, nullptr, 0, (cudaStream_t)stream);
}

int sn_ce_tanh_bwd_det(const float* logits, int pitch, const void* target, int target_layout, const sn_grad_src* src,
                       int nsrc, int n, int h, int w, int c, float weight, double* loss_acc, void* dy_hi, void* dy_lo,
                       int dy_pitch, int dy_coff, int dy_fmt, double* slots, long long slots_cap, void* stream) {
  SN_REQUIRE(slots, "ce_tanh_bwd_det: null slots");
  return ce_tanh_bwd_impl(logits, pitch, target, target_layout, src, nsrc, n, h, w, c, weight, loss_acc, dy_hi, dy_lo,
                          dy_pitch, dy_coff, dy_fmt, slots, slots_cap, (cudaStream_t)stream);
}

int sn_bce_logits_fwd_bwd(const float* pred, long long count_per_half, int halves, float t0, float t1,
                          float gscale, double* loss_acc, float* dpred, void* stream) {
  SN_REQUIRE(halves == 1 || halves == 2, "halves must be 1 or 2");
  dim3 grid(grid_for(count_per_half), halves);
  gan_loss_kernel<SN_GAN_BCE, false><<<grid, kEwThreads, 0, (cudaStream_t)stream>>>(pred, count_per_half, halves, t0, t1,
                                                                             nullptr, gscale, loss_acc, dpred, nullptr);
  LAUNCH_CHECK();
  return SN_OK;
}

int sn_bce_logits_fwd_bwd_dev(const float* pred, long long count_per_half, int halves, const float* t_dev,
                              float gscale, double* loss_acc, float* dpred, void* stream) {
  SN_REQUIRE((halves == 1 || halves == 2) && t_dev, "halves must be 1 or 2, t_dev non-null");
  dim3 grid(grid_for(count_per_half), halves);
  gan_loss_kernel<SN_GAN_BCE, false><<<grid, kEwThreads, 0, (cudaStream_t)stream>>>(pred, count_per_half, halves, 0.f, 0.f,
                                                                             t_dev, gscale, loss_acc, dpred, nullptr);
  LAUNCH_CHECK();
  return SN_OK;
}

}  // extern "C"

template <bool DET>
static void launch_gan_loss(int objective, dim3 grid, cudaStream_t s, const float* pred, long long count_per_half,
                            int halves, float t0, float t1, const float* t_dev, float gscale, double* loss_acc,
                            float* dpred, double* slots) {
  switch (objective) {
    case SN_GAN_BCE:
      gan_loss_kernel<SN_GAN_BCE, DET><<<grid, kEwThreads, 0, s>>>(pred, count_per_half, halves, t0, t1, t_dev, gscale,
                                                                   loss_acc, dpred, slots);
      break;
    case SN_GAN_MSE:
      gan_loss_kernel<SN_GAN_MSE, DET><<<grid, kEwThreads, 0, s>>>(pred, count_per_half, halves, t0, t1, t_dev, gscale,
                                                                   loss_acc, dpred, slots);
      break;
    default:
      gan_loss_kernel<SN_GAN_WGAN, DET><<<grid, kEwThreads, 0, s>>>(pred, count_per_half, halves, t0, t1, nullptr,
                                                                    gscale, loss_acc, dpred, slots);
  }
}

extern "C" {

static int gan_loss_impl(int objective, const float* pred, long long count_per_half, int halves, float t0, float t1,
                         const float* t_dev, float gscale, double* loss_acc, float* dpred, double* slots,
                         long long slots_cap, cudaStream_t s) {
  SN_REQUIRE(halves == 1 || halves == 2, "halves must be 1 or 2");
  SN_REQUIRE(pred && loss_acc && count_per_half > 0, "gan_loss: null pointer or empty prediction");
  SN_REQUIRE(objective != SN_GAN_WGAN || !t_dev, "gan_loss: the WGAN signs are passed by value (t0, t1), not t_dev");
  SN_REQUIRE(objective == SN_GAN_BCE || objective == SN_GAN_MSE || objective == SN_GAN_WGAN,
             "gan_loss: unknown objective %d", objective);
  dim3 grid(grid_for(count_per_half), halves);
  if (!slots) {
    launch_gan_loss<false>(objective, grid, s, pred, count_per_half, halves, t0, t1, t_dev, gscale, loss_acc, dpred,
                           nullptr);
    LAUNCH_CHECK();
    return SN_OK;
  }
  SN_REQUIRE((long long)grid.x * halves <= slots_cap, "gan_loss_det: slots too small");
  launch_gan_loss<true>(objective, grid, s, pred, count_per_half, halves, t0, t1, t_dev, gscale, loss_acc, dpred, slots);
  LAUNCH_CHECK();
  SN_CHECK_CUDA(det_sum_slots(slots, (int)grid.x, (long long)halves, loss_acc, s));
  LAUNCH_CHECK();
  return SN_OK;
}

int sn_gan_loss_fwd_bwd_dev(int objective, const float* pred, long long count_per_half, int halves, float t0, float t1,
                            const float* t_dev, float gscale, double* loss_acc, float* dpred, void* stream) {
  return gan_loss_impl(objective, pred, count_per_half, halves, t0, t1, t_dev, gscale, loss_acc, dpred, nullptr, 0,
                       (cudaStream_t)stream);
}

int sn_gan_loss_fwd_bwd_det(int objective, const float* pred, long long count_per_half, int halves, float t0, float t1,
                            const float* t_dev, float gscale, double* loss_acc, float* dpred, double* slots,
                            long long slots_cap, void* stream) {
  SN_REQUIRE(slots, "gan_loss_det: null slots");
  return gan_loss_impl(objective, pred, count_per_half, halves, t0, t1, t_dev, gscale, loss_acc, dpred, slots, slots_cap,
                       (cudaStream_t)stream);
}

static int l1_loss_impl(const float* a, int pitch, const float* b_nchw, int n, int h, int w, int c, float weight,
                        double* loss_acc, float* grad, int grad_pitch, double* slots, long long slots_cap,
                        cudaStream_t st) {
  const int blocks = grid_for((long long)n * h * w * c);
  if (!slots) {
    l1_loss_kernel<false><<<blocks, kEwThreads, 0, st>>>(a, pitch, b_nchw, n, h, w, c, weight, loss_acc, grad,
                                                         grad_pitch, nullptr);
    LAUNCH_CHECK();
    return SN_OK;
  }
  SN_REQUIRE(blocks <= slots_cap, "l1_loss_det: %d slots needed, %lld given", blocks, slots_cap);
  l1_loss_kernel<true><<<blocks, kEwThreads, 0, st>>>(a, pitch, b_nchw, n, h, w, c, weight, loss_acc, grad, grad_pitch,
                                                      slots);
  LAUNCH_CHECK();
  SN_CHECK_CUDA(det_sum_slots(slots, blocks, 1, loss_acc, st));
  LAUNCH_CHECK();
  return SN_OK;
}

int sn_l1_loss_fwd_bwd(const float* a, int pitch, const float* b_nchw, int n, int h, int w, int c,
                       float weight, double* loss_acc, float* grad, int grad_pitch, void* stream) {
  return l1_loss_impl(a, pitch, b_nchw, n, h, w, c, weight, loss_acc, grad, grad_pitch, nullptr, 0,
                      (cudaStream_t)stream);
}

int sn_l1_loss_fwd_bwd_det(const float* a, int pitch, const float* b_nchw, int n, int h, int w, int c, float weight,
                           double* loss_acc, float* grad, int grad_pitch, double* slots, long long slots_cap,
                           void* stream) {
  SN_REQUIRE(slots, "l1_loss_det: null slots");
  return l1_loss_impl(a, pitch, b_nchw, n, h, w, c, weight, loss_acc, grad, grad_pitch, slots, slots_cap,
                      (cudaStream_t)stream);
}

int sn_tap_gemm_simt(const sn_tap_gemm_desc* d, void* stream) {
  SN_REQUIRE(d && d->a_hi && d->b_hi && d->out, "null pointer");
  SimtArgs a;
  a.a_hi = (const uint16_t*)d->a_hi; a.a_lo = (const uint16_t*)d->a_lo;
  a.b_hi = (const uint16_t*)d->b_hi; a.b_lo = (const uint16_t*)d->b_lo;
  a.a_fmt = d->a_fmt; a.b_fmt = d->b_fmt; a.b_scale = d->b_scale;
  a.a_n = d->a_n; a.a_h = d->a_h; a.a_w = d->a_w; a.a_c = d->a_c; a.a_pitch = d->a_pitch;
  a.parity = d->a_parity;
  a.b_k = d->b_k; a.b_rows = d->b_rows;
  a.m_n = d->m_n; a.m_h = d->m_h; a.m_w = d->m_w; a.ntaps = d->ntaps; a.k_per_tap = d->k_per_tap;
  for (int t = 0; t < d->ntaps; ++t) a.taps[t] = d->taps[t];
  a.out = d->out; a.out_sn = d->out_sn; a.out_sh = d->out_sh; a.out_sw = d->out_sw;
  a.omh = d->out_mul_h; a.ooh = d->out_off_h; a.omw = d->out_mul_w; a.oow = d->out_off_w;
  a.n_valid = d->n_valid; a.bias = d->bias; a.act = d->act; a.nsplit = d->nsplit;
  const long long total = (long long)d->m_n * d->m_h * d->m_w * d->n_valid;
  tap_gemm_simt_kernel<<<grid_for(total), kEwThreads, 0, (cudaStream_t)stream>>>(a);
  LAUNCH_CHECK();
  return SN_OK;
}

}  // extern "C"
