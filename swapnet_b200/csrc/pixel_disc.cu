// swapnet_b200 — the 1x1 PixelGAN discriminator (modules/discriminators.py:138-168) as fused per-pixel passes.
//
// The network is a per-pixel MLP  x (cin <= 32) -> z1 = W1 x + b1 (64) -> a1 = lrelu(z1) -> z2 = W2 a1 (+ b2) (128)
// -> y2 = IN(z2) or z2 -> a2 = lrelu(y2) -> p = w3 . a2 (+ b3), every layer at full input resolution.  Keeping its
// activations would cost 1-2.5 KB per pixel and layer; instead every pass recomputes z1 and z2 from the 22-channel
// operand through ONE device function (recompute()), so the values — and the LeakyReLU gates — are bit-identical in
// every pass, and only the logits, per-(n, c) statistics, weight gradients and the input gradient reach memory.
//
// Products run on the tensor cores (mma.sync m16n8k16, fp32 accumulation) as split 16-bit operands (DESIGN §2):
// forward fp16-split with the weights pre-scaled by the per-tensor power of two of sn_weight_scale_multi, backward
// bf16-split and unscaled; nsplit = 1 keeps the hi x hi product only.  One warp owns 16 pixels; the C fragment of one
// GEMM is the A fragment of the next, so z1 -> z2 and dz2 -> dA1 -> dx never leave registers.  The weight gradients
// dW2 = dz2^T a1 and dW1 = g1^T x contract over pixels: the block stages its 64-pixel tile transposed in shared memory
// and accumulates both in registers across all its tiles, each tile's partial promoted with round-to-nearest adds; a
// constant-one row appended to a1 and x gives db2 and db1 from the same MMAs.
//
// Cross-block sums (statistics, weight gradients) use atomics, or per-block slots added in block order by
// det_sum_slots (deterministic mode).  Blocks take contiguous tile ranges of a grid fixed by the shapes alone.
#include "common.cuh"
#include "../../include/swapnet_b200.h"

void sn_count_launch(int n);

namespace {

constexpr int C1 = 64, C2 = 128, KX = 32;         // hidden widths, padded input channels
constexpr int kWarps = 4, kThreads = 32 * kWarps, kTile = 16 * kWarps;
constexpr int kBlocks = 2 * SN_NUM_SMS;            // grid of every pass (fixed: the deterministic slots depend on it)
// shared-memory row pitches in 32-bit words (padded so the fragment loads of the 8 row groups hit distinct banks)
constexpr int kW1P = 20, kW2P = 36, kW2bP = 68, kW1bP = 36, kSP = 36;
constexpr int kA1Rows = C1 + 8, kXRows = KX + 8;  // staged a1 / x plus the constant-one row (bias gradients)

// shared-memory layout, offsets in 32-bit words
constexpr int oW1h = 0, oW1l = oW1h + C1 * kW1P, oW2h = oW1l + C1 * kW1P, oW2l = oW2h + C2 * kW2P;
constexpr int oVec = oW2l + C2 * kW2P;             // b1[64] b2[128] w3[128] mean[128] rstd[128] mg[128] mgy[128]
constexpr int oAcc = oVec + 832;                   // doubles [kWarps][4][C2]: per-warp column sums
constexpr int oFwdEnd = oAcc + 2 * kWarps * 4 * C2;
constexpr int oW2bh = oFwdEnd, oW2bl = oW2bh + C1 * kW2bP, oW1bh = oW2bl + C1 * kW2bP, oW1bl = oW1bh + KX * kW1bP;
constexpr int oDzh = oW1bl + KX * kW1bP, oDzl = oDzh + C2 * kSP, oA1h = oDzl + C2 * kSP, oA1l = oA1h + kA1Rows * kSP;
constexpr int oG1h = oA1l + kA1Rows * kSP, oG1l = oG1h + C1 * kSP, oXh = oG1l + C1 * kSP, oXl = oXh + kXRows * kSP;
constexpr int oBwdEnd = oXl + kXRows * kSP;
static_assert(oAcc % 2 == 0, "double alignment");

enum { PASS_STATS = 0, PASS_FWD = 1, PASS_REDUCE = 2, PASS_APPLY = 3 };

template <bool BF>
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  if constexpr (BF)
    asm("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  else
    asm("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// hi x hi (+ lo x hi + hi x lo) of split operands
template <bool BF>
__device__ __forceinline__ void mma_split(float (&d)[4], const uint32_t (&ah)[4], const uint32_t (&al)[4], const uint32_t* bh,
                                          const uint32_t* bl, int nsplit) {
  mma16816<BF>(d, ah, bh[0], bh[4]);
  if (nsplit > 1) {
    mma16816<BF>(d, al, bh[0], bh[4]);
    mma16816<BF>(d, ah, bl[0], bl[4]);
  }
}

__device__ __forceinline__ void split_pair(float v0, float v1, int fmt, uint32_t& hi, uint32_t& lo) {
  uint16_t h0, l0, h1, l1;
  split16(v0, fmt, h0, l0);
  split16(v1, fmt, h1, l1);
  hi = (uint32_t)h0 | ((uint32_t)h1 << 16);
  lo = (uint32_t)l0 | ((uint32_t)l1 << 16);
}

__device__ __forceinline__ float lrelu(float v, float slope) { return v > 0.f ? v : v * slope; }
__device__ __forceinline__ float gate(float v, float slope) { return v > 0.f ? 1.f : slope; }

struct Args {
  sn_pixel_desc d;
  int tiles_per_img, tiles_per_block;
};

// z1 (C fragments, 8 n-tiles of 8 hidden channels) and z2 (16 n-tiles) of the warp's 16 pixels, rows g and g + 8.
// The single definition of the forward arithmetic: every pass calls it, so every pass sees the same bits.
__device__ __forceinline__ void recompute(const sn_pixel_desc& d, const uint32_t* sm, long long pg, long long pg8, bool vg,
                                          bool vg8, int lane, float (&z1)[8][4], float (&z2)[16][4]) {
  const int g = lane >> 2, t = lane & 3;
  const float* vec = reinterpret_cast<const float*>(sm + oVec);
  const uint16_t* xh = (const uint16_t*)d.x_hi;
  const uint16_t* xl = (const uint16_t*)d.x_lo;
#pragma unroll
  for (int nt = 0; nt < 8; ++nt)
#pragma unroll
    for (int i = 0; i < 4; ++i) z1[nt][i] = 0.f;
  for (int kc = 0; kc < d.x_c / 16; ++kc) {
    uint32_t ah[4], al[4];
    const int c = 16 * kc + 2 * t;
    const long long og = pg * d.x_pitch + c, og8 = pg8 * d.x_pitch + c;
    ah[0] = vg ? *reinterpret_cast<const uint32_t*>(xh + og) : 0u;
    ah[1] = vg8 ? *reinterpret_cast<const uint32_t*>(xh + og8) : 0u;
    ah[2] = vg ? *reinterpret_cast<const uint32_t*>(xh + og + 8) : 0u;
    ah[3] = vg8 ? *reinterpret_cast<const uint32_t*>(xh + og8 + 8) : 0u;
    al[0] = vg ? *reinterpret_cast<const uint32_t*>(xl + og) : 0u;
    al[1] = vg8 ? *reinterpret_cast<const uint32_t*>(xl + og8) : 0u;
    al[2] = vg ? *reinterpret_cast<const uint32_t*>(xl + og + 8) : 0u;
    al[3] = vg8 ? *reinterpret_cast<const uint32_t*>(xl + og8 + 8) : 0u;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const int w = (8 * nt + g) * kW1P + 8 * kc + t;
      mma_split<false>(z1[nt], ah, al, sm + oW1h + w, sm + oW1l + w, d.nsplit);
    }
  }
  const float inv1 = d.scale1[1], inv2 = d.scale2[1];
  uint32_t ah[4][4], al[4][4];   // a1 as the A fragments of the 4 k-chunks of the second GEMM
#pragma unroll
  for (int nt = 0; nt < 8; ++nt) {
    const float b0 = vec[8 * nt + 2 * t], b1 = vec[8 * nt + 2 * t + 1];
    z1[nt][0] = z1[nt][0] * inv1 + b0;
    z1[nt][1] = z1[nt][1] * inv1 + b1;
    z1[nt][2] = z1[nt][2] * inv1 + b0;
    z1[nt][3] = z1[nt][3] * inv1 + b1;
    const int kk = nt >> 1, half = nt & 1;
    split_pair(lrelu(z1[nt][0], d.slope), lrelu(z1[nt][1], d.slope), SN_FMT_F16, ah[kk][2 * half], al[kk][2 * half]);
    split_pair(lrelu(z1[nt][2], d.slope), lrelu(z1[nt][3], d.slope), SN_FMT_F16, ah[kk][2 * half + 1],
               al[kk][2 * half + 1]);
  }
  const float* b2 = vec + C1;
#pragma unroll
  for (int nt = 0; nt < 16; ++nt) {
#pragma unroll
    for (int i = 0; i < 4; ++i) z2[nt][i] = 0.f;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const int w = (8 * nt + g) * kW2P + 8 * kk + t;
      mma_split<false>(z2[nt], ah[kk], al[kk], sm + oW2h + w, sm + oW2l + w, d.nsplit);
    }
    const float c0 = d.b2 ? b2[8 * nt + 2 * t] : 0.f, c1 = d.b2 ? b2[8 * nt + 2 * t + 1] : 0.f;
    z2[nt][0] = z2[nt][0] * inv2 + c0;
    z2[nt][1] = z2[nt][1] * inv2 + c1;
    z2[nt][2] = z2[nt][2] * inv2 + c0;
    z2[nt][3] = z2[nt][3] * inv2 + c1;
  }
}

// acc[c] += sum over the warp's 16 rows of f(v, row, c) (fp64; xor butterfly over the 8 row groups, fixed order)
template <typename F>
__device__ __forceinline__ void colsum_add(double* acc, int lane, F f) {
  const int t = lane & 3;
#pragma unroll
  for (int nt = 0; nt < 16; ++nt) {
    double s0 = f(nt, 0) + f(nt, 2), s1 = f(nt, 1) + f(nt, 3);
#pragma unroll
    for (int o = 4; o < 32; o <<= 1) {
      s0 += __shfl_xor_sync(0xffffffffu, s0, o);
      s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    }
    if (lane < 4) {
      acc[8 * nt + 2 * t] += s0;
      acc[8 * nt + 2 * t + 1] += s1;
    }
  }
}

// per-(n, c) pairs accumulated in the per-warp slots 0 and 1 -> dst[n][c][2] (atomics, or this block's slot row)
__device__ void flush_pairs(const Args& a, double* acc, int n, double* dst) {
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * C2; i += blockDim.x) {
    const int c = i >> 1, k = i & 1;
    double s = 0.0;
    for (int w = 0; w < kWarps; ++w) s += acc[(w * 4 + k) * C2 + c];
    for (int w = 0; w < kWarps; ++w) acc[(w * 4 + k) * C2 + c] = 0.0;
    const long long o = ((long long)n * C2 + c) * 2 + k;
    if (a.d.slots) a.d.slots[(long long)blockIdx.x * a.d.n * C2 * 2 + o] = s;
    else atomicAdd(dst + o, s);
  }
  __syncthreads();
}

__device__ __forceinline__ void add_wgrad(const Args& a, float* slot_region, int count, int i, float* dst, float v) {
  if (a.d.slots) slot_region[(long long)blockIdx.x * count + i] = v;
  else atomicAdd(dst + i, v);
}

// float slot regions of the weight gradients, after the [kBlocks][n][C2][2] doubles of the statistics
struct WgSlots {
  float *dw2, *db2, *dw1, *db1, *dw3, *db3;
};
__host__ __device__ inline WgSlots wg_slots(double* slots, int n, int cin) {
  float* f = reinterpret_cast<float*>(slots + (long long)kBlocks * n * C2 * 2);
  WgSlots s;
  s.dw2 = f; f += (long long)kBlocks * C2 * C1;
  s.db2 = f; f += (long long)kBlocks * C2;
  s.dw1 = f; f += (long long)kBlocks * C1 * cin;
  s.db1 = f; f += (long long)kBlocks * C1;
  s.dw3 = f; f += (long long)kBlocks * C2;
  s.db3 = f;
  return s;
}

template <int PASS, bool NORM, bool WG>
__global__ void __launch_bounds__(kThreads, 1) pixel_kernel(const Args a) {
  extern __shared__ __align__(16) uint32_t sm[];
  const sn_pixel_desc& d = a.d;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
  float* vec = reinterpret_cast<float*>(sm + oVec);
  double* acc = reinterpret_cast<double*>(sm + oAcc);
  double* wacc = acc + warp * 4 * C2;
  // ---- prologue: weights split into shared memory, per-block column sums zeroed ----
  const float s1 = d.scale1[0], s2 = d.scale2[0];
  for (int i = threadIdx.x; i < C1 * (KX / 2); i += blockDim.x) {
    const int r = i / (KX / 2), j = i % (KX / 2), c = 2 * j;
    const float v0 = c < d.cin ? d.w1[r * d.cin + c] * s1 : 0.f, v1 = c + 1 < d.cin ? d.w1[r * d.cin + c + 1] * s1 : 0.f;
    split_pair(v0, v1, SN_FMT_F16, sm[oW1h + r * kW1P + j], sm[oW1l + r * kW1P + j]);
  }
  for (int i = threadIdx.x; i < C2 * (C1 / 2); i += blockDim.x) {
    const int r = i / (C1 / 2), j = i % (C1 / 2);
    split_pair(d.w2[r * C1 + 2 * j] * s2, d.w2[r * C1 + 2 * j + 1] * s2, SN_FMT_F16, sm[oW2h + r * kW2P + j],
               sm[oW2l + r * kW2P + j]);
  }
  for (int i = threadIdx.x; i < C1; i += blockDim.x) vec[i] = d.b1[i];
  for (int i = threadIdx.x; i < C2; i += blockDim.x) {
    vec[C1 + i] = d.b2 ? d.b2[i] : 0.f;
    vec[C1 + C2 + i] = d.w3[i];
  }
  for (int i = threadIdx.x; i < kWarps * 4 * C2; i += blockDim.x) acc[i] = 0.0;
  if constexpr (PASS == PASS_APPLY) {
    // backward weights, bf16-split and unscaled: W2^T as [c1][c2 pairs], W1^T as [cin][c1 pairs]
    for (int i = threadIdx.x; i < C1 * (C2 / 2); i += blockDim.x) {
      const int r = i / (C2 / 2), j = i % (C2 / 2);
      split_pair(d.w2[(2 * j) * C1 + r], d.w2[(2 * j + 1) * C1 + r], SN_FMT_BF16, sm[oW2bh + r * kW2bP + j],
                 sm[oW2bl + r * kW2bP + j]);
    }
    for (int i = threadIdx.x; i < KX * (C1 / 2); i += blockDim.x) {
      const int r = i / (C1 / 2), j = i % (C1 / 2);
      const float v0 = r < d.cin ? d.w1[(2 * j) * d.cin + r] : 0.f, v1 = r < d.cin ? d.w1[(2 * j + 1) * d.cin + r] : 0.f;
      split_pair(v0, v1, SN_FMT_BF16, sm[oW1bh + r * kW1bP + j], sm[oW1bl + r * kW1bP + j]);
    }
    if constexpr (WG) {
      // the constant rows of the staged a1 / x: row C1 (KX) is 1 (bias gradients), the 7 after it 0
      for (int i = threadIdx.x; i < 8 * kSP; i += blockDim.x) {
        const uint32_t one = (i / kSP == 0) ? 0x3F803F80u : 0u;   // bf16 1.0 in both halves
        sm[oA1h + C1 * kSP + i] = one;
        sm[oA1l + C1 * kSP + i] = 0u;
        sm[oXh + KX * kSP + i] = one;
        sm[oXl + KX * kSP + i] = 0u;
      }
    }
  }
  __syncthreads();

  // weight-gradient accumulators of this warp: dW2 rows [32 warp, +32) x 72 columns (64 + ones), dW1 rows [16 warp, +16)
  // x 40 columns (32 + ones)
  float gw2[2][9][4], gw1[5][4];
  if constexpr (WG) {
#pragma unroll
    for (int m = 0; m < 2; ++m)
#pragma unroll
      for (int nt = 0; nt < 9; ++nt)
#pragma unroll
        for (int i = 0; i < 4; ++i) gw2[m][nt][i] = 0.f;
#pragma unroll
    for (int nt = 0; nt < 5; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) gw1[nt][i] = 0.f;
  }

  const long long total_tiles = (long long)d.n * a.tiles_per_img;
  const long long t0 = (long long)blockIdx.x * a.tiles_per_block;
  const long long t1 = t0 + a.tiles_per_block < total_tiles ? t0 + a.tiles_per_block : total_tiles;
  int cur_n = -1;
  const float* mean = vec + C1 + 2 * C2;
  const float* rstd = mean + C2;
  const float* mg = rstd + C2;
  const float* mgy = mg + C2;
  for (long long tile = t0; tile < t1; ++tile) {
    const int n = (int)(tile / a.tiles_per_img);
    if (n != cur_n) {
      if constexpr (PASS == PASS_STATS) {
        if (cur_n >= 0) flush_pairs(a, acc, cur_n, d.stats);
      } else if constexpr (PASS == PASS_REDUCE && NORM) {
        if (cur_n >= 0) flush_pairs(a, acc, cur_n, d.gstats);
      } else {
        __syncthreads();
      }
      if constexpr (NORM && PASS != PASS_STATS) {
        float* mv = vec + C1 + 2 * C2;
        for (int c = threadIdx.x; c < C2; c += blockDim.x) {
          mv[c] = (float)d.stats[((long long)n * C2 + c) * 2];
          mv[C2 + c] = (float)d.stats[((long long)n * C2 + c) * 2 + 1];
          if constexpr (PASS == PASS_APPLY) {
            mv[2 * C2 + c] = (float)(d.gstats[((long long)n * C2 + c) * 2] / d.hw);
            mv[3 * C2 + c] = (float)(d.gstats[((long long)n * C2 + c) * 2 + 1] / d.hw);
          }
        }
      }
      __syncthreads();
      cur_n = n;
    }
    const int r0 = (int)(tile % a.tiles_per_img) * kTile + 16 * warp;
    const bool vg = r0 + g < d.hw, vg8 = r0 + g + 8 < d.hw;
    const long long pg = (long long)n * d.hw + r0 + g, pg8 = pg + 8;
    float z1[8][4], z2[16][4];
    recompute(d, sm, pg, pg8, vg, vg8, lane, z1, z2);
    if constexpr (PASS == PASS_STATS) {
      colsum_add(wacc, lane, [&](int nt, int i) { const bool v = i < 2 ? vg : vg8; return v ? (double)z2[nt][i] : 0.0; });
      colsum_add(wacc + C2, lane, [&](int nt, int i) {
        const bool v = i < 2 ? vg : vg8;
        return v ? (double)z2[nt][i] * (double)z2[nt][i] : 0.0;
      });
      continue;
    }
    // y2 (in z2), then a2 and the logit
#pragma unroll
    for (int nt = 0; nt < 16; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int c = 8 * nt + 2 * t + (i & 1);
        if constexpr (NORM) z2[nt][i] = (z2[nt][i] - mean[c]) * rstd[c];
      }
    const float* w3 = vec + C1 + C2;
    if constexpr (PASS == PASS_FWD) {
      float p0 = 0.f, p1 = 0.f;
#pragma unroll
      for (int nt = 0; nt < 16; ++nt) {
        const int c = 8 * nt + 2 * t;
        p0 = fmaf(w3[c], lrelu(z2[nt][0], d.slope), p0);
        p0 = fmaf(w3[c + 1], lrelu(z2[nt][1], d.slope), p0);
        p1 = fmaf(w3[c], lrelu(z2[nt][2], d.slope), p1);
        p1 = fmaf(w3[c + 1], lrelu(z2[nt][3], d.slope), p1);
      }
      p0 += __shfl_xor_sync(0xffffffffu, p0, 1);
      p1 += __shfl_xor_sync(0xffffffffu, p1, 1);
      p0 += __shfl_xor_sync(0xffffffffu, p0, 2);
      p1 += __shfl_xor_sync(0xffffffffu, p1, 2);
      const float b3 = d.b3 ? d.b3[0] : 0.f;
      if (t == 0) {
        if (vg) d.pred[pg] = p0 + b3;
        if (vg8) d.pred[pg8] = p1 + b3;
      }
      if (d.debug) {   // pre-activations z1 and y2 (tests impose the device's gates on their reference)
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
          const int c = 8 * nt + 2 * t;
          if (vg) { d.debug[pg * (C1 + C2) + c] = z1[nt][0]; d.debug[pg * (C1 + C2) + c + 1] = z1[nt][1]; }
          if (vg8) { d.debug[pg8 * (C1 + C2) + c] = z1[nt][2]; d.debug[pg8 * (C1 + C2) + c + 1] = z1[nt][3]; }
        }
#pragma unroll
        for (int nt = 0; nt < 16; ++nt) {
          const int c = C1 + 8 * nt + 2 * t;
          if (vg) { d.debug[pg * (C1 + C2) + c] = z2[nt][0]; d.debug[pg * (C1 + C2) + c + 1] = z2[nt][1]; }
          if (vg8) { d.debug[pg8 * (C1 + C2) + c] = z2[nt][2]; d.debug[pg8 * (C1 + C2) + c + 1] = z2[nt][3]; }
        }
      }
      continue;
    }
    // ---- backward: g2 = dpred w3 lrelu'(y2); dW3 = sum dpred a2, db3 = sum dpred ----
    const float dp0 = vg ? d.dpred[pg] : 0.f, dp1 = vg8 ? d.dpred[pg8] : 0.f;
    constexpr bool kW3 = (PASS == PASS_REDUCE) || (PASS == PASS_APPLY && !NORM);
    if (kW3 && d.dw3) {
      colsum_add(wacc + 2 * C2, lane, [&](int nt, int i) {
        return (double)((i < 2 ? dp0 : dp1) * lrelu(z2[nt][i], d.slope));
      });
      double s = (double)dp0 + (double)dp1;   // the 4 lanes of a row group hold the same two pixels
#pragma unroll
      for (int o = 4; o < 32; o <<= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) wacc[3 * C2] += s;
    }
    auto g2_at = [&](int nt, int i) {
      return (i < 2 ? dp0 : dp1) * w3[8 * nt + 2 * t + (i & 1)] * gate(z2[nt][i], d.slope);
    };
    if constexpr (PASS == PASS_REDUCE) {
      if constexpr (NORM) {
        colsum_add(wacc, lane, [&](int nt, int i) { return (double)g2_at(nt, i); });
        colsum_add(wacc + C2, lane, [&](int nt, int i) { return (double)g2_at(nt, i) * (double)z2[nt][i]; });
      }
      continue;
    }
    // ---- apply: dz2, dA1 = dz2 W2, g1, dx = g1 W1; stage the tile for the weight gradients ----
    uint32_t dh[8][4], dl[8][4];   // dz2 as the A fragments of dA1's 8 k-chunks
#pragma unroll
    for (int nt = 0; nt < 16; ++nt) {
      float v[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int c = 8 * nt + 2 * t + (i & 1);
        v[i] = g2_at(nt, i);
        if constexpr (NORM) v[i] = rstd[c] * (v[i] - mg[c] - z2[nt][i] * mgy[c]);
        if (!(i < 2 ? vg : vg8)) v[i] = 0.f;
      }
      const int kk = nt >> 1, half = nt & 1;
      split_pair(v[0], v[1], SN_FMT_BF16, dh[kk][2 * half], dl[kk][2 * half]);
      split_pair(v[2], v[3], SN_FMT_BF16, dh[kk][2 * half + 1], dl[kk][2 * half + 1]);
    }
    const int pl = 16 * warp + g;   // this thread's pixel rows inside the block tile: pl, pl + 8
    if constexpr (WG) {
      uint16_t* Dh = reinterpret_cast<uint16_t*>(sm + oDzh);
      uint16_t* Dl = reinterpret_cast<uint16_t*>(sm + oDzl);
      uint16_t* Ah = reinterpret_cast<uint16_t*>(sm + oA1h);
      uint16_t* Al = reinterpret_cast<uint16_t*>(sm + oA1l);
#pragma unroll
      for (int nt = 0; nt < 16; ++nt) {
        const int kk = nt >> 1, half = nt & 1, c = 8 * nt + 2 * t;
        const uint32_t h0 = dh[kk][2 * half], l0 = dl[kk][2 * half], h1 = dh[kk][2 * half + 1], l1 = dl[kk][2 * half + 1];
        Dh[c * 2 * kSP + pl] = (uint16_t)h0; Dh[(c + 1) * 2 * kSP + pl] = (uint16_t)(h0 >> 16);
        Dl[c * 2 * kSP + pl] = (uint16_t)l0; Dl[(c + 1) * 2 * kSP + pl] = (uint16_t)(l0 >> 16);
        Dh[c * 2 * kSP + pl + 8] = (uint16_t)h1; Dh[(c + 1) * 2 * kSP + pl + 8] = (uint16_t)(h1 >> 16);
        Dl[c * 2 * kSP + pl + 8] = (uint16_t)l1; Dl[(c + 1) * 2 * kSP + pl + 8] = (uint16_t)(l1 >> 16);
      }
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const int c = 8 * nt + 2 * t;
        uint32_t h, l;
        split_pair(lrelu(z1[nt][0], d.slope), lrelu(z1[nt][1], d.slope), SN_FMT_BF16, h, l);
        Ah[c * 2 * kSP + pl] = (uint16_t)h; Ah[(c + 1) * 2 * kSP + pl] = (uint16_t)(h >> 16);
        Al[c * 2 * kSP + pl] = (uint16_t)l; Al[(c + 1) * 2 * kSP + pl] = (uint16_t)(l >> 16);
        split_pair(lrelu(z1[nt][2], d.slope), lrelu(z1[nt][3], d.slope), SN_FMT_BF16, h, l);
        Ah[c * 2 * kSP + pl + 8] = (uint16_t)h; Ah[(c + 1) * 2 * kSP + pl + 8] = (uint16_t)(h >> 16);
        Al[c * 2 * kSP + pl + 8] = (uint16_t)l; Al[(c + 1) * 2 * kSP + pl + 8] = (uint16_t)(l >> 16);
      }
    }
    float g1[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
      for (int i = 0; i < 4; ++i) g1[nt][i] = 0.f;
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        const int w = (8 * nt + g) * kW2bP + 8 * kk + t;
        mma_split<true>(g1[nt], dh[kk], dl[kk], sm + oW2bh + w, sm + oW2bl + w, d.nsplit);
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) g1[nt][i] *= gate(z1[nt][i], d.slope);
    }
    uint32_t gh[4][4], gl[4][4];   // g1 as the A fragments of dx's 4 k-chunks
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const int kk = nt >> 1, half = nt & 1;
      split_pair(g1[nt][0], g1[nt][1], SN_FMT_BF16, gh[kk][2 * half], gl[kk][2 * half]);
      split_pair(g1[nt][2], g1[nt][3], SN_FMT_BF16, gh[kk][2 * half + 1], gl[kk][2 * half + 1]);
    }
    if (d.dx) {
#pragma unroll
      for (int nt = 0; nt < KX / 8; ++nt) {
        float o[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          const int w = (8 * nt + g) * kW1bP + 8 * kk + t;
          mma_split<true>(o, gh[kk], gl[kk], sm + oW1bh + w, sm + oW1bl + w, d.nsplit);
        }
        const int c = 8 * nt + 2 * t;
        if (vg && c < d.cin) d.dx[pg * d.dx_pitch + c] = o[0];
        if (vg && c + 1 < d.cin) d.dx[pg * d.dx_pitch + c + 1] = o[1];
        if (vg8 && c < d.cin) d.dx[pg8 * d.dx_pitch + c] = o[2];
        if (vg8 && c + 1 < d.cin) d.dx[pg8 * d.dx_pitch + c + 1] = o[3];
      }
    }
    if constexpr (WG) {
      uint16_t* Gh = reinterpret_cast<uint16_t*>(sm + oG1h);
      uint16_t* Gl = reinterpret_cast<uint16_t*>(sm + oG1l);
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const int kk = nt >> 1, half = nt & 1, c = 8 * nt + 2 * t;
        const uint32_t h0 = gh[kk][2 * half], l0 = gl[kk][2 * half], h1 = gh[kk][2 * half + 1], l1 = gl[kk][2 * half + 1];
        Gh[c * 2 * kSP + pl] = (uint16_t)h0; Gh[(c + 1) * 2 * kSP + pl] = (uint16_t)(h0 >> 16);
        Gl[c * 2 * kSP + pl] = (uint16_t)l0; Gl[(c + 1) * 2 * kSP + pl] = (uint16_t)(l0 >> 16);
        Gh[c * 2 * kSP + pl + 8] = (uint16_t)h1; Gh[(c + 1) * 2 * kSP + pl + 8] = (uint16_t)(h1 >> 16);
        Gl[c * 2 * kSP + pl + 8] = (uint16_t)l1; Gl[(c + 1) * 2 * kSP + pl + 8] = (uint16_t)(l1 >> 16);
      }
      // x (bf16 twin) of the warp's 16 pixels, transposed: lane = channel
      uint16_t* Xh = reinterpret_cast<uint16_t*>(sm + oXh);
      uint16_t* Xl = reinterpret_cast<uint16_t*>(sm + oXl);
      const uint16_t* xbh = (const uint16_t*)d.xb_hi;
      const uint16_t* xbl = (const uint16_t*)d.xb_lo;
      for (int r = 0; r < 16; ++r) {
        const bool v = r0 + r < d.hw;
        const long long p = (long long)n * d.hw + r0 + r;
        const bool in = v && lane < d.x_c;
        Xh[lane * 2 * kSP + 16 * warp + r] = in ? xbh[p * d.x_pitch + lane] : (uint16_t)0;
        Xl[lane * 2 * kSP + 16 * warp + r] = in ? xbl[p * d.x_pitch + lane] : (uint16_t)0;
      }
      __syncthreads();
      // dW2 (+ db2) += dz2^T [a1; 1]   and   dW1 (+ db1) += g1^T [x; 1]   over the tile's 64 pixels.  Each output
      // fragment's 64-pixel partial runs in a fresh MMA accumulator (the tensor cores' adds truncate) and is then
      // promoted into the block's sums with round-to-nearest adds, so the error stays flat over the hundreds of tiles a
      // block sums at training shapes.
      auto tile_partial = [&](float (&acc)[4], int a_h, int a_l, int r, int b_h, int b_l, int nt) {
        float p[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int kc = 0; kc < kTile / 16; ++kc) {
          uint32_t ah[4], al[4];
          const int row = r * kSP + 8 * kc + t;
          ah[0] = sm[a_h + row]; ah[1] = sm[a_h + row + 8 * kSP];
          ah[2] = sm[a_h + row + 4]; ah[3] = sm[a_h + row + 8 * kSP + 4];
          al[0] = sm[a_l + row]; al[1] = sm[a_l + row + 8 * kSP];
          al[2] = sm[a_l + row + 4]; al[3] = sm[a_l + row + 8 * kSP + 4];
          const int w = (8 * nt + g) * kSP + 8 * kc + t;
          mma_split<true>(p, ah, al, sm + b_h + w, sm + b_l + w, d.nsplit);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[i] = __fadd_rn(acc[i], p[i]);
      };
#pragma unroll
      for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int nt = 0; nt < 9; ++nt) tile_partial(gw2[m][nt], oDzh, oDzl, 32 * warp + 16 * m + g, oA1h, oA1l, nt);
#pragma unroll
      for (int nt = 0; nt < 5; ++nt) tile_partial(gw1[nt], oG1h, oG1l, 16 * warp + g, oXh, oXl, nt);
      __syncthreads();   // the staging buffers are rewritten by the next tile
    }
  }
  // ---- epilogue: the block's remaining sums ----
  if constexpr (PASS == PASS_STATS) {
    if (cur_n >= 0) flush_pairs(a, acc, cur_n, d.stats);
    return;
  }
  if constexpr (PASS == PASS_REDUCE && NORM) {
    if (cur_n >= 0) flush_pairs(a, acc, cur_n, d.gstats);
  }
  const WgSlots S = wg_slots(d.slots, d.n, d.cin);
  constexpr bool kW3 = (PASS == PASS_REDUCE) || (PASS == PASS_APPLY && !NORM);
  if (kW3 && d.dw3) {
    __syncthreads();
    for (int c = threadIdx.x; c <= C2; c += blockDim.x) {
      const int slot = c < C2 ? 2 * C2 + c : 3 * C2;
      double s = 0.0;
      for (int w = 0; w < kWarps; ++w) s += acc[w * 4 * C2 + slot];
      if (c < C2) add_wgrad(a, S.dw3, C2, c, d.dw3, (float)s);
      else if (d.db3) add_wgrad(a, S.db3, 1, 0, d.db3, (float)s);
    }
  }
  if constexpr (WG) {
#pragma unroll
    for (int m = 0; m < 2; ++m)
#pragma unroll
      for (int nt = 0; nt < 9; ++nt)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int r = 32 * warp + 16 * m + g + (i >= 2 ? 8 : 0), c = 8 * nt + 2 * t + (i & 1);
          if (c < C1) add_wgrad(a, S.dw2, C2 * C1, r * C1 + c, d.dw2, gw2[m][nt][i]);
          else if (c == C1 && d.db2) add_wgrad(a, S.db2, C2, r, d.db2, gw2[m][nt][i]);
        }
#pragma unroll
    for (int nt = 0; nt < 5; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int r = 16 * warp + g + (i >= 2 ? 8 : 0), c = 8 * nt + 2 * t + (i & 1);
        if (c < d.cin) add_wgrad(a, S.dw1, C1 * d.cin, r * d.cin + c, d.dw1, gw1[nt][i]);
        else if (c == KX) add_wgrad(a, S.db1, C1, r, d.db1, gw1[nt][i]);
      }
  }
}

template <int PASS, bool NORM, bool WG>
int launch(const sn_pixel_desc* d, cudaStream_t st) {
  Args a;
  a.d = *d;
  a.tiles_per_img = (d->hw + kTile - 1) / kTile;
  const long long tiles = (long long)d->n * a.tiles_per_img;
  a.tiles_per_block = (int)((tiles + kBlocks - 1) / kBlocks);
  const size_t smem = (size_t)(PASS == PASS_APPLY ? oBwdEnd : oFwdEnd) * 4;
  // set on every launch (a host-side call, no stream work): the attribute is per device, and a process may drive several
  SN_CHECK_CUDA(cudaFuncSetAttribute(pixel_kernel<PASS, NORM, WG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  pixel_kernel<PASS, NORM, WG><<<kBlocks, kThreads, smem, st>>>(a);
  sn_count_launch(1);
  SN_CHECK_CUDA(cudaGetLastError());
  return SN_OK;
}

int check_desc(const sn_pixel_desc* d, const char* what) {
  SN_REQUIRE(d && d->x_hi && d->x_lo && d->w1 && d->b1 && d->w2 && d->w3 && d->scale1 && d->scale2,
             "%s: null pointer", what);
  SN_REQUIRE(d->n >= 1 && d->hw >= 1 && d->cin >= 1 && d->cin <= d->x_c && (d->x_c == 16 || d->x_c == KX) &&
                 d->x_pitch >= d->x_c && d->x_pitch % 2 == 0,
             "%s: cin %d, x_c %d (16 or 32), pitch %d", what, d->cin, d->x_c, d->x_pitch);
  // x and its twin are read as 32-bit words (channel pairs): an odd channel offset would issue misaligned loads
  SN_REQUIRE(((uintptr_t)d->x_hi | (uintptr_t)d->x_lo | (uintptr_t)d->xb_hi | (uintptr_t)d->xb_lo) % 4 == 0,
             "%s: x and its bf16 twin must be 4-byte aligned (an even channel offset)", what);
  SN_REQUIRE(d->nsplit == 1 || d->nsplit == 3, "%s: nsplit must be 1 or 3", what);
  SN_REQUIRE(!d->norm || d->stats, "%s: instance norm needs the statistics buffer", what);
  SN_REQUIRE(!d->slots || d->slots_cap >= sn_pixel_det_slots(d->n, d->cin), "%s: %lld slots given, %lld needed", what,
             d->slots_cap, sn_pixel_det_slots(d->n, d->cin));
  return SN_OK;
}

}  // namespace

extern "C" {

long long sn_pixel_det_slots(int n, int cin) {
  // doubles: the statistics' [blocks][n][C2][2], then the weight gradients' float regions
  const long long floats = (long long)kBlocks * (C2 * C1 + C2 + C1 * cin + C1 + C2 + 1);
  return (long long)kBlocks * n * C2 * 2 + (floats + 1) / 2;
}

int sn_pixel_fwd_stats(const sn_pixel_desc* d, void* stream) {
  if (int rc = check_desc(d, "pixel_fwd_stats")) return rc;
  SN_REQUIRE(d->norm, "pixel_fwd_stats: only with instance norm");
  cudaStream_t st = (cudaStream_t)stream;
  const long long count = (long long)d->n * C2 * 2;
  SN_CHECK_CUDA(cudaMemsetAsync(d->stats, 0, count * sizeof(double), st));
  if (d->slots) SN_CHECK_CUDA(cudaMemsetAsync(d->slots, 0, (size_t)kBlocks * count * sizeof(double), st));
  if (int rc = launch<PASS_STATS, true, false>(d, st)) return rc;
  if (d->slots) {
    SN_CHECK_CUDA(det_sum_slots(d->slots, kBlocks, count, d->stats, st));
    sn_count_launch(1);
  }
  return sn_stats_finalize(d->stats, d->n * C2, d->hw, d->eps, stream);
}

int sn_pixel_fwd(const sn_pixel_desc* d, void* stream) {
  if (int rc = check_desc(d, "pixel_fwd")) return rc;
  SN_REQUIRE(d->pred, "pixel_fwd: null pred");
  cudaStream_t st = (cudaStream_t)stream;
  return d->norm ? launch<PASS_FWD, true, false>(d, st) : launch<PASS_FWD, false, false>(d, st);
}

int sn_pixel_bwd_reduce(const sn_pixel_desc* d, void* stream) {
  if (int rc = check_desc(d, "pixel_bwd_reduce")) return rc;
  SN_REQUIRE(d->norm && d->gstats && d->dpred, "pixel_bwd_reduce: instance norm, gstats and dpred");
  cudaStream_t st = (cudaStream_t)stream;
  const long long count = (long long)d->n * C2 * 2;
  SN_CHECK_CUDA(cudaMemsetAsync(d->gstats, 0, count * sizeof(double), st));
  if (d->slots) SN_CHECK_CUDA(cudaMemsetAsync(d->slots, 0, (size_t)kBlocks * count * sizeof(double), st));
  if (int rc = launch<PASS_REDUCE, true, false>(d, st)) return rc;
  if (d->slots) {
    SN_CHECK_CUDA(det_sum_slots(d->slots, kBlocks, count, d->gstats, st));
    sn_count_launch(1);
    const WgSlots S = wg_slots(d->slots, d->n, d->cin);
    if (d->dw3) {
      SN_CHECK_CUDA(det_sum_slots(S.dw3, kBlocks, C2, d->dw3, st));
      sn_count_launch(1);
    }
    if (d->db3) {
      SN_CHECK_CUDA(det_sum_slots(S.db3, kBlocks, 1, d->db3, st));
      sn_count_launch(1);
    }
  }
  return SN_OK;
}

int sn_pixel_bwd_apply(const sn_pixel_desc* d, void* stream) {
  if (int rc = check_desc(d, "pixel_bwd_apply")) return rc;
  SN_REQUIRE(d->dpred && (!d->norm || d->gstats), "pixel_bwd_apply: dpred (and gstats with instance norm)");
  const bool wg = d->dw1 != nullptr;
  SN_REQUIRE(wg == (d->dw2 != nullptr) && (!wg || (d->db1 && d->xb_hi && d->xb_lo)),
             "pixel_bwd_apply: dw1, db1, dw2 and the bf16 twin of x go together");
  SN_REQUIRE(wg || d->dx, "pixel_bwd_apply: nothing to compute");
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  if (d->norm) rc = wg ? launch<PASS_APPLY, true, true>(d, st) : launch<PASS_APPLY, true, false>(d, st);
  else rc = wg ? launch<PASS_APPLY, false, true>(d, st) : launch<PASS_APPLY, false, false>(d, st);
  if (rc) return rc;
  if (d->slots) {
    // the slots this pass wrote: dW1 / dW2 with the weight gradients, dw3 / db3 here only without instance norm (the
    // reduce pass sums them otherwise), with or without dW1 / dW2
    const WgSlots S = wg_slots(d->slots, d->n, d->cin);
    struct { const float* s; long long count; float* dst; } sums[] = {
        {S.dw2, C2 * C1, wg ? d->dw2 : nullptr}, {S.db2, C2, wg ? d->db2 : nullptr},
        {S.dw1, (long long)C1 * d->cin, wg ? d->dw1 : nullptr}, {S.db1, C1, wg ? d->db1 : nullptr},
        {S.dw3, C2, d->norm ? nullptr : d->dw3}, {S.db3, 1, d->norm ? nullptr : d->db3}};
    for (auto& s : sums) {
      if (!s.dst) continue;
      SN_CHECK_CUDA(det_sum_slots(s.s, kBlocks, s.count, s.dst, st));
      sn_count_launch(1);
    }
  }
  return SN_OK;
}

}  // extern "C"
