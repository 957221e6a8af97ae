// swapnet_b200 — the one-output-channel conv (PatchGAN logits, modules/discriminators.py:131:
// Conv2d(ndf*8, 1, kernel_size=4, stride=1, padding=1)).
//
// A conv with ONE output channel is an HBM-bound op (1 GMAC over a 260 MB input at batch 32): a GEMM with N = 1 (or the
// N = 16 of the tap factorisation) leaves the tensor core idle behind its operand loads.  It runs on the CUDA cores at
// stream speed through the factorisation
//   P[px, t]  = sum_c x[px, c] * W[0, c, t]                (to_one_fwd_kernel: x is read once)
//   y[o]      = bias + sum_t P[o + off_t, t]               (tap_sum_fwd)
// and backward through its adjoint, with dP[px, t] = dy[px - off_t] gathered on the fly:
//   dW[0,c,t] = sum_px x[px, c] dP[px, t]                  (to_one_wgrad_kernel)
//   dx[px, c] = sum_t dP[px, t] W[0, c, t]                 (to_one_dgrad_kernel)
// x arrives as fp16-split planes (hi + lo = 22 mantissa bits), products and sums are fp32 FMAs.
#include "common.cuh"
#include "../../include/swapnet_b200.h"

void sn_count_launch(int n);

namespace {

constexpr int kThreads = 256;

inline int grid_for(long long total) {
  long long g = (total + kThreads - 1) / kThreads;
  if (g > SN_NUM_SMS * 16) g = SN_NUM_SMS * 16;
  return g < 1 ? 1 : (int)g;
}

__global__ void tap_sum_fwd_kernel(const float* __restrict__ P, int ppitch, int N, int H, int W, int K, int pad,
                                   const float* __restrict__ bias, float* __restrict__ y, int ypitch) {
  const int OH = H + 2 * pad - K + 1, OW = W + 2 * pad - K + 1;
  const long long total = (long long)N * OH * OW;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int ow = (int)(i % OW), oh = (int)((i / OW) % OH);
    const long long n = i / ((long long)OW * OH);
    float acc = 0.f;
    for (int kh = 0; kh < K; ++kh) {
      const int h = oh + kh - pad;
      if (h < 0 || h >= H) continue;
      for (int kw = 0; kw < K; ++kw) {
        const int w = ow + kw - pad;
        if (w < 0 || w >= W) continue;
        acc += P[((n * H + h) * W + w) * ppitch + kh * K + kw];
      }
    }
    y[i * ypitch] = acc + (bias ? bias[0] : 0.f);
  }
}

// ---- CUDA-core kernels -----------------------------------------------------------------------------------------
// decode 8 consecutive 16-bit words (hi + lo) into floats
__device__ __forceinline__ void load8(const uint16_t* __restrict__ hi, const uint16_t* __restrict__ lo, long long off,
                                      int fmt, float v[8]) {
  const uint4 a = *reinterpret_cast<const uint4*>(hi + off);
  const uint4 b = lo ? *reinterpret_cast<const uint4*>(lo + off) : make_uint4(0, 0, 0, 0);
  const uint32_t wa[4] = {a.x, a.y, a.z, a.w}, wb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    v[2 * j] = decode16((uint16_t)(wa[j] & 0xFFFF), fmt) + (lo ? decode16((uint16_t)(wb[j] & 0xFFFF), fmt) : 0.f);
    v[2 * j + 1] = decode16((uint16_t)(wa[j] >> 16), fmt) + (lo ? decode16((uint16_t)(wb[j] >> 16), fmt) : 0.f);
  }
}

// P[px, t] = sum_c x[px, c] W[c*T + t]; one warp = kPx pixels, lane = 8 channels of every 256-channel chunk.
// smem: W transposed to [t][C] so that a lane's 8 channels are two conflict-free LDS.128.
constexpr int kPx = 2;
template <int T>
__global__ void __launch_bounds__(256) to_one_fwd_kernel(const uint16_t* __restrict__ xhi, const uint16_t* __restrict__ xlo,
                                                         int xpitch, int xfmt, long long npix, int C,
                                                         const float* __restrict__ W, float* __restrict__ P, int ppitch) {
  extern __shared__ float Ws[];   // [T][C]
  for (int i = threadIdx.x; i < C * T; i += blockDim.x) Ws[(i % T) * C + i / T] = W[i];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  for (long long p0 = ((long long)blockIdx.x * wpb + warp) * kPx; p0 < npix; p0 += (long long)gridDim.x * wpb * kPx) {
    float acc[kPx][T];
#pragma unroll
    for (int q = 0; q < kPx; ++q)
#pragma unroll
      for (int t = 0; t < T; ++t) acc[q][t] = 0.f;
    for (int c0 = lane * 8; c0 < C; c0 += 256) {
      float xv[kPx][8];
#pragma unroll
      for (int q = 0; q < kPx; ++q) {
        if (p0 + q < npix) load8(xhi, xlo, (p0 + q) * xpitch + c0, xfmt, xv[q]);
        else {
#pragma unroll
          for (int j = 0; j < 8; ++j) xv[q][j] = 0.f;
        }
      }
#pragma unroll
      for (int t = 0; t < T; ++t) {
        const float4 w0 = *reinterpret_cast<const float4*>(Ws + t * C + c0);
        const float4 w1 = *reinterpret_cast<const float4*>(Ws + t * C + c0 + 4);
        const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
        for (int q = 0; q < kPx; ++q)
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[q][t] = fmaf(xv[q][j], wv[j], acc[q][t]);
      }
    }
#pragma unroll
    for (int q = 0; q < kPx; ++q)
#pragma unroll
      for (int t = 0; t < T; ++t) {
        float v = acc[q][t];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == t && p0 + q < npix) P[(p0 + q) * ppitch + t] = v;
      }
  }
}

// dP[(n,h,w), (kh,kw)] = dy[n, h - kh + pad, w - kw + pad] (0 outside), dy = channel 0 of split planes
struct DyView { const uint16_t* hi; const uint16_t* lo; int pitch, fmt, H, W, OH, OW, K, pad; };
__device__ __forceinline__ float dp_at(const DyView& d, long long n, int h, int w, int kh, int kw) {
  const int oh = h - kh + d.pad, ow = w - kw + d.pad;
  if (oh < 0 || oh >= d.OH || ow < 0 || ow >= d.OW) return 0.f;
  const long long o = ((n * d.OH + oh) * d.OW + ow) * d.pitch;
  return decode16(d.hi[o], d.fmt) + (d.lo ? decode16(d.lo[o], d.fmt) : 0.f);
}

// dW[c*T + t] += sum over this block's pixels of x[px, c] dP[px, t].  block = (C/4 threads.x, rows threads.y):
// thread = 4 channels, strided over the block's pixel range; T accumulators per channel.  The block first gathers its
// pixels' dP values (T per pixel) into shared memory, so the main loop is 2 vector loads + T broadcast LDS + 4T FMAs.
// DET: the block's sums go to slots[blockIdx.x][c*T + t] instead (det_sum_slots adds them in block order).
constexpr int kWgPix = 256;     // pixels staged per round
template <int K, bool DET>
__global__ void __launch_bounds__(256) to_one_wgrad_kernel(const uint16_t* __restrict__ xhi, const uint16_t* __restrict__ xlo,
                                                           int xpitch, int xfmt, long long npix, int C, const DyView d,
                                                           float* __restrict__ dW, float* __restrict__ slots) {
  constexpr int T = K * K;
  extern __shared__ float smem[];
  float* dps = smem;                       // [kWgPix][T]
  float* red = smem + kWgPix * T;          // [rows - 1][C*T] partial sums of the pixel rows > 0
  const int c = threadIdx.x * 4;
  const int tid = threadIdx.y * blockDim.x + threadIdx.x, nthr = blockDim.x * blockDim.y;
  const long long per = (npix + gridDim.x - 1) / gridDim.x;
  const long long p0 = blockIdx.x * per, p1 = p0 + per < npix ? p0 + per : npix;
  float acc[4][T];
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int t = 0; t < T; ++t) acc[j][t] = 0.f;
  const long long HW = (long long)d.H * d.W;
  for (long long q0 = p0; q0 < p1; q0 += kWgPix) {
    const int cnt = (int)(p1 - q0 < kWgPix ? p1 - q0 : kWgPix);
    __syncthreads();
    for (int i = tid; i < cnt * T; i += nthr) {
      const long long p = q0 + i / T;
      const int t = i % T;
      const long long n = p / HW;
      const int r = (int)(p - n * HW), h = r / d.W, w = r - h * d.W;
      dps[i] = dp_at(d, n, h, w, t / K, t % K);
    }
    __syncthreads();
    for (int pl = threadIdx.y; pl < cnt; pl += blockDim.y) {
      const long long p = q0 + pl;
      const uint2 a = *reinterpret_cast<const uint2*>(xhi + p * xpitch + c);
      const uint2 b = xlo ? *reinterpret_cast<const uint2*>(xlo + p * xpitch + c) : make_uint2(0, 0);
      float xv[4];
      xv[0] = decode16((uint16_t)(a.x & 0xFFFF), xfmt) + (xlo ? decode16((uint16_t)(b.x & 0xFFFF), xfmt) : 0.f);
      xv[1] = decode16((uint16_t)(a.x >> 16), xfmt) + (xlo ? decode16((uint16_t)(b.x >> 16), xfmt) : 0.f);
      xv[2] = decode16((uint16_t)(a.y & 0xFFFF), xfmt) + (xlo ? decode16((uint16_t)(b.y & 0xFFFF), xfmt) : 0.f);
      xv[3] = decode16((uint16_t)(a.y >> 16), xfmt) + (xlo ? decode16((uint16_t)(b.y >> 16), xfmt) : 0.f);
      const float4* g4 = reinterpret_cast<const float4*>(dps + pl * T);
#pragma unroll
      for (int tq = 0; tq < T / 4; ++tq) {
        const float4 g = g4[tq];             // the same address for the whole pixel row: a broadcast
        const float gg[4] = {g.x, g.y, g.z, g.w};
#pragma unroll
        for (int u = 0; u < 4; ++u)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[j][tq * 4 + u] = fmaf(xv[j], gg[u], acc[j][tq * 4 + u]);
      }
    }
  }
  // rows 1.. hand their partial sums to row 0 through smem, row 0 adds its own and issues one atomic per (c, t)
  const int CT = C * T;
  __syncthreads();
  if (threadIdx.y > 0) {
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int t = 0; t < T; ++t) red[(threadIdx.y - 1) * CT + (c + j) * T + t] = acc[j][t];
  }
  __syncthreads();
  if (threadIdx.y == 0) {
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int t = 0; t < T; ++t) {
        float v = acc[j][t];
        for (int r = 0; r + 1 < (int)blockDim.y; ++r) v += red[r * CT + (c + j) * T + t];
        if constexpr (DET) slots[(long long)blockIdx.x * CT + (c + j) * T + t] = v;
        else atomicAdd(dW + (c + j) * T + t, v);
      }
  }
}

// dx[px, c] = sum_t dP[px, t] W[c*T + t]; one warp = one pixel (its T gathered dy values are shared by all lanes),
// lane = channel quads lane, lane + 32, ... (512-B coalesced stores)
template <int K>
__global__ void __launch_bounds__(256) to_one_dgrad_kernel(const DyView d, long long npix, int C, const float* __restrict__ W,
                                                           float* __restrict__ dx, int dxpitch) {
  constexpr int T = K * K;
  extern __shared__ float Ws[];   // [T][C]
  for (int i = threadIdx.x; i < C * T; i += blockDim.x) Ws[(i % T) * C + i / T] = W[i];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const int Q = C >> 2;
  const long long HW = (long long)d.H * d.W;
  for (long long p = (long long)blockIdx.x * wpb + warp; p < npix; p += (long long)gridDim.x * wpb) {
    const long long n = p / HW;
    const int r = (int)(p - n * HW), h = r / d.W, w = r - h * d.W;
    float g[T];
#pragma unroll
    for (int kh = 0; kh < K; ++kh)
#pragma unroll
      for (int kw = 0; kw < K; ++kw) g[kh * K + kw] = dp_at(d, n, h, w, kh, kw);
    for (int q = lane; q < Q; q += 32) {
      const int c = q << 2;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int t = 0; t < T; ++t) {
        const float4 wv = *reinterpret_cast<const float4*>(Ws + t * C + c);
        acc.x = fmaf(g[t], wv.x, acc.x); acc.y = fmaf(g[t], wv.y, acc.y);
        acc.z = fmaf(g[t], wv.z, acc.z); acc.w = fmaf(g[t], wv.w, acc.w);
      }
      *reinterpret_cast<float4*>(dx + p * dxpitch + c) = acc;
    }
  }
}

}  // namespace

#define LAUNCH_CHECK()                         \
  do {                                         \
    sn_count_launch(1);                        \
    SN_CHECK_CUDA(cudaGetLastError());         \
  } while (0)

extern "C" {

int sn_tap_sum_fwd(const float* p, int p_pitch, int n, int h, int w, int k, int pad, const float* bias, float* y,
                   int y_pitch, void* stream) {
  SN_REQUIRE(p && y && k >= 1 && k * k <= p_pitch, "tap_sum: bad arguments");
  const long long total = (long long)n * (h + 2 * pad - k + 1) * (w + 2 * pad - k + 1);
  tap_sum_fwd_kernel<<<grid_for(total), kThreads, 0, (cudaStream_t)stream>>>(p, p_pitch, n, h, w, k, pad, bias, y,
                                                                             y_pitch);
  LAUNCH_CHECK();
  return SN_OK;
}

static int fill_dy(DyView* d, const void* dy_hi, const void* dy_lo, int dy_pitch, int dy_fmt, int h, int w, int k, int pad) {
  d->hi = (const uint16_t*)dy_hi; d->lo = (const uint16_t*)dy_lo; d->pitch = dy_pitch; d->fmt = dy_fmt;
  d->H = h; d->W = w; d->OH = h + 2 * pad - k + 1; d->OW = w + 2 * pad - k + 1; d->K = k; d->pad = pad;
  return SN_OK;
}

int sn_to_one_fwd(const void* x_hi, const void* x_lo, int x_pitch, int x_fmt, long long npix, int c, const float* weight,
                  int k, float* p, int p_pitch, void* stream) {
  SN_REQUIRE(x_hi && weight && p && k == 4 && c % 8 == 0 && x_pitch % 8 == 0 && p_pitch >= 16 &&
                 ((uintptr_t)x_hi & 15) == 0 && ((uintptr_t)x_lo & 15) == 0,
             "to_one_fwd: k = 4, channels %% 8 == 0, 16-B aligned planes");
  const size_t smem = (size_t)c * 16 * sizeof(float);
  static bool attr = false;
  if (!attr) {
    SN_CHECK_CUDA(cudaFuncSetAttribute(to_one_fwd_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    SN_CHECK_CUDA(cudaFuncSetAttribute(to_one_dgrad_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    SN_CHECK_CUDA(cudaFuncSetAttribute(to_one_wgrad_kernel<4, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr = true;
  }
  SN_REQUIRE(smem <= 96 * 1024, "to_one_fwd: too many channels (%d)", c);
  long long blocks = (npix + 8 * kPx - 1) / (8 * kPx);
  if (blocks > SN_NUM_SMS * 4) blocks = SN_NUM_SMS * 4;
  to_one_fwd_kernel<16><<<(int)blocks, 256, smem, (cudaStream_t)stream>>>((const uint16_t*)x_hi, (const uint16_t*)x_lo, x_pitch,
                                                                        x_fmt, npix, c, weight, p, p_pitch);
  LAUNCH_CHECK();
  return SN_OK;
}

static int to_one_wgrad_impl(const void* x_hi, const void* x_lo, int x_pitch, int x_fmt, int n, int h, int w, int c,
                             const void* dy_hi, const void* dy_lo, int dy_pitch, int dy_fmt, int k, int pad, float* dw,
                             float* slots, long long slots_cap, cudaStream_t stream) {
  SN_REQUIRE(x_hi && dy_hi && dw && k == 4 && c % 4 == 0 && c <= 1024 && x_pitch % 4 == 0 &&
                 ((uintptr_t)x_hi & 7) == 0 && ((uintptr_t)x_lo & 7) == 0,
             "to_one_wgrad: k = 4, channels %% 4 == 0 and <= 1024");
  DyView d;
  fill_dy(&d, dy_hi, dy_lo, dy_pitch, dy_fmt, h, w, k, pad);
  const int bx = c / 4;
  int by = 256 / bx;
  if (by < 1) by = 1;
  const long long npix = (long long)n * h * w;
  const size_t smem = ((size_t)(by - 1) * c * 16 + (size_t)kWgPix * 16) * sizeof(float);
  SN_REQUIRE(smem <= 200 * 1024, "to_one_wgrad: reduction scratch too large");
  if (smem > 48 * 1024) {   // attribute set by the first forward call; set here too for backward-only use
    static bool attr = false;
    if (!attr) {
      SN_CHECK_CUDA(cudaFuncSetAttribute(to_one_wgrad_kernel<4, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
      SN_CHECK_CUDA(cudaFuncSetAttribute(to_one_wgrad_kernel<4, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
      attr = true;
    }
  }
  long long blocks = npix / kWgPix;
  if (blocks > SN_NUM_SMS * 4) blocks = SN_NUM_SMS * 4;
  if (blocks < 1) blocks = 1;
  if (!slots) {
    to_one_wgrad_kernel<4, false><<<(int)blocks, dim3(bx, by), smem, stream>>>(
        (const uint16_t*)x_hi, (const uint16_t*)x_lo, x_pitch, x_fmt, npix, c, d, dw, nullptr);
    LAUNCH_CHECK();
    return SN_OK;
  }
  SN_REQUIRE(blocks * c * 16 <= slots_cap, "to_one_wgrad_det: %lld slots needed, %lld given", blocks * c * 16, slots_cap);
  to_one_wgrad_kernel<4, true><<<(int)blocks, dim3(bx, by), smem, stream>>>(
      (const uint16_t*)x_hi, (const uint16_t*)x_lo, x_pitch, x_fmt, npix, c, d, dw, slots);
  LAUNCH_CHECK();
  SN_CHECK_CUDA(det_sum_slots(slots, (int)blocks, (long long)c * 16, dw, stream));
  LAUNCH_CHECK();
  return SN_OK;
}

int sn_to_one_wgrad(const void* x_hi, const void* x_lo, int x_pitch, int x_fmt, int n, int h, int w, int c,
                    const void* dy_hi, const void* dy_lo, int dy_pitch, int dy_fmt, int k, int pad, float* dw,
                    void* stream) {
  return to_one_wgrad_impl(x_hi, x_lo, x_pitch, x_fmt, n, h, w, c, dy_hi, dy_lo, dy_pitch, dy_fmt, k, pad, dw, nullptr, 0,
                           (cudaStream_t)stream);
}

int sn_to_one_wgrad_det(const void* x_hi, const void* x_lo, int x_pitch, int x_fmt, int n, int h, int w, int c,
                        const void* dy_hi, const void* dy_lo, int dy_pitch, int dy_fmt, int k, int pad, float* dw,
                        float* slots, long long slots_cap, void* stream) {
  SN_REQUIRE(slots, "to_one_wgrad_det: null slots");
  return to_one_wgrad_impl(x_hi, x_lo, x_pitch, x_fmt, n, h, w, c, dy_hi, dy_lo, dy_pitch, dy_fmt, k, pad, dw, slots,
                           slots_cap, (cudaStream_t)stream);
}

long long sn_to_one_wgrad_det_slots(int c) { return (long long)SN_NUM_SMS * 4 * c * 16; }

int sn_to_one_dgrad(const void* dy_hi, const void* dy_lo, int dy_pitch, int dy_fmt, int n, int h, int w, int c,
                    const float* weight, int k, int pad, float* dx, int dx_pitch, void* stream) {
  SN_REQUIRE(dy_hi && weight && dx && k == 4 && c % 4 == 0 && dx_pitch % 4 == 0 && ((uintptr_t)dx & 15) == 0,
             "to_one_dgrad: k = 4, channels %% 4 == 0, 16-B aligned dx");
  DyView d;
  fill_dy(&d, dy_hi, dy_lo, dy_pitch, dy_fmt, h, w, k, pad);
  const size_t smem = (size_t)c * 16 * sizeof(float);
  SN_REQUIRE(smem <= 96 * 1024, "to_one_dgrad: too many channels (%d)", c);
  static bool attr = false;
  if (!attr) {
    SN_CHECK_CUDA(cudaFuncSetAttribute(to_one_dgrad_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    attr = true;
  }
  const long long npix = (long long)n * h * w;
  long long blocks = (npix + 7) / 8;
  if (blocks > SN_NUM_SMS * 8) blocks = SN_NUM_SMS * 8;
  to_one_dgrad_kernel<4><<<(int)blocks, kThreads, smem, (cudaStream_t)stream>>>(d, npix, c, weight, dx, dx_pitch);
  LAUNCH_CHECK();
  return SN_OK;
}

}  // extern "C"
