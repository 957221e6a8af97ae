// swapnet_b200 — element-wise kernels of the VGG16 perceptual loss (sm_90a).
//
// Reference: modules/losses/perceptual.py:6-79 as used by models/texture_model.py:68-69,171-176.
//   get_features:  x <- 2x - 1; five slices of vgg16.features[0:30] (conv3x3+bias+ReLU, MaxPool2d(2));
//                  every tap is L2-normalised over channels: f = x / (sqrt(sum_c x^2) + 1e-8)
//   content loss:  sum over the 5 taps of MSELoss(f_out, f_target)
//   style loss:    5 x MSELoss(gram(out), gram(target)) with the Gram matrix of the RAW images viewed as
//                  [B*3, H*W] (perceptual.py:58-63 — not of the features)
// The 3x3 convolutions themselves run on the tap-GEMM kernel (gemm_tc.cu); this file holds the HBM-bound
// pieces around them.  All tensors NHWC fp32 with explicit pixel pitch unless noted.
#include "common.cuh"
#include "../../include/swapnet_b200.h"

void sn_count_launch(int n);

namespace {

constexpr int kThreads = 256;

inline int grid_for(long long total, int threads = kThreads) {
  long long g = (total + threads - 1) / threads;
  if (g > SN_NUM_SMS * 16) g = SN_NUM_SMS * 16;
  if (g < 1) g = 1;
  return (int)g;
}

__device__ __forceinline__ uint2 pack4(const uint16_t* x) {
  uint2 r;
  r.x = x[0] | ((uint32_t)x[1] << 16);
  r.y = x[2] | ((uint32_t)x[3] << 16);
  return r;
}

// ---------------------------------------------------------------------------------
// affine_pack: planes[n,h,w,0:c_fill] = split(mul * src + add), zero beyond c (c_fill = 16)
// ---------------------------------------------------------------------------------
__global__ void affine_pack_kernel(const float* __restrict__ src, int layout, int pitch, int N, int C, long long HW,
                                   float mul, float add, uint16_t* __restrict__ hi, uint16_t* __restrict__ lo,
                                   int dpitch, int coff, int fmt) {
  const long long total = (long long)N * HW;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long n = i / HW, p = i - n * HW;
    uint16_t h[16], l[16];
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      float v = 0.f;
      if (c < C) {
        const float s = layout == SN_LAYOUT_NCHW ? src[(n * C + c) * HW + p] : src[i * pitch + c];
        v = __fadd_rn(__fmul_rn(mul, s), add);
      }
      split16(v, fmt, h[c], l[c]);
    }
    uint4* dh = reinterpret_cast<uint4*>(hi + i * dpitch + coff);
    uint4* dl = reinterpret_cast<uint4*>(lo + i * dpitch + coff);
    auto pk8 = [](const uint16_t* x) {
      uint4 r;
      r.x = x[0] | ((uint32_t)x[1] << 16); r.y = x[2] | ((uint32_t)x[3] << 16);
      r.z = x[4] | ((uint32_t)x[5] << 16); r.w = x[6] | ((uint32_t)x[7] << 16);
      return r;
    };
    dh[0] = pk8(h); dh[1] = pk8(h + 8);
    dl[0] = pk8(l); dl[1] = pk8(l + 8);
  }
}

// ---------------------------------------------------------------------------------
// ReLU + MaxPool2d(2) forward: out[n, h/2, w/2, c] = max over the 2x2 window of relu(y)
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) relu_pool_fwd_kernel(const float* __restrict__ y, int ypitch, int N,
                                                                  int H, int W, int C, uint16_t* __restrict__ hi,
                                                                  uint16_t* __restrict__ lo, int opitch, int coff,
                                                                  int fmt) {
  const int C4 = C >> 2, OH = H >> 1, OW = W >> 1;
  const long long total = (long long)N * OH * OW * C4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4) * 4;
    const long long op = i / C4;
    const int ow = (int)(op % OW);
    const long long t = op / OW;
    const int oh = (int)(t % OH);
    const long long n = t / OH;
    const float* base = y + ((n * H + 2 * oh) * W + 2 * ow) * (long long)ypitch + c;
    const float4 a = *reinterpret_cast<const float4*>(base);
    const float4 b = *reinterpret_cast<const float4*>(base + ypitch);
    const float4 d = *reinterpret_cast<const float4*>(base + (long long)W * ypitch);
    const float4 e = *reinterpret_cast<const float4*>(base + (long long)W * ypitch + ypitch);
    float m[4];
    m[0] = fmaxf(fmaxf(fmaxf(a.x, b.x), fmaxf(d.x, e.x)), 0.f);
    m[1] = fmaxf(fmaxf(fmaxf(a.y, b.y), fmaxf(d.y, e.y)), 0.f);
    m[2] = fmaxf(fmaxf(fmaxf(a.z, b.z), fmaxf(d.z, e.z)), 0.f);
    m[3] = fmaxf(fmaxf(fmaxf(a.w, b.w), fmaxf(d.w, e.w)), 0.f);
    uint16_t h4[4], l4[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) split16(m[j], fmt, h4[j], l4[j]);
    const long long off = op * opitch + coff + c;
    *reinterpret_cast<uint2*>(hi + off) = pack4(h4);
    *reinterpret_cast<uint2*>(lo + off) = pack4(l4);
  }
}

// ReLU + MaxPool2d(2) backward: dy[n,h,w,c] = (g_direct + [first max of the window] g_pool) * (y > 0)
// (PyTorch's max_pool2d routes the gradient to the first maximum in row-major window order.)
__global__ void __launch_bounds__(kThreads) relu_pool_bwd_kernel(const float* __restrict__ y, int ypitch,
                                                                  const float* __restrict__ gp, int gppitch,
                                                                  const float* __restrict__ gd, int gdpitch, int N,
                                                                  int H, int W, int C, uint16_t* __restrict__ hi,
                                                                  uint16_t* __restrict__ lo, int dpitch, int coff,
                                                                  int fmt) {
  const int C4 = C >> 2, OH = H >> 1, OW = W >> 1;
  const long long total = (long long)N * OH * OW * C4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4) * 4;
    const long long op = i / C4;
    const int ow = (int)(op % OW);
    const long long t = op / OW;
    const int oh = (int)(t % OH);
    const long long n = t / OH;
    const long long pix0 = (n * H + 2 * oh) * W + 2 * ow;
    const long long pix[4] = {pix0, pix0 + 1, pix0 + W, pix0 + W + 1};
    float v[4][4], g[4][4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float4 a = *reinterpret_cast<const float4*>(y + pix[q] * ypitch + c);
      v[q][0] = a.x; v[q][1] = a.y; v[q][2] = a.z; v[q][3] = a.w;
      if (gd) {
        const float4 b = *reinterpret_cast<const float4*>(gd + pix[q] * gdpitch + c);
        g[q][0] = b.x; g[q][1] = b.y; g[q][2] = b.z; g[q][3] = b.w;
      } else {
        g[q][0] = g[q][1] = g[q][2] = g[q][3] = 0.f;
      }
    }
    float gpv[4] = {0.f, 0.f, 0.f, 0.f};
    if (gp) {
      const float4 b = *reinterpret_cast<const float4*>(gp + op * gppitch + c);
      gpv[0] = b.x; gpv[1] = b.y; gpv[2] = b.z; gpv[3] = b.w;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int am = 0;
      float best = fmaxf(v[0][j], 0.f);
#pragma unroll
      for (int q = 1; q < 4; ++q) {
        const float r = fmaxf(v[q][j], 0.f);
        if (r > best) { best = r; am = q; }
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) g[q][j] = (v[q][j] > 0.f) ? g[q][j] + (q == am ? gpv[j] : 0.f) : 0.f;
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      uint16_t h4[4], l4[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) split16(g[q][j], fmt, h4[j], l4[j]);
      const long long off = pix[q] * dpitch + coff + c;
      *reinterpret_cast<uint2*>(hi + off) = pack4(h4);
      *reinterpret_cast<uint2*>(lo + off) = pack4(l4);
    }
  }
}

// ---------------------------------------------------------------------------------
// feature loss: one warp per pixel.  x = relu(y); f = x / (|x|_2 + 1e-8);
//   loss += w * sum_c (f_o - f_t)^2;   dx_o = J^T (2 w (f_o - f_t)),  J = d f_o / d x_o
// NV float4 per lane (C = 128 * NV), or C = 64 with half of the lanes.
// ---------------------------------------------------------------------------------
// DET: the block's loss sum goes to slots[blockIdx.x] (det_sum_slots adds the blocks in order)
template <int NV, bool DET>
__global__ void __launch_bounds__(kThreads) feat_loss_kernel(const float* __restrict__ yo, int po,
                                                              const float* __restrict__ yt, int pt, long long npix,
                                                              int C, double weight, double gscale,
                                                              double* __restrict__ loss_acc,
                                                              float* __restrict__ dx, int pdx, double* slots) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const float w = (float)(weight * gscale);
  double local = 0.0;
  for (long long p = blockIdx.x * (long long)wpb + warp; p < npix; p += (long long)gridDim.x * wpb) {
    float xo[NV][4], xt[NV][4];
    float so = 0.f, st = 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const int c = (k * 32 + lane) * 4;
      if (c < C) {
        const float4 a = *reinterpret_cast<const float4*>(yo + p * po + c);
        const float4 b = *reinterpret_cast<const float4*>(yt + p * pt + c);
        xo[k][0] = fmaxf(a.x, 0.f); xo[k][1] = fmaxf(a.y, 0.f); xo[k][2] = fmaxf(a.z, 0.f); xo[k][3] = fmaxf(a.w, 0.f);
        xt[k][0] = fmaxf(b.x, 0.f); xt[k][1] = fmaxf(b.y, 0.f); xt[k][2] = fmaxf(b.z, 0.f); xt[k][3] = fmaxf(b.w, 0.f);
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) xo[k][j] = xt[k][j] = 0.f;
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) { so += xo[k][j] * xo[k][j]; st += xt[k][j] * xt[k][j]; }
    }
    so = warp_sum(so);
    st = warp_sum(st);
    const float no = sqrtf(so), nt = sqrtf(st);
    const float ido = 1.f / (no + 1e-8f), idt = 1.f / (nt + 1e-8f);
    float s = 0.f, l = 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float d = xo[k][j] * ido - xt[k][j] * idt;
        l += d * d;
        const float g = 2.f * w * d;
        xt[k][j] = g;                 // keep g in place of the target value
        s += g * xo[k][j];
      }
    s = warp_sum(s);
    l = warp_sum(l);
    if (lane == 0) local += (double)l;
    const float coef = no > 0.f ? s * ido * ido / no : 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const int c = (k * 32 + lane) * 4;
      if (c < C) {
        float4 r;
        r.x = xt[k][0] * ido - coef * xo[k][0];
        r.y = xt[k][1] * ido - coef * xo[k][1];
        r.z = xt[k][2] * ido - coef * xo[k][2];
        r.w = xt[k][3] * ido - coef * xo[k][3];
        *reinterpret_cast<float4*>(dx + p * pdx + c) = r;
      }
    }
  }
  __shared__ double red[kThreads / 32];
  if (lane == 0) red[warp] = local;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < wpb; ++i) t += red[i];
    if constexpr (DET) slots[blockIdx.x] = t * weight;
    else atomicAdd(loss_acc, t * weight);
  }
}

// ---------------------------------------------------------------------------------
// The style term: row blocks of the Gram matrix of R = n*c rows of npix pixels, G[i][j] = sum_p X_i[p] X_j[p], row
// r = (b, ch): X_r[p] = src[b*sn + ch*sc + p*sp].  out[i][j] = sum_p A_i[p] B_j[p] for the R_l rows of A and the R rows
// of B: the whole matrix (A = B), or one rank's rows against every rank's.  Nothing is sized by the row count: the
// output is cut into kRowT x kRowT tiles (blockIdx.x) and the pixel chunks are split over blockIdx.y.  Each 128-pixel
// chunk is summed in fp32; the chunk sums are added in fp64, so an entry's fp32 chain is one chunk long whatever the
// split.
// ---------------------------------------------------------------------------------
constexpr int kGramP = 128;                    // pixels per smem tile
constexpr int kRowT = 32;                      // rows per tile edge
constexpr int kRowBlocks = 4 * SN_NUM_SMS;     // target block count of gram_rows / gram_rows_bwd

struct RowSrc {
  const float* p;
  long long sn, sc, sp;
};

// tile[r][0:kGramP] <- rows r0 .. r0 + nr - 1 of s over pixels [p0, p0 + kGramP); zero past nr rows and npix pixels
__device__ __forceinline__ void load_row_tile(float* tile, const RowSrc& s, int C, int r0, int nr, long long p0,
                                              long long npix) {
  constexpr int TP = kGramP + 1;
  for (int i = threadIdx.x; i < kRowT * kGramP; i += blockDim.x) {
    int r, p;
    if (s.sp == 1) { r = i / kGramP; p = i - r * kGramP; } else { p = i / kRowT; r = i - p * kRowT; }
    float v = 0.f;
    if (r < nr && p0 + p < npix) {
      const int g = r0 + r, b = g / C, c = g - b * C;
      v = s.p[b * s.sn + c * s.sc + (p0 + p) * s.sp];
    }
    tile[r * TP + p] = v;
  }
}

// Thread t owns the entries (i0 + t/16 + 16u, j0 + t%16 + 16v), u, v in {0, 1}.
// DET: the block's partials go to slots[blockIdx.y][R_l * R] (det_sum_slots adds the pixel splits in order)
template <bool DET>
__global__ void __launch_bounds__(kThreads) gram_rows_kernel(RowSrc a, RowSrc b, int C, int Rl, int R,
                                                              long long npix, double* __restrict__ out,
                                                              double* __restrict__ slots) {
  constexpr int TP = kGramP + 1;
  __shared__ float ta[kRowT * TP], tb[kRowT * TP];
  const int tiles_j = (R + kRowT - 1) / kRowT;
  const int i0 = (blockIdx.x / tiles_j) * kRowT, j0 = (blockIdx.x % tiles_j) * kRowT;
  const int ni = min(kRowT, Rl - i0), nj = min(kRowT, R - j0);
  const int ti = threadIdx.x >> 4, tj = threadIdx.x & 15;
  double acc[2][2] = {{0.0, 0.0}, {0.0, 0.0}};
  const long long nchunks = (npix + kGramP - 1) / kGramP;
  for (long long ch = blockIdx.y; ch < nchunks; ch += gridDim.y) {
    const long long p0 = ch * kGramP;
    __syncthreads();
    load_row_tile(ta, a, C, i0, ni, p0, npix);
    load_row_tile(tb, b, C, j0, nj, p0, npix);
    __syncthreads();
    const float* a0 = ta + ti * TP;
    const float* a1 = ta + (ti + 16) * TP;
    const float* b0 = tb + tj * TP;
    const float* b1 = tb + (tj + 16) * TP;
    float s00 = 0.f, s01 = 0.f, s10 = 0.f, s11 = 0.f;
#pragma unroll 8
    for (int p = 0; p < kGramP; ++p) {
      const float x0 = a0[p], x1 = a1[p], y0 = b0[p], y1 = b1[p];
      s00 += x0 * y0; s01 += x0 * y1; s10 += x1 * y0; s11 += x1 * y1;
    }
    acc[0][0] += (double)s00; acc[0][1] += (double)s01; acc[1][0] += (double)s10; acc[1][1] += (double)s11;
  }
#pragma unroll
  for (int u = 0; u < 2; ++u)
#pragma unroll
    for (int v = 0; v < 2; ++v) {
      const int i = ti + 16 * u, j = tj + 16 * v;
      if (i < ni && j < nj) {
        const long long idx = (long long)(i0 + i) * R + j0 + j;
        if constexpr (DET) slots[(long long)blockIdx.y * Rl * R + idx] = acc[u][v];
        else atomicAdd(&out[idx], acc[u][v]);
      }
    }
}

// loss_acc += weight * sum((Go - Gt)^2) / R^2 over an [R_l][R] row block;  M = 4 * weight * gscale * (Go - Gt) / R^2
// (= gscale * (dL/dGo + its transpose) on those rows, the Gram matrices being symmetric).  One block, fp64 throughout:
// each thread's strided squares, a tree over the threads, one atomicAdd.  M is rounded to fp32 once, from
// (4 * weight * gscale * d) * (1 / R^2).
__global__ void gram_rows_mse_kernel(const double* __restrict__ Go, const double* __restrict__ Gt, long long n, int R,
                                     double weight, double gscale, double* __restrict__ loss_acc,
                                     float* __restrict__ M) {
  __shared__ double red[kThreads];
  double l = 0.0;
  const double inv = 1.0 / ((double)R * R);
  const double mw = 4.0 * weight * gscale;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) {
    const double d = Go[i] - Gt[i];
    l += d * d;
    M[i] = (float)(mw * d * inv);
  }
  red[threadIdx.x] = l;
  __syncthreads();
  for (int o = kThreads / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) atomicAdd(loss_acc, weight * red[0] * inv);
}

// dx[b, p, ch] (+)= sum_j M[r][j] X_j[p] for the R_l rows r = b*C + ch of M and the R rows of X.  Block (x, y): row
// tile y (kRowT rows of M), pixel chunks x, x + gridDim.x, ...; thread t owns pixel t % 128 of rows t/128 + 2k.
// The columns j are summed in order in fp32 (the zero rows past R add exact zeros): one fp32 chain of R terms per entry.
__global__ void __launch_bounds__(kThreads) gram_rows_bwd_kernel(const float* __restrict__ M, RowSrc x, int C, int Rl,
                                                                  int R, long long npix, float* __restrict__ dx,
                                                                  int pdx, int accumulate) {
  constexpr int TP = kGramP + 1, MP = kRowT + 1, KR = kRowT / (kThreads / kGramP);
  __shared__ float tx[kRowT * TP], tm[kRowT * MP];
  const int i0 = blockIdx.y * kRowT;
  const int p = threadIdx.x % kGramP, rg = threadIdx.x / kGramP;
  const long long nchunks = (npix + kGramP - 1) / kGramP;
  for (long long ch = blockIdx.x; ch < nchunks; ch += gridDim.x) {
    const long long p0 = ch * kGramP;
    float s[KR];
#pragma unroll
    for (int k = 0; k < KR; ++k) s[k] = 0.f;
    for (int j0 = 0; j0 < R; j0 += kRowT) {
      __syncthreads();
      load_row_tile(tx, x, C, j0, min(kRowT, R - j0), p0, npix);
      for (int t = threadIdx.x; t < kRowT * kRowT; t += blockDim.x) {
        const int i = t / kRowT, j = t - i * kRowT;
        tm[i * MP + j] = (i0 + i < Rl && j0 + j < R) ? M[(long long)(i0 + i) * R + j0 + j] : 0.f;
      }
      __syncthreads();
#pragma unroll 4
      for (int j = 0; j < kRowT; ++j) {
        const float xv = tx[j * TP + p];
#pragma unroll
        for (int k = 0; k < KR; ++k) s[k] += tm[(rg + 2 * k) * MP + j] * xv;
      }
    }
    if (p0 + p < npix) {
#pragma unroll
      for (int k = 0; k < KR; ++k) {
        const int r = i0 + rg + 2 * k;
        if (r < Rl) {
          const int b = r / C, c = r - b * C;
          float* d = dx + ((long long)b * npix + p0 + p) * pdx + c;
          *d = accumulate ? *d + s[k] : s[k];
        }
      }
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

int sn_affine_pack(const float* src, int src_layout, int src_pitch, int n, int c, int h, int w, float mul, float add,
                   void* dst_hi, void* dst_lo, int dst_pitch, int dst_coff, int fmt, void* stream) {
  SN_REQUIRE(src && dst_hi && dst_lo, "null pointer");
  SN_REQUIRE(c >= 1 && c <= 16 && dst_pitch % 8 == 0 && dst_coff % 8 == 0, "affine_pack: c <= 16, 16-byte aligned planes");
  const long long hw = (long long)h * w;
  affine_pack_kernel<<<grid_for((long long)n * hw), kThreads, 0, (cudaStream_t)stream>>>(
      src, src_layout, src_pitch, n, c, hw, mul, add, (uint16_t*)dst_hi, (uint16_t*)dst_lo, dst_pitch, dst_coff, fmt);
  LAUNCH_CHECK();
  return SN_OK;
}

int sn_relu_pool_fwd(const float* y, int y_pitch, int n, int h, int w, int c, void* out_hi, void* out_lo,
                     int out_pitch, int out_coff, int fmt, void* stream) {
  SN_REQUIRE(y && out_hi && out_lo, "null pointer");
  SN_REQUIRE(c % 4 == 0 && y_pitch % 4 == 0 && out_pitch % 4 == 0 && out_coff % 4 == 0 && h % 2 == 0 && w % 2 == 0,
             "relu_pool: c, pitches multiples of 4; even h, w");
  relu_pool_fwd_kernel<<<grid_for((long long)n * (h / 2) * (w / 2) * (c / 4)), kThreads, 0, (cudaStream_t)stream>>>(
      y, y_pitch, n, h, w, c, (uint16_t*)out_hi, (uint16_t*)out_lo, out_pitch, out_coff, fmt);
  LAUNCH_CHECK();
  return SN_OK;
}

int sn_relu_pool_bwd(const float* y, int y_pitch, const float* g_pool, int gp_pitch, const float* g_direct,
                     int gd_pitch, int n, int h, int w, int c, void* dy_hi, void* dy_lo, int dy_pitch, int dy_coff,
                     int dy_fmt, void* stream) {
  SN_REQUIRE(y && dy_hi && dy_lo && (g_pool || g_direct), "null pointer");
  SN_REQUIRE(c % 4 == 0 && y_pitch % 4 == 0 && dy_pitch % 4 == 0 && dy_coff % 4 == 0 && h % 2 == 0 && w % 2 == 0 &&
                 (!g_pool || gp_pitch % 4 == 0) && (!g_direct || gd_pitch % 4 == 0),
             "relu_pool_bwd: c, pitches multiples of 4; even h, w");
  relu_pool_bwd_kernel<<<grid_for((long long)n * (h / 2) * (w / 2) * (c / 4)), kThreads, 0, (cudaStream_t)stream>>>(
      y, y_pitch, g_pool, gp_pitch, g_direct, gd_pitch, n, h, w, c, (uint16_t*)dy_hi, (uint16_t*)dy_lo, dy_pitch,
      dy_coff, dy_fmt);
  LAUNCH_CHECK();
  return SN_OK;
}

}  // extern "C"

template <bool DET>
static void launch_feat_loss(int blocks, cudaStream_t st, const float* y_out, int po, const float* y_tgt, int pt,
                             long long npix, int c, double weight, double gscale, double* loss_acc, float* dx, int pdx,
                             double* slots) {
  if (c <= 128)
    feat_loss_kernel<1, DET><<<blocks, kThreads, 0, st>>>(y_out, po, y_tgt, pt, npix, c, weight, gscale, loss_acc, dx,
                                                          pdx, slots);
  else if (c <= 256)
    feat_loss_kernel<2, DET><<<blocks, kThreads, 0, st>>>(y_out, po, y_tgt, pt, npix, c, weight, gscale, loss_acc, dx,
                                                          pdx, slots);
  else
    feat_loss_kernel<4, DET><<<blocks, kThreads, 0, st>>>(y_out, po, y_tgt, pt, npix, c, weight, gscale, loss_acc, dx,
                                                          pdx, slots);
}

extern "C" {

static int feat_loss_impl(const float* y_out, int po, const float* y_tgt, int pt, long long npix, int c, double weight,
                          double gscale, double* loss_acc, float* dx, int pdx, double* slots, long long slots_cap,
                          cudaStream_t st) {
  SN_REQUIRE(y_out && y_tgt && loss_acc && dx, "null pointer");
  SN_REQUIRE(c % 4 == 0 && c <= 512 && po % 4 == 0 && pt % 4 == 0 && pdx % 4 == 0,
             "feat_loss: c multiple of 4 and <= 512, pitches multiples of 4");
  const int wpb = kThreads / 32;
  long long blocks = (npix + wpb - 1) / wpb;
  if (blocks > SN_NUM_SMS * 8) blocks = SN_NUM_SMS * 8;
  if (!slots) {
    launch_feat_loss<false>((int)blocks, st, y_out, po, y_tgt, pt, npix, c, weight, gscale, loss_acc, dx, pdx, nullptr);
    LAUNCH_CHECK();
    return SN_OK;
  }
  SN_REQUIRE(blocks <= slots_cap, "feat_loss_det: %lld slots needed, %lld given", blocks, slots_cap);
  launch_feat_loss<true>((int)blocks, st, y_out, po, y_tgt, pt, npix, c, weight, gscale, loss_acc, dx, pdx, slots);
  LAUNCH_CHECK();
  SN_CHECK_CUDA(det_sum_slots(slots, (int)blocks, 1, loss_acc, st));
  LAUNCH_CHECK();
  return SN_OK;
}

int sn_feat_loss_fwd_bwd(const float* y_out, int po, const float* y_tgt, int pt, long long npix, int c, double weight,
                         double gscale, double* loss_acc, float* dx, int pdx, void* stream) {
  return feat_loss_impl(y_out, po, y_tgt, pt, npix, c, weight, gscale, loss_acc, dx, pdx, nullptr, 0,
                        (cudaStream_t)stream);
}

int sn_feat_loss_fwd_bwd_det(const float* y_out, int po, const float* y_tgt, int pt, long long npix, int c,
                             double weight, double gscale, double* loss_acc, float* dx, int pdx, double* slots,
                             long long slots_cap, void* stream) {
  SN_REQUIRE(slots, "feat_loss_det: null slots");
  return feat_loss_impl(y_out, po, y_tgt, pt, npix, c, weight, gscale, loss_acc, dx, pdx, slots, slots_cap,
                        (cudaStream_t)stream);
}

// pixel splits of gram_rows: enough blocks for kRowBlocks whatever the tile count, at most one per chunk
static long long gram_rows_splits(long long rows_l, long long rows) {
  const long long tiles = ((rows_l + kRowT - 1) / kRowT) * ((rows + kRowT - 1) / kRowT);
  const long long p = (kRowBlocks + tiles - 1) / tiles;
  return p < 1 ? 1 : p;
}

static int gram_rows_impl(const float* a, long long a_n, long long a_c, long long a_p, int n_a, const float* b,
                          long long b_n, long long b_c, long long b_p, int n_b, int c, long long npix, double* out,
                          double* slots, long long slots_cap, cudaStream_t st) {
  SN_REQUIRE(a && b && out, "null pointer");
  SN_REQUIRE(n_a >= 1 && c >= 1 && npix >= 1 && n_a <= n_b, "gram_rows: 1 <= n_a <= n_b samples, c >= 1, npix >= 1");
  SN_REQUIRE(a_n >= 1 && a_c >= 1 && a_p >= 1 && b_n >= 1 && b_c >= 1 && b_p >= 1, "gram_rows: strides must be >= 1");
  const long long rl = (long long)n_a * c, r = (long long)n_b * c;
  SN_REQUIRE(r <= (1 << 20), "gram_rows: %lld rows, at most %d supported", r, 1 << 20);
  const long long tiles = ((rl + kRowT - 1) / kRowT) * ((r + kRowT - 1) / kRowT);
  SN_REQUIRE(tiles < (1LL << 31), "gram_rows: %lld output tiles", tiles);
  const long long chunks = (npix + kGramP - 1) / kGramP;
  long long splits = gram_rows_splits(rl, r);
  if (splits > chunks) splits = chunks;
  SN_CHECK_CUDA(cudaMemsetAsync(out, 0, sizeof(double) * rl * r, st));
  const dim3 grid((unsigned)tiles, (unsigned)splits);
  const RowSrc sa{a, a_n, a_c, a_p}, sb{b, b_n, b_c, b_p};
  if (!slots) {
    gram_rows_kernel<false><<<grid, kThreads, 0, st>>>(sa, sb, c, (int)rl, (int)r, npix, out, nullptr);
    LAUNCH_CHECK();
    return SN_OK;
  }
  SN_REQUIRE(splits * rl * r <= slots_cap, "gram_rows_det: %lld slots needed, %lld given", splits * rl * r, slots_cap);
  gram_rows_kernel<true><<<grid, kThreads, 0, st>>>(sa, sb, c, (int)rl, (int)r, npix, out, slots);
  LAUNCH_CHECK();
  SN_CHECK_CUDA(det_sum_slots(slots, (int)splits, rl * r, out, st));
  LAUNCH_CHECK();
  return SN_OK;
}

int sn_gram_rows(const float* a, long long a_n, long long a_c, long long a_p, int n_a, const float* b, long long b_n,
                 long long b_c, long long b_p, int n_b, int c, long long npix, double* out, void* stream) {
  return gram_rows_impl(a, a_n, a_c, a_p, n_a, b, b_n, b_c, b_p, n_b, c, npix, out, nullptr, 0, (cudaStream_t)stream);
}

int sn_gram_rows_det(const float* a, long long a_n, long long a_c, long long a_p, int n_a, const float* b,
                     long long b_n, long long b_c, long long b_p, int n_b, int c, long long npix, double* out,
                     double* slots, long long slots_cap, void* stream) {
  SN_REQUIRE(slots, "gram_rows_det: null slots");
  return gram_rows_impl(a, a_n, a_c, a_p, n_a, b, b_n, b_c, b_p, n_b, c, npix, out, slots, slots_cap,
                        (cudaStream_t)stream);
}

long long sn_gram_rows_det_slots(int rows_l, int rows) {
  if (rows_l < 1 || rows < 1) return 0;
  return gram_rows_splits(rows_l, rows) * rows_l * rows;
}

int sn_gram_rows_mse(const double* gram_out, const double* gram_tgt, int rows_l, int rows, double weight,
                     double gscale, double* loss_acc, float* m, void* stream) {
  SN_REQUIRE(gram_out && gram_tgt && loss_acc && m, "null pointer");
  SN_REQUIRE(rows_l >= 1 && rows_l <= rows, "gram_rows_mse: 1 <= rows_l (%d) <= rows (%d)", rows_l, rows);
  gram_rows_mse_kernel<<<1, kThreads, 0, (cudaStream_t)stream>>>(gram_out, gram_tgt, (long long)rows_l * rows, rows,
                                                                  weight, gscale, loss_acc, m);
  LAUNCH_CHECK();
  return SN_OK;
}

int sn_gram_rows_bwd(const float* m, int rows_l, const float* src, long long s_n, long long s_c, long long s_p, int n,
                     int c, long long npix, float* dx, int dx_pitch, int accumulate, void* stream) {
  SN_REQUIRE(m && src && dx, "null pointer");
  SN_REQUIRE(n >= 1 && c >= 1 && npix >= 1, "gram_rows_bwd: n, c, npix >= 1");
  SN_REQUIRE(s_n >= 1 && s_c >= 1 && s_p >= 1 && dx_pitch >= c, "gram_rows_bwd: strides >= 1, dx_pitch >= c");
  const long long r = (long long)n * c;
  SN_REQUIRE(rows_l >= 1 && rows_l <= r && rows_l % c == 0,
             "gram_rows_bwd: rows_l = %d must be whole samples of the %lld rows of src", rows_l, r);
  SN_REQUIRE(r <= (1 << 20), "gram_rows_bwd: %lld rows, at most %d supported", r, 1 << 20);
  const int row_tiles = (rows_l + kRowT - 1) / kRowT;
  const long long chunks = (npix + kGramP - 1) / kGramP;
  long long gx = (kRowBlocks + row_tiles - 1) / row_tiles;
  if (gx > chunks) gx = chunks;
  const RowSrc sx{src, s_n, s_c, s_p};
  gram_rows_bwd_kernel<<<dim3((unsigned)gx, (unsigned)row_tiles), kThreads, 0, (cudaStream_t)stream>>>(
      m, sx, c, rows_l, (int)r, npix, dx, dx_pitch, accumulate);
  LAUNCH_CHECK();
  return SN_OK;
}

}  // extern "C"
