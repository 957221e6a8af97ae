// swapnet_b200 — per-channel cloth augmentation on the device (sm_90a, HBM bound; SURVEY §8 f4).
//
// Replaces datasets/data_utils.py:346-361 `per_channel_transform` (19 PIL mode-"F" images per sample, each through
// torchvision's RandomOrder([RandomVerticalFlip, RandomHorizontalFlip, RandomAffine, RandomPerspective]) of
// datasets/__init__.py:88-110) together with the label map -> one-hot expansion of data_utils.py:330-343 that
// precedes it: the source is the uint8 label map (or a dense fp32 tensor), the result the fp32 [n, c, h, w] tensor
// `set_input` takes.  The random draws and the matrices are made on the host (swapnet_b200/data.py, through
// torchvision's own get_params); this file does the pixel work, bit-exactly as Pillow's libImaging/Geometry.c does it:
//   * FLIP_LEFT_RIGHT / FLIP_TOP_BOTTOM: index reversal;
//   * AFFINE + NEAREST (`affine_fixed`): 16.16 fixed point, source = ((a2 + x*a0 + y*a1) >> 16, (a5 + x*a3 + y*a4) >> 16),
//     coefficients already FIX()ed on the host; outside -> fill 0;
//   * PERSPECTIVE + BILINEAR (`perspective_transform` + `bilinear_filter32F`): doubles with explicit round-to-nearest
//     mul/add/div (no FMA contraction), the horizontal tap difference in float32 like the C code's FLOAT32 operands.
// Each op is a full-plane dependency of the next (Pillow resamples after every transform), so the ops of a plane run
// as passes: pass j of a plane with k ops reads what pass j-1 wrote and writes `out` when k-1-j is even, else `tmp`
// (the last pass always lands in `out`); pass 0 reads the label map itself.  One launch per pass for all planes.
#include "common.cuh"
#include "../../include/swapnet_b200.h"

void sn_count_launch(int n);

namespace {

constexpr int kAugRows = 8;   // rows of one plane per block: grid = (ceil(h / kAugRows), n * c)

struct AugArgs {
  const uint8_t* labels;   // [n, h, w] or null
  const float* dense;      // [n, c, h, w] or null
  const sn_aug_op* ops;    // [n*c, stride]
  float* out; float* tmp;  // [n, c, h, w]
  int n, c, h, w, stride, pass;
};

// source plane of a pass: the uint8 label map seen through one channel (pass 0) or an fp32 plane
template <bool LAB>
struct Src {
  const uint8_t* lab; const float* f; int ch, w;
  __device__ __forceinline__ float at(int y, int x) const {
    if (LAB) return (ch > 0 && lab[(long long)y * w + x] == ch) ? 1.f : 0.f;
    return f[(long long)y * w + x];
  }
};

// rows [r0, r1) of one plane through one op; the op's constants are hoisted out of the pixel loop and the loop nest is
// row / column, so there is no division per pixel.  The arithmetic per pixel is exactly Geometry.c's (see the header).
template <int KIND, bool LAB>
__device__ __forceinline__ void plane_rows(const Src<LAB> s, float* __restrict__ dst, const double* __restrict__ p,
                                           const int H, const int W, const int r0, const int r1) {
  long long a0 = 0, a1 = 0, a2 = 0, a3 = 0, a4 = 0, a5 = 0;
  double q0 = 0, q1 = 0, q2 = 0, q3 = 0, q4 = 0, q5 = 0, q6 = 0, q7 = 0;
  if (KIND == SN_AUG_AFFINE_NEAREST) {
    a0 = (long long)p[0]; a1 = (long long)p[1]; a2 = (long long)p[2];
    a3 = (long long)p[3]; a4 = (long long)p[4]; a5 = (long long)p[5];
  }
  if (KIND == SN_AUG_PERSPECTIVE_BILINEAR) {
    q0 = p[0]; q1 = p[1]; q2 = p[2]; q3 = p[3]; q4 = p[4]; q5 = p[5]; q6 = p[6]; q7 = p[7];
  }
  for (int y = r0; y < r1; ++y) {
    float* drow = dst + (long long)y * W;
    const long long rx = a2 + y * a1, ry = a5 + y * a4;                       // affine: row terms
    const double yc = __dadd_rn((double)y, 0.5);                              // perspective: row terms
    const double q1y = __dmul_rn(q1, yc), q4y = __dmul_rn(q4, yc), q7y = __dmul_rn(q7, yc);
    for (int x = threadIdx.x; x < W; x += blockDim.x) {
      float v = 0.f;
      if (KIND == SN_AUG_NONE) {
        v = s.at(y, x);
      } else if (KIND == SN_AUG_HFLIP) {
        v = s.at(y, W - 1 - x);
      } else if (KIND == SN_AUG_VFLIP) {
        v = s.at(H - 1 - y, x);
      } else if (KIND == SN_AUG_AFFINE_NEAREST) {
        const long long xin = (rx + x * a0) >> 16;
        const long long yin = (ry + x * a3) >> 16;
        if (xin >= 0 && xin < W && yin >= 0 && yin < H) v = s.at((int)yin, (int)xin);
      } else {  // SN_AUG_PERSPECTIVE_BILINEAR: ((q0*xc + q1*yc) + q2) / ((q6*xc + q7*yc) + 1), same for y
        const double xc = __dadd_rn((double)x, 0.5);
        const double den = __dadd_rn(__dadd_rn(__dmul_rn(q6, xc), q7y), 1.0);
        double xs = __ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(q0, xc), q1y), q2), den);
        double ys = __ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(q3, xc), q4y), q5), den);
        if (!(xs < 0.0 || xs >= (double)W || ys < 0.0 || ys >= (double)H)) {     // NaN falls through like in C
          xs = __dsub_rn(xs, 0.5); ys = __dsub_rn(ys, 0.5);
          const int x0 = (int)floor(xs), y0 = (int)floor(ys);
          const double dx = __dsub_rn(xs, (double)x0), dy = __dsub_rn(ys, (double)y0);
          const int xa = min(max(x0, 0), W - 1), xb = min(max(x0 + 1, 0), W - 1);
          const int ya = min(max(y0, 0), H - 1);
          float t0 = s.at(ya, xa), t1 = s.at(ya, xb);
          const double v1 = __dadd_rn((double)t0, __dmul_rn((double)__fsub_rn(t1, t0), dx));
          double v2 = v1;
          if (y0 + 1 >= 0 && y0 + 1 < H) {
            t0 = s.at(y0 + 1, xa); t1 = s.at(y0 + 1, xb);
            v2 = __dadd_rn((double)t0, __dmul_rn((double)__fsub_rn(t1, t0), dx));
          }
          v = __double2float_rn(__dadd_rn(v1, __dmul_rn(__dsub_rn(v2, v1), dy)));
        }
      }
      drow[x] = v;
    }
  }
}

template <bool LAB>
__device__ __forceinline__ void plane_dispatch(const int kind, const Src<LAB> s, float* dst, const double* p, const int H,
                                               const int W, const int r0, const int r1) {
  switch (kind) {                                                      // block-uniform
    case SN_AUG_HFLIP: plane_rows<SN_AUG_HFLIP, LAB>(s, dst, p, H, W, r0, r1); break;
    case SN_AUG_VFLIP: plane_rows<SN_AUG_VFLIP, LAB>(s, dst, p, H, W, r0, r1); break;
    case SN_AUG_AFFINE_NEAREST: plane_rows<SN_AUG_AFFINE_NEAREST, LAB>(s, dst, p, H, W, r0, r1); break;
    case SN_AUG_PERSPECTIVE_BILINEAR: plane_rows<SN_AUG_PERSPECTIVE_BILINEAR, LAB>(s, dst, p, H, W, r0, r1); break;
    default: plane_rows<SN_AUG_NONE, LAB>(s, dst, p, H, W, r0, r1); break;
  }
}

__global__ void __launch_bounds__(256) augment_pass_kernel(const AugArgs a) {
  const int plane = blockIdx.y;                       // b * c + ch
  const sn_aug_op* pops = a.ops + (long long)plane * a.stride;
  const int k = min(pops[0].nops, a.stride);
  const int keff = k > 0 ? k : 1;
  const int j = a.pass;
  if (j >= keff) return;
  const long long hw = (long long)a.h * a.w;
  float* dst = (((keff - 1 - j) & 1) == 0 ? a.out : a.tmp) + plane * hw;
  const int kind = k > 0 ? pops[j].kind : SN_AUG_NONE;
  const double* p = pops[j].p;
  const int r0 = blockIdx.x * kAugRows, r1 = min(r0 + kAugRows, a.h);
  if (j == 0 && a.labels) {
    Src<true> s;
    s.lab = a.labels + (long long)(plane / a.c) * hw; s.f = nullptr; s.ch = plane % a.c; s.w = a.w;
    plane_dispatch<true>(kind, s, dst, p, a.h, a.w, r0, r1);
  } else {
    Src<false> s;
    s.lab = nullptr; s.ch = 0; s.w = a.w;
    s.f = (j == 0 ? a.dense : (((keff - j) & 1) == 0 ? a.out : a.tmp)) + plane * hw;   // pass j-1 wrote there
    plane_dispatch<false>(kind, s, dst, p, a.h, a.w, r0, r1);
  }
}

}  // namespace

extern "C" int sn_augment_channels(const void* labels_u8, const float* dense_nchw, int n, int c, int h, int w,
                                   const sn_aug_op* ops_dev, int op_stride, int max_ops, float* out_nchw,
                                   float* tmp_nchw, void* stream) {
  SN_REQUIRE((labels_u8 != nullptr) != (dense_nchw != nullptr), "exactly one of labels_u8 / dense_nchw");
  SN_REQUIRE(ops_dev && out_nchw, "null pointer");
  SN_REQUIRE(n > 0 && c > 0 && h > 0 && w > 0 && (long long)n * c <= 65535, "bad shape (n*c <= 65535)");
  SN_REQUIRE(!labels_u8 || c <= 256, "a uint8 label map addresses at most 256 channels");
  SN_REQUIRE(op_stride >= 1 && max_ops >= 0 && max_ops <= op_stride && op_stride <= SN_AUG_MAX_OPS,
             "op table: 1 <= op_stride <= SN_AUG_MAX_OPS, 0 <= max_ops <= op_stride");
  SN_REQUIRE(max_ops < 2 || tmp_nchw, "two or more ops on a plane need the tmp buffer");
  SN_REQUIRE(out_nchw != tmp_nchw && (!dense_nchw || (dense_nchw != out_nchw && dense_nchw != tmp_nchw)),
             "buffers must not alias");
  AugArgs a;
  a.labels = (const uint8_t*)labels_u8; a.dense = dense_nchw; a.ops = ops_dev;
  a.out = out_nchw; a.tmp = tmp_nchw;
  a.n = n; a.c = c; a.h = h; a.w = w; a.stride = op_stride;
  const int gx = (h + kAugRows - 1) / kAugRows;
  const int passes = max_ops > 0 ? max_ops : 1;
  for (int j = 0; j < passes; ++j) {
    a.pass = j;
    augment_pass_kernel<<<dim3(gx, n * c), 256, 0, (cudaStream_t)stream>>>(a);
    sn_count_launch(1);
  }
  SN_CHECK_CUDA(cudaGetLastError());
  return SN_OK;
}
