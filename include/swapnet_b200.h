/* swapnet_b200 — C ABI of the B200-native SwapNet hot path (libswapnet_b200.so).
 *
 * The reference (andrewjong/SwapNet) has no FFI: its plugin boundary is the Python class
 * protocol of models/__init__.py:5-44.  This header is the NEW lower boundary under that
 * protocol: what a maintainer binds (ctypes, see INTEGRATION.md) to replace the eager
 * torch ops of
 *     modules/layers.py:12-63,126-144        (UNetDown / UNetUp / DualUNetUp / ResidualBlock)
 *     modules/swapnet_modules.py:85-90,92-151,209-260 (head conv, WarpModule, TextureModule)
 *     modules/pix2pix_modules.py:180-262     (UnetSkipConnectionBlock)
 *     modules/discriminators.py:91-136       (NLayerDiscriminator / PatchGAN)
 *     modules/loss.py:110-130, models/warp_model.py:147-150, models/texture_model.py:168-170
 *     torchvision.ops.roi_align as called at modules/swapnet_modules.py:166-168,234
 *
 * Conventions
 *   - every pointer is a caller-owned DEVICE pointer (torch tensor.data_ptr()); the library
 *     allocates nothing persistent except plan handles;
 *   - every call takes the CUDA stream to run on (a cudaStream_t passed as void*), is
 *     asynchronous, and returns 0 on success or a negative code (message: sn_last_error());
 *   - activations are NHWC ("channels-last") fp32 with an explicit pixel pitch (elements per
 *     pixel in memory >= channels) so that a tensor can live inside a channel slice of a
 *     wider concat buffer;
 *   - a GEMM operand is a "split plane pair": two 16-bit-float NHWC tensors hi = r16(v),
 *     lo = r16(v - hi) in format SN_FMT_F16 or SN_FMT_BF16 (fp32 carried as 2 x 16 bit; products are
 *     evaluated as hi*hi + lo*hi + hi*lo on the tensor cores (sm_90a wgmma) with fp32 accumulation).
 *     Both operands of one contraction must use the same format: forward GEMMs run fp16-split
 *     (activations x scaled weights), backward GEMMs bf16-split (gradients x bf16 copies).
 */
#ifndef SWAPNET_B200_H
#define SWAPNET_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SN_MAX_TAPS 32
#define SN_MAX_SRC 3

enum { SN_ACT_NONE = 0, SN_ACT_TANH = 1, SN_ACT_LRELU = 2, SN_ACT_RELU = 3 };
/* SN_LAYOUT_LABEL_U8 / SN_LAYOUT_MASK_I32: compact encodings of the 0/1-valued cloth segmentation tensors — the wire
 * format the reference's dataset expands on the host (datasets/data_utils.py:311-343 `to_onehot_tensor`: label L > 0 ->
 * channel L one-hot, label 0 (background) -> the all-zero vector; after the per-channel augmentation of
 * data_utils.py:346-361 the channels are independent 0/1 masks).  LABEL_U8: uint8 [n,h,w] label map; MASK_I32: int32
 * [n,h,w] with bit c = channel c.  The kernels below that take a `layout` expand them on the fly, so the batch travels
 * over PCIe as 1-4 bytes per pixel instead of 76 (SURVEY 8f rank 4). */
enum { SN_LAYOUT_NCHW = 0, SN_LAYOUT_NHWC = 1, SN_LAYOUT_LABEL_U8 = 2, SN_LAYOUT_MASK_I32 = 3 };
/* 16-bit float format of a split plane pair: bf16 (8+8 mantissa bits, fp32 range: gradients) or
 * fp16 (11+11 bits: activations, pre-scaled weights).  A and B of one GEMM must agree. */
#define SN_FMT_BF16 0
#define SN_FMT_F16 1

const char* sn_version(void);
const char* sn_last_error(void);
/* number of kernel launches issued by this library since process start (bench.py: gpu_launches) */
long long sn_launch_count(void);
/* a CUDA-graph replay executes launches that were counted once, at capture: the host adds them per replay */
void sn_count_replayed(long long n);

/* ------------------------------------------------------------------------------------------
 * tensor-core contractions
 * ---------------------------------------------------------------------------------------- */
typedef struct sn_tap {
  int c_off;  /* channel offset inside the A tensor view (parity view: pw * pitch) */
  int kb_off; /* K offset of this tap in the packed weight matrix (tap GEMM only) */
  int dw, dh; /* GEMM-row (h, w) -> source pixel (h + dh, w + dw); out of range = zero */
  int hp;     /* parity view only: h parity plane (0/1); 0 otherwise */
} sn_tap;

/* D[(n,h,w), j] = sum_t sum_c A[n, h+dh_t, w+dw_t, c_off_t + c] * B[j, kb_off_t + c]  (+bias, act)
 * Lowers Conv2d / ConvTranspose2d forward and their dgrad; see swapnet_b200/lowering.py. */
typedef struct sn_tap_gemm_desc {
  const void* a_hi; const void* a_lo;   /* split planes, logical [a_n, a_h, a_w, a_c], pitch a_pitch */
  int a_n, a_h, a_w, a_c, a_pitch;
  int a_parity;                          /* 1: address through the 2x2 parity view (stride-2) */
  int a_fmt;                             /* SN_FMT_* of the A planes */
  int a_chunk;                           /* channels per TMA row: 64 (default when 0), 32 or 16.  Narrow
                                            operands (3/19/22-channel images, 1/3/19-channel gradients)
                                            are padded to 16/32 instead of 64: then k_per_tap == a_chunk,
                                            64/a_chunk taps share one pipeline stage, ntaps %% (64/a_chunk) == 0 */
  const void* b_hi; const void* b_lo;   /* packed weights [b_rows][b_k] 16-bit, K contiguous */
  int b_rows; long long b_k;
  int b_fmt;                             /* SN_FMT_* of the packed weights */
  const float* b_scale;                  /* optional device float[2] = (s, 1/s) written by
                                            sn_weight_scale_multi: weights were packed as w*s, the
                                            epilogue multiplies the accumulator by 1/s */
  int m_n, m_h, m_w;                     /* GEMM row grid */
  int ntaps; int k_per_tap;              /* k_per_tap % 64 == 0 (or == a_chunk when narrow) */
  sn_tap taps[SN_MAX_TAPS];
  float* out;                            /* fp32, element strides below, channel stride 1 */
  long long out_sn, out_sh, out_sw;
  int out_mul_h, out_off_h, out_mul_w, out_off_w; /* row (h,w) -> out pixel (h*mul+off, ...) */
  int n_valid;                           /* output channels actually written */
  int block_n;                           /* N tile: multiple of 16, <= 128 */
  const float* bias;                     /* optional [n_valid] */
  int act;                               /* SN_ACT_NONE | SN_ACT_TANH */
  int nsplit;                            /* 3 = fp32-faithful split product, 1 = bf16 fast mode */
  int nphase;                            /* 0/1: one contraction.  4: the taps are 4 equal groups, one per
                                            output parity phase (py, px) = (z >> 1, z & 1) of a stride-2 transposed
                                            structure; phase z writes pixel (h*mul_h + off_h + py, w*mul_w + off_w + px)
                                            — ONE launch (grid.z = 4) instead of four under-filled ones */
  int stack_slot, stack_c;               /* stack_slot > 0: the N columns are 4 output-parity phases STACKED side by side,
                                            stack_slot columns apiece of which the first stack_c are real: column
                                            j = phase*stack_slot + c goes to pixel (h*mul_h + py, w*mul_w + px), channel c
                                            (bias[c]).  The up-sample+pad head (swapnet_modules.py:85-90) as ONE 9-tap GEMM
                                            with N = 4 x 24: its 192-channel input is read 9 times instead of 25.
                                            Needs n_valid = 4*stack_slot, nphase <= 1, out_mul = 2. */
  double* stats;                         /* optional [m_n][n_valid][2]: the launch ALSO accumulates (sum, sum of squares) of
                                            its output per (image, channel) — the InstanceNorm statistics of layers.py:17,
                                            33,134 — zeroing the buffer first; sn_stats_finalize turns them into (mean,
                                            rstd).  Only honoured when a tile never spans two images and n_valid % 16 == 0
                                            (sn_plan_has_stats tells); otherwise call sn_plane_stats. */
} sn_tap_gemm_desc;

/* G[i*s_row + j*s_col + tap_off[t]] += sum_{(n,h,w)} X[n, h+dh_t, w+dw_t, xc_t + i] * Y[n, h+dh'_t, w+dw'_t, yc_t + j]
 * Lowers every weight gradient (atomic accumulation into a zeroed fp32 buffer, which can be the
 * torch-layout .grad tensor itself). */
typedef struct sn_wgrad_desc {
  const void* x_hi; const void* x_lo; int x_n, x_h, x_w, x_c, x_pitch, x_parity, x_fmt;
  const void* y_hi; const void* y_lo; int y_n, y_h, y_w, y_c, y_pitch, y_parity, y_fmt;
  int m_n, m_h, m_w;                     /* pixel grid the reduction runs over */
  int ntaps;
  sn_tap xtaps[SN_MAX_TAPS];
  sn_tap ytaps[SN_MAX_TAPS];
  long long tap_off[SN_MAX_TAPS];
  float* out; long long s_row, s_col;
  int rows_valid, cols_valid;
  int block_n;                           /* 64 or 128; == y_chunk when Y is narrow */
  int y_chunk;                           /* channels per TMA row of Y: 64 (default when 0), 32 or 16 */
  /* narrow Y only: taps that share the same X tap are grouped, one CTA handles a group and reads X once:
   * group g = taps [group_start[g], +group_size[g]), each tap one y_chunk-wide column block of the
   * block_n = max_group * y_chunk accumulator.  ngroups == 0: every tap is its own launch slice. */
  int ngroups; int group_start[SN_MAX_TAPS]; int group_size[SN_MAX_TAPS];
  int ksplit;                            /* 0 = auto */
  int nsplit;
  int deterministic;                     /* 1: the ksplit partials go to a workspace owned by the plan and are added into
                                            out in split order by a second kernel (bit-identical on every run); the auto
                                            ksplit is then computed for SN_NUM_SMS SMs whatever the device, so the
                                            summation order depends on the shapes alone.  Needs distinct tap_off. */
} sn_wgrad_desc;

typedef struct sn_plan sn_plan; /* opaque; owns the encoded TMA descriptors of one launch */

int sn_tap_gemm_plan_create(const sn_tap_gemm_desc* desc, sn_plan** out);
int sn_wgrad_plan_create(const sn_wgrad_desc* desc, sn_plan** out);
int sn_plan_run(const sn_plan* plan, void* stream);
void sn_plan_destroy(sn_plan* plan);
/* 1 when the plan accumulates the fused InstanceNorm statistics requested through sn_tap_gemm_desc.stats */
int sn_plan_has_stats(const sn_plan* plan);
/* launch geometry of a plan, for per-plan timing tables: out[0] = kind (0 tap GEMM, 1 weight gradient), then
 * tap GEMM: M tiles, N tiles, phases, block_n, A row chunk; weight gradient: grid x, y, z, block_n, Y row chunk */
int sn_plan_geometry(const sn_plan* plan, int* out);
/* device workspace bytes a plan owns (the split-K partials of a deterministic weight-gradient plan; 0 otherwise) */
long long sn_plan_workspace_bytes(const sn_plan* plan);
/* the split-K count sn_wgrad_plan_create would choose for desc on a device with sm_count SMs (host only) */
int sn_wgrad_ksplit(const sn_wgrad_desc* desc, int sm_count);

/* ------------------------------------------------------------------------------------------
 * operand packing
 * ---------------------------------------------------------------------------------------- */
/* fp32 image tensor (NCHW contiguous, or NHWC with src_pitch; or a LABEL_U8 / MASK_I32 map expanded to c channels) -> split planes at channel
 * offset dst_coff of an NHWC plane pair with pitch dst_pitch.  Replaces the torch.cat /
 * .to(device) glue of warp_model.py:99-116 and swapnet_modules.py:258. */
int sn_pack_planes(const float* src, int src_layout, int src_pitch, int n, int c, int h, int w,
                   void* dst_hi, void* dst_lo, int dst_pitch, int dst_coff, int fmt, void* stream);

/* one pass: `lead` zero channels, then up to two fp32 sources (src1 may be NULL) concatenated along channels and
 * zero-filled to c_fill channels -> planes (dst_*) and, optionally, a second-format copy (dst2_*, e.g. the bf16 twin).
 * dst_coff, c_fill, dst_pitch multiples of 8; lead any count >= 0 (pix2pix's cat(zeros[B, 36], cloths),
 * pix2pix_model.py:158-159).  (cat((bodys, fakes), 1) of warp_model.py:115 etc.) */
int sn_pack_concat(int lead, const float* src0, int layout0, int pitch0, int c0, const float* src1, int layout1,
                   int pitch1, int c1, int n, int h, int w, int c_fill, void* dst_hi, void* dst_lo, void* dst2_hi,
                   void* dst2_lo, int dst_pitch, int dst_coff, int fmt, int fmt2, void* stream);

/* weight packing: torch conv weights -> kernel-layout split planes, a whole network in one launch per entry.  The item
 * tables live in DEVICE memory and are built once per engine.
 * sn_weight_scale_multi: scale2 <- (s, 1/s) of every tensor, s the exact power of two that brings max|w| into
 *   [2^13, 2^14) (1 when max|w| is 0).  Every w 16-byte aligned (float4 loads).  scratch: 2 * nitems zeroed uint32
 *   (left zeroed).
 * sn_pack_weights_multi: every item writes packed [rows][taps_pitch][k_pad] split planes (taps_pitch >= taps: extra
 *   tap slots stay zero, see a_chunk).  Source element (row r, tap t, k) is read at src[r*s_row + k*s_k + t] (taps
 *   contiguous, as in torch OIHW / IOHW) and written to tap slot slot[t], times scale2[0] when scale2 is not NULL;
 *   k >= k_real is zero.  taps <= 16, k_pad % 8 == 0, hi / lo 16-byte aligned.  block_begin = running sum of
 *   ceil(rows / sn_pack_rows_per_block()) * ceil(k_pad / sn_pack_k_per_block()), total_blocks its end. */
typedef struct sn_scale_item { const float* w; long long count; float* scale2; } sn_scale_item;
typedef struct sn_pack_item {
  const float* src; long long s_row, s_k;
  int rows, taps, taps_pitch, k_real, k_pad, fmt;
  void* hi; void* lo; const float* scale2;
  int slot[16];
  int block_begin;
} sn_pack_item;
int sn_weight_scale_multi(const sn_scale_item* items_dev, int nitems, unsigned int* scratch_dev, void* stream);
int sn_pack_weights_multi(const sn_pack_item* items_dev, int nitems, int total_blocks, int max_taps, void* stream);
int sn_pack_rows_per_block(void);
int sn_pack_k_per_block(void);

/* head conv (swapnet_modules.py:85-90): nearest x2 upsample + ZeroPad2d((1,0,1,0)) + Conv2d(k4,p1)
 * folded into 4 output-parity phases with 2/3 effective taps per dim (25 taps in total).
 *   fwd pack:  dst[phase][row=co (rows_pad)][teff][ci (k_pad)]   (rows >= cout are zero)
 *   dgrad pack: dst[row=ci][ (phase,teff) : taps_pitch >= 25 ][co (k_pad)]
 * src is torch OIHW [cout][cin][4][4]. */
int sn_pack_head_weights(const float* src, int cout, int cin, int rows_pad, int k_pad, int dgrad, int taps_pitch,
                         void* dst_hi, void* dst_lo, int fmt, const float* scale2, void* stream);
/* the same effective taps laid out for the phase-stacked 9-tap GEMM (sn_tap_gemm_desc.stack_slot):
 *   dst[row = phase*slot + co][tap = (sy+1)*3 + (sx+1)][ci (k_pad)], zero where the phase has no tap at that shift
 *   (parity 0 reads shifts -1, 0; parity 1 reads -1, 0, +1) and for co >= cout; rows = 4*slot. */
int sn_pack_head_stacked(const float* src, int cout, int cin, int slot, int k_pad, void* dst_hi, void* dst_lo, int fmt,
                         const float* scale2, void* stream);
/* fold the 25 effective-tap gradients [cout][25][cin] back onto dW [cout][cin][4][4] (+=) */
int sn_fold_head_wgrad(const float* geff, int cout, int cin, float* dw, void* stream);

/* ------------------------------------------------------------------------------------------
 * InstanceNorm / activation / dropout blocks (layers.py:17-20,32-36,133-138)
 * ---------------------------------------------------------------------------------------- */
/* per-(n,c) InstanceNorm statistics over the plane -> stats[n][c] = (mean, 1/sqrt(var_biased + eps))
 * as doubles (accumulated in fp64). */
int sn_plane_stats(const float* y, int pitch, int n, int hw, int c, float eps, double* stats,
                   void* stream);
/* (sum, sum of squares) over hw pixels -> (mean, 1/sqrt(var_biased + eps)) in place, `count` = n*c pairs */
int sn_stats_finalize(double* stats, int count, int hw, float eps, void* stream);
/* per-(n,c) (sum, sum of squares) over the plane, accumulated in fp64, without sn_stats_finalize's conversion */
int sn_plane_sums(const float* y, int pitch, int n, int hw, int c, double* stats, void* stream);

/* Deterministic variants (the *_det entry points, sn_norm_act_bwd_desc.det_slots): where the plain entry point adds
 * per-block partial sums with floating-point atomics, these store each block's partial to its own slot of the
 * caller's workspace `slots` (slots_cap doubles) and a second kernel adds the slots in index order, so the result is
 * bit-identical on every run.  Two launches that may overlap must not share a workspace.  sn_det_slots(n, c): doubles
 * of workspace enough for any of them whose output is [n][c] per-channel values (or a loss of n*c <= 2 terms). */
long long sn_det_slots(int n, int c);
int sn_plane_sums_det(const float* y, int pitch, int n, int hw, int c, double* stats, double* slots,
                      long long slots_cap, void* stream);
int sn_plane_stats_det(const float* y, int pitch, int n, int hw, int c, float eps, double* stats, double* slots,
                       long long slots_cap, void* stream);

/* BatchNorm2d(affine, track_running_stats) statistics (pix2pix / PatchGAN `--norm batch`).  The n samples form `groups`
 * consecutive groups of n/groups samples, each normalised as a call of its own (the discriminator's fake and real
 * halves).  Reductions over the samples run in sample order on one thread per channel: no atomics.
 * sn_bn_finalize (train mode): stats[n][c] = (sum, sum of squares) over hw pixels (a fused GEMM epilogue or
 * sn_plane_sums) -> (mean, 1/sqrt(var_biased + eps)) of the sample's group, in place; then, group after group,
 * running_mean/var <- (1 - momentum) * running + momentum * (mean, unbiased variance) and num_batches_tracked += groups
 * (running buffers and counter may be NULL: not tracked).
 * sn_bn_eval_stats (eval mode): stats[n][c] = (running_mean, 1/sqrt(running_var + eps)); nothing is updated. */
int sn_bn_finalize(double* stats, int n, int c, int groups, int hw, float eps, float momentum, float* running_mean,
                   float* running_var, long long* num_batches_tracked, void* stream);
int sn_bn_eval_stats(double* stats, int n, int c, const float* running_mean, const float* running_var, float eps,
                     void* stream);
/* Cross-rank batch statistics (data parallelism): every rank normalises with the statistics of each group's samples on
 * all ranks.  sn_bn_group_sums turns per-(n, c) pair sums — the forward's (sum, sum of squares) or the backward's
 * (sum g, sum g*xhat), see sn_norm_act_bwd_desc.bn_phase — into this rank's partials part[groups][c][3] =
 * (element count n/groups * hw, sum, sum of squares), summing the samples in sample order.  The caller gathers every
 * rank's part in rank order into gathered[world][groups][c][3] (the element count travels with the sums: shards may
 * differ in size).  sn_bn_finalize_gathered sums those slices in rank order, writes the (mean, rstd) of each local
 * sample's group to stats[n][c] and updates the running buffers as sn_bn_finalize does, with the unbiased variance over
 * the global count: every rank computes the same bits.  With world 1 both give sn_bn_finalize's results exactly. */
int sn_bn_group_sums(const double* stats, int n, int c, int groups, int hw, double* part, void* stream);
int sn_bn_finalize_gathered(double* stats, int n, int c, int groups, const double* gathered, int world, float eps,
                            float momentum, float* running_mean, float* running_var, long long* num_batches_tracked,
                            void* stream);

typedef struct sn_norm_act_desc {
  const float* y; int y_pitch;           /* conv output, [n, h, w, c] */
  int n, h, w, c;
  const double* stats;                   /* (mean, rstd) [n][c][2] or NULL (no InstanceNorm) */
  int act; float slope;                  /* SN_ACT_NONE / LRELU / RELU */
  float drop_p; unsigned long long drop_seed; /* drop_p == 0: no dropout */
  unsigned long long drop_offset;        /* added to the NHWC element index of the keep-mask: global sample index *
                                            h*w*c of the first local sample (data-parallel shards draw the masks of
                                            the samples they hold, SURVEY 8e ii) */
  const float* drop_step_seed_dev; unsigned int drop_stage_id; /* non-NULL: the 32-bit step seed is read on the device
                                            as two exact 16-bit halves (lo, hi) of the float step-parameter buffer
                                            (sn_set_step_params) and the seed is mix(step_seed, drop_stage_id): a captured
                                            CUDA graph replays with fresh masks; drop_seed is ignored */
  const float* residual; int res_pitch;  /* optional: out = residual + xhat (ResidualBlock tail) */
  void* out_hi; void* out_lo; int out_pitch, out_coff; /* optional split planes */
  int out_fmt;
  void* out2_hi; void* out2_lo; int out2_fmt; /* optional companion planes, same geometry (the
                                            bf16-split copy read by the weight-gradient GEMM: A and B
                                            of one wgmma must share a format) */
  int out_reflect_pad;                   /* 1: planes are [n, h+2, w+2] with ReflectionPad2d(1) */
  float* out_f32; int f32_pitch;         /* optional fp32 copy (residual stream) */
  const float* gamma; const float* beta; /* optional [c] BatchNorm weight / bias: the normalised value is
                                            gamma * xhat + beta (activation gate included); needs stats, c % 4 == 0 */
} sn_norm_act_desc;
int sn_norm_act_fwd(const sn_norm_act_desc* d, void* stream);

typedef struct sn_grad_src {
  const float* ptr; int pitch; int c_off;
  int reflect_padded;                    /* 1: [n, h+2, w+2] gradient of a reflect-padded operand */
  int up;                                /* >1: source is [n, h*up, w*up]; gradient of a nearest-upsampled
                                            copy (F.interpolate, swapnet_modules.py:244-247): block-summed */
  int act;                               /* -1: the block's activation; else SN_ACT_* of THIS consumer: the
                                            pix2pix skip reads relu() of a tensor whose other consumer reads
                                            leaky_relu() (pix2pix_modules.py:220-222,262) */
} sn_grad_src;

typedef struct sn_norm_act_bwd_desc {
  sn_grad_src src[SN_MAX_SRC]; int nsrc; /* upstream gradients w.r.t. the block output (summed) */
  const float* y; int y_pitch;
  int n, h, w, c;
  const double* stats;
  int act; float slope;
  float drop_p; unsigned long long drop_seed;
  unsigned long long drop_offset; const float* drop_step_seed_dev; unsigned int drop_stage_id;
  double* gstats;                        /* scratch [n][c][2] (needed when stats != NULL) */
  void* dy_hi; void* dy_lo; int dy_pitch, dy_coff; /* split planes of dL/dy */
  int dy_fmt;
  float* bias_grad;                      /* optional [c], c in {256, 512, 1024}: += sum over pixels of dL/dy (the bias
                                            gradient of the conv that produced y), fused into the apply pass */
  const float* gamma; const float* beta; /* BatchNorm (both NULL: InstanceNorm / none).  stats hold the (mean, rstd) of
                                            sn_bn_finalize or sn_bn_eval_stats */
  int bn_groups;                         /* sample groups of the forward call (sn_bn_finalize) */
  int bn_train;                          /* 1: batch statistics (dL/dy subtracts the group means); 0: running statistics */
  float* gamma_grad; float* beta_grad;   /* optional [c]: += d(loss)/d(gamma), d(loss)/d(beta) */
  double* det_slots; long long det_slots_cap; /* non-NULL: deterministic gstats reduction (see sn_det_slots; no
                                            fused bias_grad) */
  int bn_phase;                          /* BatchNorm, train mode, statistics across ranks: the call is split so that the
                                            gather of the gradient sums sits between its halves.  0: the whole backward
                                            (all fields below zero).  1: the reduction only; gstats is left holding the
                                            per-(n, c) (sum g, sum g*xhat) for sn_bn_group_sums.  2: group means from
                                            bn_gathered, then the apply pass */
  const double* bn_gathered; int bn_world; int bn_rank; /* phase 2: [bn_world][bn_groups][c][3] gathered partials,
                                            this rank's index: d(gamma), d(beta) add its slice only */
} sn_norm_act_bwd_desc;
int sn_norm_act_bwd(const sn_norm_act_bwd_desc* d, void* stream);

/* bias gradient db[c] = sum over the npix pixels of dL/dy (split planes); scratch: double[c] */
int sn_bias_grad(const void* dy_hi, const void* dy_lo, int pitch, int coff, int fmt, long long npix, int c,
                 double* scratch, float* db, void* stream);
int sn_bias_grad_det(const void* dy_hi, const void* dy_lo, int pitch, int coff, int fmt, long long npix, int c,
                     double* scratch, float* db, double* slots, long long slots_cap, void* stream);

/* dst[n,h,w,c] = sum_i src_i (fp32), e.g. the residual-stream gradient of a ResidualBlock */
int sn_sum_grads(const sn_grad_src* src, int nsrc, int n, int h, int w, int c, float* dst,
                 int dst_pitch, void* stream);

/* dL/dy of a tanh output: (sum_i src_i) * (1 - out^2) -> split planes */
int sn_tanh_bwd(const sn_grad_src* src, int nsrc, const float* out, int out_pitch, int n, int h,
                int w, int c, void* dy_hi, void* dy_lo, int dy_pitch, int dy_coff, int dy_fmt, void* stream);

/* nearest-neighbour up-sampling of split planes (16-bit words are copied, hi and lo):
 * dst[n, h, w, dst_coff + c] = src[n, h / f, w / f, src_coff + c] */
int sn_upsample_planes(const void* src_hi, const void* src_lo, int src_pitch, int src_coff, int n, int h, int w,
                       int c, int factor, void* dst_hi, void* dst_lo, int dst_pitch, int dst_coff, void* stream);

/* fused AdamW step over flat fp32 buffers (torch.optim.AdamW semantics as optimizers/__init__.py:48-59
 * builds it: decoupled weight decay, bias correction, eps outside the sqrt); step is 1-based. */
int sn_adamw_step(float* p, const float* g, float* m, float* v, long long n, double lr, double beta1, double beta2,
                  double eps, double weight_decay, int step, void* stream);
/* the same update with its scalars read from DEVICE memory, so that a captured CUDA graph of the training step replays
 * with the current step's bias corrections: hyper[8] = { 1 - lr*wd, 1 - beta1, beta2, 1 - beta2, lr / (1 - beta1^t),
 * 1 / sqrt(1 - beta2^t), eps, gscale } with gscale multiplied into every gradient as it is read (1/world under data
 * parallelism: the all-reduce leaves the SUM in g).  sn_adamw_hyper fills the 8 floats on the host. */
int sn_adamw_step_dev(float* p, const float* g, float* m, float* v, long long n, const float* hyper_dev, void* stream);
void sn_adamw_hyper(double lr, double beta1, double beta2, double eps, double weight_decay, int step, double gscale,
                    float hyper_out[8]);

/* fused AdaBound step over flat fp32 buffers (Luo et al., "Adaptive Gradient Methods with Dynamic Bound of Learning
 * Rate", ICLR 2019; the update of adabound.AdaBound as optimizers/__init__.py:55-59 builds it, amsbound off), t = step:
 *   g += wd * p;  m = b1 m + (1 - b1) g;  v = b2 v + (1 - b2) g g;
 *   p -= clamp(lr sqrt(1 - b2^t) / (1 - b1^t) / (sqrt(v) + eps), lower, upper) * m
 *   lower = F (1 - 1 / (gamma t + 1)),  upper = F (1 + 1 / (gamma t)),  F = final_lr * lr / base_lr
 * base_lr is the lr the optimizer was created with (> 0); gamma > 0, final_lr >= 0, step is 1-based. */
int sn_adabound_step(float* p, const float* g, float* m, float* v, long long n, double lr, double base_lr, double beta1,
                     double beta2, double eps, double weight_decay, double final_lr, double gamma, int step,
                     void* stream);
/* the same update with its scalars read from DEVICE memory (see sn_adamw_step_dev): hyper[8] = { 1 - beta1, 1 - beta2,
 * eps, wd, lr sqrt(1 - beta2^t) / (1 - beta1^t), lower, upper, gscale }, gscale multiplied into every gradient as it
 * is read and BEFORE the decay term is added.  sn_adabound_hyper fills the 8 floats on the host. */
int sn_adabound_step_dev(float* p, const float* g, float* m, float* v, long long n, const float* hyper_dev,
                         void* stream);
void sn_adabound_hyper(double lr, double base_lr, double beta1, double beta2, double eps, double weight_decay,
                       double final_lr, double gamma, int step, double gscale, float hyper_out[8]);

/* per-step scalars of the training step (smooth GAN labels, AdamW scalars, the dropout step seed) live in one small
 * device buffer: dst[0..n) <- vals (n <= 64 floats, passed BY VALUE through the launch, so the host array may be reused
 * immediately); launched once per step ahead of the (possibly graph-replayed) step kernels. */
int sn_set_step_params(float* dst, const float* vals, int n, void* stream);

/* deterministic dropout keep-mask shared by forward, backward and the test oracle:
 * keep(seed, idx) with idx the linear NHWC element index; returns 0/1 bytes. */
int sn_dropout_mask(unsigned long long seed, float p, long long count, uint8_t* out, void* stream);

/* ------------------------------------------------------------------------------------------
 * losses (value + gradient in one pass)
 * ---------------------------------------------------------------------------------------- */
/* CrossEntropyLoss(logits, argmax(target,1)) * weight  (warp_model.py:147-150).
 * logits NHWC [n,h,w,c] (pitch), target NCHW [n,c,h,w] — or, with target_layout = SN_LAYOUT_LABEL_U8, the uint8
 * label map [n,h,w] itself (argmax of its one-hot expansion: the label; 0 for background); loss accumulated into
 * *loss_acc (double, caller zeroes); grad NHWC fp32 (pitch c). */
int sn_ce_loss_fwd_bwd(const float* logits, int pitch, const void* target, int target_layout, int n, int h, int w,
                       int c, float weight, double* loss_acc, float* grad, int grad_pitch, void* stream);
/* the same cross entropy fused with the backward of the tanh head it is applied to (warp_model.py:147-150: CE on the
 * tanh OUTPUTS): dy = (weight * dCE/do + sum_i src_i) * (1 - o^2) as split planes, loss value accumulated; the extra
 * sources carry the other loss terms' gradients w.r.t. o (the GAN term).  Replaces sn_ce_loss_fwd_bwd + sn_tanh_bwd. */
int sn_ce_tanh_bwd(const float* logits, int pitch, const void* target, int target_layout, const sn_grad_src* src,
                   int nsrc, int n, int h, int w, int c, float weight, double* loss_acc, void* dy_hi, void* dy_lo,
                   int dy_pitch, int dy_coff, int dy_fmt, void* stream);
int sn_ce_tanh_bwd_det(const float* logits, int pitch, const void* target, int target_layout, const sn_grad_src* src,
                       int nsrc, int n, int h, int w, int c, float weight, double* loss_acc, void* dy_hi, void* dy_lo,
                       int dy_pitch, int dy_coff, int dy_fmt, double* slots, long long slots_cap, void* stream);
/* BCEWithLogitsLoss(pred, t) over two consecutive halves of `count` elements each with its own
 * target (loss.py:58,110-122): loss_acc[half] += mean, dpred = gscale * (sigmoid(x) - t)/count. */
int sn_bce_logits_fwd_bwd(const float* pred, long long count_per_half, int halves, float t0, float t1,
                          float gscale, double* loss_acc, float* dpred, void* stream);
/* targets read from device memory: t_dev[0] (first half) and t_dev[1] (second half) */
int sn_bce_logits_fwd_bwd_dev(const float* pred, long long count_per_half, int halves, const float* t_dev,
                              float gscale, double* loss_acc, float* dpred, void* stream);
/* GANLoss objectives (loss.py:53-62,110-130), the --gan_mode values that need no gradient penalty. */
enum { SN_GAN_BCE = 0, SN_GAN_MSE = 1, SN_GAN_WGAN = 2 };
/* One GAN objective over `halves` (1 or 2) consecutive blocks of count_per_half predictions, each with its own scalar:
 * loss_acc[half] += the unweighted batch mean, dpred = gscale * d(mean)/d(pred) (dpred may be null).
 *   SN_GAN_BCE   vanilla: BCEWithLogitsLoss(pred, t)     t = t_dev[half] if t_dev is non-null, else t0 / t1
 *   SN_GAN_MSE   lsgan:   MSELoss(pred, t)               t as for SN_GAN_BCE
 *   SN_GAN_WGAN  wgan:    t * mean(pred), t0 / t1 = +1 (fake) or -1 (real); t_dev must be null
 * SN_GAN_BCE runs the kernel of sn_bce_logits_fwd_bwd(_dev). */
int sn_gan_loss_fwd_bwd_dev(int objective, const float* pred, long long count_per_half, int halves, float t0, float t1,
                            const float* t_dev, float gscale, double* loss_acc, float* dpred, void* stream);
int sn_gan_loss_fwd_bwd_det(int objective, const float* pred, long long count_per_half, int halves, float t0, float t1,
                            const float* t_dev, float gscale, double* loss_acc, float* dpred, double* slots,
                            long long slots_cap, void* stream);
/* L1Loss(a, b) * weight (texture_model.py:168-170); a NHWC (pitch), b NCHW; grad wrt a. */
int sn_l1_loss_fwd_bwd(const float* a, int pitch, const float* b_nchw, int n, int h, int w, int c,
                       float weight, double* loss_acc, float* grad, int grad_pitch, void* stream);
int sn_l1_loss_fwd_bwd_det(const float* a, int pitch, const float* b_nchw, int n, int h, int w, int c, float weight,
                           double* loss_acc, float* grad, int grad_pitch, double* slots, long long slots_cap,
                           void* stream);

/* ------------------------------------------------------------------------------------------
 * one-output-channel conv (PatchGAN logits, discriminators.py:131) over a per-tap
 * product image P[n,h,w,t] = sum_c x[n,h,w,c] W[0,c,t] (the input is read once instead of once per tap):
 *   y[n,oh,ow] = bias + sum_{kh,kw} P[n, oh+kh-pad, ow+kw-pad, kh*k+kw]
 * ---------------------------------------------------------------------------------------- */
int sn_tap_sum_fwd(const float* p, int p_pitch, int n, int h, int w, int k, int pad, const float* bias, float* y,
                   int y_pitch, void* stream);

/* the one-output-channel conv on the CUDA cores at stream speed (csrc/patch_logits.cu; k = 4, stride 1):
 *   sn_to_one_fwd:   p[px][t] = sum_c x[px][c] * weight[c*16 + t]      x: split planes [npix][x_pitch], weight: the torch
 *                                                                      [1][c][4][4] parameter itself (no packing)
 *   sn_to_one_wgrad: dw[c*16 + t] += sum_px x[px][c] * dy[px - off_t]  dy: channel 0 of split planes [n][h+2p-3][w+2p-3]
 *   sn_to_one_dgrad: dx[px][c]  = sum_t dy[px - off_t] * weight[c*16 + t]   (fp32 NHWC, pitch dx_pitch) */
int sn_to_one_fwd(const void* x_hi, const void* x_lo, int x_pitch, int x_fmt, long long npix, int c, const float* weight,
                  int k, float* p, int p_pitch, void* stream);
int sn_to_one_wgrad(const void* x_hi, const void* x_lo, int x_pitch, int x_fmt, int n, int h, int w, int c,
                    const void* dy_hi, const void* dy_lo, int dy_pitch, int dy_fmt, int k, int pad, float* dw,
                    void* stream);
/* deterministic sn_to_one_wgrad: per-block partials of dw in `slots` (float, slots_cap of them;
 * sn_to_one_wgrad_det_slots(c) are enough), added into dw in block order */
int sn_to_one_wgrad_det(const void* x_hi, const void* x_lo, int x_pitch, int x_fmt, int n, int h, int w, int c,
                        const void* dy_hi, const void* dy_lo, int dy_pitch, int dy_fmt, int k, int pad, float* dw,
                        float* slots, long long slots_cap, void* stream);
long long sn_to_one_wgrad_det_slots(int c);
int sn_to_one_dgrad(const void* dy_hi, const void* dy_lo, int dy_pitch, int dy_fmt, int n, int h, int w, int c,
                    const float* weight, int k, int pad, float* dx, int dx_pitch, void* stream);

/* ------------------------------------------------------------------------------------------
 * VGG16 perceptual loss (modules/losses/perceptual.py:6-79, used by texture_model.py:68-69,171-176).
 * The 13 conv3x3(+bias) layers run as tap-GEMM plans; these are the element-wise pieces.
 * ---------------------------------------------------------------------------------------- */
/* planes[n,h,w,0:16] = split(mul * src + add), channels >= c zero  (get_features' x <- 2x - 1, :70). c <= 16. */
int sn_affine_pack(const float* src, int src_layout, int src_pitch, int n, int c, int h, int w, float mul, float add,
                   void* dst_hi, void* dst_lo, int dst_pitch, int dst_coff, int fmt, void* stream);
/* nn.ReLU + nn.MaxPool2d(2) of vgg16.features (indices 3-4, 8-9, 15-16, 22-23): y fp32 [n,h,w,c] ->
 * split planes [n,h/2,w/2,c]. */
int sn_relu_pool_fwd(const float* y, int y_pitch, int n, int h, int w, int c, void* out_hi, void* out_lo,
                     int out_pitch, int out_coff, int fmt, void* stream);
/* its adjoint: dy = (g_direct + [first max of the 2x2 window] g_pool) * (y > 0) as split planes.
 * g_pool [n,h/2,w/2,c] and g_direct [n,h,w,c] fp32, either may be NULL. */
int sn_relu_pool_bwd(const float* y, int y_pitch, const float* g_pool, int gp_pitch, const float* g_direct,
                     int gd_pitch, int n, int h, int w, int c, void* dy_hi, void* dy_lo, int dy_pitch, int dy_coff,
                     int dy_fmt, void* stream);
/* one tap of the content loss (perceptual.py:53-57,72-78): x = relu(y), f = x / (|x|_2 over c + 1e-8),
 * *loss_acc += weight * sum (f_out - f_tgt)^2  (weight = lambda / numel), dx = gscale * d(loss)/d(x_out)
 * (gradient w.r.t. the post-ReLU feature; gscale carries the 2 of x <- 2x - 1). c in {64..512}, c % 4 == 0. */
int sn_feat_loss_fwd_bwd(const float* y_out, int po, const float* y_tgt, int pt, long long npix, int c, double weight,
                         double gscale, double* loss_acc, float* dx, int pdx, void* stream);
/* deterministic variant (see sn_det_slots: sn_det_slots(1, 1) slots are enough) */
int sn_feat_loss_fwd_bwd_det(const float* y_out, int po, const float* y_tgt, int pt, long long npix, int c,
                             double weight, double gscale, double* loss_acc, float* dx, int pdx, double* slots,
                             long long slots_cap, void* stream);
/* gram_matrix (perceptual.py:6-10) of the rows r = (b, ch): X_r[p] = src[b*s_n + ch*s_c + p*s_p];
 * gram: double [n*c][n*c] (zeroed here).  n*c <= 96. */
int sn_gram(const float* src, long long s_n, long long s_c, long long s_p, int n, int c, long long npix, double* gram,
            void* stream);
/* deterministic variant: per-block partial Gram matrices in `slots` (sn_gram_det_slots(n*c) doubles are enough), added
 * in block order.  sn_gram_mse is one block and needs no variant. */
int sn_gram_det(const float* src, long long s_n, long long s_c, long long s_p, int n, int c, long long npix,
                double* gram, double* slots, long long slots_cap, void* stream);
long long sn_gram_det_slots(int rows);

/* ------------------------------------------------------------------------------------------
 * 1x1 PixelGAN discriminator (discriminators.py:138-168, csrc/pixel_disc.cu): per pixel
 *   z1 = W1 x + b1 (64), a1 = lrelu(z1), z2 = W2 a1 (+ b2) (128), y2 = InstanceNorm(z2) or z2, a2 = lrelu(y2),
 *   pred = w3 . a2 (+ b3).
 * Every pass recomputes z1 and z2 from x through one device function (bit-identical in every pass); nothing of the
 * hidden layers is stored.  Weights are the torch parameters themselves ([64][cin], [128][64], [1][128]).
 * ---------------------------------------------------------------------------------------- */
typedef struct sn_pixel_desc {
  const void* x_hi; const void* x_lo;     /* fp16-split operand planes [n*hw][x_pitch] (forward products) */
  const void* xb_hi; const void* xb_lo;   /* their bf16-split twin (dW1 in sn_pixel_bwd_apply) */
  int x_pitch, x_c;                        /* x_c = 16 or 32 channels read, zero from cin on */
  int n, hw, cin;
  const float* w1; const float* b1; const float* w2; const float* b2; const float* w3; const float* b3;  /* b2, b3 may be
                                            NULL (--norm none: no bias on net.2 / net.5) */
  const float* scale1; const float* scale2;  /* device (s, 1/s) of w1 and w2 from sn_weight_scale_multi */
  int norm;                                /* 1: InstanceNorm2d(affine=False) after net.2, 0: none */
  int nsplit;                              /* 3 = split products, 1 = hi x hi only */
  float slope, eps;                        /* LeakyReLU slope (0.2), InstanceNorm eps */
  double* stats;                           /* [n][128][2]: (mean, rstd) of z2 per (image, channel) */
  double* gstats;                          /* [n][128][2]: (sum g2, sum g2 * y2) */
  float* pred;                             /* [n*hw] logits */
  const float* dpred;                      /* [n*hw] dL/dpred */
  float* dw1; float* db1; float* dw2; float* db2; float* dw3; float* db3;   /* += gradients; NULL: not computed */
  float* dx; int dx_pitch;                 /* optional fp32 NHWC [n*hw][dx_pitch]: dL/dx, channels < cin */
  float* debug;                            /* optional [n*hw][64 + 128]: z1 and y2 (sn_pixel_fwd) */
  double* slots; long long slots_cap;      /* non-NULL: deterministic reductions (sn_pixel_det_slots doubles) */
} sn_pixel_desc;
/* stats <- (mean, rstd): per-(n, c) sum z2 and sum z2^2 in fp64, then sn_stats_finalize (norm = 1 only) */
int sn_pixel_fwd_stats(const sn_pixel_desc* d, void* stream);
/* pred (and debug) */
int sn_pixel_fwd(const sn_pixel_desc* d, void* stream);
/* gstats <- (sum g2, sum g2 * y2), g2 = dpred w3 lrelu'(y2); dw3 += sum dpred a2, db3 += sum dpred (norm = 1 only) */
int sn_pixel_bwd_reduce(const sn_pixel_desc* d, void* stream);
/* dz2 (the InstanceNorm backward, or g2), dw2/db2, g1 = (W2^T dz2) lrelu'(z1), dw1/db1, dx = W1^T g1; with norm = 0 also
 * dw3/db3 */
int sn_pixel_bwd_apply(const sn_pixel_desc* d, void* stream);
long long sn_pixel_det_slots(int n, int cin);
/* *loss_acc += weight * MSELoss(gram_out, gram_tgt);  m[r][j] = d(that)/d(gram_out) + transpose (fp32). */
int sn_gram_mse(const double* gram_out, const double* gram_tgt, int rows, double weight, double* loss_acc, float* m,
                void* stream);
/* dx[b, p, ch] (+)= sum_j m[b*c + ch][j] X_j[p]  — the style-loss gradient w.r.t. the raw image; dx NHWC fp32. */
int sn_gram_bwd(const float* m, const float* src, long long s_n, long long s_c, long long s_p, int n, int c,
                long long npix, float* dx, int dx_pitch, int accumulate, void* stream);

/* ------------------------------------------------------------------------------------------
 * ROIAlign + channel repack (swapnet_modules.py:209-240, torchvision roi_align aligned=False,
 * spatial_scale=1, sampling_ratio=1, output 128x128): tex NCHW [b,3,h,w], rois [b,nroi,4]
 * (x1,y1,x2,y2) -> fp32 NHWC [b,pool,pool,3*nroi] and/or split planes.
 * ---------------------------------------------------------------------------------------- */
int sn_roi_align_pack_fwd(const float* tex_nchw, int b, int ch, int h, int w, const float* rois,
                          int nroi, int pool, float* out_f32, int out_pitch, void* out_hi,
                          void* out_lo, int plane_pitch, int plane_coff, int plane_fmt, void* stream);

/* ------------------------------------------------------------------------------------------
 * Per-channel cloth augmentation on the device (SURVEY §8 f4): replaces datasets/data_utils.py:346-361
 * `per_channel_transform` — every channel of the one-hot cloth tensor through its own random
 * RandomOrder([RandomVerticalFlip, RandomHorizontalFlip, RandomAffine, RandomPerspective]) (datasets/__init__.py:88-110,
 * call site datasets/warp_dataset.py:133-134) — fused with the label map -> one-hot expansion of
 * data_utils.py:330-343.  The draws are made on the host (torchvision's get_params); an op is one Pillow
 * resampling, restated bit-exactly (libImaging/Geometry.c): flips, AFFINE+NEAREST in 16.16 fixed point
 * (p[0..5] = the FIX()ed integer coefficients a0..a5 as doubles), PERSPECTIVE+BILINEAR on mode "F"
 * (p[0..7] = the 8 coefficients of Image.transform).
 *   ops_dev[(b*c + ch) * op_stride + j] = j-th op of that plane, `nops` (same in every entry of the plane) of them;
 *   source = uint8 label map [n,h,w] (label L > 0 -> channel L, 0 -> nothing) or dense fp32 [n,c,h,w];
 *   out/tmp fp32 [n,c,h,w]; tmp may be null when max_ops < 2.  max_ops = max over planes of nops (passes launched).
 * ---------------------------------------------------------------------------------------- */
#define SN_AUG_NONE 0
#define SN_AUG_HFLIP 1
#define SN_AUG_VFLIP 2
#define SN_AUG_AFFINE_NEAREST 3
#define SN_AUG_PERSPECTIVE_BILINEAR 4
#define SN_AUG_MAX_OPS 8
typedef struct sn_aug_op {
  int kind;     /* SN_AUG_* */
  int nops;     /* number of ops of this plane */
  double p[8];
} sn_aug_op;
int sn_augment_channels(const void* labels_u8, const float* dense_nchw, int n, int c, int h, int w,
                        const sn_aug_op* ops_dev, int op_stride, int max_ops, float* out_nchw, float* tmp_nchw,
                        void* stream);

/* ------------------------------------------------------------------------------------------
 * reference-free fp32 CUDA-core contraction with the tap-GEMM semantics (no tensor cores).
 * Used by the tests as an on-device cross-check of the wgmma path, never by the plugin.
 * ---------------------------------------------------------------------------------------- */
int sn_tap_gemm_simt(const sn_tap_gemm_desc* desc, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SWAPNET_B200_H */
