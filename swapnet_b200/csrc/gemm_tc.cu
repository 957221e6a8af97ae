// swapnet_b200 — wgmma implicit-GEMM kernels (sm_90a).
//
// Every dense contraction of the SwapNet hot path (reference call sites:
// modules/layers.py:15,31,131-138  Conv2d 4x4 s2 / ConvTranspose2d 4x4 s2 /
// reflect-pad Conv2d 3x3; modules/swapnet_modules.py:85-90 upsample+pad+conv
// head; modules/discriminators.py:111-131 PatchGAN convs; and their autograd
// dgrad / wgrad) is lowered by the host onto ONE generic contraction:
//
//   "tap GEMM" (conv mode, K-major operands)
//     D[(n,h,w), j] = sum_{t < ntaps} sum_{c < k_per_tap}
//                       A[n, h + dh_t, w + dw_t, (hp_t), c_off_t + c] * Wp[j, kb_off_t + c]
//   A is an NHWC activation tensor carried as split-bf16 planes (hi, lo); the
//   128-row M tile is a th x tw x nb patch of GEMM rows, so the A tile of one
//   (tap, 64-channel chunk) is a single 5-D TMA box whose out-of-bounds part is
//   zero-filled by the TMA unit (= the conv zero padding).  Stride-2 gathers go
//   through a 2x2 "parity view" of the same memory (dims c', w/2, h%2, h/2, n).
//
//   "wgrad GEMM" (MN-major operands)
//     G[i, j] (+)= sum_{pixels (n,h,w)} X[n, h + dh, w + dw, i] * Y[n, h + dh', w + dw', j]
//   both operands are activation patches; the reduction runs over pixels.
//
// Arithmetic: 16-bit tensor-core MMAs (wgmma.mma_async, bf16 or f16) with fp32
// accumulation in registers.  NSPLIT = 3 evaluates hi*hi + lo*hi + hi*lo, i.e. an
// fp32-faithful product (~2^-16 relative) as the 1e-3 fp32 parity bar requires;
// NSPLIT = 1 is the single-pass bf16 fast mode.
//
// Warp roles (288 threads): warps 0..7 = two MMA warpgroups (64 rows of the
// 128-row tile each; they also run the epilogue, registers -> global), warp 8 =
// TMA producer.
#include "common.cuh"
#include "plan.h"

namespace {

constexpr int kBlockM = 128;
constexpr int kTileRing = 4;
constexpr int kTileBytes = 16384;  // 128 rows x 128 B (one operand plane of one stage)
constexpr int kConsumerWarps = 8;  // two MMA warpgroups, 64 of the 128 tile rows each
constexpr int kProducerWarp = kConsumerWarps;
constexpr int kThreads = (kConsumerWarps + 1) * 32;

template <int NSPLIT>
struct Cfg {
  static constexpr int kPlanes = NSPLIT == 3 ? 2 : 1;
  static constexpr int kStages = NSPLIT == 3 ? 3 : 6;
  static constexpr int kStageBytes = kPlanes * 2 * kTileBytes;
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024;  // + alignment slack
};

__device__ __forceinline__ float apply_act(float v, int act) {
  if (act == SN_ACT_TANH) return tanhf(v);
  return v;
}

// Sum over the 8 rows held by lanes with the same (lane % 4): after the call every lane holds its column's total over
// the warp's 16 accumulator rows (given v = the sum of the lane's two rows).
__device__ __forceinline__ float quad_col_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 4);
  v += __shfl_xor_sync(0xffffffffu, v, 8);
  v += __shfl_xor_sync(0xffffffffu, v, 16);
  return v;
}

// ============================================================================
// conv mode
// ============================================================================
// CW = channels per A row (64 / 32 / 16) and BN = MMA N (>= block_n): template parameters so that the MMA loop
// carries no runtime index arithmetic.  F16: both operands f16 (else bf16).
template <int NSPLIT, int CW, int BN, bool F16>
__global__ void __launch_bounds__(kThreads, 1)
tap_gemm_kernel(const __grid_constant__ TapGemmParams p, const int m_tiles, const int n_tiles, const int total_tiles) {
  // Persistent: one CTA per SM walks tiles blockIdx.x, blockIdx.x + gridDim.x, ... (N tile fastest, then M tile,
  // then output-parity phase).  The smem ring keeps running across tiles, so the producer loads the next tile's
  // stages while the MMA warpgroups run the epilogue of the current one, and the pipeline prologue is paid once per
  // CTA instead of once per tile.
  // N tile fastest: the resident CTAs cover all N tiles of ~132 / n_tiles M tiles, so the activation rows they read
  // (~10 MB for a resblock conv) stay in L2 from one tap to the next.  M tile fastest spread them over 132 M tiles:
  // the whole 75 MB operand, beyond the 50 MB L2, so every tap re-read it from HBM.
  const auto tile_coords = [&](int tile, int& mt, int& nt, int& z) {
    nt = tile % n_tiles;
    const int rest = tile / n_tiles;
    mt = rest % m_tiles;
    z = rest / m_tiles;
  };
  using C = Cfg<NSPLIT>;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[C::kStages];
  __shared__ __align__(8) uint64_t empty_bar[C::kStages];
  // dynamic tile schedule: the producer draws tile numbers from a device counter (p.tile_counter) and hands them
  // to the MMA warps through a 4-deep ring, so a CTA that becomes resident late (SMs held by NCCL or by the
  // weight-gradient stream's CTAs) finds only the tiles nobody has taken yet instead of a fixed 1/gridDim share
  __shared__ __align__(8) uint64_t tr_full[kTileRing];
  __shared__ __align__(8) uint64_t tr_empty[kTileRing];
  __shared__ int tile_ring[kTileRing];

  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (smem_base - smem_u32(smem_raw));
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  constexpr int cw = CW;                    // channels per A row: 64, 32 or 16
  constexpr int tps = 64 / cw;              // taps sharing one 64-deep stage (1, 2 or 4)
  // output parity phase z (merged 4-phase launches) owns taps [z*tpp, (z+1)*tpp)
  const int tpp = p.ntaps / p.nphase;
  const int k_iters = cw == 64 ? tpp * p.chunks : tpp / tps;

  if (threadIdx.x == 0) {
    for (int s = 0; s < C::kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);    // one arrival per MMA warpgroup
    }
    for (int r = 0; r < kTileRing; ++r) {
      mbar_init(&tr_full[r], 1);
      mbar_init(&tr_empty[r], kConsumerWarps);
    }
    mbar_fence_init();
  }
  if (warp == kProducerWarp && lane == 0) {
    for (int pl = 0; pl < C::kPlanes; ++pl) {
      tma_prefetch_desc(&p.tmA[pl]);
      tma_prefetch_desc(&p.tmB[pl]);
    }
  }
  __syncthreads();

  if (warp == kProducerWarp) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      const uint32_t stage_tx = C::kPlanes * (p.a_rows * 128 + p.block_n * 128);
      uint32_t it = 0, tcount = 0;
      for (int tile = blockIdx.x;; ++tcount) {
        // the first tile is static; every further one a ticket.  The ticket for the NEXT tile is drawn now (its latency
        // hides behind this tile's loads), the tile number goes to the other warps through the ring
        const int next = tile < total_tiles ? (int)gridDim.x + atomicAdd(p.tile_counter, 1) : total_tiles;
        const uint32_t slot = tcount % kTileRing, rph = (tcount / kTileRing) & 1;
        mbar_wait(&tr_empty[slot], rph ^ 1);
        tile_ring[slot] = tile < total_tiles ? tile : -1;
        mbar_arrive(&tr_full[slot]);
        if (tile >= total_tiles) break;
        int mt, nt, z;
        tile_coords(tile, mt, nt, z);
        const int ncol0 = nt * p.block_n;
        const int tap0 = z * tpp;
        const int w0 = (mt % p.tiles_w) * p.tw;
        const int h0 = ((mt / p.tiles_w) % p.tiles_h) * p.th;
        const int n0 = (mt / (p.tiles_w * p.tiles_h)) * p.nb;
        for (int k = 0; k < k_iters; ++k, ++it) {
          const uint32_t s = it % C::kStages;
          const uint32_t ph = (it / C::kStages) & 1;
          mbar_wait(&empty_bar[s], ph ^ 1);
          mbar_expect_tx(&full_bar[s], stage_tx);
          uint8_t* st = smem + s * C::kStageBytes;
          if (cw == 64) {
            const int t = k / p.chunks;
            const int ch = k - t * p.chunks;
            const TapDesc tap = p.taps[tap0 + t];
            if (p.a_merged) {   // dims (c, w, h, n, plane): hi tile, then lo tile
              tma_load_5d(&p.tmA[0], &full_bar[s], st, tap.c_off + ch * 64, w0 + tap.dw, h0 + tap.dh, n0, 0);
            } else {
#pragma unroll
              for (int pl = 0; pl < C::kPlanes; ++pl)
                tma_load_5d(&p.tmA[pl], &full_bar[s], st + pl * kTileBytes, tap.c_off + ch * 64,
                            w0 + tap.dw, tap.hp, h0 + tap.dh, n0);
            }
            if (p.b_merged) {   // dims (k, row, plane)
              tma_load_3d(&p.tmB[0], &full_bar[s], st + C::kPlanes * kTileBytes, tap.kb_off + ch * 64, ncol0, 0);
            } else {
#pragma unroll
              for (int pl = 0; pl < C::kPlanes; ++pl)
                tma_load_2d(&p.tmB[pl], &full_bar[s], st + (C::kPlanes + pl) * kTileBytes,
                            tap.kb_off + ch * 64, ncol0);
            }
          } else {
            // narrow operand: 64/cw taps, each a [128 rows][cw channels] sub-tile, fill one stage; the
            // weights of consecutive taps are contiguous in K, so B is still one 64-deep box
            constexpr int sub = 128 * cw * 2;
#pragma unroll
            for (int j = 0; j < tps; ++j) {
              const TapDesc tap = p.taps[tap0 + k * tps + j];
#pragma unroll
              for (int pl = 0; pl < C::kPlanes; ++pl)
                tma_load_5d(&p.tmA[pl], &full_bar[s], st + pl * kTileBytes + j * sub, tap.c_off,
                            w0 + tap.dw, tap.hp, h0 + tap.dh, n0);
            }
            const int kb = p.taps[tap0 + k * tps].kb_off;
            if (p.b_merged) {
              tma_load_3d(&p.tmB[0], &full_bar[s], st + C::kPlanes * kTileBytes, kb, ncol0, 0);
            } else {
#pragma unroll
              for (int pl = 0; pl < C::kPlanes; ++pl)
                tma_load_2d(&p.tmB[pl], &full_bar[s], st + (C::kPlanes + pl) * kTileBytes, kb, ncol0);
            }
          }
        }
        tile = next;
      }
    }
  } else {
    // ===================== MMA warpgroups + epilogue =====================
    const int wg = warp >> 2;                              // rows [64 wg, 64 wg + 64) of the tile
    const int quad = lane & 3;
    const int row0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // this thread's rows: row0 and row0 + 8
    int w_i[2], h_i[2], n_i[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = row0 + 8 * h;
      w_i[h] = row % p.tw;
      h_i[h] = (row / p.tw) % p.th;
      n_i[h] = row / (p.tw * p.th);
    }
    const float oscale = p.b_scale ? p.b_scale[1] : 1.f;  // undo the power-of-two weight scale (exact)
    float acc[BN / 2];
    uint32_t it = 0;
    for (uint32_t tcount = 0;; ++tcount) {
      const uint32_t slot = tcount % kTileRing, rph = (tcount / kTileRing) & 1;
      mbar_wait(&tr_full[slot], rph);
      const int tile = tile_ring[slot];
      __syncwarp();
      if (lane == 0) mbar_arrive(&tr_empty[slot]);
      if (tile < 0) break;
      for (int k = 0; k < k_iters; ++k, ++it) {
        const uint32_t s = it % C::kStages;
        const uint32_t ph = (it / C::kStages) & 1;
        mbar_wait(&full_bar[s], ph);
        const uint32_t st = smem_base + s * C::kStageBytes;
        // K-major, rows of cw channels: SWIZZLE_128B/64B/32B, SBO = 8 rows; this warpgroup's 64 rows start
        // 64 rows into every A sub-tile
        constexpr uint32_t a_layout = cw >= 64 ? 1u : (cw == 32 ? 2u : 3u);
        constexpr uint32_t a_sbo = 8u * cw * 2u;
        const uint32_t a_row0 = (uint32_t)wg * 64u * cw * 2u;
        const uint64_t a_hi = gmma_smem_desc(st + a_row0, 16, a_sbo, a_layout);
        const uint64_t b_hi = gmma_smem_desc(st + C::kPlanes * kTileBytes, 16, 1024);
        const uint64_t a_lo = gmma_smem_desc(st + p.a_lo_off + a_row0, 16, a_sbo, a_layout);
        const uint64_t b_lo = gmma_smem_desc(st + C::kPlanes * kTileBytes + p.b_lo_off, 16, 1024);
        constexpr uint32_t sub16 = (uint32_t)(128 * cw * 2) >> 4;  // sub-tile stride in 16-B units
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {  // 4 x (K = 16 elements = 32 B) per 64-deep stage
          const uint64_t badv = (uint64_t)(kk * 2);
          // A: k-step kk lives in sub-tile (16kk / cw), at byte offset ((16kk) % cw) * 2 of its rows
          const uint64_t aadv = (uint64_t)(((kk * 16) / cw) * sub16 + (((kk * 16) % cw) >> 3));
          Wgmma<BN, F16>::template mma<0, 0>(acc, a_hi + aadv, b_hi + badv, (k | kk) != 0);
          if (NSPLIT == 3) {
            Wgmma<BN, F16>::template mma<0, 0>(acc, a_lo + aadv, b_hi + badv, 1);
            Wgmma<BN, F16>::template mma<0, 0>(acc, a_hi + aadv, b_lo + badv, 1);
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_acc(acc);
        // frees the smem stage (the other warpgroup's MMAs on it may still be running: two arrivals)
        if ((threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[s]);
      }

      // ---- epilogue: registers -> global ----
      int mt, nt, z;
      tile_coords(tile, mt, nt, z);
      const int ncol0 = nt * p.block_n;
      const int ph_h = p.nphase == 4 ? (z >> 1) : 0, ph_w = p.nphase == 4 ? (z & 1) : 0;
      int gw[2], gh[2], gn[2];
      bool valid[2];
      float* optr[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        gw[h] = (mt % p.tiles_w) * p.tw + w_i[h];
        gh[h] = ((mt / p.tiles_w) % p.tiles_h) * p.th + h_i[h];
        gn[h] = (mt / (p.tiles_w * p.tiles_h)) * p.nb + n_i[h];
        valid[h] = (row0 + 8 * h < p.a_rows) && (gw[h] < p.m_w) && (gh[h] < p.m_h) && (gn[h] < p.m_n);
        optr[h] = p.out + (long long)gn[h] * p.out_sn + (long long)(gh[h] * p.omh + p.ooh + ph_h) * p.out_sh +
                  (long long)(gw[h] * p.omw + p.oow + ph_w) * p.out_sw + ncol0;
      }
#pragma unroll
      for (int i = 0; i < BN / 8; ++i) {
        const int c = 8 * i + 2 * quad;    // this thread's column pair (c, c + 1) of the tile
        if (BN > 16 && 8 * i >= p.block_n) break;   // MMA columns past block_n: not this tile's output
        if (p.stack_slot) {
          // phase-stacked head: column -> (phase, channel); every phase lands on its own output pixel
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            if (!valid[h]) continue;
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int col = ncol0 + c + e;
              const int ph = col / p.stack_slot, ch = col - ph * p.stack_slot;
              if (ph < 4 && ch < p.stack_c) {
                float v = acc[4 * i + 2 * h + e] * oscale;
                if (p.bias) v += p.bias[ch];
                float* o = p.out + (long long)gn[h] * p.out_sn + (long long)(gh[h] * p.omh + (ph >> 1)) * p.out_sh +
                           (long long)(gw[h] * p.omw + (ph & 1)) * p.out_sw + ch;
                *o = apply_act(v, p.act);
              }
            }
          }
        } else if (p.stats) {
          // InstanceNorm statistics fused into the producer (layers.py:17,33,134): every tile row belongs to one image
          // (nb == 1, checked by the host), so the warp's 16 rows reduce to per-column sums of y and y^2 — one fp64
          // atomic pair per column per warp into stats[n][c] = (sum, sum of squares), finalised by stats_finalize.
          // n_valid % 16 == 0 in this mode: an 8-column group is either wholly valid or wholly past the last channel.
          if (ncol0 + 8 * i >= p.n_valid) continue;
          float v[2][2];
#pragma unroll
          for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              float t = acc[4 * i + 2 * h + e] * oscale;
              if (p.bias) t += p.bias[ncol0 + c + e];
              v[h][e] = valid[h] ? t : 0.f;
            }
            if (valid[h]) *reinterpret_cast<float2*>(optr[h] + c) = make_float2(v[h][0], v[h][1]);
          }
          const float s0 = quad_col_sum(v[0][0] + v[1][0]);
          const float s1 = quad_col_sum(v[0][1] + v[1][1]);
          const float q0 = quad_col_sum(v[0][0] * v[0][0] + v[1][0] * v[1][0]);
          const float q1 = quad_col_sum(v[0][1] * v[0][1] + v[1][1] * v[1][1]);
          if (lane < 4) {
            const int tn = (mt / (p.tiles_w * p.tiles_h)) * p.nb;      // the tile's image (uniform over the CTA)
            double* sp = p.stats + ((long long)tn * p.n_valid + ncol0 + c) * 2;
            atomicAdd(sp, (double)s0);
            atomicAdd(sp + 1, (double)q0);
            atomicAdd(sp + 2, (double)s1);
            atomicAdd(sp + 3, (double)q1);
          }
        } else {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            if (!valid[h]) continue;
            float v0 = acc[4 * i + 2 * h] * oscale, v1 = acc[4 * i + 2 * h + 1] * oscale;
            const int col = ncol0 + c;
            if (p.vec4 && col + 1 < p.n_valid) {
              if (p.bias) {
                const float2 bb = *reinterpret_cast<const float2*>(p.bias + col);
                v0 += bb.x; v1 += bb.y;
              }
              *reinterpret_cast<float2*>(optr[h] + c) = make_float2(apply_act(v0, p.act), apply_act(v1, p.act));
            } else {
              if (col < p.n_valid) optr[h][c] = apply_act(p.bias ? v0 + p.bias[col] : v0, p.act);
              if (col + 1 < p.n_valid) optr[h][c + 1] = apply_act(p.bias ? v1 + p.bias[col + 1] : v1, p.act);
            }
          }
        }
      }
    }
  }

  __syncthreads();
  if (threadIdx.x == 0) {
    // the last CTA to finish re-arms the counters for the next launch of this plan (every CTA's tickets are drawn
    // before it gets here; launches of one plan never overlap)
    __threadfence();
    if (atomicAdd(p.tile_counter + 1, 1) == (int)gridDim.x - 1) {
      p.tile_counter[0] = 0;
      p.tile_counter[1] = 0;
      __threadfence();
    }
  }
}

// ============================================================================
// wgrad mode
// ============================================================================
// DET: instead of atomically adding its partial into out, CTA (tile, split z) stores it to the plan's workspace
// det_ws[z][tap][row][col] (plain stores, every valid element of the CTA's tile); wgrad_det_sum_kernel then adds the
// splits in index order into out.
template <int NSPLIT, int BN, bool F16, bool DET>
__global__ void __launch_bounds__(kThreads, 1)
wgrad_gemm_kernel(const __grid_constant__ WgradParams p) {
  using C = Cfg<NSPLIT>;
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[C::kStages];
  __shared__ __align__(8) uint64_t empty_bar[C::kStages];

  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (smem_base - smem_u32(smem_raw));
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  const int m_tile = blockIdx.x / p.n_tiles;
  const int n_tile = blockIdx.x - m_tile * p.n_tiles;
  // grid.y = tap (wide Y) or tap group (narrow Y: the group's taps are column blocks of one accumulator
  // and share the X tile, which is then read once per pixel tile instead of once per tap)
  const bool grouped = p.ngroups > 0;
  const int tap_i = grouped ? p.gstart[blockIdx.y] : blockIdx.y;
  const int gsize = grouped ? p.gsize[blockIdx.y] : 1;
  const int m0 = m_tile * kBlockM;
  const int ncol0 = n_tile * p.block_n;
  const int total = p.tiles_w * p.tiles_h * p.tiles_n;
  const int kt0 = (int)(((long long)total * blockIdx.z) / gridDim.z);
  const int kt1 = (int)(((long long)total * (blockIdx.z + 1)) / gridDim.z);
  const int k_iters = kt1 - kt0;
  const int ycw = p.y_chunk;                               // channels per Y row: 64, 32, 16
  const int y_blocks = ycw == 64 ? p.block_n / 64 : gsize; // narrow Y: one ycw-wide atom per grouped tap
  const int y_block_bytes = 64 * ycw * 2;                  // 64 pixels x ycw channels

  if (threadIdx.x == 0) {
    for (int s = 0; s < C::kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);    // one arrival per MMA warpgroup
    }
    mbar_fence_init();
  }
  if (warp == kProducerWarp && lane == 0) {
    for (int pl = 0; pl < C::kPlanes; ++pl) {
      tma_prefetch_desc(&p.tmX[pl]);
      tma_prefetch_desc(&p.tmY[pl]);
    }
  }
  __syncthreads();

  if (k_iters > 0) {
    if (warp == kProducerWarp) {
      if (lane == 0) {
        const TapDesc xt = p.xtaps[tap_i];
        const uint32_t stage_tx = C::kPlanes * (2 * 8192 + y_blocks * y_block_bytes);
        // every CTA walks the pixel tiles in the same order (a narrow wavefront shared through L2)
        for (int it = 0; it < k_iters; ++it) {
          const int s = it % C::kStages;
          const uint32_t ph = (it / C::kStages) & 1;
          mbar_wait(&empty_bar[s], ph ^ 1);
          mbar_expect_tx(&full_bar[s], stage_tx);
          const int kt = kt0 + it;
          const int tw_i = kt % p.tiles_w;
          const int th_i = (kt / p.tiles_w) % p.tiles_h;
          const int tn_i = kt / (p.tiles_w * p.tiles_h);
          const int w0 = tw_i * p.tw, h0 = th_i * p.th, n0 = tn_i * p.nb;
          uint8_t* st = smem + s * C::kStageBytes;
          if (p.x_merged) {   // one box per 64-channel block: [hi 8 KB][lo 8 KB]
            for (int b = 0; b < 2; ++b)
              tma_load_5d(&p.tmX[0], &full_bar[s], st + b * 16384, xt.c_off + m0 + b * 64, w0 + xt.dw, h0 + xt.dh,
                          n0, 0);
          } else {
#pragma unroll
            for (int pl = 0; pl < C::kPlanes; ++pl)
              for (int b = 0; b < 2; ++b)
                tma_load_5d(&p.tmX[pl], &full_bar[s], st + pl * kTileBytes + b * 8192,
                            xt.c_off + m0 + b * 64, w0 + xt.dw, xt.hp, h0 + xt.dh, n0);
          }
          if (p.y_merged) {
            const TapDesc yt = p.ytaps[tap_i];
            for (int b = 0; b < y_blocks; ++b)
              tma_load_5d(&p.tmY[0], &full_bar[s], st + C::kPlanes * kTileBytes + b * 16384,
                          yt.c_off + ncol0 + b * 64, w0 + yt.dw, h0 + yt.dh, n0, 0);
          } else {
#pragma unroll
            for (int pl = 0; pl < C::kPlanes; ++pl)
              for (int b = 0; b < y_blocks; ++b) {
                const TapDesc yt = p.ytaps[grouped ? tap_i + b : tap_i];
                tma_load_5d(&p.tmY[pl], &full_bar[s],
                            st + (C::kPlanes + pl) * kTileBytes + b * y_block_bytes,
                            yt.c_off + (grouped ? 0 : ncol0 + b * 64), w0 + yt.dw, yt.hp, h0 + yt.dh, n0);
              }
          }
        }
      }
    } else if (warp < kProducerWarp) {
      // MMA warpgroup wg: X channels [m0 + 64 wg, m0 + 64 wg + 64) = the wg-th 64-channel block of the X tile
      const int wg = warp >> 2;
      // The reduction runs over up to millions of pixels per CTA: each 64-pixel stage goes into a fresh tensor-core
      // accumulator `part` (12 MMA updates), which is then added into `acc` with round-to-nearest fp32 adds — the
      // tensor core's accumulator truncates, so its error grows with the number of updates it absorbs.
      float acc[BN / 2], part[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      // MN-major SWIZZLE_128B: SBO = stride between 8-pixel groups (1024 B); one 64-channel atom per warpgroup
      const uint32_t y_layout = gmma_layout_of_chunk(ycw);
      const uint32_t y_sbo = 8u * ycw * 2u;              // 8 pixel rows of the narrow / full atom
      // merged planes: the 64-channel blocks are [hi 8 KB][lo 8 KB] pairs, 16 KB apart
      const uint32_t x_lbo = p.x_merged ? 16384u : 8192u;
      const uint32_t x_lo_off = p.x_merged ? 8192u : (uint32_t)kTileBytes;
      const uint32_t y_lbo = p.y_merged ? 16384u : (uint32_t)y_block_bytes;
      const uint32_t y_lo_off = p.y_merged ? 8192u : (uint32_t)kTileBytes;
      for (int it = 0; it < k_iters; ++it) {
        const int s = it % C::kStages;
        const uint32_t ph = (it / C::kStages) & 1;
        mbar_wait(&full_bar[s], ph);
        const uint32_t st = smem_base + s * C::kStageBytes;
        const uint64_t x_hi = gmma_smem_desc(st + wg * x_lbo, x_lbo, 1024);
        // LBO = stride between the N atoms (64-channel blocks, or the grouped taps' narrow blocks)
        const uint64_t y_hi = gmma_smem_desc(st + C::kPlanes * kTileBytes, y_lbo, y_sbo, y_layout);
        const uint64_t x_lo = gmma_smem_desc(st + x_lo_off + wg * x_lbo, x_lbo, 1024);
        const uint64_t y_lo = gmma_smem_desc(st + C::kPlanes * kTileBytes + y_lo_off, y_lbo, y_sbo, y_layout);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {  // 4 x 16 pixels; 16 pixel rows = 2048 B (X), 16 * ycw * 2 B (Y)
          const uint64_t xadv = (uint64_t)(k * 128);
          const uint64_t yadv = (uint64_t)((k * 16 * ycw * 2) >> 4);
          Wgmma<BN, F16>::template mma<1, 1>(part, x_hi + xadv, y_hi + yadv, k != 0);
          if (NSPLIT == 3) {
            Wgmma<BN, F16>::template mma<1, 1>(part, x_lo + xadv, y_hi + yadv, 1);
            Wgmma<BN, F16>::template mma<1, 1>(part, x_hi + xadv, y_lo + yadv, 1);
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_acc(part);
        if ((threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[s]);
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] += part[i];
      }
      const int quad = lane & 3;
      const int row0 = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = row0 + 8 * h;
        if (row >= p.rows_valid) continue;
        float* orow = p.out + (long long)row * p.s_row;
        float* wrow = DET ? p.det_ws + (long long)blockIdx.z * p.det_count + (long long)row * p.cols_valid : nullptr;
#pragma unroll
        for (int i = 0; i < BN / 8; ++i) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int c = 8 * i + 2 * quad + e;
            const float v = acc[4 * i + 2 * h + e];
            if (!grouped) {
              const int col = ncol0 + c;
              if (c < p.block_n && col < p.cols_valid) {
                if constexpr (DET) wrow[(long long)tap_i * p.rows_valid * p.cols_valid + col] = v;
                else atomicAdd(orow + p.tap_off[tap_i] + (long long)col * p.s_col, v);
              }
            } else {
              const int b = c / ycw;               // which grouped tap this column belongs to
              const int cbase = c - b * ycw;
              if (b < gsize && cbase < p.cols_valid) {
                if constexpr (DET) wrow[(long long)(tap_i + b) * p.rows_valid * p.cols_valid + cbase] = v;
                else atomicAdd(orow + p.tap_off[tap_i + b] + (long long)cbase * p.s_col, v);
              }
            }
          }
        }
      }
    }
  }
}

// out[row*s_row + tap_off[tap] + col*s_col] += sum over the splits z (in order) of det_ws[z][tap][row][col]
__global__ void __launch_bounds__(256) wgrad_det_sum_kernel(const __grid_constant__ WgradParams p, int ksplit) {
  const long long rc = (long long)p.rows_valid * p.cols_valid;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < p.det_count;
       e += (long long)gridDim.x * blockDim.x) {
    float s = p.det_ws[e];
    for (int z = 1; z < ksplit; ++z) s += p.det_ws[(long long)z * p.det_count + e];
    const int tap = (int)(e / rc);
    const long long r = e - tap * rc;
    const int row = (int)(r / p.cols_valid), col = (int)(r - (long long)row * p.cols_valid);
    p.out[(long long)row * p.s_row + p.tap_off[tap] + (long long)col * p.s_col] += s;
  }
}

}  // namespace

// ============================================================================
// host side
// ============================================================================
void sn_count_launch(int n);
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !ptr) return nullptr;
    fn = reinterpret_cast<PFN_encodeTiled>(ptr);
  }
  return fn;
}

// 5-D map over a split-bf16 NHWC plane.  dims (c', w, hp, h, n); see file header.
// plane_stride > 0 (non-parity only): one extra outermost dimension of 2 planes (hi, lo) `plane_stride`
// bytes apart -> dims (c, w, h, n, plane); otherwise dims (c', w, h parity, h, n).
int sn_make_act_map(CUtensorMap* tm, const void* base, int N, int H, int W, int C, int pitch,
                    int parity, int box_w, int box_h, int box_n, int chunk = 64, long long plane_stride = 0) {
  PFN_encodeTiled enc = get_encode_fn();
  SN_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled driver entry point unavailable");
  SN_REQUIRE(pitch % 8 == 0 && ((uintptr_t)base % 16) == 0,
             "activation plane needs 16-B aligned base and pitch %% 8 == 0 (pitch=%d)", pitch);
  SN_REQUIRE(box_w >= 1 && box_h >= 1 && box_n >= 1 && box_w <= 256 && box_h <= 256 && box_n <= 256,
             "bad TMA box %d x %d x %d", box_w, box_h, box_n);
  cuuint64_t dims[5];
  cuuint64_t strides[4];
  const cuuint64_t e = 2;  // bytes per bf16
  cuuint32_t box[5] = {(cuuint32_t)chunk, (cuuint32_t)box_w, 1, (cuuint32_t)box_h, (cuuint32_t)box_n};
  if (plane_stride > 0) {
    SN_REQUIRE(plane_stride % 16 == 0, "merged planes: 16-B aligned plane stride");
    if (!parity) {
      dims[0] = C; dims[1] = W; dims[2] = H; dims[3] = N; dims[4] = 2;
      strides[0] = (cuuint64_t)pitch * e;
      strides[1] = (cuuint64_t)W * pitch * e;
    } else {
      // parity view with BOTH parities folded into the channel coordinate: c' = hp*W*pitch + pw*pitch + c
      // (overlapping dimensions are fine for loads), dims (c', w/2, h/2, n, plane)
      SN_REQUIRE(H % 2 == 0 && W % 2 == 0, "parity view needs even H, W (got %d x %d)", H, W);
      dims[0] = (cuuint64_t)(W + 1) * pitch + C; dims[1] = W / 2; dims[2] = H / 2; dims[3] = N; dims[4] = 2;
      strides[0] = (cuuint64_t)2 * pitch * e;
      strides[1] = (cuuint64_t)2 * W * pitch * e;
    }
    strides[2] = (cuuint64_t)H * W * pitch * e;
    strides[3] = (cuuint64_t)plane_stride;
    box[2] = (cuuint32_t)box_h; box[3] = (cuuint32_t)box_n; box[4] = 2;
  } else if (!parity) {
    dims[0] = C; dims[1] = W; dims[2] = 1; dims[3] = H; dims[4] = N;
    strides[0] = (cuuint64_t)pitch * e;
    strides[1] = (cuuint64_t)W * pitch * e;
    strides[2] = (cuuint64_t)W * pitch * e;
    strides[3] = (cuuint64_t)H * W * pitch * e;
  } else {
    SN_REQUIRE(H % 2 == 0 && W % 2 == 0, "parity view needs even H, W (got %d x %d)", H, W);
    dims[0] = (cuuint64_t)pitch + C; dims[1] = W / 2; dims[2] = 2; dims[3] = H / 2; dims[4] = N;
    strides[0] = (cuuint64_t)2 * pitch * e;
    strides[1] = (cuuint64_t)W * pitch * e;
    strides[2] = (cuuint64_t)2 * W * pitch * e;
    strides[3] = (cuuint64_t)H * W * pitch * e;
  }
  SN_REQUIRE(chunk == 64 || chunk == 32 || chunk == 16, "row chunk must be 64, 32 or 16 channels (got %d)", chunk);
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  const CUtensorMapSwizzle swz = chunk == 64 ? CU_TENSOR_MAP_SWIZZLE_128B
                                 : chunk == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B;
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(base), dims, strides,
                   box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SN_REQUIRE(r == CUDA_SUCCESS,
             "cuTensorMapEncodeTiled(act) failed: %d (N=%d H=%d W=%d C=%d pitch=%d parity=%d box=%dx%dx%d)",
             (int)r, N, H, W, C, pitch, parity, box_w, box_h, box_n);
  return SN_OK;
}

// 2-D map over packed weights [rows][k_total] bf16, K contiguous.
int sn_make_weight_map(CUtensorMap* tm, const void* base, int rows, long long k_total, int box_rows,
                       long long plane_stride = 0) {
  PFN_encodeTiled enc = get_encode_fn();
  SN_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled driver entry point unavailable");
  SN_REQUIRE(k_total % 64 == 0 && ((uintptr_t)base % 16) == 0, "packed weights need K %% 64 == 0");
  cuuint64_t dims[3] = {(cuuint64_t)k_total, (cuuint64_t)rows, 2};
  cuuint64_t strides[2] = {(cuuint64_t)k_total * 2, (cuuint64_t)plane_stride};
  cuuint32_t box[3] = {64, (cuuint32_t)box_rows, 2};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, plane_stride > 0 ? 3 : 2, const_cast<void*>(base), dims, strides,
                   box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SN_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(weights) failed: %d (rows=%d K=%lld box_rows=%d)",
             (int)r, rows, k_total, box_rows);
  return SN_OK;
}

static void pick_patch(int m_h, int m_w, int rows, int* th, int* tw, int* nb) {
  // rows = 128 (conv mode) or 64 (wgrad mode); dims are powers of two except the
  // PatchGAN 63/62 planes, which take the largest patch and rely on masking.
  int w = 16;
  while (w > 1 && w / 2 >= m_w) w /= 2;
  if (w > rows) w = rows;
  int h = rows / w;
  while (h > 1 && h / 2 >= m_h) h /= 2;
  *tw = w;
  *th = h;
  *nb = rows / (w * h);
}

// conv mode: any th x tw x nb patch with <= 128 GEMM rows works (rows the TMA box does not write
// are never stored), so pick the patch that wastes the fewest rows on this plane — e.g. 7 x 17 on the
// 34 x 34 padded resblock-gradient grid (90 % instead of 60 % with 8 x 16).  Ties: squarer patch
// (smaller halo re-read across taps).
static void pick_patch_conv(int m_n, int m_h, int m_w, int* th, int* tw, int* nb) {
  double best_eff = -1.0;
  int best_perim = 1 << 30, best_rows = 0, best_area = 0;
  const long long useful = (long long)m_n * m_h * m_w;
  for (int w = 1; w <= m_w && w <= 128; ++w) {
    for (int h = 1; h <= m_h && h * w <= 128; ++h) {
      // planes of >= 128 pixels: purely spatial patches (halo locality); smaller planes: whole
      // planes of several images per tile
      int n = 1;
      if (m_h * m_w < 128) {
        if (w != m_w || h != m_h) continue;
        n = 128 / (w * h);
        if (n > m_n) n = m_n;
        if (n > 256) n = 256;
      }
      const long long tiles = (long long)((m_w + w - 1) / w) * ((m_h + h - 1) / h) * ((m_n + n - 1) / n);
      const double eff = (double)useful / (double)(tiles * 128);
      const int rows = w * h * n, perim = w + h, area = w * h;
      // ties: more rows per tile, then the larger spatial patch (fewer images per tile), then the squarer one
      const bool better =
          eff > best_eff + 1e-9 ||
          (eff > best_eff - 1e-9 &&
           (rows > best_rows ||
            (rows == best_rows && (area > best_area || (area == best_area && (perim < best_perim || (perim == best_perim && w > *tw)))))));
      if (better) {
        best_eff = eff; best_rows = rows; best_perim = perim; best_area = area;
        *tw = w; *th = h; *nb = n;
      }
    }
  }
}

int sn_tap_gemm_plan_init(TapGemmPlan* plan, const sn_tap_gemm_desc* d) {
  memset(plan, 0, sizeof(*plan));
  TapGemmParams& p = plan->p;
  SN_REQUIRE(d->nsplit == 1 || d->nsplit == 3, "nsplit must be 1 or 3");
  SN_REQUIRE(d->ntaps >= 1 && d->ntaps <= SN_MAX_TAPS, "ntaps out of range: %d", d->ntaps);
  const int a_chunk = d->a_chunk ? d->a_chunk : 64;
  SN_REQUIRE(a_chunk == 64 || a_chunk == 32 || a_chunk == 16, "a_chunk must be 64, 32 or 16");
  if (a_chunk == 64) {
    SN_REQUIRE(d->k_per_tap > 0 && d->k_per_tap % 64 == 0, "k_per_tap must be a multiple of 64");
  } else {
    SN_REQUIRE(d->k_per_tap == a_chunk && d->ntaps % (64 / a_chunk) == 0,
               "narrow operand: k_per_tap must equal a_chunk (%d) and ntaps (%d) be a multiple of %d", a_chunk,
               d->ntaps, 64 / a_chunk);
  }
  p.a_chunk = a_chunk;
  SN_REQUIRE(d->block_n >= 16 && d->block_n <= 128 && d->block_n % 16 == 0,
             "block_n must be a multiple of 16 in [16,128]");
  SN_REQUIRE(d->a_hi && d->b_hi && d->out, "null operand");
  SN_REQUIRE(d->nsplit == 1 || (d->a_lo && d->b_lo), "nsplit=3 needs lo planes");
  SN_REQUIRE(d->a_fmt == d->b_fmt, "A and B of one wgmma must share a 16-bit format (a=%d b=%d)",
             d->a_fmt, d->b_fmt);
  int th, tw, nb;
  pick_patch_conv(d->m_n, d->m_h, d->m_w, &th, &tw, &nb);
  p.a_rows = th * tw * nb;
  p.tw = tw; p.th = th; p.nb = nb;
  p.tiles_w = (d->m_w + tw - 1) / tw;
  p.tiles_h = (d->m_h + th - 1) / th;
  p.tiles_n = (d->m_n + nb - 1) / nb;
  p.m_w = d->m_w; p.m_h = d->m_h; p.m_n = d->m_n;
  p.ntaps = d->ntaps;
  p.chunks = a_chunk == 64 ? d->k_per_tap / 64 : 1;
  for (int t = 0; t < d->ntaps; ++t) {
    p.taps[t].c_off = d->taps[t].c_off;
    p.taps[t].kb_off = d->taps[t].kb_off;
    p.taps[t].dw = (short)d->taps[t].dw;
    p.taps[t].dh = (short)d->taps[t].dh;
    p.taps[t].hp = (short)d->taps[t].hp;
  }
  p.block_n = d->block_n;
  p.n_valid = d->n_valid;
  p.out = d->out;
  p.out_sn = d->out_sn; p.out_sh = d->out_sh; p.out_sw = d->out_sw;
  p.omh = d->out_mul_h; p.ooh = d->out_off_h; p.omw = d->out_mul_w; p.oow = d->out_off_w;
  p.nphase = d->nphase == 4 ? 4 : 1;
  SN_REQUIRE(d->nphase == 0 || d->nphase == 1 || d->nphase == 4, "nphase must be 1 or 4");
  if (p.nphase == 4) {
    SN_REQUIRE(d->ntaps % 4 == 0, "4-phase launch: ntaps must split into 4 equal groups");
    const int tpp = d->ntaps / 4;
    SN_REQUIRE(a_chunk == 64 || tpp % (64 / a_chunk) == 0, "4-phase launch: taps per phase must fill whole stages");
  }
  p.bias = d->bias;
  p.stack_slot = d->stack_slot; p.stack_c = d->stack_c;
  p.stats = nullptr;
  if (d->stack_slot > 0)
    SN_REQUIRE(d->nphase <= 1 && d->n_valid == 4 * d->stack_slot && d->stack_c >= 1 && d->stack_c <= d->stack_slot &&
                   d->out_mul_h == 2 && d->out_mul_w == 2,
               "phase-stacked output: n_valid = 4*stack_slot, nphase 1, out_mul 2 (slot=%d c=%d n_valid=%d)",
               d->stack_slot, d->stack_c, d->n_valid);
  p.b_scale = d->b_scale;
  p.a_fmt = d->a_fmt;
  p.b_fmt = d->b_fmt;
  p.act = d->act;
  p.vec4 = ((uintptr_t)d->out % 16 == 0) && (d->out_sn % 4 == 0) && (d->out_sh % 4 == 0) &&
           (d->out_sw % 4 == 0) && (!d->bias || (uintptr_t)d->bias % 16 == 0);
  // fused InstanceNorm statistics: whole tile inside one image, 16-column chunks fully valid, plain vectorised stores
  if (d->stats && nb == 1 && p.vec4 && d->n_valid % 16 == 0 && d->act == 0 && d->stack_slot == 0 && d->m_n * 1 >= 1)
    p.stats = d->stats;
  plan->stats_bytes = p.stats ? sizeof(double) * 2 * (size_t)d->m_n * d->n_valid : 0;
  p.tile_counter = nullptr;
  SN_CHECK_CUDA(cudaMalloc(&p.tile_counter, 2 * sizeof(int)));
  SN_CHECK_CUDA(cudaMemset(p.tile_counter, 0, 2 * sizeof(int)));
  int rc;
  const void* a_pl[2] = {d->a_hi, d->a_lo};
  const void* b_pl[2] = {d->b_hi, d->b_lo};
  const long long a_ps = d->nsplit == 3 ? (const char*)d->a_lo - (const char*)d->a_hi : 0;
  const long long b_ps = d->nsplit == 3 ? (const char*)d->b_lo - (const char*)d->b_hi : 0;
  // the lo tile must start on a swizzle-atom boundary (8 rows x 128 B)
  p.a_merged = a_chunk == 64 && a_ps > 0 && a_ps % 16 == 0 && p.a_rows % 8 == 0;
  if (p.a_merged && d->a_parity)   // h parity moves into the channel coordinate of the merged parity map
    for (int t = 0; t < d->ntaps; ++t) p.taps[t].c_off += p.taps[t].hp * d->a_w * d->a_pitch;
  p.b_merged = b_ps > 0 && b_ps % 16 == 0 && d->block_n % 8 == 0;
  p.a_lo_off = p.a_merged ? p.a_rows * 128 : kTileBytes;
  p.b_lo_off = p.b_merged ? d->block_n * 128 : kTileBytes;
  for (int pl = 0; pl < (d->nsplit == 3 ? 2 : 1); ++pl) {
    if (!(p.a_merged && pl == 1)) {
      rc = sn_make_act_map(&p.tmA[pl], a_pl[pl], d->a_n, d->a_h, d->a_w, d->a_c, d->a_pitch,
                           d->a_parity, tw, th, nb, a_chunk, p.a_merged ? a_ps : 0);
      if (rc) return rc;
    }
    if (!(p.b_merged && pl == 1)) {
      rc = sn_make_weight_map(&p.tmB[pl], b_pl[pl], d->b_rows, d->b_k, d->block_n, p.b_merged ? b_ps : 0);
      if (rc) return rc;
    }
  }
  if (p.a_merged) p.tmA[1] = p.tmA[0];
  if (p.b_merged) p.tmB[1] = p.tmB[0];
  plan->nsplit = d->nsplit;
  plan->grid = dim3(p.tiles_w * p.tiles_h * p.tiles_n, (d->n_valid + d->block_n - 1) / d->block_n, p.nphase);
  return SN_OK;
}

// MMA N of a plan: the smallest instantiated wgmma N >= block_n (the extra columns are computed and not stored)
static int mma_n(int block_n) {
  return block_n <= 16 ? 16 : block_n <= 32 ? 32 : block_n <= 64 ? 64 : block_n <= 96 ? 96 : 128;
}

template <int NSPLIT, int CW, int BN, bool F16>
static int launch_tap(const TapGemmPlan* plan, cudaStream_t stream) {
  static bool attr_done = false;
  if (!attr_done) {
    SN_CHECK_CUDA(cudaFuncSetAttribute(tap_gemm_kernel<NSPLIT, CW, BN, F16>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       Cfg<NSPLIT>::kSmemBytes));
    attr_done = true;
  }
  // persistent launch: at most one CTA per SM; plan->grid = (M tiles, N tiles, phases)
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    SN_CHECK_CUDA(cudaGetDevice(&dev));
    SN_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  }
  const int m_tiles = (int)plan->grid.x, n_tiles = (int)plan->grid.y;
  const int total = m_tiles * n_tiles * (int)plan->grid.z;
  if (plan->p.stats) SN_CHECK_CUDA(cudaMemsetAsync(plan->p.stats, 0, plan->stats_bytes, stream));
  const int ctas = total < sms ? total : sms;
  tap_gemm_kernel<NSPLIT, CW, BN, F16>
      <<<ctas, kThreads, Cfg<NSPLIT>::kSmemBytes, stream>>>(plan->p, m_tiles, n_tiles, total);
  SN_CHECK_CUDA(cudaGetLastError());
  return SN_OK;
}

template <int NSPLIT, int CW, bool F16>
static int launch_tap_n(const TapGemmPlan* plan, cudaStream_t stream) {
  switch (mma_n(plan->p.block_n)) {
    case 16: return launch_tap<NSPLIT, CW, 16, F16>(plan, stream);
    case 32: return launch_tap<NSPLIT, CW, 32, F16>(plan, stream);
    case 64: return launch_tap<NSPLIT, CW, 64, F16>(plan, stream);
    case 96: return launch_tap<NSPLIT, CW, 96, F16>(plan, stream);
    default: return launch_tap<NSPLIT, CW, 128, F16>(plan, stream);
  }
}

template <int NSPLIT, bool F16>
static int launch_tap_cw(const TapGemmPlan* plan, cudaStream_t stream) {
  const int cw = plan->p.a_chunk;
  if (cw == 64) return launch_tap_n<NSPLIT, 64, F16>(plan, stream);
  if (cw == 32) return launch_tap_n<NSPLIT, 32, F16>(plan, stream);
  return launch_tap_n<NSPLIT, 16, F16>(plan, stream);
}

int sn_tap_gemm_plan_launch(const TapGemmPlan* plan, cudaStream_t stream) {
  const bool f16 = plan->p.a_fmt == SN_FMT_F16;
  if (plan->nsplit == 3) return f16 ? launch_tap_cw<3, true>(plan, stream) : launch_tap_cw<3, false>(plan, stream);
  return f16 ? launch_tap_cw<1, true>(plan, stream) : launch_tap_cw<1, false>(plan, stream);
}

// split-K count: ~3 waves of CTAs on sm_count SMs, at least 8 k-iterations (64-pixel tiles) per CTA; a deterministic
// plan sizes it for SN_NUM_SMS whatever the device, so that its summation order follows from the shapes alone
static int wgrad_ksplit(const sn_wgrad_desc* d, int base_ctas, int total, int sm_count) {
  if (d->deterministic) sm_count = SN_NUM_SMS;
  int ks = d->ksplit;
  if (ks <= 0) {
    ks = (3 * sm_count + base_ctas - 1) / base_ctas;
    int max_ks = total / 8;
    if (max_ks < 1) max_ks = 1;
    if (ks > max_ks) ks = max_ks;
    if (ks < 1) ks = 1;
  }
  if (ks > total) ks = total;
  return ks;
}

int sn_wgrad_plan_init(WgradPlan* plan, const sn_wgrad_desc* d, int sm_count) {
  memset(plan, 0, sizeof(*plan));
  WgradParams& p = plan->p;
  SN_REQUIRE(d->nsplit == 1 || d->nsplit == 3, "nsplit must be 1 or 3");
  SN_REQUIRE(d->ntaps >= 1 && d->ntaps <= SN_MAX_TAPS, "ntaps out of range: %d", d->ntaps);
  const int y_chunk = d->y_chunk ? d->y_chunk : 64;
  SN_REQUIRE(y_chunk == 64 || y_chunk == 32 || y_chunk == 16, "y_chunk must be 64, 32 or 16");
  p.y_chunk = y_chunk;
  p.ngroups = 0;
  int grid_y = d->ntaps;
  if (y_chunk == 64) {
    SN_REQUIRE(d->block_n == 64 || d->block_n == 128, "wgrad block_n must be 64 or 128 for 64-channel Y rows");
  } else {
    SN_REQUIRE(d->cols_valid <= y_chunk, "narrow Y: cols_valid must fit one %d-channel block", y_chunk);
    if (d->ngroups > 0) {
      int maxg = 0, covered = 0;
      for (int g = 0; g < d->ngroups; ++g) {
        SN_REQUIRE(d->group_size[g] >= 1 && d->group_start[g] >= 0 &&
                       d->group_start[g] + d->group_size[g] <= d->ntaps, "bad tap group %d", g);
        if (d->group_size[g] > maxg) maxg = d->group_size[g];
        covered += d->group_size[g];
        p.gstart[g] = (short)d->group_start[g];
        p.gsize[g] = (short)d->group_size[g];
      }
      SN_REQUIRE(covered == d->ntaps && maxg * y_chunk <= 128 && d->block_n == maxg * y_chunk,
                 "tap groups must cover all taps and block_n == max group * y_chunk <= 128");
      p.ngroups = d->ngroups;
      grid_y = d->ngroups;
    } else {
      SN_REQUIRE(d->block_n == y_chunk, "narrow Y without groups: block_n must equal y_chunk");
    }
  }
  SN_REQUIRE(d->x_hi && d->y_hi && d->out, "null operand");
  SN_REQUIRE(d->nsplit == 1 || (d->x_lo && d->y_lo), "nsplit=3 needs lo planes");
  SN_REQUIRE(d->x_fmt == d->y_fmt, "X and Y of one wgmma must share a 16-bit format (x=%d y=%d)",
             d->x_fmt, d->y_fmt);
  int th, tw, nb;
  pick_patch(d->m_h, d->m_w, 64, &th, &tw, &nb);
  p.tw = tw; p.th = th; p.nb = nb;
  p.tiles_w = (d->m_w + tw - 1) / tw;
  p.tiles_h = (d->m_h + th - 1) / th;
  p.tiles_n = (d->m_n + nb - 1) / nb;
  p.ntaps = d->ntaps;
  for (int t = 0; t < d->ntaps; ++t) {
    p.xtaps[t].c_off = d->xtaps[t].c_off; p.xtaps[t].dw = (short)d->xtaps[t].dw;
    p.xtaps[t].dh = (short)d->xtaps[t].dh; p.xtaps[t].hp = (short)d->xtaps[t].hp;
    p.ytaps[t].c_off = d->ytaps[t].c_off; p.ytaps[t].dw = (short)d->ytaps[t].dw;
    p.ytaps[t].dh = (short)d->ytaps[t].dh; p.ytaps[t].hp = (short)d->ytaps[t].hp;
    p.tap_off[t] = d->tap_off[t];
  }
  p.block_n = d->block_n;
  p.m_tiles = (d->rows_valid + kBlockM - 1) / kBlockM;
  p.n_tiles = y_chunk == 64 ? (d->cols_valid + d->block_n - 1) / d->block_n : 1;
  p.rows_valid = d->rows_valid;
  p.cols_valid = d->cols_valid;
  p.out = d->out;
  p.s_row = d->s_row;
  p.s_col = d->s_col;
  p.x_fmt = d->x_fmt;
  p.y_fmt = d->y_fmt;
  int rc;
  const void* x_pl[2] = {d->x_hi, d->x_lo};
  const void* y_pl[2] = {d->y_hi, d->y_lo};
  {
    const long long x_ps = d->nsplit == 3 ? (const char*)d->x_lo - (const char*)d->x_hi : 0;
    const long long y_ps = d->nsplit == 3 ? (const char*)d->y_lo - (const char*)d->y_hi : 0;
    p.x_merged = x_ps > 0 && x_ps % 16 == 0 && tw * th * nb == 64;
    p.y_merged = y_ps > 0 && y_ps % 16 == 0 && tw * th * nb == 64 && y_chunk == 64 && d->ngroups == 0;
    for (int t = 0; t < d->ntaps; ++t) {   // h parity -> channel coordinate of the merged parity maps
      if (p.x_merged && d->x_parity) p.xtaps[t].c_off += p.xtaps[t].hp * d->x_w * d->x_pitch;
      if (p.y_merged && d->y_parity) p.ytaps[t].c_off += p.ytaps[t].hp * d->y_w * d->y_pitch;
    }
    for (int pl = 0; pl < (d->nsplit == 3 ? 2 : 1); ++pl) {
      if (!(p.x_merged && pl == 1)) {
        rc = sn_make_act_map(&p.tmX[pl], x_pl[pl], d->x_n, d->x_h, d->x_w, d->x_c, d->x_pitch,
                             d->x_parity, tw, th, nb, 64, p.x_merged ? x_ps : 0);
        if (rc) return rc;
      }
      if (!(p.y_merged && pl == 1)) {
        rc = sn_make_act_map(&p.tmY[pl], y_pl[pl], d->y_n, d->y_h, d->y_w, d->y_c, d->y_pitch,
                             d->y_parity, tw, th, nb, y_chunk, p.y_merged ? y_ps : 0);
        if (rc) return rc;
      }
    }
    if (p.x_merged) p.tmX[1] = p.tmX[0];
    if (p.y_merged) p.tmY[1] = p.tmY[0];
  }
  plan->nsplit = d->nsplit;
  const int base_ctas = p.m_tiles * p.n_tiles * grid_y;
  const int total = p.tiles_w * p.tiles_h * p.tiles_n;
  const int ks = wgrad_ksplit(d, base_ctas, total, sm_count);
  plan->grid = dim3(p.m_tiles * p.n_tiles, grid_y, ks);
  p.det_ws = nullptr;
  p.det_count = 0;
  plan->ws_bytes = 0;
  if (d->deterministic) {
    // the finalize kernel writes out[tap_off[t] + ...] from one thread per element: taps must not share outputs
    for (int t = 0; t < d->ntaps; ++t)
      for (int u = 0; u < t; ++u)
        SN_REQUIRE(d->tap_off[t] != d->tap_off[u], "deterministic wgrad: taps %d and %d share tap_off", u, t);
    p.det_count = (long long)d->ntaps * d->rows_valid * d->cols_valid;
    plan->ws_bytes = sizeof(float) * (size_t)ks * p.det_count;
    SN_CHECK_CUDA(cudaMalloc(&p.det_ws, plan->ws_bytes));
  }
  return SN_OK;
}

int sn_wgrad_plan_ksplit(const sn_wgrad_desc* d, int sm_count) {
  SN_REQUIRE(d && d->ntaps >= 1 && d->ntaps <= SN_MAX_TAPS, "wgrad_ksplit: bad descriptor");
  int th, tw, nb;
  pick_patch(d->m_h, d->m_w, 64, &th, &tw, &nb);
  const int total = ((d->m_w + tw - 1) / tw) * ((d->m_h + th - 1) / th) * ((d->m_n + nb - 1) / nb);
  const int y_chunk = d->y_chunk ? d->y_chunk : 64;
  const int grid_y = (y_chunk != 64 && d->ngroups > 0) ? d->ngroups : d->ntaps;
  const int m_tiles = (d->rows_valid + kBlockM - 1) / kBlockM;
  const int n_tiles = y_chunk == 64 ? (d->cols_valid + d->block_n - 1) / d->block_n : 1;
  return wgrad_ksplit(d, m_tiles * n_tiles * grid_y, total, sm_count);
}

template <int NSPLIT, int BN, bool F16, bool DET>
static int launch_wgrad_k(const WgradPlan* plan, cudaStream_t stream) {
  static bool attr_done = false;
  if (!attr_done) {
    SN_CHECK_CUDA(cudaFuncSetAttribute(wgrad_gemm_kernel<NSPLIT, BN, F16, DET>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<NSPLIT>::kSmemBytes));
    attr_done = true;
  }
  wgrad_gemm_kernel<NSPLIT, BN, F16, DET><<<plan->grid, kThreads, Cfg<NSPLIT>::kSmemBytes, stream>>>(plan->p);
  SN_CHECK_CUDA(cudaGetLastError());
  return SN_OK;
}

template <int NSPLIT, int BN, bool F16>
static int launch_wgrad(const WgradPlan* plan, cudaStream_t stream) {
  if (!plan->p.det_ws) return launch_wgrad_k<NSPLIT, BN, F16, false>(plan, stream);
  const int rc = launch_wgrad_k<NSPLIT, BN, F16, true>(plan, stream);
  if (rc) return rc;
  long long g = (plan->p.det_count + 255) / 256;
  if (g > SN_NUM_SMS * 8) g = SN_NUM_SMS * 8;
  wgrad_det_sum_kernel<<<(int)g, 256, 0, stream>>>(plan->p, (int)plan->grid.z);
  SN_CHECK_CUDA(cudaGetLastError());
  sn_count_launch(1);
  return SN_OK;
}

template <int NSPLIT, bool F16>
static int launch_wgrad_n(const WgradPlan* plan, cudaStream_t stream) {
  switch (mma_n(plan->p.block_n)) {
    case 16: return launch_wgrad<NSPLIT, 16, F16>(plan, stream);
    case 32: return launch_wgrad<NSPLIT, 32, F16>(plan, stream);
    case 64: return launch_wgrad<NSPLIT, 64, F16>(plan, stream);
    case 96: return launch_wgrad<NSPLIT, 96, F16>(plan, stream);
    default: return launch_wgrad<NSPLIT, 128, F16>(plan, stream);
  }
}

int sn_wgrad_plan_launch(const WgradPlan* plan, cudaStream_t stream) {
  const bool f16 = plan->p.x_fmt == SN_FMT_F16;
  if (plan->nsplit == 3) return f16 ? launch_wgrad_n<3, true>(plan, stream) : launch_wgrad_n<3, false>(plan, stream);
  return f16 ? launch_wgrad_n<1, true>(plan, stream) : launch_wgrad_n<1, false>(plan, stream);
}
