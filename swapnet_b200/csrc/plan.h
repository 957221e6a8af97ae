// swapnet_b200 — internal kernel-parameter structs and plan objects.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include "../../include/swapnet_b200.h"

struct TapDesc {
  int c_off;   // channel (c') offset of this tap inside the A tensor map
  int kb_off;  // K offset of this tap inside the packed weight matrix
  short dw, dh, hp, _pad;
};

struct alignas(64) TapGemmParams {
  CUtensorMap tmA[2];  // hi, lo activation planes
  CUtensorMap tmB[2];  // hi, lo packed weights
  TapDesc taps[SN_MAX_TAPS];
  int ntaps, chunks;
  int tiles_w, tiles_h, tiles_n;
  int tw, th, nb;
  int a_rows;  // th * tw * nb <= 128 GEMM rows actually loaded / stored per tile
  int m_w, m_h, m_n;
  int block_n, n_valid;
  float* out;
  long long out_sn, out_sh, out_sw;
  int omh, ooh, omw, oow;
  const float* bias;
  const float* b_scale;  // device (s, 1/s) of the packed weights, or null
  int act;
  int vec4;
  int a_fmt, b_fmt;
  int a_chunk;  // 64 / 32 / 16 channels per A row
  int nphase;   // 1 or 4 (grid.z = output parity phase; taps split in nphase equal groups)
  // merged planes: hi and lo of an operand live `plane stride` apart in one buffer and come in ONE TMA box
  // (an extra outermost box dimension of 2) — the TMA unit is bound by the number of box operations, not bytes
  int a_merged, b_merged;
  int a_lo_off, b_lo_off;   // byte offset of the lo tile behind the hi tile inside a stage
  int stack_slot, stack_c;  // > 0: N = 4 output-parity phases side by side (sn_tap_gemm_desc.stack_slot)
  double* stats;            // non-null: accumulate per-(image, channel) sum / sum of squares of the output (fused IN stats)
  int* tile_counter;        // dynamic tile schedule: [0] next ticket, [1] CTAs finished (self-resetting)
};

struct alignas(64) WgradParams {
  CUtensorMap tmX[2];
  CUtensorMap tmY[2];
  TapDesc xtaps[SN_MAX_TAPS];
  TapDesc ytaps[SN_MAX_TAPS];
  long long tap_off[SN_MAX_TAPS];
  int ntaps;
  int tiles_w, tiles_h, tiles_n;
  int tw, th, nb;
  int m_tiles, n_tiles, block_n;
  int rows_valid, cols_valid;
  float* out;
  long long s_row, s_col;
  int x_fmt, y_fmt;
  int y_chunk;  // 64 / 32 / 16 channels per Y row
  int ngroups;  // > 0: narrow-Y tap groups (grid.y = group)
  int x_merged, y_merged;   // hi+lo of a 64-channel block in one TMA box (see TapGemmParams)
  short gstart[SN_MAX_TAPS], gsize[SN_MAX_TAPS];
  float* det_ws;            // deterministic plans: split partials [ksplit][ntaps][rows_valid][cols_valid] (plan-owned)
  long long det_count;      // ntaps * rows_valid * cols_valid
};

struct TapGemmPlan {
  TapGemmParams p;
  dim3 grid;
  int nsplit;
  size_t stats_bytes;       // bytes of p.stats zeroed ahead of every launch
};
struct WgradPlan {
  WgradParams p;
  dim3 grid;
  int nsplit;
  size_t ws_bytes;          // bytes of p.det_ws
};

int sn_tap_gemm_plan_init(TapGemmPlan* plan, const sn_tap_gemm_desc* d);
int sn_tap_gemm_plan_launch(const TapGemmPlan* plan, cudaStream_t stream);
int sn_wgrad_plan_init(WgradPlan* plan, const sn_wgrad_desc* d, int sm_count);
int sn_wgrad_plan_launch(const WgradPlan* plan, cudaStream_t stream);
int sn_wgrad_plan_ksplit(const sn_wgrad_desc* d, int sm_count);
