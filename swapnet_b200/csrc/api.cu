// swapnet_b200 — C-ABI glue: error state, plan handles, launch counter.
#include <stdarg.h>
#include <atomic>
#include "common.cuh"
#include "plan.h"

static thread_local char g_err[1024] = "";
std::atomic<long long> g_launches{0};

void sn_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void sn_count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

struct sn_plan {
  int kind;  // 0 tap gemm, 1 wgrad
  TapGemmPlan tg;
  WgradPlan wg;
};

static int g_sm_count = 0;
static int sm_count() {
  if (!g_sm_count) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_sm_count, cudaDevAttrMultiProcessorCount, dev);
    if (g_sm_count <= 0) g_sm_count = SN_NUM_SMS;
  }
  return g_sm_count;
}

extern "C" {

const char* sn_version(void) { return "swapnet_b200 0.1.0 (sm_90a, wgmma split-bf16)"; }
const char* sn_last_error(void) { return g_err; }
long long sn_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }
void sn_count_replayed(long long n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int sn_tap_gemm_plan_create(const sn_tap_gemm_desc* desc, sn_plan** out) {
  SN_REQUIRE(desc && out, "null argument");
  sn_plan* p = new sn_plan();
  p->kind = 0;
  int rc = sn_tap_gemm_plan_init(&p->tg, desc);
  if (rc) {
    delete p;
    return rc;
  }
  *out = p;
  return SN_OK;
}

int sn_wgrad_plan_create(const sn_wgrad_desc* desc, sn_plan** out) {
  SN_REQUIRE(desc && out, "null argument");
  sn_plan* p = new sn_plan();
  p->kind = 1;
  int rc = sn_wgrad_plan_init(&p->wg, desc, sm_count());
  if (rc) {
    delete p;
    return rc;
  }
  *out = p;
  return SN_OK;
}

int sn_plan_run(const sn_plan* plan, void* stream) {
  SN_REQUIRE(plan, "null plan");
  sn_count_launch(1);
  if (plan->kind == 0) return sn_tap_gemm_plan_launch(&plan->tg, (cudaStream_t)stream);
  return sn_wgrad_plan_launch(&plan->wg, (cudaStream_t)stream);
}

int sn_plan_has_stats(const sn_plan* plan) { return plan && plan->kind == 0 && plan->tg.p.stats != nullptr; }

int sn_plan_geometry(const sn_plan* plan, int* out) {
  SN_REQUIRE(plan && out, "null argument");
  const dim3 g = plan->kind == 0 ? plan->tg.grid : plan->wg.grid;
  out[0] = plan->kind;
  out[1] = (int)g.x;
  out[2] = (int)g.y;
  out[3] = (int)g.z;
  out[4] = plan->kind == 0 ? plan->tg.p.block_n : plan->wg.p.block_n;
  out[5] = plan->kind == 0 ? plan->tg.p.a_chunk : plan->wg.p.y_chunk;
  return SN_OK;
}

long long sn_plan_workspace_bytes(const sn_plan* plan) {
  return plan && plan->kind == 1 ? (long long)plan->wg.ws_bytes : 0;
}

int sn_wgrad_ksplit(const sn_wgrad_desc* desc, int sm_count) { return sn_wgrad_plan_ksplit(desc, sm_count); }

void sn_plan_destroy(sn_plan* plan) {
  if (plan && plan->kind == 0 && plan->tg.p.tile_counter) cudaFree(plan->tg.p.tile_counter);
  if (plan && plan->kind == 1 && plan->wg.p.det_ws) cudaFree(plan->wg.p.det_ws);
  delete plan;
}

}  // extern "C"
