// Library-level entry points of libnudf.so: error reporting, ABI version, engine selection.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/nudf.h"
#include "common.cuh"

namespace nudf {

static thread_local char g_err[512] = "";
static int g_engine = -1;
static unsigned long long g_launches = 0;
void count_launch() { __atomic_fetch_add(&g_launches, 1ull, __ATOMIC_RELAXED); }

// ---- per-family launch timing (bench.py) ----
static bool g_timing = false;
static const int kMaxTimed = 8192;
static cudaEvent_t g_ev[kMaxTimed][2];
static int g_ev_family[kMaxTimed];
static int g_ev_created = 0, g_ev_used = 0;
bool launch_timing_on() { return g_timing; }
int launch_timer_begin(int family, cudaStream_t st) {
  if (g_ev_used >= kMaxTimed) return -1;
  const int slot = g_ev_used;
  if (slot >= g_ev_created) {
    if (cudaEventCreate(&g_ev[slot][0]) != cudaSuccess || cudaEventCreate(&g_ev[slot][1]) != cudaSuccess) return -1;
    g_ev_created = slot + 1;
  }
  g_ev_family[slot] = family;
  if (cudaEventRecord(g_ev[slot][0], st) != cudaSuccess) return -1;
  g_ev_used = slot + 1;
  return slot;
}
void launch_timer_end(int slot, cudaStream_t st) { cudaEventRecord(g_ev[slot][1], st); }

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// NUDF_TC_MASK: which chains may run on the tensor engine (bits: 1 UDF value chain -- hidden layers and feature rows with three
// bf16 planes, the udf-head row in exact fp32 --, 2 reverse sweep, 4 tangent, 8 backward, 16 weight gradients, 32 colour-net
// backward, 64 NeRF++ backward, 128 colour / NeRF++ forward with THREE bf16 planes / six products per layer, 3.5e-7: the
// two-plane split's 4e-6 flips ~60x more ReLU gates than the reference's own fp32 rounding and fails the gradient parity
// tests, the three-plane one passes them).  The three-plane split is relative to each element (about 24 significant bits),
// so small softplus outputs next to O(1) ones in the same row keep their precision.
// Default: every chain (255).
static int g_tc_mask = -1;
static const int kDefaultTcMask = 1 | 2 | 4 | 8 | 16 | 32 | 64 | 128;
int tc_mask() {
  if (g_tc_mask < 0) {
    const char* e = getenv("NUDF_TC_MASK");
    g_tc_mask = e ? atoi(e) : kDefaultTcMask;
  }
  return g_tc_mask;
}

// Workspace of the deterministic split-K reductions (common.cuh): one per device, kept for the life of the process.
float* split_workspace(cudaStream_t st) {
  static float* ws[64] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) {
    set_error("split_workspace: no current CUDA device");
    return nullptr;
  }
  if (ws[dev] == nullptr) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(st, &cs) != cudaSuccess || cs != cudaStreamCaptureStatusNone) {
      set_error("split_workspace: first use inside a CUDA-graph capture (run one step eagerly first)");
      return nullptr;
    }
    if (cudaMalloc(&ws[dev], sizeof(float) * SPLIT_WS_FLOATS) != cudaSuccess) {
      ws[dev] = nullptr;
      set_error("split_workspace: cudaMalloc of %lld floats failed", (long long)SPLIT_WS_FLOATS);
      return nullptr;
    }
  }
  return ws[dev];
}

int get_engine() {
  if (g_engine < 0) {
    const char* e = getenv("NUDF_ENGINE");
    g_engine = (e && e[0] == '0') ? 0 : 1;
  }
  return g_engine;
}

}  // namespace nudf

extern "C" {

int nudf_abi_version(void) { return NUDF_ABI_VERSION; }
const char* nudf_last_error(void) { return nudf::g_err; }
int nudf_set_engine(int engine) {
  if (engine != 0 && engine != 1) {
    nudf::set_error("nudf_set_engine: engine must be 0 (fp32 FFMA) or 1 (tensor cores, split bf16)");
    return -1;
  }
  nudf::g_engine = engine;
  return 0;
}
int nudf_get_engine(void) { return nudf::get_engine(); }
int nudf_set_tc_mask(int mask) { nudf::g_tc_mask = mask & 255; return 0; }
int nudf_get_tc_mask(void) { return nudf::tc_mask(); }
int nudf_default_tc_mask(void) { return nudf::kDefaultTcMask; }
int64_t nudf_launch_count(void) { return (int64_t)__atomic_load_n(&nudf::g_launches, __ATOMIC_RELAXED); }

int nudf_launch_family_count(void) { return nudf::FAM_COUNT; }
int nudf_set_launch_timing(int on) {
  nudf::g_timing = on != 0;
  nudf::g_ev_used = 0;
  return 0;
}
int nudf_read_launch_timing(float* ms_per_family, int32_t* launches_per_family) {
  for (int f = 0; f < nudf::FAM_COUNT; ++f) { ms_per_family[f] = 0.f; launches_per_family[f] = 0; }
  for (int i = 0; i < nudf::g_ev_used; ++i) {
    if (cudaEventSynchronize(nudf::g_ev[i][1]) != cudaSuccess) { nudf::set_error("nudf_read_launch_timing: event sync failed"); return -2; }
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, nudf::g_ev[i][0], nudf::g_ev[i][1]) != cudaSuccess) { nudf::set_error("nudf_read_launch_timing: elapsed failed"); return -2; }
    ms_per_family[nudf::g_ev_family[i]] += ms;
    launches_per_family[nudf::g_ev_family[i]] += 1;
  }
  nudf::g_ev_used = 0;
  return 0;
}

}  // extern "C"
