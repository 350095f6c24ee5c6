// Error reporting + launch accounting for libofk.so.
#include <atomic>
#include <cstdlib>
#include <string>

#include <cuda_runtime.h>

#include "ofk_internal.h"

static thread_local std::string g_err;
static std::atomic<long long> g_launches{0};

int ofk_set_error(int code, const char* msg) {
  g_err = msg ? msg : "";
  return code;
}
void ofk_count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

extern "C" const char* ofk_last_error(void) { return g_err.c_str(); }
extern "C" int ofk_abi_version(void) { return OFK_ABI_VERSION; }
extern "C" long long ofk_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

// Attention implementation switch: wgmma kernels by default, the mma.sync kernels when OFK_ATTN_LEGACY=1 is set at load
// time or ofk_attn_force_legacy(1) was called (A/B measurements and the parity tests that compare the two).
static std::atomic<int> g_attn_legacy{-1};
static std::atomic<long long> g_attn_wgmma_calls{0};
bool ofk_attn_use_wgmma() {
  int v = g_attn_legacy.load(std::memory_order_relaxed);
  if (v < 0) {
    const char* e = getenv("OFK_ATTN_LEGACY");
    v = (e && atoi(e) != 0) ? 1 : 0;
    g_attn_legacy.store(v, std::memory_order_relaxed);
  }
  return v == 0;
}
void ofk_attn_count_wgmma() { g_attn_wgmma_calls.fetch_add(1, std::memory_order_relaxed); }
extern "C" int ofk_attn_force_legacy(int on) {
  const int prev = ofk_attn_use_wgmma() ? 0 : 1;
  g_attn_legacy.store(on ? 1 : 0, std::memory_order_relaxed);
  return prev;
}
extern "C" long long ofk_attn_tc_launch_count(void) { return g_attn_wgmma_calls.load(std::memory_order_relaxed); }
