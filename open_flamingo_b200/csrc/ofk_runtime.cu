// Error reporting + launch accounting for libofk.so.
#include <atomic>
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
