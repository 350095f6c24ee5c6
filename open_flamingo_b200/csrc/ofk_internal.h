// Internal helpers shared by the .cu translation units of libofk.so.
#pragma once
#include "../../include/ofk.h"

// Records the message returned by ofk_last_error() (thread-local) and returns `code`.
int ofk_set_error(int code, const char* msg);
void ofk_count_launch();
// Attention: true unless the mma.sync kernels were forced (ofk_attn_force_legacy / OFK_ATTN_LEGACY=1); every entry-point
// call served by the wgmma kernels is counted (ofk_attn_tc_launch_count).
bool ofk_attn_use_wgmma();
void ofk_attn_count_wgmma();

#define OFK_CHECK_LAUNCH()                                                        \
  do {                                                                            \
    cudaError_t e__ = cudaGetLastError();                                         \
    if (e__ != cudaSuccess) return ofk_set_error(OFK_ERR_CUDA, cudaGetErrorString(e__)); \
    ofk_count_launch();                                                           \
  } while (0)
