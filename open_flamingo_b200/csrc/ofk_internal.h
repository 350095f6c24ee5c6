// Internal helpers shared by the .cu translation units of libofk.so.
#pragma once
#include "../../include/ofk.h"

// Records the message returned by ofk_last_error() (thread-local) and returns `code`.
int ofk_set_error(int code, const char* msg);
void ofk_count_launch();

#define OFK_CHECK_LAUNCH()                                                        \
  do {                                                                            \
    cudaError_t e__ = cudaGetLastError();                                         \
    if (e__ != cudaSuccess) return ofk_set_error(OFK_ERR_CUDA, cudaGetErrorString(e__)); \
    ofk_count_launch();                                                           \
  } while (0)
