// RMSNorm forward / backward of the LLaMA decoder blocks (HF LlamaRMSNorm), fp32 statistics, HBM-bound.
// One 256-thread block per row; thread t owns the 8-column groups (g * 256 + t) * 8, so a row of up to 8192 columns
// stays in registers.  Row sums add each thread's columns in order, the lanes of a warp by a butterfly and the eight
// warps in index order: the same bits on every launch.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "ofk_internal.h"
#include "ofk_ptx.cuh"

namespace ofk {

constexpr int RMS_THREADS = 256;
constexpr int RMS_MAX_D = 8192;

__device__ __forceinline__ float rms_block_sum(float v, float* s_red) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int w = 0; w < RMS_THREADS / 32; ++w) s += s_red[w];
  return s;
}

__device__ __forceinline__ void load8(const float* p, float (&v)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

__device__ __forceinline__ void ldg8(const float* p, float (&v)[8]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p + 4));
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

// y = bf16(gamma * (x * rstd)), rstd = rsqrt(mean(x^2) + eps): LlamaRMSNorm's product order, rounded once where
// autocast rounds its fp32 output as the next Linear's operand.
template <int G>
__global__ void __launch_bounds__(RMS_THREADS) rmsnorm_fwd_kernel(const float* __restrict__ x, long long ldx,
                                                                  const float* __restrict__ gamma, float eps, int D,
                                                                  __nv_bfloat16* __restrict__ y, long long ldy,
                                                                  float* __restrict__ rstd_out) {
  __shared__ float s_red[RMS_THREADS / 32];
  const int row = blockIdx.x, t = threadIdx.x;
  const float* xr = x + (long long)row * ldx;
  float v[G][8];
  float s = 0.f;
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const int c = (g * RMS_THREADS + t) * 8;
    if (c < D) {
      load8(xr + c, v[g]);
#pragma unroll
      for (int j = 0; j < 8; ++j) s += v[g][j] * v[g][j];
    }
  }
  const float rstd = rsqrtf(rms_block_sum(s, s_red) / (float)D + eps);
  if (t == 0 && rstd_out) rstd_out[row] = rstd;
  __nv_bfloat16* yr = y + (long long)row * ldy;
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const int c = (g * RMS_THREADS + t) * 8;
    if (c < D) {
      float gm[8];
      ldg8(gamma + c, gm);
      uint32_t o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j)
        o[j] = pack_bf16x2(gm[2 * j] * (v[g][2 * j] * rstd), gm[2 * j + 1] * (v[g][2 * j + 1] * rstd));
      *reinterpret_cast<uint4*>(yr + c) = make_uint4(o[0], o[1], o[2], o[3]);
    }
  }
}

// dx = rstd * (gamma * dy - xhat * mean(gamma * dy * xhat)) (+ dx_add), xhat = x * rstd.  dx_add may alias dx: each
// element is read and written by the same thread.
template <int G>
__global__ void __launch_bounds__(RMS_THREADS) rmsnorm_bwd_kernel(const __nv_bfloat16* __restrict__ dy, long long lddy,
                                                                  const float* __restrict__ x, long long ldx,
                                                                  const float* __restrict__ gamma,
                                                                  const float* __restrict__ rstd, int D, float* dx,
                                                                  long long lddx, const float* dx_add, long long ldadd) {
  __shared__ float s_red[RMS_THREADS / 32];
  const int row = blockIdx.x, t = threadIdx.x;
  const float rs = rstd[row];
  float gd[G][8], xh[G][8];
  float s = 0.f;
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const int c = (g * RMS_THREADS + t) * 8;
    if (c < D) {
      const uint4 u = *reinterpret_cast<const uint4*>(dy + (long long)row * lddy + c);
      const float d[8] = {bf16_lo(u.x), bf16_hi(u.x), bf16_lo(u.y), bf16_hi(u.y),
                          bf16_lo(u.z), bf16_hi(u.z), bf16_lo(u.w), bf16_hi(u.w)};
      float gm[8];
      ldg8(gamma + c, gm);
      load8(x + (long long)row * ldx + c, xh[g]);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        gd[g][j] = d[j] * gm[j];
        xh[g][j] *= rs;
        s += gd[g][j] * xh[g][j];
      }
    }
  }
  const float m = rms_block_sum(s, s_red) / (float)D;
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const int c = (g * RMS_THREADS + t) * 8;
    if (c < D) {
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = rs * (gd[g][j] - xh[g][j] * m);
      if (dx_add) {
        float a[8];
        load8(dx_add + (long long)row * ldadd + c, a);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] += a[j];
      }
      float* dr = dx + (long long)row * lddx + c;
      *reinterpret_cast<float4*>(dr) = make_float4(o[0], o[1], o[2], o[3]);
      *reinterpret_cast<float4*>(dr + 4) = make_float4(o[4], o[5], o[6], o[7]);
    }
  }
}

static bool misaligned(const void* p, unsigned bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) != 0; }

static bool bad_width(int D) { return D <= 0 || D % 8 != 0 || D > RMS_MAX_D; }

}  // namespace ofk

extern "C" int ofk_rmsnorm_fwd(const float* x, long long ldx, const float* gamma, float eps, int rows, int D, void* y,
                               long long ldy, float* rstd, void* stream_) {
  using namespace ofk;
  if (!x || !gamma || !y) return ofk_set_error(OFK_ERR_ARG, "rmsnorm: null pointer");
  if (rows < 1) return ofk_set_error(OFK_ERR_ARG, "rmsnorm: rows must be >= 1");
  if (bad_width(D)) return ofk_set_error(OFK_ERR_ARG, "rmsnorm: D must be a positive multiple of 8, <= 8192");
  if (ldx < D || ldy < D) return ofk_set_error(OFK_ERR_ARG, "rmsnorm: row strides must be >= D");
  if (ldx % 4 != 0 || ldy % 8 != 0) return ofk_set_error(OFK_ERR_ALIGN, "rmsnorm: ldx must be a multiple of 4, ldy of 8");
  if (misaligned(x, 16) || misaligned(gamma, 16) || misaligned(y, 16) || misaligned(rstd, 4))
    return ofk_set_error(OFK_ERR_ALIGN, "rmsnorm: x, gamma and y must be 16-byte aligned, rstd 4-byte");
  cudaStream_t s = (cudaStream_t)stream_;
  __nv_bfloat16* yb = reinterpret_cast<__nv_bfloat16*>(y);
  if (D <= 2048)
    rmsnorm_fwd_kernel<1><<<rows, RMS_THREADS, 0, s>>>(x, ldx, gamma, eps, D, yb, ldy, rstd);
  else if (D <= 4096)
    rmsnorm_fwd_kernel<2><<<rows, RMS_THREADS, 0, s>>>(x, ldx, gamma, eps, D, yb, ldy, rstd);
  else
    rmsnorm_fwd_kernel<4><<<rows, RMS_THREADS, 0, s>>>(x, ldx, gamma, eps, D, yb, ldy, rstd);
  OFK_CHECK_LAUNCH();
  return 0;
}

extern "C" int ofk_rmsnorm_bwd(const void* dy, long long lddy, const float* x, long long ldx, const float* gamma,
                               const float* rstd, int rows, int D, float* dx, long long lddx, const float* dx_add,
                               long long ldadd, void* stream_) {
  using namespace ofk;
  if (!dy || !x || !gamma || !rstd || !dx) return ofk_set_error(OFK_ERR_ARG, "rmsnorm bwd: null pointer");
  if (rows < 1) return ofk_set_error(OFK_ERR_ARG, "rmsnorm bwd: rows must be >= 1");
  if (bad_width(D)) return ofk_set_error(OFK_ERR_ARG, "rmsnorm bwd: D must be a positive multiple of 8, <= 8192");
  if (lddy < D || ldx < D || lddx < D || (dx_add && ldadd < D))
    return ofk_set_error(OFK_ERR_ARG, "rmsnorm bwd: row strides must be >= D");
  if (lddy % 8 != 0 || ldx % 4 != 0 || lddx % 4 != 0 || (dx_add && ldadd % 4 != 0))
    return ofk_set_error(OFK_ERR_ALIGN, "rmsnorm bwd: lddy must be a multiple of 8, ldx, lddx and ldadd of 4");
  if (misaligned(dy, 16) || misaligned(x, 16) || misaligned(gamma, 16) || misaligned(dx, 16) ||
      misaligned(dx_add, 16) || misaligned(rstd, 4))
    return ofk_set_error(OFK_ERR_ALIGN, "rmsnorm bwd: dy, x, gamma, dx and dx_add must be 16-byte aligned, rstd 4-byte");
  cudaStream_t s = (cudaStream_t)stream_;
  const __nv_bfloat16* db = reinterpret_cast<const __nv_bfloat16*>(dy);
  if (D <= 2048)
    rmsnorm_bwd_kernel<1><<<rows, RMS_THREADS, 0, s>>>(db, lddy, x, ldx, gamma, rstd, D, dx, lddx, dx_add, ldadd);
  else if (D <= 4096)
    rmsnorm_bwd_kernel<2><<<rows, RMS_THREADS, 0, s>>>(db, lddy, x, ldx, gamma, rstd, D, dx, lddx, dx_add, ldadd);
  else
    rmsnorm_bwd_kernel<4><<<rows, RMS_THREADS, 0, s>>>(db, lddy, x, ldx, gamma, rstd, D, dx, lddx, dx_add, ldadd);
  OFK_CHECK_LAUNCH();
  return 0;
}
