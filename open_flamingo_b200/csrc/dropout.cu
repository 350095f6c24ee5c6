// Residual dropout of the OPT decoder block (HF OPTDecoderLayer: residual + dropout(branch, p) under autocast, with
// the branch a bf16 Linear output), fused with the fp32 residual add, and its backward.
//
// The keep mask is a counter-based draw: Philox-4x32-10 keyed by the 64-bit seed, on the counter
// (column / 4, row, offset low, offset high); lane column % 4 of the result is element (row, column)'s 32-bit draw,
// and the element is kept when that draw is >= floor(p * 2^32).  So the mask depends on (seed, offset, row, column)
// only -- not on the grid, the strides or which thread drew it -- and the backward regenerates it instead of reading a
// stored one.  Seed and offset are read from a device int64 pair, so a captured CUDA graph that advances the offset on
// the device draws a fresh mask at every replay.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "ofk_internal.h"
#include "ofk_ptx.cuh"

namespace ofk {

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return c;
}

// Keep bits of columns [c, c + 8) of row r (c a multiple of 8): bit j set = column c + j kept.
__device__ __forceinline__ uint32_t keep_bits8(uint64_t seed, uint64_t offset, long long r, int c, uint32_t thresh) {
  const uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  const uint32_t o0 = (uint32_t)offset, o1 = (uint32_t)(offset >> 32);
  const uint4 a = philox4x32_10(make_uint4((uint32_t)(c >> 2), (uint32_t)r, o0, o1), k0, k1);
  const uint4 b = philox4x32_10(make_uint4((uint32_t)(c >> 2) + 1u, (uint32_t)r, o0, o1), k0, k1);
  return (uint32_t)(a.x >= thresh) | (uint32_t)(a.y >= thresh) << 1 | (uint32_t)(a.z >= thresh) << 2 |
         (uint32_t)(a.w >= thresh) << 3 | (uint32_t)(b.x >= thresh) << 4 | (uint32_t)(b.y >= thresh) << 5 |
         (uint32_t)(b.z >= thresh) << 6 | (uint32_t)(b.w >= thresh) << 7;
}

// out = x + (kept ? bf16(branch * scale) : 0), a dropped element keeps x's bits.  One 8-column group per item.
// thresh == 0 (p = 0) keeps everything and reads no seed.
__global__ void __launch_bounds__(256) dropout_resid_fwd_kernel(
    const float* x, long long ldx, const __nv_bfloat16* __restrict__ br, long long ldb, int cols,
    uint32_t thresh, float scale, const long long* __restrict__ seed_offset, float* out, long long ldo,
    long long n8) {
  const int c8 = cols / 8;
  uint64_t seed = 0, offset = 0;
  if (thresh != 0) {
    seed = (uint64_t)__ldg(seed_offset);
    offset = (uint64_t)__ldg(seed_offset + 1);
  }
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += stride) {
    const long long r = i / c8;
    const int c = (int)(i % c8) * 8;
    const uint32_t keep = thresh != 0 ? keep_bits8(seed, offset, r, c, thresh) : 0xffu;
    const float4* xp = reinterpret_cast<const float4*>(x + r * ldx + c);
    const float4 x0 = xp[0], x1 = xp[1];
    const uint4 b = *reinterpret_cast<const uint4*>(br + r * ldb + c);
    const float xv[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
    const float bv[8] = {bf16_lo(b.x), bf16_hi(b.x), bf16_lo(b.y), bf16_hi(b.y),
                         bf16_lo(b.z), bf16_hi(b.z), bf16_lo(b.w), bf16_hi(b.w)};
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = (keep >> j) & 1u ? xv[j] + bf16_round(bv[j] * scale) : xv[j];
    float4* op = reinterpret_cast<float4*>(out + r * ldo + c);
    op[0] = make_float4(o[0], o[1], o[2], o[3]);
    op[1] = make_float4(o[4], o[5], o[6], o[7]);
  }
}

// dbranch = kept ? bf16(bf16(dout) * scale) : 0: the gradient autograd gives the bf16 branch through the fp32 residual
// add (a bf16 cast) and the dropout (a multiply by mask * scale in bf16).
__global__ void __launch_bounds__(256) dropout_resid_bwd_kernel(
    const float* __restrict__ dout, long long ldd, int cols, uint32_t thresh, float scale,
    const long long* __restrict__ seed_offset, __nv_bfloat16* __restrict__ dbr, long long lddb, long long n8) {
  const int c8 = cols / 8;
  uint64_t seed = 0, offset = 0;
  if (thresh != 0) {
    seed = (uint64_t)__ldg(seed_offset);
    offset = (uint64_t)__ldg(seed_offset + 1);
  }
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += stride) {
    const long long r = i / c8;
    const int c = (int)(i % c8) * 8;
    const uint32_t keep = thresh != 0 ? keep_bits8(seed, offset, r, c, thresh) : 0xffu;
    const float4* dp = reinterpret_cast<const float4*>(dout + r * ldd + c);
    const float4 d0 = dp[0], d1 = dp[1];
    const float dv[8] = {d0.x, d0.y, d0.z, d0.w, d1.x, d1.y, d1.z, d1.w};
    float g[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) g[j] = (keep >> j) & 1u ? bf16_round(dv[j]) * scale : 0.0f;
    *reinterpret_cast<uint4*>(dbr + r * lddb + c) =
        make_uint4(pack_bf16x2(g[0], g[1]), pack_bf16x2(g[2], g[3]), pack_bf16x2(g[4], g[5]), pack_bf16x2(g[6], g[7]));
  }
}

}  // namespace ofk

using namespace ofk;

static bool misaligned(const void* p, unsigned bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) != 0; }

static int grid_for8(long long n8) {
  long long b = (n8 + 255) / 256;
  if (b > 132LL * 16) b = 132LL * 16;
  return (int)(b < 1 ? 1 : b);
}

// The keep threshold floor(p * 2^32) and torch's dropout scale: 1 / (1 - p) with 1 - p taken in double and rounded
// to float before the division (at::native_dropout's fused kernel), the division in double, then rounded to float.
static void dropout_consts(double p, uint32_t* thresh, float* scale) {
  *thresh = (uint32_t)(p * 4294967296.0);
  *scale = (float)(1.0 / (double)(float)(1.0 - p));
}

// Checks both directions share, in the order of the header: p, the seed pair, rows and cols, then the strides.
static int dropout_check(const char* what, int rows, int cols, double p, const long long* seed_offset,
                         long long ld_f32, long long ld_f32b, long long ld_bf16) {
  if (!(p >= 0.0 && p < 1.0)) return ofk_set_error(OFK_ERR_ARG, what);
  if (p > 0.0 && !seed_offset) return ofk_set_error(OFK_ERR_ARG, what);
  if (rows < 1 || cols < 1 || cols % 8 != 0) return ofk_set_error(OFK_ERR_ARG, what);
  if (ld_f32 < cols || ld_f32b < cols || ld_bf16 < cols) return ofk_set_error(OFK_ERR_ARG, what);
  if (ld_f32 % 4 != 0 || ld_f32b % 4 != 0 || ld_bf16 % 8 != 0) return ofk_set_error(OFK_ERR_ALIGN, what);
  if (misaligned(seed_offset, 8)) return ofk_set_error(OFK_ERR_ALIGN, what);
  return 0;
}

extern "C" int ofk_dropout_resid_fwd(const float* x, long long ldx, const void* branch, long long ldb, int rows,
                                     int cols, double p, const long long* seed_offset, float* out, long long ldo,
                                     void* stream) {
  if (!x || !branch || !out) return ofk_set_error(OFK_ERR_ARG, "dropout_resid_fwd: null pointer");
  if (int rc = dropout_check("dropout_resid_fwd: p in [0, 1), a seed pair when p > 0, rows >= 1, cols a positive "
                             "multiple of 8, ldx, ldb and ldo >= cols, ldx and ldo multiples of 4, ldb of 8, seed pair "
                             "8-byte aligned", rows, cols, p, seed_offset, ldx, ldo, ldb))
    return rc;
  if (misaligned(x, 16) || misaligned(branch, 16) || misaligned(out, 16))
    return ofk_set_error(OFK_ERR_ALIGN, "dropout_resid_fwd: x, branch and out must be 16-byte aligned");
  uint32_t thresh;
  float scale;
  dropout_consts(p, &thresh, &scale);
  const long long n8 = (long long)rows * (cols / 8);
  dropout_resid_fwd_kernel<<<grid_for8(n8), 256, 0, (cudaStream_t)stream>>>(
      x, ldx, (const __nv_bfloat16*)branch, ldb, cols, thresh, scale, seed_offset, out, ldo, n8);
  OFK_CHECK_LAUNCH();
  return 0;
}

extern "C" int ofk_dropout_resid_bwd(const float* dout, long long ldd, int rows, int cols, double p,
                                     const long long* seed_offset, void* dbranch, long long lddb, void* stream) {
  if (!dout || !dbranch) return ofk_set_error(OFK_ERR_ARG, "dropout_resid_bwd: null pointer");
  if (int rc = dropout_check("dropout_resid_bwd: p in [0, 1), a seed pair when p > 0, rows >= 1, cols a positive "
                             "multiple of 8, ldd and lddb >= cols, ldd a multiple of 4, lddb of 8, seed pair 8-byte "
                             "aligned", rows, cols, p, seed_offset, ldd, ldd, lddb))
    return rc;
  if (misaligned(dout, 16) || misaligned(dbranch, 16))
    return ofk_set_error(OFK_ERR_ALIGN, "dropout_resid_bwd: dout and dbranch must be 16-byte aligned");
  uint32_t thresh;
  float scale;
  dropout_consts(p, &thresh, &scale);
  const long long n8 = (long long)rows * (cols / 8);
  dropout_resid_bwd_kernel<<<grid_for8(n8), 256, 0, (cudaStream_t)stream>>>(
      dout, ldd, cols, thresh, scale, seed_offset, (__nv_bfloat16*)dbranch, lddb, n8);
  OFK_CHECK_LAUNCH();
  return 0;
}
