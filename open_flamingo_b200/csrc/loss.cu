// Fused shifted causal-LM cross-entropy on the LM head's logits (the loss `Flamingo.forward` returns when labels
// are given: flamingo.py:111-117 -> HF `ForCausalLMLoss`: logits.float(), labels shifted left by one with -100
// padding, cross_entropy(mean over non-ignored)).  The reference path materialises an fp32 copy of the
// [B*T, vocab] logits, its log-softmax and, in backward, the softmax gradient (several 1.6 GB round trips at
// OF-3B); here the forward reads the logits once (row max / log-sum-exp / target logit) and the backward reads
// them once more and writes d(logits) directly.  HBM-bound, one 256-thread block per row.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "ofk_internal.h"
#include "ofk_ptx.cuh"

namespace ofk {

__device__ __forceinline__ float load_logit(const void* base, int is_f32, long long idx) {
  return is_f32 ? reinterpret_cast<const float*>(base)[idx]
                : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(base)[idx]);
}

__device__ __forceinline__ long long row_target(const long long* labels, int T, long long row, int shift) {
  const long long b = row / T, t = row % T;
  if (shift) return (t + 1 < T) ? labels[b * T + t + 1] : -100;
  return labels[row];
}

// lse[row] (natural log) of every row.
// vec: the rows may be read 8 bf16 at a time (see vec8_rows).
__global__ void __launch_bounds__(256) ce_fwd_kernel(const void* __restrict__ logits, int is_f32, int vec, long long ld,
                                                     int V, float* __restrict__ lse) {
  __shared__ float s_m[8], s_l[8];
  const long long row = blockIdx.x;
  float m = -INFINITY, l = 0.f;
  // The running max is subtracted as 0 while it is still -inf (every logit so far was -inf): -inf - -inf would be NaN.
  if (vec) {
    const uint4* p = reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(logits) + row * ld);
    for (int i = threadIdx.x; i < V / 8; i += 256) {
      const uint4 u = p[i];
      const float v[8] = {bf16_lo(u.x), bf16_hi(u.x), bf16_lo(u.y), bf16_hi(u.y), bf16_lo(u.z), bf16_hi(u.z), bf16_lo(u.w), bf16_hi(u.w)};
      float mx = m;
#pragma unroll
      for (int j = 0; j < 8; ++j) mx = fmaxf(mx, v[j]);
      const float ms = mx == -INFINITY ? 0.f : mx;
      float acc = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) acc += __expf(v[j] - ms);
      l = l * __expf(m - ms) + acc;
      m = mx;
    }
  } else {
    for (int i = threadIdx.x; i < V; i += 256) {
      const float v = load_logit(logits, is_f32, row * ld + i);
      const float mx = fmaxf(m, v);
      const float ms = mx == -INFINITY ? 0.f : mx;
      l = l * __expf(m - ms) + __expf(v - ms);
      m = mx;
    }
  }
  // block combine of (m, l)
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), l2 = __shfl_xor_sync(0xffffffffu, l, o);
    const float mx = fmaxf(m, m2);
    l = (m == -INFINITY ? 0.f : l * __expf(m - mx)) + (m2 == -INFINITY ? 0.f : l2 * __expf(m2 - mx));
    m = mx;
  }
  if ((threadIdx.x & 31) == 0) { s_m[threadIdx.x >> 5] = m; s_l[threadIdx.x >> 5] = l; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float M = -INFINITY, Ls = 0.f;
    for (int w = 0; w < 8; ++w) M = fmaxf(M, s_m[w]);
    for (int w = 0; w < 8; ++w) Ls += (s_m[w] == -INFINITY) ? 0.f : s_l[w] * __expf(s_m[w] - M);
    const float L = M + logf(Ls);
    lse[row] = L;
  }
}

// *loss_sum += sum over non-ignored rows of (lse - logit[target]); *count += their number.  One block, fixed order
// (no atomics), so the loss does not depend on which row finished first.
__global__ void __launch_bounds__(256) ce_sum_kernel(const void* __restrict__ logits, int is_f32, long long ld, long long rows,
                                                     int V, const long long* __restrict__ labels, int T, int shift,
                                                     long long ignore_index, const float* __restrict__ lse,
                                                     float* __restrict__ loss_sum, float* __restrict__ count) {
  __shared__ float s_l[8], s_c[8];
  float acc = 0.f, cnt = 0.f;
  for (long long row = threadIdx.x; row < rows; row += 256) {
    const long long tgt = row_target(labels, T, row, shift);
    if (tgt != ignore_index && tgt >= 0 && tgt < V) {
      acc += lse[row] - load_logit(logits, is_f32, row * ld + tgt);
      cnt += 1.0f;
    }
  }
  acc = warp_sum(acc);
  cnt = warp_sum(cnt);
  if ((threadIdx.x & 31) == 0) { s_l[threadIdx.x >> 5] = acc; s_c[threadIdx.x >> 5] = cnt; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, b = 0.f;
    for (int w = 0; w < 8; ++w) { a += s_l[w]; b += s_c[w]; }
    *loss_sum += a;
    *count += b;
  }
}

// dlogits[row, v] = (softmax(row)[v] - [v == target]) * (*gscale) / (*count) for non-ignored rows, else 0.
__global__ void __launch_bounds__(256) ce_bwd_kernel(const void* __restrict__ logits, int is_f32, int vec, long long ld, int V,
                                                     const long long* __restrict__ labels, int T, int shift,
                                                     long long ignore_index, const float* __restrict__ lse,
                                                     const float* __restrict__ gscale, const float* __restrict__ count,
                                                     void* __restrict__ dlogits, long long ldd) {
  const long long row = blockIdx.x;
  const long long tgt = row_target(labels, T, row, shift);
  const bool valid = tgt != ignore_index && tgt >= 0 && tgt < V;
  const float sc = valid ? __ldg(gscale) / fmaxf(__ldg(count), 1.0f) : 0.f;
  const float L = lse[row];
  if (vec) {
    const uint4* p = reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(logits) + row * ld);
    uint4* d = reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(dlogits) + row * ldd);
    for (int i = threadIdx.x; i < V / 8; i += 256) {
      const uint4 u = p[i];
      float v[8] = {bf16_lo(u.x), bf16_hi(u.x), bf16_lo(u.y), bf16_hi(u.y), bf16_lo(u.z), bf16_hi(u.z), bf16_lo(u.w), bf16_hi(u.w)};
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float pj = __expf(v[j] - L);
        v[j] = (pj - ((long long)i * 8 + j == tgt ? 1.0f : 0.0f)) * sc;
      }
      d[i] = make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
    }
  } else {
    for (int i = threadIdx.x; i < V; i += 256) {
      const float pj = __expf(load_logit(logits, is_f32, row * ld + i) - L);
      const float g = (pj - (i == tgt ? 1.0f : 0.0f)) * sc;
      if (is_f32) reinterpret_cast<float*>(dlogits)[row * ldd + i] = g;
      else reinterpret_cast<__nv_bfloat16*>(dlogits)[row * ldd + i] = __float2bfloat16_rn(g);
    }
  }
}

// The 8-wide bf16 path reads (and writes) each row as uint4: it needs every row start 16-byte aligned.  Any other
// layout takes the scalar path, which is correct for every pointer and stride.
static int vec8_rows(const void* p, int is_f32, long long ld, int V) {
  return !is_f32 && V % 8 == 0 && ld % 8 == 0 && (reinterpret_cast<uintptr_t>(p) & 15) == 0;
}

}  // namespace ofk

extern "C" int ofk_ce_fwd(const void* logits, int logits_is_f32, long long ld, long long rows, int vocab,
                          const long long* labels, int T, int shift_labels, long long ignore_index, float* lse,
                          float* loss_sum, float* count, void* stream) {
  if (!logits || !labels || !lse || !loss_sum || !count) return ofk_set_error(OFK_ERR_ARG, "ce_fwd: null pointer");
  if (rows <= 0) return 0;
  if (vocab <= 0 || T <= 0 || rows % T != 0) return ofk_set_error(OFK_ERR_ARG, "ce_fwd: rows must be a multiple of T");
  const int vec = ofk::vec8_rows(logits, logits_is_f32, ld, vocab);
  ofk::ce_fwd_kernel<<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>(logits, logits_is_f32, vec, ld, vocab, lse);
  OFK_CHECK_LAUNCH();
  ofk::ce_sum_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(logits, logits_is_f32, ld, rows, vocab, labels, T, shift_labels,
                                                          ignore_index, lse, loss_sum, count);
  OFK_CHECK_LAUNCH();
  return 0;
}

extern "C" int ofk_ce_bwd(const void* logits, int logits_is_f32, long long ld, long long rows, int vocab,
                          const long long* labels, int T, int shift_labels, long long ignore_index, const float* lse,
                          const float* grad_scale, const float* count, void* dlogits, long long ldd, void* stream) {
  if (!logits || !labels || !lse || !grad_scale || !count || !dlogits) return ofk_set_error(OFK_ERR_ARG, "ce_bwd: null pointer");
  if (rows <= 0) return 0;
  if (vocab <= 0 || T <= 0 || rows % T != 0) return ofk_set_error(OFK_ERR_ARG, "ce_bwd: rows must be a multiple of T");
  const int vec = ofk::vec8_rows(logits, logits_is_f32, ld, vocab) && ofk::vec8_rows(dlogits, logits_is_f32, ldd, vocab);
  ofk::ce_bwd_kernel<<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>(logits, logits_is_f32, vec, ld, vocab, labels, T,
                                                                        shift_labels, ignore_index, lse, grad_scale, count,
                                                                        dlogits, ldd);
  OFK_CHECK_LAUNCH();
  return 0;
}
