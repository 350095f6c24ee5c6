// Self-attention core of the frozen LM's decoder blocks (SURVEY.md section 8f rank 1: HF MptAttention, reached
// through flamingo_lm.py:63-65), head_dim 64 or 128, bf16 in/out, fp32 online softmax:
//
//   S = scale * Q K^T + slope[h] * key_index          (ALiBi; MPT's bias is slope * (key - (nk-1)), and softmax
//                                                      is invariant to the per-row constant)
//   S[masked] = "finfo.min"                           (explicit bool mask [B, nq, nk], True = masked, and/or
//                                                      the causal rule key <= query + nk - nq)
//   O = softmax(S) V
//
// Masked scores are set to a large finite negative (not -inf), exactly like masked_fill(finfo.min): a row whose
// keys are all masked (a padded query) therefore gets the reference's uniform attention, not NaN/zeros.
// Backward (dgrad only -- the LM is frozen): dQ kernel + dK/dV kernel, both recomputing P from the saved LSE.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "attention_tile.cuh"
#include "ofk_internal.h"

namespace ofk {
namespace dense {

constexpr float MASKED = -30000.0f;  // log2-domain stand-in for finfo.min: exp2(MASKED - m) == 0 for any real m

struct Params {
  const __nv_bfloat16 *q, *k, *v, *o, *d_o;
  __nv_bfloat16 *out, *dq, *dk, *dv;
  float* lse;
  float* delta;
  const unsigned char* mask;  // [B, nq, nk] 1 = masked, or NULL
  const float* slopes;        // [heads] or NULL
  const int* pure_causal;     // device flag or NULL: nonzero => the mask is exactly the causal rule (ignore `mask`,
                              // apply causal, skip key tiles above the diagonal) -- decided on the device, no host sync
  int batch, heads, nq, nk, causal;
  long long q_bs, ldq, k_bs, ldk, v_bs, ldv, o_bs, ldo, dq_bs, lddq, dk_bs, lddk, dv_bs, lddv;
  float scale;
};

// P as hi + lo bf16 fragments (lo = P - bf16(P), exact in fp32): O += P_hi V + P_lo V carries P to ~16 mantissa bits
// instead of 8.  A single bf16 rounding of P here, compounded over the LM's decoder blocks, was measured to bias the
// gradient reaching the first gated block by 1-2 % against fp32 (the gate-gradient parity test).
__device__ __forceinline__ void c_to_a_split(float (&c)[8][4], uint32_t (&hi)[4][4], uint32_t (&lo)[4][4]) {
  c_to_a(c, hi);
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int e = 0; e < 4; ++e) c[i][e] -= bf16_round(c[i][e]);
  c_to_a(c, lo);
}

// log2-domain score of (row, key) given the raw dot product.
__device__ __forceinline__ float score(const Params& p, float dot, float sl2, float slope2, int b, int row, int key) {
  if (key >= p.nk) return -INFINITY;
  bool masked = p.causal && key > row + (p.nk - p.nq);
  if (!masked && p.mask && row < p.nq) masked = p.mask[((long long)b * p.nq + row) * p.nk + key] != 0;
  return masked ? MASKED : fmaf(dot, sl2, slope2 * (float)key);
}
__device__ __forceinline__ bool is_masked(const Params& p, int b, int row, int key) {
  if (p.causal && key > row + (p.nk - p.nq)) return true;
  if (p.mask && row < p.nq) return p.mask[((long long)b * p.nq + row) * p.nk + key] != 0;
  return false;
}
// key tiles a query block needs when only the causal rule applies
__device__ __forceinline__ int causal_tiles(const Params& p, int q0) {
  const int total = (p.nk + BKV - 1) / BKV;
  if (!p.causal || p.mask) return total;
  const int last_key = min(p.nk - 1, q0 + BQ - 1 + (p.nk - p.nq));
  return last_key < 0 ? 0 : min(total, last_key / BKV + 1);
}

// Tile classes for the fast paths: with no explicit mask, an in-bounds key tile entirely at or below the diagonal
// of ALL rows this thread touches needs no per-score predicate (that is ~3/4 of the causal work at T = 256).
__device__ __forceinline__ bool tile_unmasked(const Params& p, int key_last, int row_first) {
  if (p.mask != nullptr || key_last >= p.nk) return false;
  return !p.causal || key_last <= row_first + (p.nk - p.nq);
}

// ================================================================ forward
template <int HD>
__global__ void __launch_bounds__(THREADS) fwd_kernel(const Params p_in) {
  Params p = p_in;
  if (p.pure_causal != nullptr && *p.pure_causal != 0) { p.mask = nullptr; p.causal = 1; }
  using T = Tile<HD>;
  uint8_t* sQ = tile_at<HD>(0);
  auto sK = [](int buf) { return tile_at<HD>(1 + buf); };
  auto sV = [](int buf) { return tile_at<HD>(3 + buf); };

  const int q0 = blockIdx.x * BQ, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const __nv_bfloat16* qp = p.q + b * p.q_bs + h * HD;
  const __nv_bfloat16* kp = p.k + b * p.k_bs + h * HD;
  const __nv_bfloat16* vp = p.v + b * p.v_bs + h * HD;
  const int nblk = causal_tiles(p, q0);

  load_tile<HD>(sQ, qp, p.ldq, q0, p.nq);
  if (nblk > 0) { load_tile<HD>(sK(0), kp, p.ldk, 0, p.nk); load_tile<HD>(sV(0), vp, p.ldv, 0, p.nk); }
  cp_commit();

  const int row_a = q0 + warp * 16 + g, row_b = row_a + 8;
  const float sl2 = p.scale * LOG2E;
  const float slope2 = p.slopes ? p.slopes[h] * LOG2E : 0.f;
  float o[T::NT][4];
#pragma unroll
  for (int i = 0; i < T::NT; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
  float m_a = -INFINITY, m_b = -INFINITY, l_a = 0.f, l_b = 0.f;

  for (int j = 0; j < nblk; ++j) {
    const int buf = j & 1;
    if (j + 1 < nblk) {
      load_tile<HD>(sK(buf ^ 1), kp, p.ldk, (j + 1) * BKV, p.nk);
      load_tile<HD>(sV(buf ^ 1), vp, p.ldv, (j + 1) * BKV, p.nk);
      cp_commit();
      cp_wait<1>();
    } else {
      cp_wait<0>();
    }
    fence_proxy_async_smem();   // cp.async (generic proxy) -> wgmma reads
    __syncthreads();
    float s[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; }
    mma_rows_x_tileT<HD>(s, sQ, sK(buf));
    float mx_a = -INFINITY, mx_b = -INFINITY;
    if (tile_unmasked(p, j * BKV + BKV - 1, q0 + warp * 16)) {
      const float kb = slope2 * (float)(j * BKV + 2 * t);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float b0 = kb + slope2 * (float)(i * 8), b1 = b0 + slope2;
        s[i][0] = fmaf(s[i][0], sl2, b0); s[i][1] = fmaf(s[i][1], sl2, b1);
        s[i][2] = fmaf(s[i][2], sl2, b0); s[i][3] = fmaf(s[i][3], sl2, b1);
        mx_a = fmaxf(mx_a, fmaxf(s[i][0], s[i][1]));
        mx_b = fmaxf(mx_b, fmaxf(s[i][2], s[i][3]));
      }
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int key = j * BKV + i * 8 + 2 * t;
        s[i][0] = score(p, s[i][0], sl2, slope2, b, row_a, key);
        s[i][1] = score(p, s[i][1], sl2, slope2, b, row_a, key + 1);
        s[i][2] = score(p, s[i][2], sl2, slope2, b, row_b, key);
        s[i][3] = score(p, s[i][3], sl2, slope2, b, row_b, key + 1);
        mx_a = fmaxf(mx_a, fmaxf(s[i][0], s[i][1]));
        mx_b = fmaxf(mx_b, fmaxf(s[i][2], s[i][3]));
      }
    }
    softmax_step(s, mx_a, mx_b, m_a, m_b, l_a, l_b, o);
    uint32_t pa[4][4], pl[4][4];
    c_to_a_split(s, pa, pl);
    mma_p_x_tile<HD>(o, pa, sV(buf));
    mma_p_x_tile<HD>(o, pl, sV(buf));
    __syncthreads();
  }
  if (nblk == 0) cp_wait<0>();

  l_a = quad_sum(l_a); l_b = quad_sum(l_b);
  const float inv_a = l_a > 0.f ? 1.f / l_a : 0.f, inv_b = l_b > 0.f ? 1.f / l_b : 0.f;
  store_rows(p.out + b * p.o_bs + h * HD, p.ldo, o, inv_a, inv_b, row_a, row_b, p.nq, t);
  if (p.lse != nullptr && t == 0) store_lse(p.lse + ((long long)b * p.heads + h) * p.nq, m_a, l_a, m_b, l_b, row_a, row_b, p.nq);
}

// ================================================================ dQ (CTA = 64 queries, loop key tiles)
template <int HD>
__global__ void __launch_bounds__(THREADS) bwd_dq_kernel(const Params p_in) {
  Params p = p_in;
  if (p.pure_causal != nullptr && *p.pure_causal != 0) { p.mask = nullptr; p.causal = 1; }
  using T = Tile<HD>;
  uint8_t* sQ = tile_at<HD>(0);
  uint8_t* sdO = tile_at<HD>(1);
  auto sK = [](int buf) { return tile_at<HD>(2 + buf); };
  auto sV = [](int buf) { return tile_at<HD>(4 + buf); };

  const int q0 = blockIdx.x * BQ, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const __nv_bfloat16* qp = p.q + b * p.q_bs + h * HD;
  const __nv_bfloat16* kp = p.k + b * p.k_bs + h * HD;
  const __nv_bfloat16* vp = p.v + b * p.v_bs + h * HD;
  const __nv_bfloat16* dop = p.d_o + b * p.o_bs + h * HD;
  const int nblk = causal_tiles(p, q0);

  load_tile<HD>(sQ, qp, p.ldq, q0, p.nq);
  load_tile<HD>(sdO, dop, p.ldo, q0, p.nq);
  if (nblk > 0) { load_tile<HD>(sK(0), kp, p.ldk, 0, p.nk); load_tile<HD>(sV(0), vp, p.ldv, 0, p.nk); }
  cp_commit();

  const int row_a = q0 + warp * 16 + g, row_b = row_a + 8;
  const float* lp = p.lse + ((long long)b * p.heads + h) * p.nq;
  const float* dp = p.delta + ((long long)b * p.heads + h) * p.nq;
  const float lse_a = row_a < p.nq ? lp[row_a] : 0.f, lse_b = row_b < p.nq ? lp[row_b] : 0.f;
  const float del_a = row_a < p.nq ? dp[row_a] : 0.f, del_b = row_b < p.nq ? dp[row_b] : 0.f;
  const float sl2 = p.scale * LOG2E;
  const float slope2 = p.slopes ? p.slopes[h] * LOG2E : 0.f;
  float dq[T::NT][4];
#pragma unroll
  for (int i = 0; i < T::NT; ++i) { dq[i][0] = dq[i][1] = dq[i][2] = dq[i][3] = 0.f; }

  for (int j = 0; j < nblk; ++j) {
    const int buf = j & 1;
    if (j + 1 < nblk) {
      load_tile<HD>(sK(buf ^ 1), kp, p.ldk, (j + 1) * BKV, p.nk);
      load_tile<HD>(sV(buf ^ 1), vp, p.ldv, (j + 1) * BKV, p.nk);
      cp_commit();
      cp_wait<1>();
    } else {
      cp_wait<0>();
    }
    fence_proxy_async_smem();   // cp.async (generic proxy) -> wgmma reads
    __syncthreads();
    float s[8][4], dpv[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; dpv[i][0] = dpv[i][1] = dpv[i][2] = dpv[i][3] = 0.f; }
    mma_rows_x_tileT<HD>(s, sQ, sK(buf));     // S  = Q K^T
    mma_rows_x_tileT<HD>(dpv, sdO, sV(buf));  // dP = dO V^T
    if (tile_unmasked(p, j * BKV + BKV - 1, q0 + warp * 16)) {
      const float kb = slope2 * (float)(j * BKV + 2 * t);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float b0 = kb + slope2 * (float)(i * 8), b1 = b0 + slope2;
        s[i][0] = ex2_approx(fmaf(s[i][0], sl2, b0) - lse_a) * (dpv[i][0] - del_a) * p.scale;
        s[i][1] = ex2_approx(fmaf(s[i][1], sl2, b1) - lse_a) * (dpv[i][1] - del_a) * p.scale;
        s[i][2] = ex2_approx(fmaf(s[i][2], sl2, b0) - lse_b) * (dpv[i][2] - del_b) * p.scale;
        s[i][3] = ex2_approx(fmaf(s[i][3], sl2, b1) - lse_b) * (dpv[i][3] - del_b) * p.scale;
      }
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int key = j * BKV + i * 8 + 2 * t + (e & 1);
          const int row = (e & 2) ? row_b : row_a;
          const float sc = score(p, s[i][e], sl2, slope2, b, row, key);
          const float pv = ex2_approx(sc - ((e & 2) ? lse_b : lse_a));
          const bool live = key < p.nk && !is_masked(p, b, row, key);   // masked_fill passes no gradient to the scores
          s[i][e] = live ? pv * (dpv[i][e] - ((e & 2) ? del_b : del_a)) * p.scale : 0.f;
        }
      }
    }
    uint32_t dsa[4][4];
    c_to_a(s, dsa);
    mma_p_x_tile<HD>(dq, dsa, sK(buf));                  // dQ += dS K
    __syncthreads();
  }
  if (nblk == 0) cp_wait<0>();

  store_rows(p.dq + b * p.dq_bs + h * HD, p.lddq, dq, 1.f, 1.f, row_a, row_b, p.nq, t);
}

// ================================================================ dK, dV (CTA = 64 keys, loop query tiles)
template <int HD>
__global__ void __launch_bounds__(THREADS) bwd_dkv_kernel(const Params p_in) {
  Params p = p_in;
  if (p.pure_causal != nullptr && *p.pure_causal != 0) { p.mask = nullptr; p.causal = 1; }
  using T = Tile<HD>;
  uint8_t* sK = tile_at<HD>(0);
  uint8_t* sV = tile_at<HD>(1);
  auto sQ = [](int buf) { return tile_at<HD>(2 + buf); };
  auto sdO = [](int buf) { return tile_at<HD>(4 + buf); };
  __shared__ float s_lse[2][BQ], s_del[2][BQ];

  const int k0 = blockIdx.x * BKV, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const __nv_bfloat16* qp = p.q + b * p.q_bs + h * HD;
  const __nv_bfloat16* kp = p.k + b * p.k_bs + h * HD;
  const __nv_bfloat16* vp = p.v + b * p.v_bs + h * HD;
  const __nv_bfloat16* dop = p.d_o + b * p.o_bs + h * HD;
  const float* lp = p.lse + ((long long)b * p.heads + h) * p.nq;
  const float* dlp = p.delta + ((long long)b * p.heads + h) * p.nq;
  const int nqb = (p.nq + BQ - 1) / BQ;
  // pure-causal: query blocks entirely before this key block see none of its keys
  int qb0 = 0;
  if (p.causal && !p.mask) qb0 = max(0, (k0 - (p.nk - p.nq)) / BQ);
  const float sl2 = p.scale * LOG2E;
  const float slope2 = p.slopes ? p.slopes[h] * LOG2E : 0.f;

  auto stage_rows = [&](int buf, int qb) {
    if (threadIdx.x < BQ) {
      const int row = qb * BQ + threadIdx.x;
      s_lse[buf][threadIdx.x] = row < p.nq ? lp[row] : 0.f;
      s_del[buf][threadIdx.x] = row < p.nq ? dlp[row] : 0.f;
    }
  };

  load_tile<HD>(sK, kp, p.ldk, k0, p.nk);
  load_tile<HD>(sV, vp, p.ldv, k0, p.nk);
  if (qb0 < nqb) { load_tile<HD>(sQ(0), qp, p.ldq, qb0 * BQ, p.nq); load_tile<HD>(sdO(0), dop, p.ldo, qb0 * BQ, p.nq); }
  cp_commit();
  if (qb0 < nqb) stage_rows(0, qb0);

  float dk[T::NT][4], dv[T::NT][4];
#pragma unroll
  for (int i = 0; i < T::NT; ++i) { dk[i][0] = dk[i][1] = dk[i][2] = dk[i][3] = 0.f; dv[i][0] = dv[i][1] = dv[i][2] = dv[i][3] = 0.f; }
  const int key_a = k0 + warp * 16 + g, key_b = key_a + 8;

  for (int qb = qb0; qb < nqb; ++qb) {
    const int buf = (qb - qb0) & 1;
    if (qb + 1 < nqb) {
      load_tile<HD>(sQ(buf ^ 1), qp, p.ldq, (qb + 1) * BQ, p.nq);
      load_tile<HD>(sdO(buf ^ 1), dop, p.ldo, (qb + 1) * BQ, p.nq);
      cp_commit();
      stage_rows(buf ^ 1, qb + 1);
      cp_wait<1>();
    } else {
      cp_wait<0>();
    }
    fence_proxy_async_smem();   // cp.async (generic proxy) -> wgmma reads
    __syncthreads();
    float st[8][4], dpt[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) { st[i][0] = st[i][1] = st[i][2] = st[i][3] = 0.f; dpt[i][0] = dpt[i][1] = dpt[i][2] = dpt[i][3] = 0.f; }
    mma_rows_x_tileT<HD>(st, sK, sQ(buf));     // S^T  = K Q^T   [16 keys x 64 queries]
    mma_rows_x_tileT<HD>(dpt, sV, sdO(buf));   // dP^T = V dO^T
    float dst[8][4];
    // fast path: the whole 64 x 64 (query, key) tile is in bounds and unmasked
    const bool fast = p.mask == nullptr && k0 + BKV <= p.nk && qb * BQ + BQ <= p.nq &&
                      (!p.causal || k0 + BKV - 1 <= qb * BQ + (p.nk - p.nq));
    if (fast) {
      const float ba = slope2 * (float)key_a, bb = slope2 * (float)key_b;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int qc = i * 8 + 2 * t + (e & 1);
          const float pv = ex2_approx(fmaf(st[i][e], sl2, (e & 2) ? bb : ba) - s_lse[buf][qc]);
          st[i][e] = pv;
          dst[i][e] = pv * (dpt[i][e] - s_del[buf][qc]) * p.scale;
        }
      }
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int qc = i * 8 + 2 * t + (e & 1);
          const int row = qb * BQ + qc;
          const int key = (e & 2) ? key_b : key_a;
          const bool inb = row < p.nq;
          const float sc = score(p, st[i][e], sl2, slope2, b, row, key);
          const float pv = inb ? ex2_approx(sc - s_lse[buf][qc]) : 0.f;
          const bool live = inb && key < p.nk && !is_masked(p, b, row, key);
          st[i][e] = pv;                                                   // P^T
          dst[i][e] = live ? pv * (dpt[i][e] - s_del[buf][qc]) * p.scale : 0.f;   // dS^T
        }
      }
    }
    uint32_t pa[4][4], dsa[4][4];
    c_to_a(st, pa);
    c_to_a(dst, dsa);
    mma_p_x_tile<HD>(dv, pa, sdO(buf));     // dV += P^T dO
    mma_p_x_tile<HD>(dk, dsa, sQ(buf));     // dK += dS^T Q
    __syncthreads();
  }
  if (qb0 >= nqb) cp_wait<0>();

  store_rows(p.dk + b * p.dk_bs + h * HD, p.lddk, dk, 1.f, 1.f, key_a, key_b, p.nk, t);
  store_rows(p.dv + b * p.dv_bs + h * HD, p.lddv, dv, 1.f, 1.f, key_a, key_b, p.nk, t);
}

// q/k/v/o/dO move 16 bytes at a time per row (32 bits in the delta kernel); dq/dk/dv are written 32 bits at a time;
// lse, delta, slopes and the flag are 4-byte scalars.  The causal rule key <= row + nk - nq leaves whole query blocks
// without a key when nq > nk, and the tile skipping would give those rows zeros instead of the finfo.min rule's uniform
// attention; no caller needs that case, so it is rejected.  Called before any CUDA call.
static int validate(const Params& p, int head_dim, bool bwd) {
  if (head_dim != 64 && head_dim != 128) return ofk_set_error(OFK_ERR_ARG, "dense attention: head_dim must be 64 or 128");
  if (p.batch <= 0 || p.heads <= 0 || p.nq <= 0 || p.nk <= 0) return ofk_set_error(OFK_ERR_ARG, "dense attention: empty problem");
  if (p.batch > 65535 || p.heads > 65535) return ofk_set_error(OFK_ERR_ARG, "dense attention: batch/heads exceed grid limits");
  if ((p.causal || p.pure_causal) && p.nq > p.nk)
    return ofk_set_error(OFK_ERR_ARG, "dense attention: the causal rule needs nq <= nk");
  const void* io = bwd ? static_cast<const void*>(p.o) : static_cast<const void*>(p.out);
  if (!aligned(p.q, 16) || !aligned(p.k, 16) || !aligned(p.v, 16) || !aligned(io, 16) || (bwd && !aligned(p.d_o, 16)))
    return ofk_set_error(OFK_ERR_ALIGN, "dense attention: q/k/v/o/dO must be 16-byte aligned");
  if ((p.q_bs | p.ldq | p.k_bs | p.ldk | p.v_bs | p.ldv | p.o_bs | p.ldo) % 8 != 0)
    return ofk_set_error(OFK_ERR_ALIGN, "dense attention: batch and row strides of q/k/v/o must be multiples of 8");
  if (!aligned(p.lse, 4) || !aligned(p.delta, 4) || !aligned(p.slopes, 4) || !aligned(p.pure_causal, 4))
    return ofk_set_error(OFK_ERR_ALIGN, "dense attention: lse/delta/slopes/pure_causal_flag must be 4-byte aligned");
  if (bwd) {
    if (!aligned(p.dq, 4) || !aligned(p.dk, 4) || !aligned(p.dv, 4))
      return ofk_set_error(OFK_ERR_ALIGN, "dense attention bwd: dq/dk/dv must be 4-byte aligned");
    if ((p.dq_bs | p.lddq | p.dk_bs | p.lddk | p.dv_bs | p.lddv) % 2 != 0)
      return ofk_set_error(OFK_ERR_ALIGN, "dense attention bwd: grad strides must be even");
  }
  return 0;
}

template <int HD>
static int launch_fwd(const Params& p, cudaStream_t s) {
  constexpr int SMEM = 5 * Tile<HD>::BYTES + 1024;
  static bool done = false;
  if (!done) { cudaFuncSetAttribute(fwd_kernel<HD>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM); done = true; }
  dim3 grid((p.nq + BQ - 1) / BQ, p.heads, p.batch);
  fwd_kernel<HD><<<grid, THREADS, SMEM, s>>>(p);
  OFK_CHECK_LAUNCH();
  return 0;
}
template <int HD>
static int launch_bwd(const Params& p, cudaStream_t s) {
  constexpr int SMEM = 6 * Tile<HD>::BYTES + 1024;
  static bool done = false;
  if (!done) {
    cudaFuncSetAttribute(bwd_dq_kernel<HD>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    cudaFuncSetAttribute(bwd_dkv_kernel<HD>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    done = true;
  }
  const long long rows = (long long)p.batch * p.heads * p.nq;
  delta_kernel<HD><<<(unsigned)((rows + 7) / 8), 256, 0, s>>>(p.o, p.d_o, p.delta, p.batch, p.heads, p.nq, p.o_bs, p.ldo);
  OFK_CHECK_LAUNCH();
  dim3 gq((p.nq + BQ - 1) / BQ, p.heads, p.batch);
  bwd_dq_kernel<HD><<<gq, THREADS, SMEM, s>>>(p);
  OFK_CHECK_LAUNCH();
  dim3 gk((p.nk + BKV - 1) / BKV, p.heads, p.batch);
  bwd_dkv_kernel<HD><<<gk, THREADS, SMEM, s>>>(p);
  OFK_CHECK_LAUNCH();
  return 0;
}
}  // namespace dense
}  // namespace ofk

extern "C" int ofk_attn_dense_fwd(const void* q, const void* k, const void* v, void* o, float* lse, int batch, int heads,
                                  int head_dim, int nq, int nk, long long q_bstride, long long ldq, long long k_bstride,
                                  long long ldk, long long v_bstride, long long ldv, long long o_bstride, long long ldo,
                                  float scale, int causal, const unsigned char* mask, const float* slopes,
                                  const int* pure_causal_flag, void* stream) {
  using namespace ofk::dense;
  Params p{};
  p.q = (const __nv_bfloat16*)q; p.k = (const __nv_bfloat16*)k; p.v = (const __nv_bfloat16*)v; p.out = (__nv_bfloat16*)o;
  p.lse = lse; p.mask = mask; p.slopes = slopes; p.pure_causal = pure_causal_flag; p.batch = batch; p.heads = heads; p.nq = nq; p.nk = nk; p.causal = causal;
  p.q_bs = q_bstride; p.ldq = ldq; p.k_bs = k_bstride; p.ldk = ldk; p.v_bs = v_bstride; p.ldv = ldv; p.o_bs = o_bstride; p.ldo = ldo;
  p.scale = scale;
  if (!q || !k || !v || !o) return ofk_set_error(OFK_ERR_ARG, "dense attention: null pointer");
  if (int rc = validate(p, head_dim, false)) return rc;
  return head_dim == 64 ? launch_fwd<64>(p, (cudaStream_t)stream) : launch_fwd<128>(p, (cudaStream_t)stream);
}

extern "C" int ofk_attn_dense_bwd(const void* q, const void* k, const void* v, const void* o, const void* d_o,
                                  const float* lse, float* delta, void* dq, void* dk, void* dv, int batch, int heads,
                                  int head_dim, int nq, int nk, long long q_bstride, long long ldq, long long k_bstride,
                                  long long ldk, long long v_bstride, long long ldv, long long o_bstride, long long ldo,
                                  long long dq_bstride, long long lddq, long long dk_bstride, long long lddk,
                                  long long dv_bstride, long long lddv, float scale, int causal, const unsigned char* mask,
                                  const float* slopes, const int* pure_causal_flag, void* stream) {
  using namespace ofk::dense;
  Params p{};
  p.q = (const __nv_bfloat16*)q; p.k = (const __nv_bfloat16*)k; p.v = (const __nv_bfloat16*)v; p.o = (const __nv_bfloat16*)o;
  p.d_o = (const __nv_bfloat16*)d_o; p.lse = const_cast<float*>(lse); p.delta = delta;
  p.dq = (__nv_bfloat16*)dq; p.dk = (__nv_bfloat16*)dk; p.dv = (__nv_bfloat16*)dv;
  p.mask = mask; p.slopes = slopes; p.pure_causal = pure_causal_flag; p.batch = batch; p.heads = heads; p.nq = nq; p.nk = nk; p.causal = causal;
  p.q_bs = q_bstride; p.ldq = ldq; p.k_bs = k_bstride; p.ldk = ldk; p.v_bs = v_bstride; p.ldv = ldv; p.o_bs = o_bstride; p.ldo = ldo;
  p.dq_bs = dq_bstride; p.lddq = lddq; p.dk_bs = dk_bstride; p.lddk = lddk; p.dv_bs = dv_bstride; p.lddv = lddv; p.scale = scale;
  if (!q || !k || !v || !o || !d_o || !lse || !delta || !dq || !dk || !dv) return ofk_set_error(OFK_ERR_ARG, "dense attention bwd: null pointer");
  if (int rc = validate(p, head_dim, true)) return rc;
  return head_dim == 64 ? launch_bwd<64>(p, (cudaStream_t)stream) : launch_bwd<128>(p, (cudaStream_t)stream);
}
