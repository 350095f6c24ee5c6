// Attention cores for the OpenFlamingo hot path, head_dim = 64, bf16 in/out, fp32 online softmax.
//
//   forward : O = softmax(scale * Q K^T + media_mask) V, LSE saved
//   backward: dK/dV kernel (parallel over key blocks) + dQ kernel (parallel over query blocks);
//             both recompute P from the saved LSE -- the [nq, nk] score matrix never touches HBM.
//
// Replaces (reference, open_flamingo/src/helpers.py):
//   PerceiverAttention core  :55-64   (q*scale, einsum QK^T, -amax, softmax, einsum PV, head merge)
//   MaskedCrossAttention core :190-232 (same + text_time/media_time mask :196-218, zero-row rule :223-229)
// and the ViT nn.MultiheadAttention core (open_clip, third party).  Head split/merge
// ("b n (h d) -> b h n d") is pure addressing here: heads are column slices of the [rows, h*64] buffers.
//
// Mask semantics (mask_mode 1 = torch.eq, 2 = torch.ge), keys grouped by media in blocks of kpm:
//   allowed(row, key) = text_time[row] (==|>=) key / kpm + 1
//   a row with no allowed key: mode 1 and text_time == 0 -> exact zeros (helpers.py:223-229);
//   otherwise the reference's masked_fill(-finfo.max) + softmax yields a UNIFORM row over all keys,
//   with no gradient to q/k (helpers.py:218-221) -- reproduced here ("uniform" rows).
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "attention_tile.cuh"
#include "ofk_internal.h"

namespace ofk {

constexpr int HD = 64;    // head dim

struct AttnParams {
  const __nv_bfloat16 *q, *k, *v, *o, *d_o;
  __nv_bfloat16 *out, *dq, *dk, *dv;
  float* lse;
  float* delta;
  const int* text_time;
  int batch, heads, nq, nk;
  long long q_bs, ldq, k_bs, ldk, v_bs, ldv, o_bs, ldo;
  long long dq_bs, lddq, dk_bs, lddk, dv_bs, lddv;
  float scale;
  int mask_mode, kpm;
};

// Row classification for the media mask.
//   kind 0: normal masked row; 1: zero row; 2: uniform row (all keys, S = 0, no grad to q/k); 3: unmasked
struct RowInfo { int tt; int kind; };
__device__ __forceinline__ RowInfo classify_row(const AttnParams& p, int b, int row) {
  RowInfo r; r.tt = 0; r.kind = 3;
  if (p.mask_mode == 0) return r;
  if (row >= p.nq) { r.kind = 1; return r; }
  const int tt = p.text_time[(long long)b * p.nq + row];
  const int n_media = p.nk / p.kpm;
  r.tt = tt;
  bool has = (p.mask_mode == 1) ? (tt >= 1 && tt <= n_media) : (tt >= 1);
  if (has) r.kind = 0;
  else if (p.mask_mode == 1 && tt == 0) r.kind = 1;
  else r.kind = 2;
  return r;
}
__device__ __forceinline__ bool key_allowed(const AttnParams& p, const RowInfo& r, int key) {
  if (r.kind == 3 || r.kind == 2) return true;
  if (r.kind == 1) return false;
  const int media = key / p.kpm + 1;
  return p.mask_mode == 1 ? (r.tt == media) : (r.tt >= media);
}
// Same predicate with the media index (key / kpm + 1) already known -- it is constant over an 8-key n-tile
// (kpm % 16 == 0), so the integer division is done once per n-tile, not once per score.
__device__ __forceinline__ bool media_allowed(const AttnParams& p, const RowInfo& r, int media) {
  if (r.kind >= 2) return true;
  if (r.kind == 1) return false;
  return p.mask_mode == 1 ? (r.tt == media) : (r.tt >= media);
}

// Key range [lo, hi) (in keys) a 64-row query block needs; computed cooperatively by the CTA.
__device__ __forceinline__ void block_key_range(const AttnParams& p, int b, int q0, int* s_red, int& lo, int& hi) {
  if (p.mask_mode == 0) { lo = 0; hi = p.nk; return; }
  int tmin = 1 << 30, tmax = -1; int any_uniform = 0;
  if (threadIdx.x < BQ) {
    RowInfo r = classify_row(p, b, q0 + threadIdx.x);
    if (r.kind == 0) { tmin = r.tt; tmax = r.tt; }
    if (r.kind == 2) any_uniform = 1;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    tmin = min(tmin, __shfl_xor_sync(0xffffffffu, tmin, o));
    tmax = max(tmax, __shfl_xor_sync(0xffffffffu, tmax, o));
    any_uniform |= __shfl_xor_sync(0xffffffffu, any_uniform, o);
  }
  if ((threadIdx.x & 31) == 0) {
    s_red[(threadIdx.x >> 5) * 3 + 0] = tmin; s_red[(threadIdx.x >> 5) * 3 + 1] = tmax;
    s_red[(threadIdx.x >> 5) * 3 + 2] = any_uniform;
  }
  __syncthreads();
  tmin = min(min(s_red[0], s_red[3]), min(s_red[6], s_red[9]));
  tmax = max(max(s_red[1], s_red[4]), max(s_red[7], s_red[10]));
  any_uniform = s_red[2] | s_red[5] | s_red[8] | s_red[11];
  __syncthreads();
  if (any_uniform) { lo = 0; hi = p.nk; return; }
  if (tmax < 0) { lo = 0; hi = 0; return; }
  lo = (p.mask_mode == 1) ? (tmin - 1) * p.kpm : 0;
  hi = min(p.nk, tmax * p.kpm);
  lo = (lo / BKV) * BKV;
}

// ================================================================ forward
using T = Tile<HD>;
constexpr int FWD_SMEM = 5 * T::BYTES + 1024;
__global__ void __launch_bounds__(THREADS) attn_fwd_kernel(const AttnParams p) {
  uint8_t* sQ = tile_at<HD>(0);
  auto sK = [](int buf) { return tile_at<HD>(1 + buf); };
  auto sV = [](int buf) { return tile_at<HD>(3 + buf); };
  __shared__ int s_red[12];

  const int q0 = blockIdx.x * BQ, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const __nv_bfloat16* qp = p.q + b * p.q_bs + h * HD;
  const __nv_bfloat16* kp = p.k + b * p.k_bs + h * HD;
  const __nv_bfloat16* vp = p.v + b * p.v_bs + h * HD;

  int klo, khi;
  block_key_range(p, b, q0, s_red, klo, khi);
  const int nblk = (khi - klo + BKV - 1) / BKV;

  load_tile<HD>(sQ, qp, p.ldq, q0, p.nq);
  if (nblk > 0) { load_tile<HD>(sK(0), kp, p.ldk, klo, p.nk); load_tile<HD>(sV(0), vp, p.ldv, klo, p.nk); }
  cp_commit();

  const int row_a = q0 + warp * 16 + g, row_b = row_a + 8;
  const RowInfo ra = classify_row(p, b, row_a), rb = classify_row(p, b, row_b);

  float o[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
  float m_a = -INFINITY, m_b = -INFINITY, l_a = 0.f, l_b = 0.f;
  const float sl2 = p.scale * LOG2E;

  for (int j = 0; j < nblk; ++j) {
    const int buf = j & 1;
    if (j + 1 < nblk) {
      load_tile<HD>(sK(buf ^ 1), kp, p.ldk, klo + (j + 1) * BKV, p.nk);
      load_tile<HD>(sV(buf ^ 1), vp, p.ldv, klo + (j + 1) * BKV, p.nk);
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

    // mask + scale (log2 domain)
    const int key0 = klo + j * BKV;
    float mx_a = -INFINITY, mx_b = -INFINITY;
    if (p.mask_mode == 0 && key0 + BKV <= p.nk) {
      // fast path (Perceiver / ViT interior tiles): no predicate at all
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        s[i][0] *= sl2; s[i][1] *= sl2; s[i][2] *= sl2; s[i][3] *= sl2;
        mx_a = fmaxf(mx_a, fmaxf(s[i][0], s[i][1]));
        mx_b = fmaxf(mx_b, fmaxf(s[i][2], s[i][3]));
      }
    } else {
      const bool one_media = p.mask_mode != 0 && (p.kpm % BKV) == 0;      // all 64 keys of the tile share a media
      int media = p.mask_mode != 0 ? key0 / p.kpm + 1 : 0;
      bool aa = media_allowed(p, ra, media), ab = media_allowed(p, rb, media);
      const float za = ra.kind == 2 ? 0.f : sl2, zb = rb.kind == 2 ? 0.f : sl2;  // uniform rows: S = 0
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int key = key0 + i * 8 + 2 * t;
        if (p.mask_mode != 0 && !one_media) {
          media = (key0 + i * 8) / p.kpm + 1;
          aa = media_allowed(p, ra, media); ab = media_allowed(p, rb, media);
        }
        const bool inb0 = key < p.nk, inb1 = (key + 1) < p.nk;
        s[i][0] = (inb0 && aa) ? s[i][0] * za : -INFINITY;
        s[i][1] = (inb1 && aa) ? s[i][1] * za : -INFINITY;
        s[i][2] = (inb0 && ab) ? s[i][2] * zb : -INFINITY;
        s[i][3] = (inb1 && ab) ? s[i][3] * zb : -INFINITY;
        mx_a = fmaxf(mx_a, fmaxf(s[i][0], s[i][1]));
        mx_b = fmaxf(mx_b, fmaxf(s[i][2], s[i][3]));
      }
    }
    softmax_step(s, mx_a, mx_b, m_a, m_b, l_a, l_b, o);
    uint32_t pa[4][4];
    c_to_a(s, pa);
    mma_p_x_tile<HD>(o, pa, sV(buf));
    __syncthreads();
  }
  if (nblk == 0) { cp_wait<0>(); }

  l_a = quad_sum(l_a); l_b = quad_sum(l_b);
  const float inv_a = l_a > 0.f ? 1.f / l_a : 0.f, inv_b = l_b > 0.f ? 1.f / l_b : 0.f;
  store_rows(p.out + b * p.o_bs + h * HD, p.ldo, o, inv_a, inv_b, row_a, row_b, p.nq, t);
  if (p.lse != nullptr && t == 0) store_lse(p.lse + ((long long)b * p.heads + h) * p.nq, m_a, l_a, m_b, l_b, row_a, row_b, p.nq);
}

// Recompute P (C layout, rows = queries) for one 16x64 tile given raw S = Q K^T.
__device__ __forceinline__ void recompute_p(const AttnParams& p, float (&s)[8][4], const RowInfo& ra, const RowInfo& rb,
                                            float lse_a, float lse_b, int key0, int t) {
  // exp(scale*s - lse) == exp2(scale*log2e*s - lse*log2e)
  const float sl2 = p.scale * LOG2E;
  const float za = ra.kind == 2 ? 0.f : sl2, zb = rb.kind == 2 ? 0.f : sl2;
  const float la = lse_a, lb = lse_b;   // LSE is stored in the log2 domain
  if (p.mask_mode == 0 && key0 + BKV <= p.nk) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      s[i][0] = ex2_approx(fmaf(s[i][0], sl2, -la)); s[i][1] = ex2_approx(fmaf(s[i][1], sl2, -la));
      s[i][2] = ex2_approx(fmaf(s[i][2], sl2, -lb)); s[i][3] = ex2_approx(fmaf(s[i][3], sl2, -lb));
    }
    return;
  }
  const bool one_media = p.mask_mode != 0 && (p.kpm % BKV) == 0;
  int media = p.mask_mode != 0 ? key0 / p.kpm + 1 : 0;
  bool aa = media_allowed(p, ra, media), ab = media_allowed(p, rb, media);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int key = key0 + i * 8 + 2 * t;
    if (p.mask_mode != 0 && !one_media) {
      media = (key0 + i * 8) / p.kpm + 1;
      aa = media_allowed(p, ra, media); ab = media_allowed(p, rb, media);
    }
    const bool inb0 = key < p.nk, inb1 = (key + 1) < p.nk;
    s[i][0] = (inb0 && aa) ? ex2_approx(fmaf(s[i][0], za, -la)) : 0.f;
    s[i][1] = (inb1 && aa) ? ex2_approx(fmaf(s[i][1], za, -la)) : 0.f;
    s[i][2] = (inb0 && ab) ? ex2_approx(fmaf(s[i][2], zb, -lb)) : 0.f;
    s[i][3] = (inb1 && ab) ? ex2_approx(fmaf(s[i][3], zb, -lb)) : 0.f;
  }
}

// ================================================================ backward: dQ  (CTA = 64 queries, loop over key tiles)
constexpr int BWD_SMEM = 6 * T::BYTES + 1024;

__global__ void __launch_bounds__(THREADS) attn_bwd_dq_kernel(const AttnParams p) {
  uint8_t* sQ = tile_at<HD>(0);
  uint8_t* sdO = tile_at<HD>(1);
  auto sK = [](int buf) { return tile_at<HD>(2 + buf); };
  auto sV = [](int buf) { return tile_at<HD>(4 + buf); };
  __shared__ int s_red[12];

  const int q0 = blockIdx.x * BQ, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const __nv_bfloat16* qp = p.q + b * p.q_bs + h * HD;
  const __nv_bfloat16* kp = p.k + b * p.k_bs + h * HD;
  const __nv_bfloat16* vp = p.v + b * p.v_bs + h * HD;
  const __nv_bfloat16* dop = p.d_o + b * p.o_bs + h * HD;

  int klo, khi;
  block_key_range(p, b, q0, s_red, klo, khi);
  const int nblk = (khi - klo + BKV - 1) / BKV;

  load_tile<HD>(sQ, qp, p.ldq, q0, p.nq);
  load_tile<HD>(sdO, dop, p.ldo, q0, p.nq);
  if (nblk > 0) { load_tile<HD>(sK(0), kp, p.ldk, klo, p.nk); load_tile<HD>(sV(0), vp, p.ldv, klo, p.nk); }
  cp_commit();

  const int row_a = q0 + warp * 16 + g, row_b = row_a + 8;
  const RowInfo ra = classify_row(p, b, row_a), rb = classify_row(p, b, row_b);
  const float* lp = p.lse + ((long long)b * p.heads + h) * p.nq;
  const float* dp = p.delta + ((long long)b * p.heads + h) * p.nq;
  const float lse_a = row_a < p.nq ? lp[row_a] : 0.f, lse_b = row_b < p.nq ? lp[row_b] : 0.f;
  const float del_a = row_a < p.nq ? dp[row_a] : 0.f, del_b = row_b < p.nq ? dp[row_b] : 0.f;

  float dq[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i) { dq[i][0] = dq[i][1] = dq[i][2] = dq[i][3] = 0.f; }

  for (int j = 0; j < nblk; ++j) {
    const int buf = j & 1;
    if (j + 1 < nblk) {
      load_tile<HD>(sK(buf ^ 1), kp, p.ldk, klo + (j + 1) * BKV, p.nk);
      load_tile<HD>(sV(buf ^ 1), vp, p.ldv, klo + (j + 1) * BKV, p.nk);
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
    mma_rows_x_tileT<HD>(s, sQ, sK(buf));      // S  = Q K^T
    mma_rows_x_tileT<HD>(dpv, sdO, sV(buf));   // dP = dO V^T
    recompute_p(p, s, ra, rb, lse_a, lse_b, klo + j * BKV, t);
    const float ga = ra.kind == 2 ? 0.f : p.scale, gb = rb.kind == 2 ? 0.f : p.scale;
#pragma unroll
    for (int i = 0; i < 8; ++i) {     // dS = P * (dP - delta) * scale
      s[i][0] = s[i][0] * (dpv[i][0] - del_a) * ga; s[i][1] = s[i][1] * (dpv[i][1] - del_a) * ga;
      s[i][2] = s[i][2] * (dpv[i][2] - del_b) * gb; s[i][3] = s[i][3] * (dpv[i][3] - del_b) * gb;
    }
    uint32_t dsa[4][4];
    c_to_a(s, dsa);
    mma_p_x_tile<HD>(dq, dsa, sK(buf));     // dQ += dS K
    __syncthreads();
  }
  if (nblk == 0) { cp_wait<0>(); }

  store_rows(p.dq + b * p.dq_bs + h * HD, p.lddq, dq, 1.f, 1.f, row_a, row_b, p.nq, t);
}

// ================================================================ backward: dK, dV (CTA = 64 keys, loop over query tiles)
// Works on transposed tiles: S^T = K Q^T (rows = keys), so P^T / dS^T are directly the A operands of
// dV += P^T dO and dK += dS^T Q.
__global__ void __launch_bounds__(THREADS) attn_bwd_dkv_kernel(const AttnParams p) {
  uint8_t* sK = tile_at<HD>(0);
  uint8_t* sV = tile_at<HD>(1);
  auto sQ = [](int buf) { return tile_at<HD>(2 + buf); };
  auto sdO = [](int buf) { return tile_at<HD>(4 + buf); };
  __shared__ float s_lse[2][BQ], s_del[2][BQ];
  __shared__ int s_tt[2][BQ], s_kind[2][BQ];

  const int k0 = blockIdx.x * BKV, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const __nv_bfloat16* qp = p.q + b * p.q_bs + h * HD;
  const __nv_bfloat16* kp = p.k + b * p.k_bs + h * HD;
  const __nv_bfloat16* vp = p.v + b * p.v_bs + h * HD;
  const __nv_bfloat16* dop = p.d_o + b * p.o_bs + h * HD;
  const float* lp = p.lse + ((long long)b * p.heads + h) * p.nq;
  const float* dlp = p.delta + ((long long)b * p.heads + h) * p.nq;
  const int nqb = (p.nq + BQ - 1) / BQ;

  auto stage_rows = [&](int buf, int qb) {
    if (threadIdx.x < BQ) {
      const int row = qb * BQ + threadIdx.x;
      RowInfo r = classify_row(p, b, row);
      s_tt[buf][threadIdx.x] = r.tt; s_kind[buf][threadIdx.x] = (row < p.nq) ? r.kind : 1;
      s_lse[buf][threadIdx.x] = row < p.nq ? lp[row] : 0.f;
      s_del[buf][threadIdx.x] = row < p.nq ? dlp[row] : 0.f;
    }
  };

  load_tile<HD>(sK, kp, p.ldk, k0, p.nk);
  load_tile<HD>(sV, vp, p.ldv, k0, p.nk);
  load_tile<HD>(sQ(0), qp, p.ldq, 0, p.nq);
  load_tile<HD>(sdO(0), dop, p.ldo, 0, p.nq);
  cp_commit();
  stage_rows(0, 0);

  float dk[8][4], dv[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i) { dk[i][0] = dk[i][1] = dk[i][2] = dk[i][3] = 0.f; dv[i][0] = dv[i][1] = dv[i][2] = dv[i][3] = 0.f; }
  const int key_a = k0 + warp * 16 + g, key_b = key_a + 8;
  const bool inb_ka = key_a < p.nk, inb_kb = key_b < p.nk;
  const int media_ka = p.mask_mode != 0 ? key_a / p.kpm + 1 : 0, media_kb = p.mask_mode != 0 ? key_b / p.kpm + 1 : 0;
  const float sl2 = p.scale * LOG2E;

  for (int qb = 0; qb < nqb; ++qb) {
    const int buf = qb & 1;
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
    {
      // skip (query block, key block) pairs the media mask rules out entirely
      int need = 0;
      if (threadIdx.x < BQ) {
        const int kind = s_kind[buf][threadIdx.x], tt = s_tt[buf][threadIdx.x];
        if (kind >= 2) need = 1;
        else if (kind == 0) {
          const int m_lo = k0 / p.kpm + 1, m_hi = min(p.nk - 1, k0 + BKV - 1) / p.kpm + 1;
          need = (p.mask_mode == 1) ? (tt >= m_lo && tt <= m_hi) : (tt >= m_lo);
        }
      }
      if (!__syncthreads_or(need)) continue;
    }

    float st[8][4], dpt[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) { st[i][0] = st[i][1] = st[i][2] = st[i][3] = 0.f; dpt[i][0] = dpt[i][1] = dpt[i][2] = dpt[i][3] = 0.f; }
    mma_rows_x_tileT<HD>(st, sK, sQ(buf));     // S^T  = K Q^T   [16 keys x 64 queries]
    mma_rows_x_tileT<HD>(dpt, sV, sdO(buf));   // dP^T = V dO^T
    float dst[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int qc = i * 8 + 2 * t + (e & 1);      // query column in this tile
        RowInfo r; r.tt = s_tt[buf][qc]; r.kind = s_kind[buf][qc];
        const bool ok = ((e & 2) ? inb_kb : inb_ka) && media_allowed(p, r, (e & 2) ? media_kb : media_ka);
        const float z = r.kind == 2 ? 0.f : sl2;
        const float pv = ok ? ex2_approx(fmaf(st[i][e], z, -s_lse[buf][qc])) : 0.f;
        st[i][e] = pv;                                                                      // P^T
        dst[i][e] = pv * (dpt[i][e] - s_del[buf][qc]) * (r.kind == 2 ? 0.f : p.scale);     // dS^T
      }
    }
    uint32_t pa[4][4], dsa[4][4];
    c_to_a(st, pa);
    c_to_a(dst, dsa);
    mma_p_x_tile<HD>(dv, pa, sdO(buf));     // dV += P^T dO
    mma_p_x_tile<HD>(dk, dsa, sQ(buf));     // dK += dS^T Q
    __syncthreads();
  }

  store_rows(p.dk + b * p.dk_bs + h * HD, p.lddk, dk, 1.f, 1.f, key_a, key_b, p.nk, t);
  store_rows(p.dv + b * p.dv_bs + h * HD, p.lddv, dv, 1.f, 1.f, key_a, key_b, p.nk, t);
}

// q/k/v/o/dO are read (and o written) 16 bytes at a time per row and 32 bits at a time by the delta kernel; dq/dk/dv
// are written 32 bits at a time; lse/delta/text_time are f32/int32 arrays.  Called before any CUDA call.
static int check_common(const AttnParams& p, bool bwd) {
  if (p.batch <= 0 || p.heads <= 0 || p.nq <= 0 || p.nk <= 0) return ofk_set_error(OFK_ERR_ARG, "attention: empty problem");
  if (p.mask_mode < 0 || p.mask_mode > 2) return ofk_set_error(OFK_ERR_ARG, "attention: bad mask_mode");
  if (p.mask_mode != 0) {
    if (!p.text_time) return ofk_set_error(OFK_ERR_ARG, "attention: media mask needs text_time");
    if (p.kpm <= 0 || p.kpm % 16 != 0 || p.nk % p.kpm != 0)
      return ofk_set_error(OFK_ERR_ARG, "attention: keys_per_media must be a multiple of 16 dividing nk");
  }
  if (p.batch > 65535 || p.heads > 65535) return ofk_set_error(OFK_ERR_ARG, "attention: batch/heads exceed grid limits");
  const void* io = bwd ? static_cast<const void*>(p.o) : static_cast<const void*>(p.out);
  if (!aligned(p.q, 16) || !aligned(p.k, 16) || !aligned(p.v, 16) || !aligned(io, 16) || (bwd && !aligned(p.d_o, 16)))
    return ofk_set_error(OFK_ERR_ALIGN, "attention: q/k/v/o/dO must be 16-byte aligned");
  if ((p.q_bs | p.ldq | p.k_bs | p.ldk | p.v_bs | p.ldv | p.o_bs | p.ldo) % 8 != 0)
    return ofk_set_error(OFK_ERR_ALIGN, "attention: batch and row strides of q/k/v/o must be multiples of 8");
  if (!aligned(p.lse, 4) || !aligned(p.delta, 4) || !aligned(p.text_time, 4))
    return ofk_set_error(OFK_ERR_ALIGN, "attention: lse/delta/text_time must be 4-byte aligned");
  if (bwd) {
    if (!aligned(p.dq, 4) || !aligned(p.dk, 4) || !aligned(p.dv, 4))
      return ofk_set_error(OFK_ERR_ALIGN, "attention bwd: dq/dk/dv must be 4-byte aligned");
    if ((p.dq_bs | p.lddq | p.dk_bs | p.lddk | p.dv_bs | p.lddv) % 2 != 0)
      return ofk_set_error(OFK_ERR_ALIGN, "attention bwd: grad strides must be even");
  }
  return 0;
}

}  // namespace ofk

extern "C" int ofk_attn_fwd(const void* q, const void* k, const void* v, void* o, float* lse, int batch, int heads,
                            int nq, int nk, long long q_bstride, long long ldq, long long k_bstride, long long ldk,
                            long long v_bstride, long long ldv, long long o_bstride, long long ldo, float scale,
                            int mask_mode, const int* text_time, int keys_per_media, void* stream_) {
  using namespace ofk;
  AttnParams p{};
  p.q = (const __nv_bfloat16*)q; p.k = (const __nv_bfloat16*)k; p.v = (const __nv_bfloat16*)v;
  p.out = (__nv_bfloat16*)o; p.lse = lse; p.text_time = text_time;
  p.batch = batch; p.heads = heads; p.nq = nq; p.nk = nk;
  p.q_bs = q_bstride; p.ldq = ldq; p.k_bs = k_bstride; p.ldk = ldk; p.v_bs = v_bstride; p.ldv = ldv;
  p.o_bs = o_bstride; p.ldo = ldo; p.scale = scale; p.mask_mode = mask_mode; p.kpm = keys_per_media;
  if (!q || !k || !v || !o) return ofk_set_error(OFK_ERR_ARG, "attention: null pointer");
  if (int rc = check_common(p, false)) return rc;
  dim3 grid((nq + BQ - 1) / BQ, heads, batch);
  attn_fwd_kernel<<<grid, THREADS, FWD_SMEM, (cudaStream_t)stream_>>>(p);
  OFK_CHECK_LAUNCH();
  return 0;
}

extern "C" int ofk_attn_bwd(const void* q, const void* k, const void* v, const void* o, const void* d_o,
                            const float* lse, float* delta, void* dq, void* dk, void* dv, int batch, int heads, int nq,
                            int nk, long long q_bstride, long long ldq, long long k_bstride, long long ldk,
                            long long v_bstride, long long ldv, long long o_bstride, long long ldo,
                            long long dq_bstride, long long lddq, long long dk_bstride, long long lddk,
                            long long dv_bstride, long long lddv, float scale, int mask_mode, const int* text_time,
                            int keys_per_media, void* stream_) {
  using namespace ofk;
  AttnParams p{};
  p.q = (const __nv_bfloat16*)q; p.k = (const __nv_bfloat16*)k; p.v = (const __nv_bfloat16*)v;
  p.o = (const __nv_bfloat16*)o; p.d_o = (const __nv_bfloat16*)d_o; p.lse = const_cast<float*>(lse); p.delta = delta;
  p.dq = (__nv_bfloat16*)dq; p.dk = (__nv_bfloat16*)dk; p.dv = (__nv_bfloat16*)dv; p.text_time = text_time;
  p.batch = batch; p.heads = heads; p.nq = nq; p.nk = nk;
  p.q_bs = q_bstride; p.ldq = ldq; p.k_bs = k_bstride; p.ldk = ldk; p.v_bs = v_bstride; p.ldv = ldv;
  p.o_bs = o_bstride; p.ldo = ldo; p.dq_bs = dq_bstride; p.lddq = lddq; p.dk_bs = dk_bstride; p.lddk = lddk;
  p.dv_bs = dv_bstride; p.lddv = lddv; p.scale = scale; p.mask_mode = mask_mode; p.kpm = keys_per_media;
  if (!q || !k || !v || !o || !d_o || !lse || !delta || !dq || !dk || !dv)
    return ofk_set_error(OFK_ERR_ARG, "attention bwd: null pointer");
  if (int rc = check_common(p, true)) return rc;
  cudaStream_t stream = (cudaStream_t)stream_;
  const long long rows = (long long)batch * heads * nq;
  delta_kernel<HD><<<(unsigned)((rows + 7) / 8), 256, 0, stream>>>(p.o, p.d_o, p.delta, batch, heads, nq, p.o_bs, p.ldo);
  OFK_CHECK_LAUNCH();
  dim3 gq((nq + BQ - 1) / BQ, heads, batch);
  static bool attr_done = false;
  if (!attr_done) {
    cudaFuncSetAttribute(attn_bwd_dq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, BWD_SMEM);
    cudaFuncSetAttribute(attn_bwd_dkv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, BWD_SMEM);
    attr_done = true;
  }
  dim3 gk((nk + BKV - 1) / BKV, heads, batch);
  attn_bwd_dq_kernel<<<gq, THREADS, BWD_SMEM, stream>>>(p);
  OFK_CHECK_LAUNCH();
  attn_bwd_dkv_kernel<<<gk, THREADS, BWD_SMEM, stream>>>(p);
  OFK_CHECK_LAUNCH();
  return 0;
}
