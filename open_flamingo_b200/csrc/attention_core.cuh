// The training attention kernels, each written once over a rule set R: attention.cu instantiates them with MediaRules
// (head_dim 64) and attention_dense.cu with DenseRules<64> and DenseRules<128>.  The kernels own the grid indexing, the
// shared-memory tile layout, the cp.async double-buffered pipeline with its fences and barriers, both wgmma products
// of every step, the lse/delta staging and the epilogues.  R says which (query, key) pairs a family scores and how:
//
//   R::HD, R::Params                      head dim; the family's AttnProblem plus its mask arguments
//   R::prepare(p)                         the launch's parameters as the kernel applies them
//   R::key_tiles(p, b, q0, klo, nblk)     key tiles [klo, klo + 64 nblk) query block q0 reads (may use a CTA barrier)
//   R::first_qblock(p, k0)                first query block that can see key block k0 (dK/dV kernel)
//   R(p, b, h)                            per-CTA constants (scale, ALiBi slope)
//   query_rows(rows) / key_rows(keys)     per-thread state of its two query rows / two key rows
//   fwd_scores(s, key0, rows, rs, mx)     raw S -> log2-domain scores and this thread's partial row maxima
//   P_TERMS, pack_p(s, pa)                P as P_TERMS bf16 A-fragment sets, summed by P_TERMS PV products
//   dq_scores(s, dp, key0, ...)           raw S and dP -> dS in place (dQ kernel)
//   stage_row(buf, row)                   extra per-query-row state staged beside lse/delta (dK/dV kernel)
//   qblock_needed(buf, k0)                whether a staged query block has any pair with key block k0
//   dkv_scores(st, dpt, dst, ...)         raw S^T and dP^T -> P^T and dS^T (dK/dV kernel)
// A hook that is constant for a family (dense: every query block is needed) compiles to nothing.
#pragma once
#include <string>

#include "attention_tile.cuh"
#include "ofk_internal.h"

namespace ofk {

// What every training attention entry point takes besides its mask arguments.
struct AttnProblem {
  const __nv_bfloat16 *q, *k, *v, *o, *d_o;
  __nv_bfloat16 *out, *dq, *dk, *dv;
  float* lse;
  float* delta;
  int batch, heads, nq, nk;
  long long q_bs, ldq, k_bs, ldk, v_bs, ldv, o_bs, ldo, dq_bs, lddq, dk_bs, lddk, dv_bs, lddv;
  float scale;
};

inline AttnProblem fwd_problem(const void* q, const void* k, const void* v, void* o, float* lse, int batch, int heads,
                               int nq, int nk, long long q_bs, long long ldq, long long k_bs, long long ldk,
                               long long v_bs, long long ldv, long long o_bs, long long ldo, float scale) {
  AttnProblem a{};
  a.q = (const __nv_bfloat16*)q; a.k = (const __nv_bfloat16*)k; a.v = (const __nv_bfloat16*)v;
  a.out = (__nv_bfloat16*)o; a.lse = lse;
  a.batch = batch; a.heads = heads; a.nq = nq; a.nk = nk;
  a.q_bs = q_bs; a.ldq = ldq; a.k_bs = k_bs; a.ldk = ldk; a.v_bs = v_bs; a.ldv = ldv; a.o_bs = o_bs; a.ldo = ldo;
  a.scale = scale;
  return a;
}

inline AttnProblem bwd_problem(const void* q, const void* k, const void* v, const void* o, const void* d_o,
                               const float* lse, float* delta, void* dq, void* dk, void* dv, int batch, int heads,
                               int nq, int nk, long long q_bs, long long ldq, long long k_bs, long long ldk,
                               long long v_bs, long long ldv, long long o_bs, long long ldo, long long dq_bs,
                               long long lddq, long long dk_bs, long long lddk, long long dv_bs, long long lddv,
                               float scale) {
  AttnProblem a = fwd_problem(q, k, v, nullptr, const_cast<float*>(lse), batch, heads, nq, nk, q_bs, ldq, k_bs, ldk,
                              v_bs, ldv, o_bs, ldo, scale);
  a.o = (const __nv_bfloat16*)o; a.d_o = (const __nv_bfloat16*)d_o; a.delta = delta;
  a.dq = (__nv_bfloat16*)dq; a.dk = (__nv_bfloat16*)dk; a.dv = (__nv_bfloat16*)dv;
  a.dq_bs = dq_bs; a.lddq = lddq; a.dk_bs = dk_bs; a.lddk = lddk; a.dv_bs = dv_bs; a.lddv = lddv;
  return a;
}

// This thread's two accumulator rows a = first + g and b = a + 8 (queries, or keys in the dK/dV kernel) of the warp's
// 16 starting at `first`, and its lane t within the quad sharing a row.
struct RowPair { int first, a, b, t; };

// ================================================================ forward (CTA = 64 queries, loop over key tiles)
template <class R>
__global__ void __launch_bounds__(THREADS) attn_fwd_kernel(const typename R::Params p_in) {
  constexpr int HD = R::HD;
  using T = Tile<HD>;
  uint8_t* sQ = tile_at<HD>(0);
  auto sK = [](int buf) { return tile_at<HD>(1 + buf); };
  auto sV = [](int buf) { return tile_at<HD>(3 + buf); };

  const int q0 = blockIdx.x * BQ, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const typename R::Params p = R::prepare(p_in);
  const __nv_bfloat16* qp = p.q + b * p.q_bs + h * HD;
  const __nv_bfloat16* kp = p.k + b * p.k_bs + h * HD;
  const __nv_bfloat16* vp = p.v + b * p.v_bs + h * HD;

  int klo, nblk;
  R::key_tiles(p, b, q0, klo, nblk);

  load_tile<HD>(sQ, qp, p.ldq, q0, p.nq);
  if (nblk > 0) { load_tile<HD>(sK(0), kp, p.ldk, klo, p.nk); load_tile<HD>(sV(0), vp, p.ldv, klo, p.nk); }
  cp_commit();

  const R r(p, b, h);
  const RowPair rows{q0 + warp * 16, q0 + warp * 16 + g, q0 + warp * 16 + g + 8, t};
  const typename R::Rows rs = r.query_rows(rows);

  float o[T::NT][4];
#pragma unroll
  for (int i = 0; i < T::NT; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
  float m_a = -INFINITY, m_b = -INFINITY, l_a = 0.f, l_b = 0.f;

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
    float mx_a = -INFINITY, mx_b = -INFINITY;
    r.fwd_scores(s, klo + j * BKV, rows, rs, mx_a, mx_b);
    softmax_step(s, mx_a, mx_b, m_a, m_b, l_a, l_b, o);
    uint32_t pa[R::P_TERMS][4][4];
    R::pack_p(s, pa);
#pragma unroll
    for (int i = 0; i < R::P_TERMS; ++i) mma_p_x_tile<HD>(o, pa[i], sV(buf));
    __syncthreads();
  }
  if (nblk == 0) cp_wait<0>();

  l_a = quad_sum(l_a); l_b = quad_sum(l_b);
  const float inv_a = l_a > 0.f ? 1.f / l_a : 0.f, inv_b = l_b > 0.f ? 1.f / l_b : 0.f;
  store_rows(p.out + b * p.o_bs + h * HD, p.ldo, o, inv_a, inv_b, rows.a, rows.b, p.nq, t);
  if (p.lse != nullptr && t == 0)
    store_lse(p.lse + ((long long)b * p.heads + h) * p.nq, m_a, l_a, m_b, l_b, rows.a, rows.b, p.nq);
}

// ================================================================ backward: dQ (CTA = 64 queries, loop over key tiles)
template <class R>
__global__ void __launch_bounds__(THREADS) attn_bwd_dq_kernel(const typename R::Params p_in) {
  constexpr int HD = R::HD;
  using T = Tile<HD>;
  uint8_t* sQ = tile_at<HD>(0);
  uint8_t* sdO = tile_at<HD>(1);
  auto sK = [](int buf) { return tile_at<HD>(2 + buf); };
  auto sV = [](int buf) { return tile_at<HD>(4 + buf); };

  const int q0 = blockIdx.x * BQ, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const typename R::Params p = R::prepare(p_in);
  const __nv_bfloat16* qp = p.q + b * p.q_bs + h * HD;
  const __nv_bfloat16* kp = p.k + b * p.k_bs + h * HD;
  const __nv_bfloat16* vp = p.v + b * p.v_bs + h * HD;
  const __nv_bfloat16* dop = p.d_o + b * p.o_bs + h * HD;

  int klo, nblk;
  R::key_tiles(p, b, q0, klo, nblk);

  load_tile<HD>(sQ, qp, p.ldq, q0, p.nq);
  load_tile<HD>(sdO, dop, p.ldo, q0, p.nq);
  if (nblk > 0) { load_tile<HD>(sK(0), kp, p.ldk, klo, p.nk); load_tile<HD>(sV(0), vp, p.ldv, klo, p.nk); }
  cp_commit();

  const R r(p, b, h);
  const RowPair rows{q0 + warp * 16, q0 + warp * 16 + g, q0 + warp * 16 + g + 8, t};
  const typename R::Rows rs = r.query_rows(rows);
  const float* lp = p.lse + ((long long)b * p.heads + h) * p.nq;
  const float* dp = p.delta + ((long long)b * p.heads + h) * p.nq;
  const float lse_a = rows.a < p.nq ? lp[rows.a] : 0.f, lse_b = rows.b < p.nq ? lp[rows.b] : 0.f;
  const float del_a = rows.a < p.nq ? dp[rows.a] : 0.f, del_b = rows.b < p.nq ? dp[rows.b] : 0.f;

  float dq[T::NT][4];
#pragma unroll
  for (int i = 0; i < T::NT; ++i) { dq[i][0] = dq[i][1] = dq[i][2] = dq[i][3] = 0.f; }

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
    r.dq_scores(s, dpv, klo + j * BKV, rows, rs, lse_a, lse_b, del_a, del_b);
    uint32_t dsa[4][4];
    c_to_a(s, dsa);
    mma_p_x_tile<HD>(dq, dsa, sK(buf));        // dQ += dS K
    __syncthreads();
  }
  if (nblk == 0) cp_wait<0>();

  store_rows(p.dq + b * p.dq_bs + h * HD, p.lddq, dq, 1.f, 1.f, rows.a, rows.b, p.nq, t);
}

// ================================================================ backward: dK, dV (CTA = 64 keys, loop over query tiles)
// Works on transposed tiles: S^T = K Q^T (rows = keys), so P^T / dS^T are directly the A operands of
// dV += P^T dO and dK += dS^T Q.
template <class R>
__global__ void __launch_bounds__(THREADS) attn_bwd_dkv_kernel(const typename R::Params p_in) {
  constexpr int HD = R::HD;
  using T = Tile<HD>;
  uint8_t* sK = tile_at<HD>(0);
  uint8_t* sV = tile_at<HD>(1);
  auto sQ = [](int buf) { return tile_at<HD>(2 + buf); };
  auto sdO = [](int buf) { return tile_at<HD>(4 + buf); };
  __shared__ float s_lse[2][BQ], s_del[2][BQ];

  const int k0 = blockIdx.x * BKV, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const typename R::Params p = R::prepare(p_in);
  const __nv_bfloat16* qp = p.q + b * p.q_bs + h * HD;
  const __nv_bfloat16* kp = p.k + b * p.k_bs + h * HD;
  const __nv_bfloat16* vp = p.v + b * p.v_bs + h * HD;
  const __nv_bfloat16* dop = p.d_o + b * p.o_bs + h * HD;
  const float* lp = p.lse + ((long long)b * p.heads + h) * p.nq;
  const float* dlp = p.delta + ((long long)b * p.heads + h) * p.nq;
  __builtin_assume(p.nq > 0);   // checked on the host; without it ptxas keeps more registers live in the media core
  const int nqb = (p.nq + BQ - 1) / BQ;
  const int qb0 = R::first_qblock(p, k0);
  const R r(p, b, h);

  auto stage_rows = [&](int buf, int qb) {
    if (threadIdx.x < BQ) {
      const int row = qb * BQ + threadIdx.x;
      r.stage_row(buf, row);
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
  const RowPair keys{k0 + warp * 16, k0 + warp * 16 + g, k0 + warp * 16 + g + 8, t};
  const typename R::Keys ks = r.key_rows(keys);

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
    if (!r.qblock_needed(buf, k0)) continue;

    float st[8][4], dpt[8][4], dst[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) { st[i][0] = st[i][1] = st[i][2] = st[i][3] = 0.f; dpt[i][0] = dpt[i][1] = dpt[i][2] = dpt[i][3] = 0.f; }
    mma_rows_x_tileT<HD>(st, sK, sQ(buf));     // S^T  = K Q^T   [16 keys x 64 queries]
    mma_rows_x_tileT<HD>(dpt, sV, sdO(buf));   // dP^T = V dO^T
    r.dkv_scores(st, dpt, dst, qb, k0, keys, ks, buf, s_lse[buf], s_del[buf]);
    uint32_t pa[4][4], dsa[4][4];
    c_to_a(st, pa);
    c_to_a(dst, dsa);
    mma_p_x_tile<HD>(dv, pa, sdO(buf));     // dV += P^T dO
    mma_p_x_tile<HD>(dk, dsa, sQ(buf));     // dK += dS^T Q
    __syncthreads();
  }
  if (qb0 >= nqb) cp_wait<0>();

  store_rows(p.dk + b * p.dk_bs + h * HD, p.lddk, dk, 1.f, 1.f, keys.a, keys.b, p.nk, t);
  store_rows(p.dv + b * p.dv_bs + h * HD, p.lddv, dv, 1.f, 1.f, keys.a, keys.b, p.nk, t);
}

// ================================================================ host side
static inline int attn_error(int code, const char* family, const char* what) {
  return ofk_set_error(code, (std::string(family) + ": " + what).c_str());
}

// The checks both families share, after a family's own argument checks and before its own alignment checks, so every
// OFK_ERR_ARG comes before any OFK_ERR_ALIGN.  q/k/v/o/dO are read (and o written) 16 bytes at a time per row and 32
// bits at a time by the delta kernel; dq/dk/dv are written 32 bits at a time; lse/delta are f32 arrays.
static int check_problem(const AttnProblem& p, bool bwd, const char* family) {
  if (!p.q || !p.k || !p.v || !(bwd ? p.o : p.out) ||
      (bwd && (!p.d_o || !p.lse || !p.delta || !p.dq || !p.dk || !p.dv)))
    return attn_error(OFK_ERR_ARG, family, "null pointer");
  if (p.batch <= 0 || p.heads <= 0 || p.nq <= 0 || p.nk <= 0) return attn_error(OFK_ERR_ARG, family, "empty problem");
  if (p.batch > 65535 || p.heads > 65535) return attn_error(OFK_ERR_ARG, family, "batch/heads exceed grid limits");
  const void* io = bwd ? static_cast<const void*>(p.o) : static_cast<const void*>(p.out);
  if (!aligned(p.q, 16) || !aligned(p.k, 16) || !aligned(p.v, 16) || !aligned(io, 16) || (bwd && !aligned(p.d_o, 16)))
    return attn_error(OFK_ERR_ALIGN, family, "q/k/v/o/dO must be 16-byte aligned");
  if ((p.q_bs | p.ldq | p.k_bs | p.ldk | p.v_bs | p.ldv | p.o_bs | p.ldo) % 8 != 0)
    return attn_error(OFK_ERR_ALIGN, family, "batch and row strides of q/k/v/o must be multiples of 8");
  if (!aligned(p.lse, 4) || !aligned(p.delta, 4)) return attn_error(OFK_ERR_ALIGN, family, "lse/delta must be 4-byte aligned");
  if (bwd) {
    if (!aligned(p.dq, 4) || !aligned(p.dk, 4) || !aligned(p.dv, 4))
      return attn_error(OFK_ERR_ALIGN, family, "dq/dk/dv must be 4-byte aligned");
    if ((p.dq_bs | p.lddq | p.dk_bs | p.lddk | p.dv_bs | p.lddv) % 2 != 0)
      return attn_error(OFK_ERR_ALIGN, family, "grad strides must be even");
  }
  return 0;
}

template <class R>
static int launch_fwd(const typename R::Params& p, cudaStream_t s) {
  constexpr int SMEM = 5 * Tile<R::HD>::BYTES + 1024;
  static bool done = false;
  if (!done) { cudaFuncSetAttribute(attn_fwd_kernel<R>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM); done = true; }
  dim3 grid((p.nq + BQ - 1) / BQ, p.heads, p.batch);
  attn_fwd_kernel<R><<<grid, THREADS, SMEM, s>>>(p);
  OFK_CHECK_LAUNCH();
  return 0;
}

template <class R>
static int launch_bwd(const typename R::Params& p, cudaStream_t s) {
  constexpr int SMEM = 6 * Tile<R::HD>::BYTES + 1024;
  static bool done = false;
  if (!done) {
    cudaFuncSetAttribute(attn_bwd_dq_kernel<R>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    cudaFuncSetAttribute(attn_bwd_dkv_kernel<R>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    done = true;
  }
  const long long rows = (long long)p.batch * p.heads * p.nq;
  delta_kernel<R::HD><<<(unsigned)((rows + 7) / 8), 256, 0, s>>>(p.o, p.d_o, p.delta, p.batch, p.heads, p.nq, p.o_bs, p.ldo);
  OFK_CHECK_LAUNCH();
  dim3 gq((p.nq + BQ - 1) / BQ, p.heads, p.batch);
  attn_bwd_dq_kernel<R><<<gq, THREADS, SMEM, s>>>(p);
  OFK_CHECK_LAUNCH();
  dim3 gk((p.nk + BKV - 1) / BKV, p.heads, p.batch);
  attn_bwd_dkv_kernel<R><<<gk, THREADS, SMEM, s>>>(p);
  OFK_CHECK_LAUNCH();
  return 0;
}

}  // namespace ofk
