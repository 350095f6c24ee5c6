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
//
// The kernels are those of attention_core.cuh; this file holds the MPT rules they run with.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "attention_core.cuh"

namespace ofk {

constexpr float MASKED = -30000.0f;  // log2-domain stand-in for finfo.min: exp2(MASKED - m) == 0 for any real m

struct DenseParams : AttnProblem {
  const unsigned char* mask;  // [B, nq, nk] 1 = masked, or NULL
  const float* slopes;        // [heads] or NULL
  const int* pure_causal;     // device flag or NULL: nonzero => the mask is exactly the causal rule (ignore `mask`,
                              // apply causal, skip key tiles above the diagonal) -- decided on the device, no host sync
  int causal;
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
__device__ __forceinline__ float score(const DenseParams& p, float dot, float sl2, float slope2, int b, int row, int key) {
  if (key >= p.nk) return -INFINITY;
  bool masked = p.causal && key > row + (p.nk - p.nq);
  if (!masked && p.mask && row < p.nq) masked = p.mask[((long long)b * p.nq + row) * p.nk + key] != 0;
  return masked ? MASKED : fmaf(dot, sl2, slope2 * (float)key);
}
__device__ __forceinline__ bool is_masked(const DenseParams& p, int b, int row, int key) {
  if (p.causal && key > row + (p.nk - p.nq)) return true;
  if (p.mask && row < p.nq) return p.mask[((long long)b * p.nq + row) * p.nk + key] != 0;
  return false;
}
// key tiles a query block needs when only the causal rule applies
__device__ __forceinline__ int causal_tiles(const DenseParams& p, int q0) {
  const int total = (p.nk + BKV - 1) / BKV;
  if (!p.causal || p.mask) return total;
  const int last_key = min(p.nk - 1, q0 + BQ - 1 + (p.nk - p.nq));
  return last_key < 0 ? 0 : min(total, last_key / BKV + 1);
}

// Tile classes for the fast paths: with no explicit mask, an in-bounds key tile entirely at or below the diagonal
// of ALL rows this thread touches needs no per-score predicate (that is ~3/4 of the causal work at T = 256).
__device__ __forceinline__ bool tile_unmasked(const DenseParams& p, int key_last, int row_first) {
  if (p.mask != nullptr || key_last >= p.nk) return false;
  return !p.causal || key_last <= row_first + (p.nk - p.nq);
}

template <int HD_>
struct DenseRules {
  static constexpr int HD = HD_;
  using Params = DenseParams;
  struct Rows {};
  struct Keys {};

  const Params p;
  int b;
  float sl2, slope2;

  __device__ static Params prepare(const Params& p_in) {
    Params p = p_in;
    if (p.pure_causal != nullptr && *p.pure_causal != 0) { p.mask = nullptr; p.causal = 1; }
    return p;
  }
  __device__ static void key_tiles(const Params& p, int, int q0, int& klo, int& nblk) { klo = 0; nblk = causal_tiles(p, q0); }
  // pure-causal: query blocks entirely before this key block see none of its keys
  __device__ static int first_qblock(const Params& p, int k0) { return p.causal && !p.mask ? max(0, (k0 - (p.nk - p.nq)) / BQ) : 0; }

  __device__ DenseRules(const Params& p_, int b_, int h)
      : p(p_), b(b_), sl2(p_.scale * LOG2E), slope2(p_.slopes ? p_.slopes[h] * LOG2E : 0.f) {}

  __device__ Rows query_rows(const RowPair&) const { return {}; }

  __device__ void fwd_scores(float (&s)[8][4], int key0, const RowPair& rows, const Rows&, float& mx_a,
                             float& mx_b) const {
    if (tile_unmasked(p, key0 + BKV - 1, rows.first)) {
      const float kb = slope2 * (float)(key0 + 2 * rows.t);
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
        const int key = key0 + i * 8 + 2 * rows.t;
        s[i][0] = score(p, s[i][0], sl2, slope2, b, rows.a, key);
        s[i][1] = score(p, s[i][1], sl2, slope2, b, rows.a, key + 1);
        s[i][2] = score(p, s[i][2], sl2, slope2, b, rows.b, key);
        s[i][3] = score(p, s[i][3], sl2, slope2, b, rows.b, key + 1);
        mx_a = fmaxf(mx_a, fmaxf(s[i][0], s[i][1]));
        mx_b = fmaxf(mx_b, fmaxf(s[i][2], s[i][3]));
      }
    }
  }

  static constexpr int P_TERMS = 2;
  __device__ static void pack_p(float (&s)[8][4], uint32_t (&pa)[2][4][4]) { c_to_a_split(s, pa[0], pa[1]); }

  __device__ void dq_scores(float (&s)[8][4], const float (&dpv)[8][4], int key0, const RowPair& rows, const Rows&,
                            float lse_a, float lse_b, float del_a, float del_b) const {
    if (tile_unmasked(p, key0 + BKV - 1, rows.first)) {
      const float kb = slope2 * (float)(key0 + 2 * rows.t);
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
          const int key = key0 + i * 8 + 2 * rows.t + (e & 1);
          const int row = (e & 2) ? rows.b : rows.a;
          const float sc = score(p, s[i][e], sl2, slope2, b, row, key);
          const float pv = ex2_approx(sc - ((e & 2) ? lse_b : lse_a));
          const bool live = key < p.nk && !is_masked(p, b, row, key);   // masked_fill passes no gradient to the scores
          s[i][e] = live ? pv * (dpv[i][e] - ((e & 2) ? del_b : del_a)) * p.scale : 0.f;
        }
      }
    }
  }

  __device__ void stage_row(int, int) const {}
  __device__ Keys key_rows(const RowPair&) const { return {}; }
  __device__ bool qblock_needed(int, int) const { return true; }

  __device__ void dkv_scores(float (&st)[8][4], const float (&dpt)[8][4], float (&dst)[8][4], int qb, int k0,
                             const RowPair& keys, const Keys&, int, const float* lse, const float* del) const {
    // fast path: the whole 64 x 64 (query, key) tile is in bounds and unmasked
    const bool fast = p.mask == nullptr && k0 + BKV <= p.nk && qb * BQ + BQ <= p.nq &&
                      (!p.causal || k0 + BKV - 1 <= qb * BQ + (p.nk - p.nq));
    if (fast) {
      const float ba = slope2 * (float)keys.a, bb = slope2 * (float)keys.b;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int qc = i * 8 + 2 * keys.t + (e & 1);
          const float pv = ex2_approx(fmaf(st[i][e], sl2, (e & 2) ? bb : ba) - lse[qc]);
          st[i][e] = pv;
          dst[i][e] = pv * (dpt[i][e] - del[qc]) * p.scale;
        }
      }
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int qc = i * 8 + 2 * keys.t + (e & 1);
          const int row = qb * BQ + qc;
          const int key = (e & 2) ? keys.b : keys.a;
          const bool inb = row < p.nq;
          const float sc = score(p, st[i][e], sl2, slope2, b, row, key);
          const float pv = inb ? ex2_approx(sc - lse[qc]) : 0.f;
          const bool live = inb && key < p.nk && !is_masked(p, b, row, key);
          st[i][e] = pv;                                                    // P^T
          dst[i][e] = live ? pv * (dpt[i][e] - del[qc]) * p.scale : 0.f;   // dS^T
        }
      }
    }
  }
};

// head_dim is 64 or 128; slopes and the flag are 4-byte scalars.  The causal rule key <= row + nk - nq leaves whole
// query blocks without a key when nq > nk, and the tile skipping would give those rows zeros instead of the finfo.min
// rule's uniform attention; no caller needs that case, so it is rejected.
static int validate(const DenseParams& p, int head_dim, bool bwd) {
  if (head_dim != 64 && head_dim != 128) return ofk_set_error(OFK_ERR_ARG, "dense attention: head_dim must be 64 or 128");
  if ((p.causal || p.pure_causal) && p.nq > p.nk)
    return ofk_set_error(OFK_ERR_ARG, "dense attention: the causal rule needs nq <= nk");
  if (int rc = check_problem(p, bwd, "dense attention")) return rc;
  if (!aligned(p.slopes, 4) || !aligned(p.pure_causal, 4))
    return ofk_set_error(OFK_ERR_ALIGN, "dense attention: slopes/pure_causal_flag must be 4-byte aligned");
  return 0;
}

}  // namespace ofk

extern "C" int ofk_attn_dense_fwd(const void* q, const void* k, const void* v, void* o, float* lse, int batch, int heads,
                                  int head_dim, int nq, int nk, long long q_bstride, long long ldq, long long k_bstride,
                                  long long ldk, long long v_bstride, long long ldv, long long o_bstride, long long ldo,
                                  float scale, int causal, const unsigned char* mask, const float* slopes,
                                  const int* pure_causal_flag, void* stream) {
  using namespace ofk;
  const DenseParams p{fwd_problem(q, k, v, o, lse, batch, heads, nq, nk, q_bstride, ldq, k_bstride, ldk, v_bstride, ldv,
                                  o_bstride, ldo, scale),
                      mask, slopes, pure_causal_flag, causal};
  if (int rc = validate(p, head_dim, false)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  return head_dim == 64 ? launch_fwd<DenseRules<64>>(p, s) : launch_fwd<DenseRules<128>>(p, s);
}

extern "C" int ofk_attn_dense_bwd(const void* q, const void* k, const void* v, const void* o, const void* d_o,
                                  const float* lse, float* delta, void* dq, void* dk, void* dv, int batch, int heads,
                                  int head_dim, int nq, int nk, long long q_bstride, long long ldq, long long k_bstride,
                                  long long ldk, long long v_bstride, long long ldv, long long o_bstride, long long ldo,
                                  long long dq_bstride, long long lddq, long long dk_bstride, long long lddk,
                                  long long dv_bstride, long long lddv, float scale, int causal, const unsigned char* mask,
                                  const float* slopes, const int* pure_causal_flag, void* stream) {
  using namespace ofk;
  const DenseParams p{bwd_problem(q, k, v, o, d_o, lse, delta, dq, dk, dv, batch, heads, nq, nk, q_bstride, ldq,
                                  k_bstride, ldk, v_bstride, ldv, o_bstride, ldo, dq_bstride, lddq, dk_bstride, lddk,
                                  dv_bstride, lddv, scale),
                      mask, slopes, pure_causal_flag, causal};
  if (int rc = validate(p, head_dim, true)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  return head_dim == 64 ? launch_bwd<DenseRules<64>>(p, s) : launch_bwd<DenseRules<128>>(p, s);
}
