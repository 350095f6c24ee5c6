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
//
// The kernels are those of attention_core.cuh; this file holds the media rules they run with.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "attention_core.cuh"

namespace ofk {

struct MediaParams : AttnProblem {
  const int* text_time;
  int mask_mode, kpm;
};

// Row classification for the media mask.
//   kind 0: normal masked row; 1: zero row; 2: uniform row (all keys, S = 0, no grad to q/k); 3: unmasked
struct RowInfo { int tt; int kind; };
__device__ __forceinline__ RowInfo classify_row(const MediaParams& p, int b, int row) {
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
// Whether a row may attend to keys of media index `media` (key / kpm + 1) -- it is constant over an 8-key n-tile
// (kpm % 16 == 0), so the integer division is done once per n-tile, not once per score.
__device__ __forceinline__ bool media_allowed(const MediaParams& p, const RowInfo& r, int media) {
  if (r.kind >= 2) return true;
  if (r.kind == 1) return false;
  return p.mask_mode == 1 ? (r.tt == media) : (r.tt >= media);
}

// Key range [lo, hi) (in keys) a 64-row query block needs; computed cooperatively by the CTA.
__device__ __forceinline__ void block_key_range(const MediaParams& p, int b, int q0, int& lo, int& hi) {
  __shared__ int s_red[12];
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

// text_time and row kind of the query blocks the dK/dV kernel has staged.
struct StagedRows { int tt[2][BQ], kind[2][BQ]; };
__device__ __forceinline__ StagedRows& staged_rows() {
  __shared__ StagedRows s;
  return s;
}

struct MediaRules {
  static constexpr int HD = 64;
  using Params = MediaParams;
  struct Rows { RowInfo a, b; };
  struct Keys { bool inb_a, inb_b; int media_a, media_b; };

  const Params p;
  int b;
  float sl2;   // exp(scale*s - lse) == exp2(scale*log2e*s - lse*log2e); LSE is stored in the log2 domain

  __device__ static Params prepare(const Params& p) { return p; }
  __device__ static void key_tiles(const Params& p, int b, int q0, int& klo, int& nblk) {
    int khi;
    block_key_range(p, b, q0, klo, khi);
    nblk = (khi - klo + BKV - 1) / BKV;
  }
  __device__ static int first_qblock(const Params&, int) { return 0; }

  __device__ MediaRules(const Params& p_, int b_, int) : p(p_), b(b_), sl2(p_.scale * LOG2E) {}
  __device__ Rows query_rows(const RowPair& rows) const { return {classify_row(p, b, rows.a), classify_row(p, b, rows.b)}; }

  __device__ void fwd_scores(float (&s)[8][4], int key0, const RowPair& rows, const Rows& rs, float& mx_a,
                             float& mx_b) const {
    if (p.mask_mode == 0 && key0 + BKV <= p.nk) {
      // fast path (Perceiver / ViT interior tiles): no predicate at all
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        s[i][0] *= sl2; s[i][1] *= sl2; s[i][2] *= sl2; s[i][3] *= sl2;
        mx_a = fmaxf(mx_a, fmaxf(s[i][0], s[i][1]));
        mx_b = fmaxf(mx_b, fmaxf(s[i][2], s[i][3]));
      }
      return;
    }
    const bool one_media = p.mask_mode != 0 && (p.kpm % BKV) == 0;      // all 64 keys of the tile share a media
    int media = p.mask_mode != 0 ? key0 / p.kpm + 1 : 0;
    bool aa = media_allowed(p, rs.a, media), ab = media_allowed(p, rs.b, media);
    const float za = rs.a.kind == 2 ? 0.f : sl2, zb = rs.b.kind == 2 ? 0.f : sl2;  // uniform rows: S = 0
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int key = key0 + i * 8 + 2 * rows.t;
      if (p.mask_mode != 0 && !one_media) {
        media = (key0 + i * 8) / p.kpm + 1;
        aa = media_allowed(p, rs.a, media); ab = media_allowed(p, rs.b, media);
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

  static constexpr int P_TERMS = 1;
  __device__ static void pack_p(const float (&s)[8][4], uint32_t (&pa)[1][4][4]) { c_to_a(s, pa[0]); }

  __device__ void dq_scores(float (&s)[8][4], const float (&dpv)[8][4], int key0, const RowPair& rows, const Rows& rs,
                            float lse_a, float lse_b, float del_a, float del_b) const {
    // P from the saved LSE
    const float za = rs.a.kind == 2 ? 0.f : sl2, zb = rs.b.kind == 2 ? 0.f : sl2;
    const float la = lse_a, lb = lse_b;
    if (p.mask_mode == 0 && key0 + BKV <= p.nk) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        s[i][0] = ex2_approx(fmaf(s[i][0], sl2, -la)); s[i][1] = ex2_approx(fmaf(s[i][1], sl2, -la));
        s[i][2] = ex2_approx(fmaf(s[i][2], sl2, -lb)); s[i][3] = ex2_approx(fmaf(s[i][3], sl2, -lb));
      }
    } else {
      const bool one_media = p.mask_mode != 0 && (p.kpm % BKV) == 0;
      int media = p.mask_mode != 0 ? key0 / p.kpm + 1 : 0;
      bool aa = media_allowed(p, rs.a, media), ab = media_allowed(p, rs.b, media);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int key = key0 + i * 8 + 2 * rows.t;
        if (p.mask_mode != 0 && !one_media) {
          media = (key0 + i * 8) / p.kpm + 1;
          aa = media_allowed(p, rs.a, media); ab = media_allowed(p, rs.b, media);
        }
        const bool inb0 = key < p.nk, inb1 = (key + 1) < p.nk;
        s[i][0] = (inb0 && aa) ? ex2_approx(fmaf(s[i][0], za, -la)) : 0.f;
        s[i][1] = (inb1 && aa) ? ex2_approx(fmaf(s[i][1], za, -la)) : 0.f;
        s[i][2] = (inb0 && ab) ? ex2_approx(fmaf(s[i][2], zb, -lb)) : 0.f;
        s[i][3] = (inb1 && ab) ? ex2_approx(fmaf(s[i][3], zb, -lb)) : 0.f;
      }
    }
    const float ga = rs.a.kind == 2 ? 0.f : p.scale, gb = rs.b.kind == 2 ? 0.f : p.scale;
#pragma unroll
    for (int i = 0; i < 8; ++i) {     // dS = P * (dP - delta) * scale
      s[i][0] = s[i][0] * (dpv[i][0] - del_a) * ga; s[i][1] = s[i][1] * (dpv[i][1] - del_a) * ga;
      s[i][2] = s[i][2] * (dpv[i][2] - del_b) * gb; s[i][3] = s[i][3] * (dpv[i][3] - del_b) * gb;
    }
  }

  __device__ void stage_row(int buf, int row) const {
    const RowInfo r = classify_row(p, b, row);
    staged_rows().tt[buf][threadIdx.x] = r.tt;
    staged_rows().kind[buf][threadIdx.x] = (row < p.nq) ? r.kind : 1;
  }
  __device__ Keys key_rows(const RowPair& keys) const {
    return {keys.a < p.nk, keys.b < p.nk, p.mask_mode != 0 ? keys.a / p.kpm + 1 : 0,
            p.mask_mode != 0 ? keys.b / p.kpm + 1 : 0};
  }
  // skip (query block, key block) pairs the media mask rules out entirely
  __device__ bool qblock_needed(int buf, int k0) const {
    int need = 0;
    if (threadIdx.x < BQ) {
      const int kind = staged_rows().kind[buf][threadIdx.x], tt = staged_rows().tt[buf][threadIdx.x];
      if (kind >= 2) need = 1;
      else if (kind == 0) {
        const int m_lo = k0 / p.kpm + 1, m_hi = min(p.nk - 1, k0 + BKV - 1) / p.kpm + 1;
        need = (p.mask_mode == 1) ? (tt >= m_lo && tt <= m_hi) : (tt >= m_lo);
      }
    }
    return __syncthreads_or(need);
  }

  __device__ void dkv_scores(float (&st)[8][4], const float (&dpt)[8][4], float (&dst)[8][4], int, int,
                             const RowPair& keys, const Keys& ks, int buf, const float* lse, const float* del) const {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int qc = i * 8 + 2 * keys.t + (e & 1);      // query column in this tile
        RowInfo r; r.tt = staged_rows().tt[buf][qc]; r.kind = staged_rows().kind[buf][qc];
        const bool ok = ((e & 2) ? ks.inb_b : ks.inb_a) && media_allowed(p, r, (e & 2) ? ks.media_b : ks.media_a);
        const float z = r.kind == 2 ? 0.f : sl2;
        const float pv = ok ? ex2_approx(fmaf(st[i][e], z, -lse[qc])) : 0.f;
        st[i][e] = pv;                                                            // P^T
        dst[i][e] = pv * (dpt[i][e] - del[qc]) * (r.kind == 2 ? 0.f : p.scale);   // dS^T
      }
    }
  }
};

// The media arguments: mask_mode, and with a media mask, text_time and a keys_per_media that tiles nk in multiples
// of 16 keys (so the media index is constant over an 8-key n-tile); text_time is an int32 array.
static int validate(const MediaParams& p, bool bwd) {
  if (p.mask_mode < 0 || p.mask_mode > 2) return ofk_set_error(OFK_ERR_ARG, "attention: bad mask_mode");
  if (p.mask_mode != 0) {
    if (!p.text_time) return ofk_set_error(OFK_ERR_ARG, "attention: media mask needs text_time");
    if (p.kpm <= 0 || p.kpm % 16 != 0 || p.nk % p.kpm != 0)
      return ofk_set_error(OFK_ERR_ARG, "attention: keys_per_media must be a multiple of 16 dividing nk");
  }
  if (int rc = check_problem(p, bwd, "attention")) return rc;
  if (!aligned(p.text_time, 4)) return ofk_set_error(OFK_ERR_ALIGN, "attention: text_time must be 4-byte aligned");
  return 0;
}

}  // namespace ofk

extern "C" int ofk_attn_fwd(const void* q, const void* k, const void* v, void* o, float* lse, int batch, int heads,
                            int nq, int nk, long long q_bstride, long long ldq, long long k_bstride, long long ldk,
                            long long v_bstride, long long ldv, long long o_bstride, long long ldo, float scale,
                            int mask_mode, const int* text_time, int keys_per_media, void* stream) {
  using namespace ofk;
  const MediaParams p{fwd_problem(q, k, v, o, lse, batch, heads, nq, nk, q_bstride, ldq, k_bstride, ldk, v_bstride, ldv,
                                  o_bstride, ldo, scale),
                      text_time, mask_mode, keys_per_media};
  if (int rc = validate(p, false)) return rc;
  return launch_fwd<MediaRules>(p, (cudaStream_t)stream);
}

extern "C" int ofk_attn_bwd(const void* q, const void* k, const void* v, const void* o, const void* d_o,
                            const float* lse, float* delta, void* dq, void* dk, void* dv, int batch, int heads, int nq,
                            int nk, long long q_bstride, long long ldq, long long k_bstride, long long ldk,
                            long long v_bstride, long long ldv, long long o_bstride, long long ldo,
                            long long dq_bstride, long long lddq, long long dk_bstride, long long lddk,
                            long long dv_bstride, long long lddv, float scale, int mask_mode, const int* text_time,
                            int keys_per_media, void* stream) {
  using namespace ofk;
  const MediaParams p{bwd_problem(q, k, v, o, d_o, lse, delta, dq, dk, dv, batch, heads, nq, nk, q_bstride, ldq,
                                  k_bstride, ldk, v_bstride, ldv, o_bstride, ldo, dq_bstride, lddq, dk_bstride, lddk,
                                  dv_bstride, lddv, scale),
                      text_time, mask_mode, keys_per_media};
  if (int rc = validate(p, true)) return rc;
  return launch_bwd<MediaRules>(p, (cudaStream_t)stream);
}
