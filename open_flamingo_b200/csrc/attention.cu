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

#include "ofk_internal.h"
#include "ofk_ptx.cuh"

namespace ofk {

constexpr int HD = 64;    // head dim
constexpr int BQ = 64;    // query rows per CTA (16 per warp)
constexpr int BKV = 64;   // keys per tile
constexpr int ATT_THREADS = 128;
constexpr float LOG2E = 1.4426950408889634f;

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

// ---------------------------------------------------------------- smem tile helpers (64 rows x 64 bf16, swizzled)
// The XOR pattern is the 128-byte swizzle wgmma descriptors expect; tiles start on 1024-byte boundaries.
__device__ __forceinline__ uint32_t tile_off(int row, int chunk) {  // chunk = 16-byte column group 0..7
  return (uint32_t)(row * 128 + ((chunk ^ (row & 7)) << 4));
}

__device__ __forceinline__ void cp_async16(uint32_t saddr, const void* g, bool valid) {
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(saddr), "l"(g), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// Load rows [row0, row0+64) x 64 columns (starting at `g`, row stride ld) into a swizzled tile; rows >= nrows -> 0.
__device__ __forceinline__ void load_tile(uint8_t* tile, const __nv_bfloat16* g, long long ld, int row0, int nrows) {
  const uint32_t base = smem_u32(tile);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int idx = threadIdx.x + i * ATT_THREADS;  // 0..511
    const int r = idx >> 3, c = idx & 7;
    const bool valid = (row0 + r) < nrows;
    const __nv_bfloat16* src = g + (long long)(valid ? (row0 + r) : 0) * ld + c * 8;
    cp_async16(base + tile_off(r, c), src, valid);
  }
}

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// A fragments (16 rows x 64 k) of a row-major tile: rows [r0, r0+16).
__device__ __forceinline__ void load_a_frags(const uint8_t* tile, int r0, uint32_t (&a)[4][4]) {
  const int lane = threadIdx.x & 31;
  const int row = r0 + (lane & 7) + ((lane >> 3) & 1) * 8;
  const uint32_t base = smem_u32(tile);
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    const int chunk = ks * 2 + (lane >> 4);
    ldsm_x4(base + tile_off(row, chunk), a[ks][0], a[ks][1], a[ks][2], a[ks][3]);
  }
}

// Tensor-core products of one CTA = one warpgroup of 4 warps x 16 rows.  WG = true: one warpgroup-wide wgmma per 16-deep
// k step over all 64 rows (A from each warp's registers, B from the 128-byte-swizzled tile through a descriptor);
// WG = false: per-warp mma.sync, kept as the A/B reference.  Both use the same accumulator and A-fragment layout, so
// the softmax / mask code around them is shared.
__device__ __forceinline__ void wgmma_pin(float* d, int n) {
  for (int i = 0; i < n; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// C[16 x 64] (+)= A[16 x 64(k)] * T^T where T is a [64 n][64 k] row-major tile  ("n rows, k contiguous").  A is the
// warp's rows of `atile` (WG: read by wgmma through a descriptor of the whole 64-row tile) or, for mma.sync, the
// fragments `a` already loaded from it.
template <bool WG>
__device__ __forceinline__ void mma_a_tileT(float (&c)[8][4], const uint32_t (&a)[4][4], const uint8_t* atile,
                                            const uint8_t* tile) {
  const uint32_t base = smem_u32(tile);
  if constexpr (WG) {
    const uint32_t abase = smem_u32(atile);
    float(&d)[32] = *reinterpret_cast<float(*)[32]>(&c[0][0]);
    wgmma_pin(d, 32);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks)
      wgmma_m64n64k16_ss(d, make_wgmma_desc_sw128(abase + ks * 32, 16, 1024), make_wgmma_desc_sw128(base + ks * 32, 16, 1024));
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_pin(d, 32);
  } else {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int np = 0; np < 4; ++np) {       // pairs of 8-wide n tiles
      const int nrow = np * 16 + (lane & 7) + (lane >> 4) * 8;
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        uint32_t b0, b1, b2, b3;
        const int chunk = ks * 2 + ((lane >> 3) & 1);
        ldsm_x4(base + tile_off(nrow, chunk), b0, b1, b2, b3);
        mma16816(c[np * 2], a[ks], b0, b1);
        mma16816(c[np * 2 + 1], a[ks], b2, b3);
      }
    }
  }
}

// C[16 x 64(n)] += P[16 x 64(k)] * T where T is a [64 k][64 n] row-major tile ("k rows, n contiguous").
template <bool WG>
__device__ __forceinline__ void mma_p_tile(float (&c)[8][4], const uint32_t (&p)[4][4], const uint8_t* tile) {
  const uint32_t base = smem_u32(tile);
  if constexpr (WG) {
    float(&d)[32] = *reinterpret_cast<float(*)[32]>(&c[0][0]);
    wgmma_pin(d, 32);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) wgmma_m64n64k16_rs<1>(d, p[ks], make_wgmma_desc_sw128(base + ks * 2048, 8192, 1024));
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_pin(d, 32);
  } else {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const int krow = ks * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
#pragma unroll
      for (int np = 0; np < 4; ++np) {
        uint32_t b0, b1, b2, b3;
        const int chunk = np * 2 + (lane >> 4);
        ldsm_x4_t(base + tile_off(krow, chunk), b0, b1, b2, b3);
        mma16816(c[np * 2], p[ks], b0, b1);
        mma16816(c[np * 2 + 1], p[ks], b2, b3);
      }
    }
  }
}

// Pack a C-layout [16 x 64] fp32 tile into A-layout bf16 fragments (k = the 64 columns).
__device__ __forceinline__ void c_to_a(const float (&c)[8][4], uint32_t (&a)[4][4]) {
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    a[ks][0] = pack_bf16x2(c[2 * ks][0], c[2 * ks][1]);
    a[ks][1] = pack_bf16x2(c[2 * ks][2], c[2 * ks][3]);
    a[ks][2] = pack_bf16x2(c[2 * ks + 1][0], c[2 * ks + 1][1]);
    a[ks][3] = pack_bf16x2(c[2 * ks + 1][2], c[2 * ks + 1][3]);
  }
}

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
// Tiles live in dynamic shared memory aligned by hand: the 128-byte swizzle wgmma reads is a function of the absolute
// shared address, so every tile must start on a 1024-byte boundary.
constexpr int FWD_SMEM = 5 * 64 * 128 + 1024;
extern __shared__ uint8_t att_dyn_smem[];
template <bool WG>
__global__ void __launch_bounds__(ATT_THREADS) attn_fwd_kernel(const AttnParams p) {
  uint8_t* fbase = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(att_dyn_smem) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = fbase;
  uint8_t* sK[2] = {fbase + 64 * 128, fbase + 2 * 64 * 128};
  uint8_t* sV[2] = {fbase + 3 * 64 * 128, fbase + 4 * 64 * 128};
  __shared__ int s_red[12];

  const int q0 = blockIdx.x * BQ, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const __nv_bfloat16* qp = p.q + b * p.q_bs + h * HD;
  const __nv_bfloat16* kp = p.k + b * p.k_bs + h * HD;
  const __nv_bfloat16* vp = p.v + b * p.v_bs + h * HD;

  int klo, khi;
  block_key_range(p, b, q0, s_red, klo, khi);
  const int nblk = (khi - klo + BKV - 1) / BKV;

  load_tile(sQ, qp, p.ldq, q0, p.nq);
  if (nblk > 0) { load_tile(sK[0], kp, p.ldk, klo, p.nk); load_tile(sV[0], vp, p.ldv, klo, p.nk); }
  cp_async_commit();

  const int row_a = q0 + warp * 16 + g, row_b = row_a + 8;
  const RowInfo ra = classify_row(p, b, row_a), rb = classify_row(p, b, row_b);

  float o[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
  float m_a = -INFINITY, m_b = -INFINITY, l_a = 0.f, l_b = 0.f;
  const float sl2 = p.scale * LOG2E;
  uint32_t qa[4][4];

  for (int j = 0; j < nblk; ++j) {
    const int buf = j & 1;
    if (j + 1 < nblk) {
      load_tile(sK[buf ^ 1], kp, p.ldk, klo + (j + 1) * BKV, p.nk);
      load_tile(sV[buf ^ 1], vp, p.ldv, klo + (j + 1) * BKV, p.nk);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    if constexpr (WG) fence_proxy_async_smem();   // cp.async (generic proxy) -> wgmma reads
    __syncthreads();
    if (!WG && j == 0) load_a_frags(sQ, warp * 16, qa);

    float s[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; }
    mma_a_tileT<WG>(s, qa, sQ, sK[buf]);

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
    mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, 1)); mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, 2));
    mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, 1)); mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, 2));
    const float mn_a = fmaxf(m_a, mx_a), mn_b = fmaxf(m_b, mx_b);
    const float sub_a = (mn_a == -INFINITY) ? 0.f : mn_a, sub_b = (mn_b == -INFINITY) ? 0.f : mn_b;
    const float corr_a = ex2_approx(m_a - sub_a), corr_b = ex2_approx(m_b - sub_b);  // m = -inf -> 0
    m_a = mn_a; m_b = mn_b;
    float rs_a = 0.f, rs_b = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      s[i][0] = ex2_approx(s[i][0] - sub_a); s[i][1] = ex2_approx(s[i][1] - sub_a);
      s[i][2] = ex2_approx(s[i][2] - sub_b); s[i][3] = ex2_approx(s[i][3] - sub_b);
      rs_a += s[i][0] + s[i][1]; rs_b += s[i][2] + s[i][3];
    }
    l_a = l_a * corr_a + rs_a; l_b = l_b * corr_b + rs_b;
#pragma unroll
    for (int i = 0; i < 8; ++i) { o[i][0] *= corr_a; o[i][1] *= corr_a; o[i][2] *= corr_b; o[i][3] *= corr_b; }
    uint32_t pa[4][4];
    c_to_a(s, pa);
    mma_p_tile<WG>(o, pa, sV[buf]);
    __syncthreads();
  }
  if (nblk == 0) { cp_async_wait<0>(); }

  l_a += __shfl_xor_sync(0xffffffffu, l_a, 1); l_a += __shfl_xor_sync(0xffffffffu, l_a, 2);
  l_b += __shfl_xor_sync(0xffffffffu, l_b, 1); l_b += __shfl_xor_sync(0xffffffffu, l_b, 2);
  const float inv_a = l_a > 0.f ? 1.f / l_a : 0.f, inv_b = l_b > 0.f ? 1.f / l_b : 0.f;
  __nv_bfloat16* op = p.out + b * p.o_bs + h * HD;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int col = i * 8 + 2 * t;
    if (row_a < p.nq) *reinterpret_cast<uint32_t*>(op + (long long)row_a * p.ldo + col) = pack_bf16x2(o[i][0] * inv_a, o[i][1] * inv_a);
    if (row_b < p.nq) *reinterpret_cast<uint32_t*>(op + (long long)row_b * p.ldo + col) = pack_bf16x2(o[i][2] * inv_b, o[i][3] * inv_b);
  }
  if (p.lse != nullptr && t == 0) {
    // log2-domain LSE of the scaled scores; rows with no mass get the sentinel 0 (P recomputes to 0 there because
    // every score is -inf).
    float* lp = p.lse + ((long long)b * p.heads + h) * p.nq;
    if (row_a < p.nq) lp[row_a] = l_a > 0.f ? m_a + log2f(l_a) : 0.f;
    if (row_b < p.nq) lp[row_b] = l_b > 0.f ? m_b + log2f(l_b) : 0.f;
  }
}

// ================================================================ backward: delta = rowsum(dO * O)
__global__ void attn_delta_kernel(const AttnParams p) {
  const int warps_per_block = blockDim.x >> 5;
  const long long row = (long long)blockIdx.x * warps_per_block + (threadIdx.x >> 5);  // over batch*heads*nq
  const long long total = (long long)p.batch * p.heads * p.nq;
  if (row >= total) return;
  const int lane = threadIdx.x & 31;
  const int qi = (int)(row % p.nq);
  const int h = (int)((row / p.nq) % p.heads);
  const int b = (int)(row / ((long long)p.nq * p.heads));
  const __nv_bfloat16* op = p.o + b * p.o_bs + (long long)qi * p.ldo + h * HD;
  const __nv_bfloat16* dop = p.d_o + b * p.o_bs + (long long)qi * p.ldo + h * HD;
  const uint32_t a = *reinterpret_cast<const uint32_t*>(op + 2 * lane);
  const uint32_t d = *reinterpret_cast<const uint32_t*>(dop + 2 * lane);
  float v = bf16_lo(a) * bf16_lo(d) + bf16_hi(a) * bf16_hi(d);
  v = warp_sum(v);
  if (lane == 0) p.delta[row] = v;
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
constexpr int BWD_SMEM = 6 * 64 * 128 + 1024;  // six 8 KiB tiles + alignment slack

template <bool WG>
__global__ void __launch_bounds__(ATT_THREADS) attn_bwd_dq_kernel(const AttnParams p) {
  uint8_t* base_ = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(att_dyn_smem) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = base_;
  uint8_t* sdO = base_ + 8192;
  uint8_t* sK[2] = {base_ + 2 * 8192, base_ + 3 * 8192};
  uint8_t* sV[2] = {base_ + 4 * 8192, base_ + 5 * 8192};
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

  load_tile(sQ, qp, p.ldq, q0, p.nq);
  load_tile(sdO, dop, p.ldo, q0, p.nq);
  if (nblk > 0) { load_tile(sK[0], kp, p.ldk, klo, p.nk); load_tile(sV[0], vp, p.ldv, klo, p.nk); }
  cp_async_commit();

  const int row_a = q0 + warp * 16 + g, row_b = row_a + 8;
  const RowInfo ra = classify_row(p, b, row_a), rb = classify_row(p, b, row_b);
  const float* lp = p.lse + ((long long)b * p.heads + h) * p.nq;
  const float* dp = p.delta + ((long long)b * p.heads + h) * p.nq;
  const float lse_a = row_a < p.nq ? lp[row_a] : 0.f, lse_b = row_b < p.nq ? lp[row_b] : 0.f;
  const float del_a = row_a < p.nq ? dp[row_a] : 0.f, del_b = row_b < p.nq ? dp[row_b] : 0.f;

  float dq[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i) { dq[i][0] = dq[i][1] = dq[i][2] = dq[i][3] = 0.f; }
  uint32_t qa[4][4], doa[4][4];

  for (int j = 0; j < nblk; ++j) {
    const int buf = j & 1;
    if (j + 1 < nblk) {
      load_tile(sK[buf ^ 1], kp, p.ldk, klo + (j + 1) * BKV, p.nk);
      load_tile(sV[buf ^ 1], vp, p.ldv, klo + (j + 1) * BKV, p.nk);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    if constexpr (WG) fence_proxy_async_smem();   // cp.async (generic proxy) -> wgmma reads
    __syncthreads();
    if (!WG && j == 0) { load_a_frags(sQ, warp * 16, qa); load_a_frags(sdO, warp * 16, doa); }

    float s[8][4], dpv[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; dpv[i][0] = dpv[i][1] = dpv[i][2] = dpv[i][3] = 0.f; }
    mma_a_tileT<WG>(s, qa, sQ, sK[buf]);      // S  = Q K^T
    mma_a_tileT<WG>(dpv, doa, sdO, sV[buf]);   // dP = dO V^T
    recompute_p(p, s, ra, rb, lse_a, lse_b, klo + j * BKV, t);
    const float ga = ra.kind == 2 ? 0.f : p.scale, gb = rb.kind == 2 ? 0.f : p.scale;
#pragma unroll
    for (int i = 0; i < 8; ++i) {     // dS = P * (dP - delta) * scale
      s[i][0] = s[i][0] * (dpv[i][0] - del_a) * ga; s[i][1] = s[i][1] * (dpv[i][1] - del_a) * ga;
      s[i][2] = s[i][2] * (dpv[i][2] - del_b) * gb; s[i][3] = s[i][3] * (dpv[i][3] - del_b) * gb;
    }
    uint32_t dsa[4][4];
    c_to_a(s, dsa);
    mma_p_tile<WG>(dq, dsa, sK[buf]);     // dQ += dS K
    __syncthreads();
  }
  if (nblk == 0) { cp_async_wait<0>(); }

  __nv_bfloat16* dqp = p.dq + b * p.dq_bs + h * HD;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int col = i * 8 + 2 * t;
    if (row_a < p.nq) *reinterpret_cast<uint32_t*>(dqp + (long long)row_a * p.lddq + col) = pack_bf16x2(dq[i][0], dq[i][1]);
    if (row_b < p.nq) *reinterpret_cast<uint32_t*>(dqp + (long long)row_b * p.lddq + col) = pack_bf16x2(dq[i][2], dq[i][3]);
  }
}

// ================================================================ backward: dK, dV (CTA = 64 keys, loop over query tiles)
// Works on transposed tiles: S^T = K Q^T (rows = keys), so P^T / dS^T are directly the A operands of
// dV += P^T dO and dK += dS^T Q.
template <bool WG>
__global__ void __launch_bounds__(ATT_THREADS) attn_bwd_dkv_kernel(const AttnParams p) {
  uint8_t* base_ = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(att_dyn_smem) + 1023) & ~uintptr_t(1023));
  uint8_t* sK = base_;
  uint8_t* sV = base_ + 8192;
  uint8_t* sQ[2] = {base_ + 2 * 8192, base_ + 3 * 8192};
  uint8_t* sdO[2] = {base_ + 4 * 8192, base_ + 5 * 8192};
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

  load_tile(sK, kp, p.ldk, k0, p.nk);
  load_tile(sV, vp, p.ldv, k0, p.nk);
  load_tile(sQ[0], qp, p.ldq, 0, p.nq);
  load_tile(sdO[0], dop, p.ldo, 0, p.nq);
  cp_async_commit();
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
      load_tile(sQ[buf ^ 1], qp, p.ldq, (qb + 1) * BQ, p.nq);
      load_tile(sdO[buf ^ 1], dop, p.ldo, (qb + 1) * BQ, p.nq);
      cp_async_commit();
      stage_rows(buf ^ 1, qb + 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    if constexpr (WG) fence_proxy_async_smem();   // cp.async (generic proxy) -> wgmma reads
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
    {
      uint32_t fa[4][4];              // A fragments are re-read from smem each time: keeps the kernel under 255 regs
      if (!WG) load_a_frags(sK, warp * 16, fa);
      mma_a_tileT<WG>(st, fa, sK, sQ[buf]);     // S^T  = K Q^T   [16 keys x 64 queries]
      if (!WG) load_a_frags(sV, warp * 16, fa);
      mma_a_tileT<WG>(dpt, fa, sV, sdO[buf]);   // dP^T = V dO^T
    }
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
    mma_p_tile<WG>(dv, pa, sdO[buf]);     // dV += P^T dO
    mma_p_tile<WG>(dk, dsa, sQ[buf]);     // dK += dS^T Q
    __syncthreads();
  }

  __nv_bfloat16* dkp = p.dk + b * p.dk_bs + h * HD;
  __nv_bfloat16* dvp = p.dv + b * p.dv_bs + h * HD;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int col = i * 8 + 2 * t;
    if (key_a < p.nk) {
      *reinterpret_cast<uint32_t*>(dkp + (long long)key_a * p.lddk + col) = pack_bf16x2(dk[i][0], dk[i][1]);
      *reinterpret_cast<uint32_t*>(dvp + (long long)key_a * p.lddv + col) = pack_bf16x2(dv[i][0], dv[i][1]);
    }
    if (key_b < p.nk) {
      *reinterpret_cast<uint32_t*>(dkp + (long long)key_b * p.lddk + col) = pack_bf16x2(dk[i][2], dk[i][3]);
      *reinterpret_cast<uint32_t*>(dvp + (long long)key_b * p.lddv + col) = pack_bf16x2(dv[i][2], dv[i][3]);
    }
  }
}

static bool aligned(const void* ptr, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(ptr) & (bytes - 1)) == 0; }

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
  if (ofk_attn_use_wgmma()) {
    attn_fwd_kernel<true><<<grid, ATT_THREADS, FWD_SMEM, (cudaStream_t)stream_>>>(p);
    OFK_CHECK_LAUNCH();
    ofk_attn_count_wgmma();
  } else {
    attn_fwd_kernel<false><<<grid, ATT_THREADS, FWD_SMEM, (cudaStream_t)stream_>>>(p);
    OFK_CHECK_LAUNCH();
  }
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
  attn_delta_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, stream>>>(p);
  OFK_CHECK_LAUNCH();
  dim3 gq((nq + BQ - 1) / BQ, heads, batch);
  static bool attr_done = false;
  if (!attr_done) {
    cudaFuncSetAttribute(attn_bwd_dq_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, BWD_SMEM);
    cudaFuncSetAttribute(attn_bwd_dkv_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, BWD_SMEM);
    cudaFuncSetAttribute(attn_bwd_dq_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, BWD_SMEM);
    cudaFuncSetAttribute(attn_bwd_dkv_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, BWD_SMEM);
    attr_done = true;
  }
  dim3 gk((nk + BKV - 1) / BKV, heads, batch);
  if (ofk_attn_use_wgmma()) {
    attn_bwd_dq_kernel<true><<<gq, ATT_THREADS, BWD_SMEM, stream>>>(p);
    OFK_CHECK_LAUNCH();
    attn_bwd_dkv_kernel<true><<<gk, ATT_THREADS, BWD_SMEM, stream>>>(p);
    OFK_CHECK_LAUNCH();
    ofk_attn_count_wgmma();
  } else {
    attn_bwd_dq_kernel<false><<<gq, ATT_THREADS, BWD_SMEM, stream>>>(p);
    OFK_CHECK_LAUNCH();
    attn_bwd_dkv_kernel<false><<<gk, ATT_THREADS, BWD_SMEM, stream>>>(p);
    OFK_CHECK_LAUNCH();
  }
  return 0;
}
