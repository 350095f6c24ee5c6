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

#include "ofk_internal.h"
#include "ofk_ptx.cuh"

namespace ofk {
namespace dense {

constexpr int BQ = 64, BKV = 64, THREADS = 128;
constexpr float LOG2E = 1.4426950408889634f;
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

template <int HD>
struct Tile {
  static constexpr int ROW_BYTES = HD * 2;
  static constexpr int CHUNKS = HD / 8;        // 16-byte chunks per row
  static constexpr int BYTES = 64 * ROW_BYTES;  // 64-row tile
  static constexpr int KSTEPS = HD / 16;       // k-steps when HD is the contraction dim
  static constexpr int NT = HD / 8;            // 8-wide n tiles when HD is the output dim
  // 64-column halves of the tile are separate 8 KiB atoms of 64 rows x 128 bytes with the 128-byte XOR swizzle: the
  // canonical layout wgmma descriptors read (tiles start on 1024-byte boundaries).
  __device__ static __forceinline__ uint32_t off(int row, int chunk) {
    return (uint32_t)((chunk >> 3) * (64 * 128) + row * 128 + (((chunk & 7) ^ (row & 7)) << 4));
  }
};

__device__ __forceinline__ void cp_async16(uint32_t saddr, const void* g, bool valid) {
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(saddr), "l"(g), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

template <int HD>
__device__ __forceinline__ void load_tile(uint8_t* tile, const __nv_bfloat16* g, long long ld, int row0, int nrows) {
  using T = Tile<HD>;
  const uint32_t base = smem_u32(tile);
#pragma unroll
  for (int i = 0; i < (64 * T::CHUNKS) / THREADS; ++i) {
    const int idx = threadIdx.x + i * THREADS;
    const int r = idx / T::CHUNKS, c = idx % T::CHUNKS;
    const bool valid = (row0 + r) < nrows;
    cp_async16(base + T::off(r, c), g + (long long)(valid ? (row0 + r) : 0) * ld + c * 8, valid);
  }
}

__device__ __forceinline__ void ldsm4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm4t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ void wgmma_pin(float* d, int n) {
  for (int i = 0; i < n; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Tensor-core products of one CTA = one warpgroup of 4 warps x 16 rows.  WG = true: warpgroup-wide wgmma over all 64
// rows, operands from the swizzled tiles through descriptors (P / dS from registers); WG = false: per-warp mma.sync,
// kept as the A/B reference.  Both share the accumulator and A-fragment layout, so the code around them is common.

// C[16 x 64] += X[rows r0.., HD(k)] * T^T, both [rows][HD] tiles (contraction over HD).
template <int HD, bool WG>
__device__ __forceinline__ void mma_rows_x_tileT(float (&c)[8][4], const uint8_t* xt, int r0, const uint8_t* tile) {
  using T = Tile<HD>;
  const uint32_t xb = smem_u32(xt), tb = smem_u32(tile);
  if constexpr (WG) {
    float(&d)[32] = *reinterpret_cast<float(*)[32]>(&c[0][0]);
    wgmma_pin(d, 32);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < T::KSTEPS; ++ks) {
      const uint32_t o = (ks >> 2) * (64 * 128) + (ks & 3) * 32;
      wgmma_m64n64k16_ss(d, make_wgmma_desc_sw128(xb + o, 16, 1024), make_wgmma_desc_sw128(tb + o, 16, 1024));
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_pin(d, 32);
  } else {
    const int lane = threadIdx.x & 31;
    const int arow = r0 + (lane & 7) + ((lane >> 3) & 1) * 8;
#pragma unroll
    for (int ks = 0; ks < T::KSTEPS; ++ks) {
      uint32_t a[4];
      ldsm4(xb + T::off(arow, ks * 2 + (lane >> 4)), a[0], a[1], a[2], a[3]);
#pragma unroll
      for (int np = 0; np < 4; ++np) {
        const int nrow = np * 16 + (lane & 7) + (lane >> 4) * 8;
        uint32_t b0, b1, b2, b3;
        ldsm4(tb + T::off(nrow, ks * 2 + ((lane >> 3) & 1)), b0, b1, b2, b3);
        mma16816(c[np * 2], a, b0, b1);
        mma16816(c[np * 2 + 1], a, b2, b3);
      }
    }
  }
}

// C[16 x HD] += P[16 x 64(k)] * T, T = [64 k][HD n] tile (contraction over the tile's 64 rows).
template <int HD, bool WG>
__device__ __forceinline__ void mma_p_x_tile(float (&c)[Tile<HD>::NT][4], const uint32_t (&p)[4][4], const uint8_t* tile) {
  using T = Tile<HD>;
  const uint32_t tb = smem_u32(tile);
  if constexpr (WG) {
    float(&d)[T::NT * 4] = *reinterpret_cast<float(*)[T::NT * 4]>(&c[0][0]);
    wgmma_pin(d, T::NT * 4);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const uint64_t bd = make_wgmma_desc_sw128(tb + ks * 2048, 64 * 128, 1024);   // MN-major: atoms 8 KiB apart
      if constexpr (HD == 64) wgmma_m64n64k16_rs<1>(d, p[ks], bd);
      else wgmma_m64n128k16_rs<1>(d, p[ks], bd);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_pin(d, T::NT * 4);
  } else {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const int krow = ks * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
#pragma unroll
      for (int np = 0; np < T::NT / 2; ++np) {
        uint32_t b0, b1, b2, b3;
        ldsm4t(tb + T::off(krow, np * 2 + (lane >> 4)), b0, b1, b2, b3);
        mma16816(c[np * 2], p[ks], b0, b1);
        mma16816(c[np * 2 + 1], p[ks], b2, b3);
      }
    }
  }
}

__device__ __forceinline__ void c_to_a(const float (&c)[8][4], uint32_t (&a)[4][4]) {
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    a[ks][0] = pack_bf16x2(c[2 * ks][0], c[2 * ks][1]);
    a[ks][1] = pack_bf16x2(c[2 * ks][2], c[2 * ks][3]);
    a[ks][2] = pack_bf16x2(c[2 * ks + 1][0], c[2 * ks + 1][1]);
    a[ks][3] = pack_bf16x2(c[2 * ks + 1][2], c[2 * ks + 1][3]);
  }
}

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

extern __shared__ uint8_t dyn_smem[];

// ================================================================ forward
template <int HD, bool WG>
__global__ void __launch_bounds__(THREADS) fwd_kernel(const Params p_in) {
  Params p = p_in;
  if (p.pure_causal != nullptr && *p.pure_causal != 0) { p.mask = nullptr; p.causal = 1; }
  using T = Tile<HD>;
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(dyn_smem) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = base;
  uint8_t* sK[2] = {base + T::BYTES, base + 2 * T::BYTES};
  uint8_t* sV[2] = {base + 3 * T::BYTES, base + 4 * T::BYTES};

  const int q0 = blockIdx.x * BQ, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const __nv_bfloat16* qp = p.q + b * p.q_bs + h * HD;
  const __nv_bfloat16* kp = p.k + b * p.k_bs + h * HD;
  const __nv_bfloat16* vp = p.v + b * p.v_bs + h * HD;
  const int nblk = causal_tiles(p, q0);

  load_tile<HD>(sQ, qp, p.ldq, q0, p.nq);
  if (nblk > 0) { load_tile<HD>(sK[0], kp, p.ldk, 0, p.nk); load_tile<HD>(sV[0], vp, p.ldv, 0, p.nk); }
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
      load_tile<HD>(sK[buf ^ 1], kp, p.ldk, (j + 1) * BKV, p.nk);
      load_tile<HD>(sV[buf ^ 1], vp, p.ldv, (j + 1) * BKV, p.nk);
      cp_commit();
      cp_wait<1>();
    } else {
      cp_wait<0>();
    }
    if constexpr (WG) fence_proxy_async_smem();   // cp.async (generic proxy) -> wgmma reads
    __syncthreads();
    float s[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; }
    mma_rows_x_tileT<HD, WG>(s, sQ, warp * 16, sK[buf]);
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
    mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, 1)); mx_a = fmaxf(mx_a, __shfl_xor_sync(0xffffffffu, mx_a, 2));
    mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, 1)); mx_b = fmaxf(mx_b, __shfl_xor_sync(0xffffffffu, mx_b, 2));
    const float mn_a = fmaxf(m_a, mx_a), mn_b = fmaxf(m_b, mx_b);
    const float sub_a = (mn_a == -INFINITY) ? 0.f : mn_a, sub_b = (mn_b == -INFINITY) ? 0.f : mn_b;
    const float corr_a = ex2_approx(m_a - sub_a), corr_b = ex2_approx(m_b - sub_b);
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
    for (int i = 0; i < T::NT; ++i) { o[i][0] *= corr_a; o[i][1] *= corr_a; o[i][2] *= corr_b; o[i][3] *= corr_b; }
    uint32_t pa[4][4], pl[4][4];
    c_to_a_split(s, pa, pl);
    mma_p_x_tile<HD, WG>(o, pa, sV[buf]);
    mma_p_x_tile<HD, WG>(o, pl, sV[buf]);
    __syncthreads();
  }
  if (nblk == 0) cp_wait<0>();

  l_a += __shfl_xor_sync(0xffffffffu, l_a, 1); l_a += __shfl_xor_sync(0xffffffffu, l_a, 2);
  l_b += __shfl_xor_sync(0xffffffffu, l_b, 1); l_b += __shfl_xor_sync(0xffffffffu, l_b, 2);
  const float inv_a = l_a > 0.f ? 1.f / l_a : 0.f, inv_b = l_b > 0.f ? 1.f / l_b : 0.f;
  __nv_bfloat16* op = p.out + b * p.o_bs + h * HD;
#pragma unroll
  for (int i = 0; i < T::NT; ++i) {
    const int col = i * 8 + 2 * t;
    if (row_a < p.nq) *reinterpret_cast<uint32_t*>(op + (long long)row_a * p.ldo + col) = pack_bf16x2(o[i][0] * inv_a, o[i][1] * inv_a);
    if (row_b < p.nq) *reinterpret_cast<uint32_t*>(op + (long long)row_b * p.ldo + col) = pack_bf16x2(o[i][2] * inv_b, o[i][3] * inv_b);
  }
  if (p.lse != nullptr && t == 0) {   // log2-domain LSE (the backward works in the same domain)
    float* lp = p.lse + ((long long)b * p.heads + h) * p.nq;
    if (row_a < p.nq) lp[row_a] = l_a > 0.f ? m_a + log2f(l_a) : 0.f;
    if (row_b < p.nq) lp[row_b] = l_b > 0.f ? m_b + log2f(l_b) : 0.f;
  }
}

// ================================================================ delta = rowsum(dO * O)
template <int HD>
__global__ void delta_kernel(const Params p) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long total = (long long)p.batch * p.heads * p.nq;
  if (row >= total) return;
  const int lane = threadIdx.x & 31;
  const int qi = (int)(row % p.nq), h = (int)((row / p.nq) % p.heads), b = (int)(row / ((long long)p.nq * p.heads));
  const __nv_bfloat16* op = p.o + b * p.o_bs + (long long)qi * p.ldo + h * HD;
  const __nv_bfloat16* dop = p.d_o + b * p.o_bs + (long long)qi * p.ldo + h * HD;
  float v = 0.f;
#pragma unroll
  for (int c = 0; c < HD / 64; ++c) {
    const uint32_t a = *reinterpret_cast<const uint32_t*>(op + c * 64 + 2 * lane);
    const uint32_t d = *reinterpret_cast<const uint32_t*>(dop + c * 64 + 2 * lane);
    v += bf16_lo(a) * bf16_lo(d) + bf16_hi(a) * bf16_hi(d);
  }
  v = warp_sum(v);
  if (lane == 0) p.delta[row] = v;
}

// ================================================================ dQ (CTA = 64 queries, loop key tiles)
template <int HD, bool WG>
__global__ void __launch_bounds__(THREADS) bwd_dq_kernel(const Params p_in) {
  Params p = p_in;
  if (p.pure_causal != nullptr && *p.pure_causal != 0) { p.mask = nullptr; p.causal = 1; }
  using T = Tile<HD>;
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(dyn_smem) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = base;
  uint8_t* sdO = base + T::BYTES;
  uint8_t* sK[2] = {base + 2 * T::BYTES, base + 3 * T::BYTES};
  uint8_t* sV[2] = {base + 4 * T::BYTES, base + 5 * T::BYTES};

  const int q0 = blockIdx.x * BQ, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const __nv_bfloat16* qp = p.q + b * p.q_bs + h * HD;
  const __nv_bfloat16* kp = p.k + b * p.k_bs + h * HD;
  const __nv_bfloat16* vp = p.v + b * p.v_bs + h * HD;
  const __nv_bfloat16* dop = p.d_o + b * p.o_bs + h * HD;
  const int nblk = causal_tiles(p, q0);

  load_tile<HD>(sQ, qp, p.ldq, q0, p.nq);
  load_tile<HD>(sdO, dop, p.ldo, q0, p.nq);
  if (nblk > 0) { load_tile<HD>(sK[0], kp, p.ldk, 0, p.nk); load_tile<HD>(sV[0], vp, p.ldv, 0, p.nk); }
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
      load_tile<HD>(sK[buf ^ 1], kp, p.ldk, (j + 1) * BKV, p.nk);
      load_tile<HD>(sV[buf ^ 1], vp, p.ldv, (j + 1) * BKV, p.nk);
      cp_commit();
      cp_wait<1>();
    } else {
      cp_wait<0>();
    }
    if constexpr (WG) fence_proxy_async_smem();   // cp.async (generic proxy) -> wgmma reads
    __syncthreads();
    float s[8][4], dpv[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; dpv[i][0] = dpv[i][1] = dpv[i][2] = dpv[i][3] = 0.f; }
    mma_rows_x_tileT<HD, WG>(s, sQ, warp * 16, sK[buf]);     // S  = Q K^T
    mma_rows_x_tileT<HD, WG>(dpv, sdO, warp * 16, sV[buf]);  // dP = dO V^T
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
    mma_p_x_tile<HD, WG>(dq, dsa, sK[buf]);                  // dQ += dS K
    __syncthreads();
  }
  if (nblk == 0) cp_wait<0>();

  __nv_bfloat16* dqp = p.dq + b * p.dq_bs + h * HD;
#pragma unroll
  for (int i = 0; i < T::NT; ++i) {
    const int col = i * 8 + 2 * t;
    if (row_a < p.nq) *reinterpret_cast<uint32_t*>(dqp + (long long)row_a * p.lddq + col) = pack_bf16x2(dq[i][0], dq[i][1]);
    if (row_b < p.nq) *reinterpret_cast<uint32_t*>(dqp + (long long)row_b * p.lddq + col) = pack_bf16x2(dq[i][2], dq[i][3]);
  }
}

// ================================================================ dK, dV (CTA = 64 keys, loop query tiles)
template <int HD, bool WG>
__global__ void __launch_bounds__(THREADS) bwd_dkv_kernel(const Params p_in) {
  Params p = p_in;
  if (p.pure_causal != nullptr && *p.pure_causal != 0) { p.mask = nullptr; p.causal = 1; }
  using T = Tile<HD>;
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(dyn_smem) + 1023) & ~uintptr_t(1023));
  uint8_t* sK = base;
  uint8_t* sV = base + T::BYTES;
  uint8_t* sQ[2] = {base + 2 * T::BYTES, base + 3 * T::BYTES};
  uint8_t* sdO[2] = {base + 4 * T::BYTES, base + 5 * T::BYTES};
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
  if (qb0 < nqb) { load_tile<HD>(sQ[0], qp, p.ldq, qb0 * BQ, p.nq); load_tile<HD>(sdO[0], dop, p.ldo, qb0 * BQ, p.nq); }
  cp_commit();
  if (qb0 < nqb) stage_rows(0, qb0);

  float dk[T::NT][4], dv[T::NT][4];
#pragma unroll
  for (int i = 0; i < T::NT; ++i) { dk[i][0] = dk[i][1] = dk[i][2] = dk[i][3] = 0.f; dv[i][0] = dv[i][1] = dv[i][2] = dv[i][3] = 0.f; }
  const int key_a = k0 + warp * 16 + g, key_b = key_a + 8;

  for (int qb = qb0; qb < nqb; ++qb) {
    const int buf = (qb - qb0) & 1;
    if (qb + 1 < nqb) {
      load_tile<HD>(sQ[buf ^ 1], qp, p.ldq, (qb + 1) * BQ, p.nq);
      load_tile<HD>(sdO[buf ^ 1], dop, p.ldo, (qb + 1) * BQ, p.nq);
      cp_commit();
      stage_rows(buf ^ 1, qb + 1);
      cp_wait<1>();
    } else {
      cp_wait<0>();
    }
    if constexpr (WG) fence_proxy_async_smem();   // cp.async (generic proxy) -> wgmma reads
    __syncthreads();
    float st[8][4], dpt[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) { st[i][0] = st[i][1] = st[i][2] = st[i][3] = 0.f; dpt[i][0] = dpt[i][1] = dpt[i][2] = dpt[i][3] = 0.f; }
    mma_rows_x_tileT<HD, WG>(st, sK, warp * 16, sQ[buf]);     // S^T  = K Q^T   [16 keys x 64 queries]
    mma_rows_x_tileT<HD, WG>(dpt, sV, warp * 16, sdO[buf]);   // dP^T = V dO^T
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
    mma_p_x_tile<HD, WG>(dv, pa, sdO[buf]);     // dV += P^T dO
    mma_p_x_tile<HD, WG>(dk, dsa, sQ[buf]);     // dK += dS^T Q
    __syncthreads();
  }
  if (qb0 >= nqb) cp_wait<0>();

  __nv_bfloat16* dkp = p.dk + b * p.dk_bs + h * HD;
  __nv_bfloat16* dvp = p.dv + b * p.dv_bs + h * HD;
#pragma unroll
  for (int i = 0; i < T::NT; ++i) {
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

static int validate(const Params& p, int head_dim) {
  if (head_dim != 64 && head_dim != 128) return ofk_set_error(OFK_ERR_ARG, "dense attention: head_dim must be 64 or 128");
  if (p.batch <= 0 || p.heads <= 0 || p.nq <= 0 || p.nk <= 0) return ofk_set_error(OFK_ERR_ARG, "dense attention: empty problem");
  if ((p.ldq | p.ldk | p.ldv | p.ldo) % 8 != 0) return ofk_set_error(OFK_ERR_ALIGN, "dense attention: row strides must be multiples of 8");
  if (p.batch > 65535 || p.heads > 65535) return ofk_set_error(OFK_ERR_ARG, "dense attention: batch/heads exceed grid limits");
  return 0;
}

template <int HD, bool WG>
static int launch_fwd_impl(const Params& p, cudaStream_t s) {
  constexpr int SMEM = 5 * Tile<HD>::BYTES + 1024;
  static bool done = false;
  if (!done) { cudaFuncSetAttribute(fwd_kernel<HD, WG>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM); done = true; }
  dim3 grid((p.nq + BQ - 1) / BQ, p.heads, p.batch);
  fwd_kernel<HD, WG><<<grid, THREADS, SMEM, s>>>(p);
  OFK_CHECK_LAUNCH();
  return 0;
}
template <int HD>
static int launch_fwd(const Params& p, cudaStream_t s) {
  if (!ofk_attn_use_wgmma()) return launch_fwd_impl<HD, false>(p, s);
  if (int rc = launch_fwd_impl<HD, true>(p, s)) return rc;
  ofk_attn_count_wgmma();
  return 0;
}

template <int HD, bool WG>
static int launch_bwd_impl(const Params& p, cudaStream_t s) {
  constexpr int SMEM = 6 * Tile<HD>::BYTES + 1024;
  static bool done = false;
  if (!done) {
    cudaFuncSetAttribute(bwd_dq_kernel<HD, WG>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    cudaFuncSetAttribute(bwd_dkv_kernel<HD, WG>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM);
    done = true;
  }
  const long long rows = (long long)p.batch * p.heads * p.nq;
  delta_kernel<HD><<<(unsigned)((rows + 7) / 8), 256, 0, s>>>(p);
  OFK_CHECK_LAUNCH();
  dim3 gq((p.nq + BQ - 1) / BQ, p.heads, p.batch);
  bwd_dq_kernel<HD, WG><<<gq, THREADS, SMEM, s>>>(p);
  OFK_CHECK_LAUNCH();
  dim3 gk((p.nk + BKV - 1) / BKV, p.heads, p.batch);
  bwd_dkv_kernel<HD, WG><<<gk, THREADS, SMEM, s>>>(p);
  OFK_CHECK_LAUNCH();
  return 0;
}
template <int HD>
static int launch_bwd(const Params& p, cudaStream_t s) {
  if (!ofk_attn_use_wgmma()) return launch_bwd_impl<HD, false>(p, s);
  if (int rc = launch_bwd_impl<HD, true>(p, s)) return rc;
  ofk_attn_count_wgmma();
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
  if (int rc = validate(p, head_dim)) return rc;
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
  if (int rc = validate(p, head_dim)) return rc;
  return head_dim == 64 ? launch_bwd<64>(p, (cudaStream_t)stream) : launch_bwd<128>(p, (cudaStream_t)stream);
}
