// Tile layer of the training attention cores: attention.cu (media rules, head_dim 64) and attention_dense.cu (MPT
// rules, head_dim 64 and 128).  One CTA is one warpgroup of 4 warps x 16 rows; 64-row tiles of Q/K/V/dO are staged by
// cp.async into 128-byte-swizzled shared memory, both products are warpgroup-wide wgmma, and every per-row quantity
// lives in the wgmma accumulator layout: thread (warp, g = lane / 4, t = lane % 4) holds rows a = 16 warp + g and
// b = a + 8, columns 8 i + 2 t and + 1 of n-tile i (c[i][0..1] for row a, c[i][2..3] for row b).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "ofk_ptx.cuh"

namespace ofk {

constexpr int BQ = 64, BKV = 64, THREADS = 128;   // query rows per CTA, keys per tile, one warpgroup
constexpr float LOG2E = 1.4426950408889634f;

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

// Load rows [row0, row0 + 64) x HD columns (starting at `g`, row stride ld) into a swizzled tile; rows >= nrows -> 0.
template <int HD>
__device__ __forceinline__ void load_tile(uint8_t* tile, const __nv_bfloat16* g, long long ld, int row0, int nrows) {
  using T = Tile<HD>;
  const uint32_t base = smem_u32(tile);
#pragma unroll
  for (int i = 0; i < (64 * T::CHUNKS) / THREADS; ++i) {
    const unsigned idx = threadIdx.x + i * THREADS;   // unsigned: the division and remainder are a shift and a mask
    const int r = idx / T::CHUNKS, c = idx % T::CHUNKS;
    const bool valid = (row0 + r) < nrows;
    cp_async16(base + T::off(r, c), g + (long long)(valid ? (row0 + r) : 0) * ld + c * 8, valid);
  }
}

// Tiles live in dynamic shared memory aligned by hand: the 128-byte swizzle wgmma reads is a function of the absolute
// shared address, so every tile must start on a 1024-byte boundary (launches reserve 1024 bytes of slack).
extern __shared__ uint8_t dyn_smem[];
__device__ __forceinline__ uint8_t* smem_base() {
  return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(dyn_smem) + 1023) & ~uintptr_t(1023));
}
// Tile i of a kernel's shared-memory layout.  Double-buffered stages are addressed as tile_at(first + buf): an address
// computed from the stage index, where an array of stage pointers indexed by buf would be kept in local memory.
template <int HD>
__device__ __forceinline__ uint8_t* tile_at(int i) { return smem_base() + i * Tile<HD>::BYTES; }

__device__ __forceinline__ void wgmma_pin(float* d, int n) {
  for (int i = 0; i < n; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// C[64 x 64] += X * T^T, X and T both [64 rows][HD] tiles (contraction over HD): QK^T-shaped.
template <int HD>
__device__ __forceinline__ void mma_rows_x_tileT(float (&c)[8][4], const uint8_t* xt, const uint8_t* tile) {
  using T = Tile<HD>;
  const uint32_t xb = smem_u32(xt), tb = smem_u32(tile);
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
}

// C[64 x HD] += P[64 x 64(k)] * T, P from registers (A-fragment layout), T = [64 k][HD n] tile.
template <int HD>
__device__ __forceinline__ void mma_p_x_tile(float (&c)[Tile<HD>::NT][4], const uint32_t (&p)[4][4], const uint8_t* tile) {
  using T = Tile<HD>;
  const uint32_t tb = smem_u32(tile);
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

// One online-softmax step over a log2-domain score tile s, given this thread's partial row maxima mx_a / mx_b: the
// maxima are completed across the 4 lanes sharing a row, s becomes exp2(s - m), its row sums are added to l, and l and
// the accumulator o are rescaled by exp2(m_old - m_new).  A row without a finite score keeps m = -inf and subtracts 0.
template <int NT>
__device__ __forceinline__ void softmax_step(float (&s)[8][4], float mx_a, float mx_b, float& m_a, float& m_b,
                                             float& l_a, float& l_b, float (&o)[NT][4]) {
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
  for (int i = 0; i < NT; ++i) { o[i][0] *= corr_a; o[i][1] *= corr_a; o[i][2] *= corr_b; o[i][3] *= corr_b; }
}

// Completes a row sum across the 4 lanes sharing the row.
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// Rows a and b of an accumulator, times sa / sb, as bf16 into out (row stride ld); rows >= nrows are not written.
template <int NT>
__device__ __forceinline__ void store_rows(__nv_bfloat16* out, long long ld, const float (&c)[NT][4], float sa, float sb,
                                           int row_a, int row_b, int nrows, int t) {
#pragma unroll
  for (int i = 0; i < NT; ++i) {
    const int col = i * 8 + 2 * t;
    if (row_a < nrows) *reinterpret_cast<uint32_t*>(out + (long long)row_a * ld + col) = pack_bf16x2(c[i][0] * sa, c[i][1] * sa);
    if (row_b < nrows) *reinterpret_cast<uint32_t*>(out + (long long)row_b * ld + col) = pack_bf16x2(c[i][2] * sb, c[i][3] * sb);
  }
}

// log2-domain LSE of rows a and b into lp[row] (the backward works in the same domain); a row with no mass gets the
// sentinel 0, which recomputes P as 0 there because every one of its scores is -inf.
__device__ __forceinline__ void store_lse(float* lp, float m_a, float l_a, float m_b, float l_b, int row_a, int row_b,
                                          int nrows) {
  if (row_a < nrows) lp[row_a] = l_a > 0.f ? m_a + log2f(l_a) : 0.f;
  if (row_b < nrows) lp[row_b] = l_b > 0.f ? m_b + log2f(l_b) : 0.f;
}

// delta[b, h, q] = rowsum(dO * O) over the head's HD columns; one warp per row.  o and d_o share strides.
template <int HD>
__global__ void delta_kernel(const __nv_bfloat16* o, const __nv_bfloat16* d_o, float* delta, int batch, int heads,
                             int nq, long long bs, long long ld) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long total = (long long)batch * heads * nq;
  if (row >= total) return;
  const int lane = threadIdx.x & 31;
  const int qi = (int)(row % nq), h = (int)((row / nq) % heads), b = (int)(row / ((long long)nq * heads));
  const __nv_bfloat16* op = o + b * bs + (long long)qi * ld + h * HD;
  const __nv_bfloat16* dop = d_o + b * bs + (long long)qi * ld + h * HD;
  float v = 0.f;
#pragma unroll
  for (int c = 0; c < HD / 64; ++c) {
    const uint32_t a = *reinterpret_cast<const uint32_t*>(op + c * 64 + 2 * lane);
    const uint32_t d = *reinterpret_cast<const uint32_t*>(dop + c * 64 + 2 * lane);
    v += bf16_lo(a) * bf16_lo(d) + bf16_hi(a) * bf16_hi(d);
  }
  v = warp_sum(v);
  if (lane == 0) delta[row] = v;
}

static inline bool aligned(const void* ptr, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(ptr) & (bytes - 1)) == 0; }

}  // namespace ofk
