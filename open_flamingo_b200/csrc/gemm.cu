// bf16 x bf16 -> fp32 GEMM for sm_90a: TMA-staged operands (128B swizzle), wgmma with the accumulator in registers,
// a warp-specialised persistent CTA (one producer warp, two consumer warpgroups), fused epilogues.
//
//   out[m, n] = epilogue( sum_k A(m, k) * B(n, k) )
//
// Operand storage ("major"):
//   K-major  : X is [rows, K] row-major (K contiguous)             -- forward  Y = X W^T
//   MN-major : X is [K, rows] row-major (rows contiguous)          -- dgrad (B = W) / wgrad (A = dY, B = X)
// so no transposed copies of weights or activations are ever materialised: wgmma reads either layout of a bf16
// operand straight from shared memory (its transpose bits).
//
// This kernel replaces every nn.Linear on the reference hot path:
//   helpers.py:15-22 (FeedForward), :35-37 / :52-54 / :65 (PerceiverAttention to_q/to_kv/to_out),
//   :153-155 / :186-189 / :233 (MaskedCrossAttention to_q/to_kv/to_out), and the gate/residual
//   arithmetic of helpers.py:267-277 in its epilogue; plus the open_clip ViT linears (third party).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <mutex>
#include <unordered_map>

#include "ofk_internal.h"
#include "ofk_ptx.cuh"

namespace ofk {

constexpr int BM = 128;       // two consumer warpgroups x wgmma M = 64
constexpr int BN = 128;       // wgmma N
constexpr int BK = 64;        // one 128-byte swizzle atom of bf16
constexpr int WGMMA_K = 16;   // fixed for 16-bit inputs
constexpr int STAGES = 4;     // TMA ring depth (32 KiB per stage)
// Warp roles: warpgroup 0 = producer (warp 0 lane 0 issues every TMA load; the other warps only take part in set-up),
// warpgroups 1 and 2 = consumers, each owning 64 accumulator rows of the 128 x 128 tile through mainloop and epilogue.
constexpr int NUM_CONSUMER_WG = 2;
constexpr int NUM_EPI_WARPS = 4 * NUM_CONSUMER_WG;
constexpr int NUM_THREADS = 128 * (1 + NUM_CONSUMER_WG);
constexpr int GROUP_M = 8;        // tile rasterisation: GROUP_M m-tiles x all n-tiles are walked together (L2 reuse)

struct GemmParams {
  int M, N, K;
  int splits;        // split-K factor (>1 only with the atomic epilogue)
  int kb_per_split;  // k-blocks per split
  void* out;
  long long ldo;
  void* out2;
  long long ldo2;
  const void* aux;
  long long ldaux;
  const float* bias;
  const float* gate;
  int stream_out;    // 1: epilogue outputs use st.global.cs (evict-first) so they do not displace the operand panels in L2
  // Grouped row maps (0 = identity): logical row r -> (r / rpg) * gs + go + r % rpg.  `out_*` places the rows of `out`
  // inside a larger interleaved buffer (the media / latent halves of PerceiverAttention's cat((x, latents), -2),
  // helpers.py:53); `ak_*` does the same for the REDUCTION rows of an MN-major A operand (wgrad over one half).
  int out_rpg, out_gs, out_go;
  int ak_rpg, ak_gs, ak_go;
};
__device__ __forceinline__ long long map_rows(long long r, int rpg, int gs, int go) {
  return rpg > 0 ? (r / rpg) * gs + go + r % rpg : r;
}

// Work item -> (m tile, n tile, k split).  Within a split, tiles are walked in groups of GROUP_M m-tiles by all
// n-tiles, m fastest, so the tiles in flight share GROUP_M row panels of A and a few column panels of B through L2.
__device__ __forceinline__ void work_to_tile(int w, int m_tiles, int n_tiles, int& mt, int& nt, int& ks) {
  const int per_split = m_tiles * n_tiles;
  ks = w / per_split;
  const int r = w - ks * per_split;
  const int group_sz = GROUP_M * n_tiles;
  const int g = r / group_sz;
  const int first_m = g * GROUP_M;
  const int gm = min(GROUP_M, m_tiles - first_m);
  const int in_g = r - g * group_sz;
  mt = first_m + in_g % gm;
  nt = in_g / gm;
}

// ----------------------------------------------------------------------------------------------
// Epilogue.  One warp drains 32 accumulator rows (lane = row) x 32 columns per round.  A lane owns a ROW, so a
// naive "each lane stores its row" epilogue issues warp stores that touch 32 different cache lines.
// Instead every global access goes through a per-warp shared-memory staging tile and is re-issued TRANSPOSED:
// consecutive lanes touch consecutive 16-byte pieces of the same row (4 or 8 rows per instruction), i.e. full
// 64/128-byte segments.  The same staging tile is used for the epilogue's reads (residual, saved pre-activation).
constexpr int STAGE_ROW = 128;                     // unpadded 128 B rows; the 16-byte piece index is XOR-swizzled with
constexpr int STAGE_BYTES_PER_WARP = 32 * STAGE_ROW;   // (row & 7) so row-wise and piece-wise accesses are conflict-free
__device__ __forceinline__ uint32_t stage_off(int row, int piece) { return (uint32_t)(row * STAGE_ROW + ((piece ^ (row & 7)) << 4)); }


__device__ __forceinline__ void st_shared_v4(uint32_t addr, uint4 v) {
  asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint4 ld_shared_v4(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
  return v;
}

// Store this warp's 32 x 32 tile (lane's row in `w`: WORDS = 32 for f32, 16 for bf16) to global, coalesced.
// MODE 0 = plain store, 1 = red.global.add.f32 (f32 only).
__device__ __forceinline__ void st_global_cs_v4(void* g, uint4 v) {
  asm volatile("st.global.cs.v4.b32 [%0], {%1,%2,%3,%4};" ::"l"(g), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

template <int ELEM_BYTES, int MODE>
__device__ __forceinline__ void warp_store_tile(uint32_t stage, const uint32_t* w, void* gbase, long long ld, int row0,
                                                int col0, int M, int N, int streaming = 0, int rpg = 0, int gs = 0,
                                                int go = 0) {
  constexpr int PIECES = ELEM_BYTES * 2;            // 16-byte pieces per 32-element row: 8 (f32) or 4 (bf16)
  constexpr int EPP = 16 / ELEM_BYTES;              // elements per piece
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int i = 0; i < PIECES; ++i)
    st_shared_v4(stage + stage_off(lane, i), make_uint4(w[4 * i], w[4 * i + 1], w[4 * i + 2], w[4 * i + 3]));
  __syncwarp();
  const int piece = lane % PIECES, rsub = lane / PIECES;
  const int col = col0 + piece * EPP;
#pragma unroll
  for (int it = 0; it < PIECES; ++it) {
    const int r = it * (32 / PIECES) + rsub;
    const uint4 v = ld_shared_v4(stage + stage_off(r, piece));
    const int row = row0 + r;
    if (row < M && col < N) {
      uint8_t* g = reinterpret_cast<uint8_t*>(gbase) + (map_rows(row, rpg, gs, go) * ld + col) * ELEM_BYTES;
      if constexpr (MODE == 0) {
        if (streaming) st_global_cs_v4(g, v);
        else *reinterpret_cast<uint4*>(g) = v;
      } else {
        asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(g), "f"(__uint_as_float(v.x)),
                     "f"(__uint_as_float(v.y)), "f"(__uint_as_float(v.z)), "f"(__uint_as_float(v.w))
                     : "memory");
      }
    }
  }
  __syncwarp();
}

// Epilogue operand (residual / saved pre-activation) tile, two-phase so the global latency is hidden:
//   aux_prefetch: coalesced global loads of this warp's 32 x 32 tile into registers (issued one round ahead)
//   aux_commit  : registers -> staging tile -> each lane reads its own row
template <int ELEM_BYTES>
__device__ __forceinline__ void aux_prefetch(uint4 (&pre)[ELEM_BYTES * 2], const void* gbase, long long ld, int row0,
                                             int col0, int M, int N) {
  constexpr int PIECES = ELEM_BYTES * 2;
  constexpr int EPP = 16 / ELEM_BYTES;
  const int lane = threadIdx.x & 31;
  const int piece = lane % PIECES, rsub = lane / PIECES;
  const int col = col0 + piece * EPP;
#pragma unroll
  for (int it = 0; it < PIECES; ++it) {
    const int row = row0 + it * (32 / PIECES) + rsub;
    pre[it] = make_uint4(0u, 0u, 0u, 0u);
    if (row < M && col < N)
      pre[it] = *reinterpret_cast<const uint4*>(reinterpret_cast<const uint8_t*>(gbase) + ((long long)row * ld + col) * ELEM_BYTES);
  }
}
template <int ELEM_BYTES>
__device__ __forceinline__ void aux_commit(uint32_t stage, const uint4 (&pre)[ELEM_BYTES * 2], uint32_t* w) {
  constexpr int PIECES = ELEM_BYTES * 2;
  const int lane = threadIdx.x & 31;
  const int piece = lane % PIECES, rsub = lane / PIECES;
#pragma unroll
  for (int it = 0; it < PIECES; ++it) st_shared_v4(stage + stage_off(it * (32 / PIECES) + rsub, piece), pre[it]);
  __syncwarp();
#pragma unroll
  for (int i = 0; i < PIECES; ++i) {
    const uint4 v = ld_shared_v4(stage + stage_off(lane, i));
    w[4 * i] = v.x; w[4 * i + 1] = v.y; w[4 * i + 2] = v.z; w[4 * i + 3] = v.w;
  }
  __syncwarp();
}

template <int EPI>
struct AuxBytes { static constexpr int value = (EPI == OFK_EPI_GATE_RESID_F32 || EPI == OFK_EPI_BIAS_RESID_F32) ? 4 : (EPI == OFK_EPI_DGELU_BF16 ? 2 : 0); };

__device__ __forceinline__ void pack32_bf16(const float (&v)[32], uint32_t (&w)[16]) {
#pragma unroll
  for (int i = 0; i < 16; ++i) w[i] = pack_bf16x2(v[2 * i], v[2 * i + 1]);
}

// One round: rows [row0, row0+32) (lane = row) x columns [col0, col0+32), accumulators in `acc`.
template <int EPI>
__device__ __forceinline__ void epilogue32(const GemmParams& p, float gate_t, uint32_t stage, int row0, int col0,
                                           const uint32_t (&acc)[32], uint32_t* aux_row) {
  float v[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) v[i] = __uint_as_float(acc[i]);
  constexpr bool HAS_BIAS = EPI == OFK_EPI_BIAS_BF16 || EPI == OFK_EPI_BIAS_QGELU_BF16 || EPI == OFK_EPI_BIAS_GELU_BF16 ||
                            EPI == OFK_EPI_BIAS_RESID_F32;
  if constexpr (HAS_BIAS) {
    // every lane needs the same 32 bias values: broadcast loads (one wavefront each)
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (col0 + 4 * i < p.N) {
        const float4 b = __ldg(reinterpret_cast<const float4*>(p.bias + col0) + i);
        v[4 * i] += b.x; v[4 * i + 1] += b.y; v[4 * i + 2] += b.z; v[4 * i + 3] += b.w;
      }
    }
  }

  if constexpr (EPI == OFK_EPI_STORE_BF16 || EPI == OFK_EPI_BIAS_BF16 || EPI == OFK_EPI_BIAS_QGELU_BF16 ||
                EPI == OFK_EPI_BIAS_GELU_BF16) {
    if constexpr (EPI == OFK_EPI_BIAS_QGELU_BF16) {
#pragma unroll
      for (int i = 0; i < 32; ++i) v[i] = quick_gelu(bf16_round(v[i]));
    }
    if constexpr (EPI == OFK_EPI_BIAS_GELU_BF16) {
#pragma unroll
      for (int i = 0; i < 32; ++i) v[i] = gelu_exact(bf16_round(v[i]));
    }
    uint32_t w[16];
    pack32_bf16(v, w);
    warp_store_tile<2, 0>(stage, w, p.out, p.ldo, row0, col0, p.M, p.N, p.stream_out, p.out_rpg, p.out_gs, p.out_go);
  } else if constexpr (EPI == OFK_EPI_STORE_F32) {
    warp_store_tile<4, 0>(stage, acc, p.out, p.ldo, row0, col0, p.M, p.N, p.stream_out, p.out_rpg, p.out_gs, p.out_go);
  } else if constexpr (EPI == OFK_EPI_ATOMIC_F32) {
    warp_store_tile<4, 1>(stage, acc, p.out, p.ldo, row0, col0, p.M, p.N);
  } else if constexpr (EPI == OFK_EPI_GELU_DUAL) {
    // z = bf16(acc) is what the reference's Linear emits under autocast; GELU is taken of that.
    uint32_t wz[16], wh[16];
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] = bf16_round(v[i]);
    pack32_bf16(v, wz);
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] = gelu_exact(v[i]);
    pack32_bf16(v, wh);
    warp_store_tile<2, 0>(stage, wz, p.out, p.ldo, row0, col0, p.M, p.N, p.stream_out);
    warp_store_tile<2, 0>(stage, wh, p.out2, p.ldo2, row0, col0, p.M, p.N, p.stream_out);
  } else if constexpr (EPI == OFK_EPI_GATE_RESID_F32 || EPI == OFK_EPI_BIAS_RESID_F32) {
    // out = branch * tanh(gate) + residual (fp32 residual stream); branch kept in bf16 for the gate grad.
    uint32_t* r = aux_row;   // this lane's 32 residual values (prefetched one round ahead)
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] = bf16_round(v[i]);
    if (p.out2 != nullptr) {
      uint32_t wb[16];
      pack32_bf16(v, wb);
      warp_store_tile<2, 0>(stage, wb, p.out2, p.ldo2, row0, col0, p.M, p.N, p.stream_out);
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) r[i] = __float_as_uint(fmaf(v[i], gate_t, __uint_as_float(r[i])));
    warp_store_tile<4, 0>(stage, r, p.out, p.ldo, row0, col0, p.M, p.N, p.stream_out);
  } else if constexpr (EPI == OFK_EPI_DGELU_BF16) {
    // out = bf16( bf16(acc) * gelu'(z) ), z = saved bf16 pre-activation
    uint32_t w[16];
    const uint32_t* z = aux_row;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      v[2 * i] = bf16_round(v[2 * i]) * gelu_exact_grad(bf16_lo(z[i]));
      v[2 * i + 1] = bf16_round(v[2 * i + 1]) * gelu_exact_grad(bf16_hi(z[i]));
    }
    pack32_bf16(v, w);
    warp_store_tile<2, 0>(stage, w, p.out, p.ldo, row0, col0, p.M, p.N, p.stream_out, p.out_rpg, p.out_gs, p.out_go);
  }
}

// ----------------------------------------------------------------------------------------------
// Shared memory: the TMA ring, then per consumer warpgroup a 64 x 64 fp32 accumulator slab (the register fragments
// of half the tile's columns, re-read lane = row by the epilogue), then the per-warp epilogue staging tiles.
struct SmemLayout {
  static constexpr int A_BYTES = BM * BK * 2;   // 16 KiB
  static constexpr int B_BYTES = BN * BK * 2;   // 16 KiB
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int ACC_PITCH = 64 + 8;      // floats; 8 mod 32 keeps the fragment stores conflict-free
  static constexpr int ACC_BYTES = 64 * ACC_PITCH * 4;
  static constexpr int ACC_OFF = STAGES * STAGE_BYTES;
  static constexpr int EPI_OFF = ACC_OFF + NUM_CONSUMER_WG * ACC_BYTES;
  static constexpr int BAR_OFF = EPI_OFF + NUM_EPI_WARPS * STAGE_BYTES_PER_WARP;
  static constexpr int TOTAL = BAR_OFF + 256 + 1024;   // + barriers + alignment slack
};
static_assert(SmemLayout::TOTAL <= 227 * 1024, "GEMM shared memory exceeds the sm_90 per-block limit");

template <int A_MN, int B_MN, int EPI>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
            const GemmParams p) {
  using L = SmemLayout;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  const int m_tiles = (p.M + BM - 1) / BM;
  const int n_tiles = (p.N + BN - 1) / BN;
  const int num_work = m_tiles * n_tiles * p.splits;
  const int total_kb = (p.K + BK - 1) / BK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tma_a);
    tma_prefetch_desc(&tma_b);
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], NUM_EPI_WARPS); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ===================== TMA producer (one thread) =====================
    // the producer warpgroup hands its registers to the consumers (40 + 2 x 232 per thread fit the 64K register file)
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    if (warp == 0 && lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int w = blockIdx.x; w < num_work; w += gridDim.x) {
        int mt, nt, ks;
        work_to_tile(w, m_tiles, n_tiles, mt, nt, ks);
        const int m0 = mt * BM, n0 = nt * BN;
        const int kb0 = ks * p.kb_per_split;
        const int kb1 = min(total_kb, kb0 + p.kb_per_split);
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * L::STAGE_BYTES;
          uint8_t* sb = sa + L::A_BYTES;
          mbar_arrive_expect_tx(&full_bar[stage], L::STAGE_BYTES);
          const int k0 = kb * BK;
          if constexpr (A_MN == 0) {
            tma_load_2d(sa, &tma_a, &full_bar[stage], k0, m0);             // box {64 k, 128 rows}
          } else {
#pragma unroll
            for (int i = 0; i < BM / 64; ++i)                               // boxes {64 mn, 64 k}
              tma_load_2d(sa + i * (BK * 128), &tma_a, &full_bar[stage], m0 + 64 * i, (int)map_rows(k0, p.ak_rpg, p.ak_gs, p.ak_go));
          }
          if constexpr (B_MN == 0) {
            tma_load_2d(sb, &tma_b, &full_bar[stage], k0, n0);             // box {64 k, 128 rows}
          } else {
#pragma unroll
            for (int i = 0; i < BN / 64; ++i)
              tma_load_2d(sb + i * (BK * 128), &tma_b, &full_bar[stage], n0 + 64 * i, k0);
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===================== consumers: wgmma mainloop + fused epilogue =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
  const int wg = warp / 4 - 1;               // consumer warpgroup: accumulator rows [64 wg, 64 wg + 64) of the tile
  const int wl = warp & 3;                   // warp within the warpgroup
  const int epi_warp = warp - 4;
  float* acc_slab = reinterpret_cast<float*>(smem + L::ACC_OFF + wg * L::ACC_BYTES);
  const uint32_t stage_addr = smem_u32(smem + L::EPI_OFF) + epi_warp * STAGE_BYTES_PER_WARP;
  float gate_t = 1.0f;
  if constexpr (EPI == OFK_EPI_GATE_RESID_F32) {
    if (p.gate != nullptr) gate_t = tanhf(__ldg(p.gate));
  }
  int stage = 0; uint32_t phase = 0;
  float d[64];
  for (int w = blockIdx.x; w < num_work; w += gridDim.x) {
    int mt, nt, ks;
    work_to_tile(w, m_tiles, n_tiles, mt, nt, ks);
    const int kb0 = ks * p.kb_per_split;
    const int kb1 = min(total_kb, kb0 + p.kb_per_split);
    int prev_stage = -1;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t sa = smem_u32(smem + stage * L::STAGE_BYTES);
      const uint32_t sb = sa + L::A_BYTES;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / WGMMA_K; ++k) {
        // K-major : this warpgroup's 64 rows start 64 * 128 B in; 8-row groups 1024 B apart (SBO); advance 32 B per
        //           WGMMA_K inside the swizzle atom.
        // MN-major: 64-wide MN chunks BK * 128 B apart (LBO; this warpgroup's rows are chunk `wg`), 8-k groups 1024 B
        //           apart (SBO); advance 2 k-groups = 2048 B per WGMMA_K.
        const uint64_t adesc = A_MN ? make_wgmma_desc_sw128(sa + wg * (BK * 128) + k * 2048, BK * 128, 1024)
                                    : make_wgmma_desc_sw128(sa + wg * (64 * 128) + k * 32, 16, 1024);
        const uint64_t bdesc = B_MN ? make_wgmma_desc_sw128(sb + k * 2048, BK * 128, 1024)
                                    : make_wgmma_desc_sw128(sb + k * 32, 16, 1024);
        wgmma_m64n128k16_bf16<A_MN, B_MN>(d, adesc, bdesc, (kb > kb0 || k > 0) ? 1u : 0u);
      }
      wgmma_commit();
      // keep one k-block of MMAs in flight; the one before it has retired, so its ring slot can be refilled
      wgmma_wait<1>();
      if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);
      prev_stage = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);

    // Epilogue, in two halves of 64 columns: fragments -> slab, then each warp re-reads one 32 x 32 block with
    // lane = row and runs the shared fused epilogue on it.
    const int rh = wl & 1, ch = wl >> 1;
    const int row0 = mt * BM + wg * 64 + rh * 32;
    constexpr int AUXB = AuxBytes<EPI>::value;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      named_bar_sync(1 + wg, 128);           // the previous half's readers are done with the slab
      const int fr = 16 * wl + lane / 4, fc = 2 * (lane % 4);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int i = 4 * (8 * h + j);
        *reinterpret_cast<float2*>(acc_slab + fr * L::ACC_PITCH + 8 * j + fc) = make_float2(d[i], d[i + 1]);
        *reinterpret_cast<float2*>(acc_slab + (fr + 8) * L::ACC_PITCH + 8 * j + fc) = make_float2(d[i + 2], d[i + 3]);
      }
      named_bar_sync(1 + wg, 128);
      uint32_t acc[32];
      const float* src = acc_slab + (rh * 32 + lane) * L::ACC_PITCH + ch * 32;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float4 v = *reinterpret_cast<const float4*>(src + 4 * i);
        acc[4 * i] = __float_as_uint(v.x); acc[4 * i + 1] = __float_as_uint(v.y);
        acc[4 * i + 2] = __float_as_uint(v.z); acc[4 * i + 3] = __float_as_uint(v.w);
      }
      const int col = nt * BN + h * 64 + ch * 32;
      if (row0 < p.M && col < p.N) {                                                 // warp-uniform
        uint32_t aux_row[AUXB ? AUXB * 8 : 1];
        if constexpr (AUXB != 0) {
          uint4 pre[AUXB * 2];
          aux_prefetch<AUXB>(pre, p.aux, p.ldaux, row0, col, p.M, p.N);
          aux_commit<AUXB>(stage_addr, pre, aux_row);
        }
        epilogue32<EPI>(p, gate_t, stage_addr, row0, col, acc, aux_row);
      }
    }
  }
}

// ----------------------------------------------------------------------------------------------
// ----------------------------------------------------------------------------------------------
// Host side: tensor-map cache + dispatch.
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(f);
  });
  return fn;
}

struct MapKey {
  const void* ptr; long long ld; int rows, cols, box_inner, box_outer;
  bool operator==(const MapKey& o) const {
    return ptr == o.ptr && ld == o.ld && rows == o.rows && cols == o.cols && box_inner == o.box_inner &&
           box_outer == o.box_outer;
  }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    size_t h = reinterpret_cast<size_t>(k.ptr);
    h = h * 1000003u ^ (size_t)k.ld; h = h * 1000003u ^ (size_t)k.rows; h = h * 1000003u ^ (size_t)k.cols;
    h = h * 1000003u ^ (size_t)(k.box_inner * 1024 + k.box_outer);
    return h;
  }
};

// 2-D bf16 row-major tensor [rows, cols] (cols contiguous, row stride ld elements), 128B swizzle.
static int get_tensor_map(const void* ptr, long long ld, int rows, int cols, int box_inner, int box_outer,
                          CUtensorMap* out) {
  static std::mutex mu;
  static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> cache;
  MapKey key{ptr, ld, rows, cols, box_inner, box_outer};
  {
    std::lock_guard<std::mutex> g(mu);
    auto it = cache.find(key);
    if (it != cache.end()) { *out = it->second; return 0; }
  }
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) return ofk_set_error(OFK_ERR_DRIVER, "cuTensorMapEncodeTiled entry point not found");
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) || ((ld * 2) & 15))
    return ofk_set_error(OFK_ERR_ALIGN, "GEMM operand must be 16-byte aligned with a 16-byte-multiple row stride");
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)box_inner, (cuuint32_t)box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUtensorMap m;
  CUresult r = enc(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[160];
    snprintf(buf, sizeof buf, "cuTensorMapEncodeTiled failed (%d) rows=%d cols=%d ld=%lld box=%dx%d", (int)r, rows,
             cols, ld, box_inner, box_outer);
    return ofk_set_error(OFK_ERR_DRIVER, buf);
  }
  {
    std::lock_guard<std::mutex> g(mu);
    if (cache.size() > 4096) cache.clear();
    cache.emplace(key, m);
  }
  *out = m;
  return 0;
}

static int g_num_sms = 0;
static int g_reserved_sms = 0;   // SMs the persistent grids leave free (ofk_gemm_reserve_sms): room for NCCL's CTAs

template <int A_MN, int B_MN, int EPI>
static int launch(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, cudaStream_t stream) {
  auto kern = gemm_kernel<A_MN, B_MN, EPI>;
  static bool attr_done = false;
  if (!attr_done) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SmemLayout::TOTAL);
    if (e != cudaSuccess) return ofk_set_error(OFK_ERR_CUDA, cudaGetErrorString(e));
    attr_done = true;
  }
  const int m_tiles = (p.M + BM - 1) / BM, n_tiles = (p.N + BN - 1) / BN;
  const int work = m_tiles * n_tiles * p.splits;
  const int avail = g_num_sms - g_reserved_sms;
  const int grid = work < avail ? work : avail;
  kern<<<grid, NUM_THREADS, SmemLayout::TOTAL, stream>>>(ta, tb, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return ofk_set_error(OFK_ERR_CUDA, cudaGetErrorString(e));
  ofk_count_launch();
  return 0;
}

template <int EPI>
static int dispatch_major(int a_mn, int b_mn, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p,
                          cudaStream_t s) {
  if (a_mn == 0 && b_mn == 0) return launch<0, 0, EPI>(ta, tb, p, s);
  if (a_mn == 0 && b_mn == 1) return launch<0, 1, EPI>(ta, tb, p, s);
  if (a_mn == 1 && b_mn == 1) return launch<1, 1, EPI>(ta, tb, p, s);
  return launch<1, 0, EPI>(ta, tb, p, s);
}

static int dispatch_epi(int epi, int a_mn, int b_mn, const CUtensorMap& ta, const CUtensorMap& tb,
                        const GemmParams& p, cudaStream_t s) {
  switch (epi) {
    case OFK_EPI_STORE_BF16: return dispatch_major<OFK_EPI_STORE_BF16>(a_mn, b_mn, ta, tb, p, s);
    case OFK_EPI_STORE_F32: return dispatch_major<OFK_EPI_STORE_F32>(a_mn, b_mn, ta, tb, p, s);
    case OFK_EPI_ATOMIC_F32: return dispatch_major<OFK_EPI_ATOMIC_F32>(a_mn, b_mn, ta, tb, p, s);
    case OFK_EPI_BIAS_BF16: return dispatch_major<OFK_EPI_BIAS_BF16>(a_mn, b_mn, ta, tb, p, s);
    case OFK_EPI_BIAS_QGELU_BF16: return dispatch_major<OFK_EPI_BIAS_QGELU_BF16>(a_mn, b_mn, ta, tb, p, s);
    case OFK_EPI_GELU_DUAL: return dispatch_major<OFK_EPI_GELU_DUAL>(a_mn, b_mn, ta, tb, p, s);
    case OFK_EPI_GATE_RESID_F32: return dispatch_major<OFK_EPI_GATE_RESID_F32>(a_mn, b_mn, ta, tb, p, s);
    case OFK_EPI_DGELU_BF16: return dispatch_major<OFK_EPI_DGELU_BF16>(a_mn, b_mn, ta, tb, p, s);
    case OFK_EPI_BIAS_RESID_F32: return dispatch_major<OFK_EPI_BIAS_RESID_F32>(a_mn, b_mn, ta, tb, p, s);
    case OFK_EPI_BIAS_GELU_BF16: return dispatch_major<OFK_EPI_BIAS_GELU_BF16>(a_mn, b_mn, ta, tb, p, s);
  }
  return ofk_set_error(OFK_ERR_ARG, "unknown GEMM epilogue");
}

}  // namespace ofk

static int gemm_impl(int epi, int a_mn_major, int b_mn_major, const void* A, long long lda, const void* B,
                     long long ldb, int M, int N, int K, int splits, int block_n, void* out, long long ldo,
                     void* out2, long long ldo2, const void* aux, long long ldaux, const float* bias,
                     const float* gate, void* stream_, int out_rpg, int out_gs, int out_go, int ak_rpg, int ak_gs,
                     int ak_go) {
  using namespace ofk;
  if (out_rpg > 0 && (epi != OFK_EPI_STORE_BF16 && epi != OFK_EPI_BIAS_BF16 && epi != OFK_EPI_STORE_F32))
    return ofk_set_error(OFK_ERR_ARG, "grouped output rows are supported by the STORE_BF16 / BIAS_BF16 / STORE_F32 epilogues");
  if (ak_rpg > 0 && (!a_mn_major || ak_rpg % 64 != 0 || K % ak_rpg != 0))
    return ofk_set_error(OFK_ERR_ARG, "grouped reduction rows need an MN-major A with rows_per_group % 64 == 0 dividing K");
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (M <= 0 || N <= 0 || K <= 0) return ofk_set_error(OFK_ERR_ARG, "GEMM dims must be positive");
  if (N % 16 != 0) return ofk_set_error(OFK_ERR_ARG, "GEMM N must be a multiple of 16");
  if (!A || !B || !out) return ofk_set_error(OFK_ERR_ARG, "GEMM null operand");
  if (block_n != 0 && block_n != 128 && block_n != 256 && block_n != 512)
    return ofk_set_error(OFK_ERR_ARG, "GEMM block_n must be 0, 128, 256 or 512");
  if (splits < 1) splits = 1;
  if (splits > 1 && epi != OFK_EPI_ATOMIC_F32) return ofk_set_error(OFK_ERR_ARG, "split-K needs the atomic epilogue");
  if ((epi == OFK_EPI_BIAS_BF16 || epi == OFK_EPI_BIAS_QGELU_BF16 || epi == OFK_EPI_BIAS_RESID_F32 ||
       epi == OFK_EPI_BIAS_GELU_BF16) && !bias)
    return ofk_set_error(OFK_ERR_ARG, "bias epilogue without bias");
  if ((epi == OFK_EPI_GATE_RESID_F32 || epi == OFK_EPI_BIAS_RESID_F32 || epi == OFK_EPI_DGELU_BF16) && !aux)
    return ofk_set_error(OFK_ERR_ARG, "epilogue needs aux operand");
  if (epi == OFK_EPI_GELU_DUAL && !out2) return ofk_set_error(OFK_ERR_ARG, "GELU_DUAL needs out2");
  if (g_num_sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (g_num_sms <= 0) return ofk_set_error(OFK_ERR_CUDA, "no CUDA device");
  }
  const int total_kb = (K + BK - 1) / BK;
  if (splits > total_kb) splits = total_kb;
  GemmParams p;
  p.M = M; p.N = N; p.K = K;
  p.kb_per_split = (total_kb + splits - 1) / splits;
  p.splits = (total_kb + p.kb_per_split - 1) / p.kb_per_split;
  p.out = out; p.ldo = ldo; p.out2 = out2; p.ldo2 = ldo2; p.aux = aux; p.ldaux = ldaux; p.bias = bias; p.gate = gate;
  p.out_rpg = out_rpg; p.out_gs = out_gs; p.out_go = out_go; p.ak_rpg = ak_rpg; p.ak_gs = ak_gs; p.ak_go = ak_go;
  const int a_rows = ak_rpg > 0 ? (K / ak_rpg) * ak_gs : K;   // physical row count of an MN-major A
  {
    static int stream_mode = -1;   // OFK_GEMM_STREAM_OUT=0/1 overrides; default: stream when the outputs exceed ~32 MB
    if (stream_mode < 0) { const char* e = getenv("OFK_GEMM_STREAM_OUT"); stream_mode = e ? atoi(e) + 2 : 0; }
    if (stream_mode >= 2) p.stream_out = stream_mode - 2;
    else p.stream_out = ((long long)M * N >= (16LL << 20)) ? 1 : 0;
  }

  // K-major: tensor [rows, K], box {64 (k), 128 rows}. MN-major: tensor [K, rows], box {64 (rows), 64 (k)}.
  CUtensorMap ta, tb;
  int rc = a_mn_major ? get_tensor_map(A, lda, a_rows, M, 64, BK, &ta) : get_tensor_map(A, lda, M, K, BK, BM, &ta);
  if (rc) return rc;
  rc = b_mn_major ? get_tensor_map(B, ldb, K, N, 64, BK, &tb) : get_tensor_map(B, ldb, N, K, BK, BN, &tb);
  if (rc) return rc;
  return dispatch_epi(epi, a_mn_major, b_mn_major, ta, tb, p, stream);
}

extern "C" int ofk_gemm_bf16(int epi, int a_mn_major, int b_mn_major, const void* A, long long lda, const void* B,
                             long long ldb, int M, int N, int K, int splits, int block_n, void* out, long long ldo,
                             void* out2, long long ldo2, const void* aux, long long ldaux, const float* bias,
                             const float* gate, void* stream_) {
  return gemm_impl(epi, a_mn_major, b_mn_major, A, lda, B, ldb, M, N, K, splits, block_n, out, ldo, out2, ldo2, aux, ldaux,
                   bias, gate, stream_, 0, 0, 0, 0, 0, 0);
}

extern "C" int ofk_gemm_reserve_sms(int n) {
  const int prev = ofk::g_reserved_sms;
  if (n < 0) n = 0;
  if (n > 64) n = 64;
  ofk::g_reserved_sms = n & ~1;   // whole TPCs (two SMs each)
  return prev;
}

extern "C" int ofk_gemm_bf16_grouped(int epi, int a_mn_major, int b_mn_major, const void* A, long long lda, const void* B,
                                     long long ldb, int M, int N, int K, int splits, int block_n, void* out,
                                     long long ldo, const float* bias, int out_rows_per_group, int out_group_stride,
                                     int out_group_offset, int a_k_rows_per_group, int a_k_group_stride,
                                     int a_k_group_offset, void* stream_) {
  return gemm_impl(epi, a_mn_major, b_mn_major, A, lda, B, ldb, M, N, K, splits, block_n, out, ldo, nullptr, 0, nullptr, 0,
                   bias, nullptr, stream_, out_rows_per_group, out_group_stride, out_group_offset, a_k_rows_per_group,
                   a_k_group_stride, a_k_group_offset);
}
