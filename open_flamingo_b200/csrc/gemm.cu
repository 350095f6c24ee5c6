// bf16 x bf16 -> fp32 GEMM for sm_90a: TMA-staged operands (128B swizzle), wgmma with the accumulator in registers,
// a warp-specialised persistent CTA (one producer warp, two consumer warpgroups), fused epilogues.
//
// Two tile shapes, chosen per launch from the problem's size (launch()):
//   wide  : 128 x 256 tiles on 2-CTA clusters.  The two CTAs compute vertically adjacent m-tiles of the same n-tile;
//           each loads its own A and one half of the shared B panel, multicast into both CTAs' shared memory, so a
//           k-block costs 32 KiB of L2 reads for 4.2 MFLOP per CTA (128 x 128 tiles: 32 KiB for 2.1 MFLOP).
//   narrow: 128 x 128 tiles, no cluster, for problems whose wide work items would not fill the GPU once (the small-M
//           GEMMs of decoding, some Perceiver shapes).
// Both reduce every output element over k in the same order, so the choice never changes a bit of the result.
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
#include <type_traits>
#include <unordered_map>

#include "ofk_internal.h"
#include "ofk_ptx.cuh"

namespace ofk {

constexpr int BM = 128;       // two consumer warpgroups x wgmma M = 64
constexpr int BN = 128;       // narrow tile width; also the B rows one CTA loads per k-block in either shape
constexpr int BN_WIDE = 256;  // wide tile width (wgmma N = 256)
constexpr int CLUSTER = 2;    // CTAs per cluster in the wide shape
constexpr int BK = 64;        // one 128-byte swizzle atom of bf16
constexpr int WGMMA_K = 16;   // fixed for 16-bit inputs
// Warp roles: warpgroup 0 = producer (warp 0 lane 0 issues every TMA load; the other warps only take part in set-up),
// warpgroups 1 and 2 = consumers, each owning 64 accumulator rows of the tile through mainloop and epilogue.
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
  int stream_out;    // 1: epilogue stores carry an L2 evict-first hint so they do not displace the operand panels in L2
  // Grouped row maps (0 = identity): logical row r -> (r / rpg) * gs + go + r % rpg.  `out_*` places the rows of `out`
  // inside a larger interleaved buffer (the media / latent halves of PerceiverAttention's cat((x, latents), -2),
  // helpers.py:53); `ak_*` does the same for the REDUCTION rows of an MN-major A operand (wgrad over one half).
  int out_rpg, out_gs, out_go;
  int ak_rpg, ak_gs, ak_go;
  int wide;          // 1: 128 x 256 tiles on 2-CTA clusters sharing B (launched with a cluster); 0: 128 x 128 tiles
  // Set by launch() for the chosen shape.  Read from the parameter bank rather than derived in the kernel, so they
  // take no registers through the main loop and the epilogue.
  int m_units;       // m-tiles (narrow) or m-tile pairs (wide)
  int n_tiles;
  int num_work;      // m_units * n_tiles * splits
  int total_kb;      // k-blocks of K
  int out_chunk;     // grouped out map: rows per TMA store (a box never crosses a group)
};
__device__ __forceinline__ long long map_rows(long long r, int rpg, int gs, int go) {
  return rpg > 0 ? (r / rpg) * gs + go + r % rpg : r;
}

// Work item -> (m unit, n tile, k split); an m unit is an m-tile (narrow) or a cluster's pair of m-tiles (wide).
// Within a split, tiles are walked in groups of GROUP_M m units by all n-tiles, m fastest, so the tiles in flight
// share GROUP_M row panels of A and a few column panels of B through L2.
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
// Epilogue.  Each consumer warpgroup finishes its 64 rows of the tile in sub-tiles of SUBN columns, straight from the
// wgmma accumulator fragments: the fused arithmetic runs in registers, the results go to an epilogue buffer in shared
// memory laid out as one box of the output's tensor map (64 rows x SUBN columns, TMA-swizzled), and one thread of the
// warpgroup writes the box with an asynchronous TMA store (a TMA reduce-add for ATOMIC_F32).  The aux operand (fp32
// residual, bf16 saved pre-activation) is TMA-loaded into the sub-tile's out buffer NBUF - 1 sub-tiles ahead (across
// the tile boundary into the next tile's first sub-tiles, so those loads overlap its main loop), and the result
// overwrites it in place.  A sub-tile's aux load completes before its store is issued, so an in-place residual
// (aux == out) is exact.  out2 has buffers of its own.
template <int EPI>
struct EpiTraits {
  static constexpr bool RESID = EPI == OFK_EPI_GATE_RESID_F32 || EPI == OFK_EPI_BIAS_RESID_F32;
  static constexpr bool F32_OUT = RESID || EPI == OFK_EPI_STORE_F32 || EPI == OFK_EPI_ATOMIC_F32;
  static constexpr bool HAS_OUT2 = RESID || EPI == OFK_EPI_GELU_DUAL;
  static constexpr bool HAS_BIAS = EPI == OFK_EPI_BIAS_BF16 || EPI == OFK_EPI_BIAS_QGELU_BF16 ||
                                   EPI == OFK_EPI_BIAS_GELU_BF16 || EPI == OFK_EPI_BIAS_RESID_F32;
  static constexpr int AUX_BYTES = RESID ? 4 : (EPI == OFK_EPI_DGELU_BF16 ? 2 : 0);
  static constexpr int OUT_BYTES = F32_OUT ? 4 : 2;
  // Columns per sub-tile and buffers per warpgroup, within 16 KiB: one-output epilogues use 128-byte box rows (one
  // 128-byte swizzle span, conflict-free fragment writes) double-buffered; GELU_DUAL two bf16 32-column boxes, each
  // double-buffered; DGELU a 32-column bf16 box four deep (its aux load runs three sub-tiles ahead); the residual
  // epilogues, the heaviest, 16 columns: fp32 out with the aux in place three deep (4 KiB each; the residual load runs
  // two sub-tiles ahead) and bf16 out2 double-buffered (2 KiB each).
  static constexpr int SUBN = RESID ? 16 : (EPI == OFK_EPI_GELU_DUAL || EPI == OFK_EPI_DGELU_BF16) ? 32 : 128 / OUT_BYTES;
  static constexpr int NBUF = EPI == OFK_EPI_DGELU_BF16 ? 4 : RESID ? 3 : 2;   // out (and aux) buffers
  static constexpr int NBUF2 = HAS_OUT2 ? 2 : 0;                                 // out2 buffers
  static constexpr int OUT_PITCH = SUBN * OUT_BYTES;    // bytes per box row = the map's swizzle span (32, 64 or 128)
  static constexpr int OUT2_PITCH = SUBN * 2;
  static constexpr int OUT_BUF_BYTES = 64 * OUT_PITCH;
  static constexpr int OUT2_BUF_BYTES = 64 * OUT2_PITCH;
  static constexpr int OUT2_BASE = NBUF * OUT_BUF_BYTES;
  static constexpr int BYTES = OUT2_BASE + NBUF2 * OUT2_BUF_BYTES;
  static_assert(OUT_BUF_BYTES % 1024 == 0 && OUT2_BUF_BYTES % 1024 == 0, "boxes start on a swizzle-pattern boundary");
  // Before a sub-tile's barrier the issuing thread lets at most PRE_WAIT stores still read their buffers, so the next
  // sub-tile's out2 buffer (and, without an aux load to wait on, its out buffer) is free after the barrier; -1: no wait
  // (an aux epilogue's out buffer is refilled only after its store has read it, see the consumer).
  static constexpr int PRE_WAIT = AUX_BYTES != 0 ? (HAS_OUT2 ? NBUF2 - 2 : -1)
                                                 : (HAS_OUT2 && NBUF2 < NBUF ? NBUF2 - 2 : NBUF - 2);
};

// Byte offset of (row, byte column) in a box with PITCH-byte rows, swizzled as the map's CU_TENSOR_MAP_SWIZZLE_<PITCH>B
// does it: the 16-byte chunk index is XORed with address bits [7, 7 + log2(PITCH / 16)) (boxes are 1024-byte aligned).
template <int PITCH>
__device__ __forceinline__ int box_off(int row, int byte_col) {
  return row * PITCH + ((((byte_col >> 4) ^ ((row * PITCH) >> 7)) & (PITCH / 16 - 1)) << 4) + (byte_col & 15);
}

__device__ __forceinline__ void st_shared_b32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_shared_b32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void st_shared_f32x2(uint32_t addr, float x, float y) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(x), "f"(y) : "memory");
}
__device__ __forceinline__ float2 ld_shared_f32x2(uint32_t addr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr) : "memory");
  return v;
}

// The fused epilogue of two adjacent accumulators, columns (c, c + 1) of row r of the sub-tile whose out / out2
// buffers are at shared addresses `buf` / `buf2` (c even); bias already added.  The operations and their rounding
// points are the same for every element wherever it sits.
template <int EPI>
__device__ __forceinline__ void epilogue_pair(const GemmParams& p, float gate_t, uint32_t buf, uint32_t buf2, int r,
                                              int c, float v0, float v1) {
  using E = EpiTraits<EPI>;
  const uint32_t o = buf + box_off<E::OUT_PITCH>(r, c * E::OUT_BYTES);
  const uint32_t o2 = buf2 + box_off<E::OUT2_PITCH>(r, c * 2);
  if constexpr (EPI == OFK_EPI_STORE_BF16 || EPI == OFK_EPI_BIAS_BF16 || EPI == OFK_EPI_BIAS_QGELU_BF16 ||
                EPI == OFK_EPI_BIAS_GELU_BF16) {
    if constexpr (EPI == OFK_EPI_BIAS_QGELU_BF16) { v0 = quick_gelu(bf16_round(v0)); v1 = quick_gelu(bf16_round(v1)); }
    if constexpr (EPI == OFK_EPI_BIAS_GELU_BF16) { v0 = gelu_exact(bf16_round(v0)); v1 = gelu_exact(bf16_round(v1)); }
    st_shared_b32(o, pack_bf16x2(v0, v1));
  } else if constexpr (EPI == OFK_EPI_STORE_F32 || EPI == OFK_EPI_ATOMIC_F32) {
    st_shared_f32x2(o, v0, v1);
  } else if constexpr (EPI == OFK_EPI_GELU_DUAL) {
    // z = bf16(acc) is what the reference's Linear emits under autocast; GELU is taken of that.
    v0 = bf16_round(v0); v1 = bf16_round(v1);
    st_shared_b32(o, pack_bf16x2(v0, v1));
    st_shared_b32(o2, pack_bf16x2(gelu_exact(v0), gelu_exact(v1)));
  } else if constexpr (E::RESID) {
    // out = branch * tanh(gate) + residual (fp32 residual stream); branch kept in bf16 for the gate grad.
    v0 = bf16_round(v0); v1 = bf16_round(v1);
    if (p.out2 != nullptr) st_shared_b32(o2, pack_bf16x2(v0, v1));
    const float2 res = ld_shared_f32x2(o);
    st_shared_f32x2(o, fmaf(v0, gate_t, res.x), fmaf(v1, gate_t, res.y));
  } else if constexpr (EPI == OFK_EPI_DGELU_BF16) {
    // out = bf16( bf16(acc) * gelu'(z) ), z = saved bf16 pre-activation
    const uint32_t z = ld_shared_b32(o);
    st_shared_b32(o, pack_bf16x2(bf16_round(v0) * gelu_exact_grad(bf16_lo(z)), bf16_round(v1) * gelu_exact_grad(bf16_hi(z))));
  }
}

// ----------------------------------------------------------------------------------------------
// Shared memory: the TMA ring of 4 stages (a stage holds A, then B), then the epilogue buffers (16 KiB per consumer
// warpgroup), then the barriers.
struct SmemLayout {
  static constexpr int A_BYTES = BM * BK * 2;                        // 16 KiB
  static constexpr int B_PART_BYTES = BN * BK * 2;                   // 16 KiB: the B rows one CTA loads
  static constexpr int NARROW_STAGE_BYTES = A_BYTES + B_PART_BYTES;  // 32 KiB
  static constexpr int WIDE_STAGE_BYTES = A_BYTES + CLUSTER * B_PART_BYTES;   // 48 KiB
  static constexpr int STAGES = 4;
  static constexpr int RING_BYTES = STAGES * WIDE_STAGE_BYTES;
  static constexpr int EPI_OFF = RING_BYTES;
  static constexpr int EPI_BYTES_PER_WG = 16 * 1024;
  static constexpr int MAX_NBUF = 4;
  static constexpr int BAR_OFF = EPI_OFF + NUM_CONSUMER_WG * EPI_BYTES_PER_WG;
  static constexpr int NUM_BARS = 2 * STAGES + NUM_CONSUMER_WG * MAX_NBUF;   // full, empty, aux per warpgroup
  static constexpr int TOTAL = BAR_OFF + 256 + 1024;   // + barriers + alignment slack
  static_assert(NUM_BARS * 8 <= 256, "barriers fit their region");
};
static_assert(SmemLayout::TOTAL <= 227 * 1024, "GEMM shared memory exceeds the sm_90 per-block limit");

template <int A_MN, int B_MN, int EPI>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
            const __grid_constant__ CUtensorMap tma_out, const __grid_constant__ CUtensorMap tma_out2,
            const __grid_constant__ CUtensorMap tma_aux, const GemmParams p) {
  using L = SmemLayout;
  using E = EpiTraits<EPI>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);
  uint64_t* empty_bar = full_bar + L::STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  // Wide: the CTAs of a cluster walk the work items together (consecutive blockIdx.x form a cluster); CTA `crank`
  // takes m-tile 2 * unit + crank and loads B rows [128 crank, 128 crank + 128) of the tile for both.  When the
  // m-tile count is odd, the last pair's second tile lies wholly past M: it still loads (TMA fills zeros) and
  // arrives, and its stores fall outside the output map, so TMA writes nothing.
  const bool wide = p.wide != 0;
  const int bn = wide ? BN_WIDE : BN;
  const int stage_bytes = wide ? L::WIDE_STAGE_BYTES : L::NARROW_STAGE_BYTES;
  const int crank = wide ? (int)cluster_ctarank() : 0;
  const int walker = wide ? blockIdx.x / CLUSTER : blockIdx.x;
  const int walkers = wide ? gridDim.x / CLUSTER : gridDim.x;
  const int m_units = p.m_units, n_tiles = p.n_tiles, num_work = p.num_work, total_kb = p.total_kb;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tma_a);
    tma_prefetch_desc(&tma_b);
    tma_prefetch_desc(&tma_out);
    if constexpr (E::HAS_OUT2) tma_prefetch_desc(&tma_out2);
    if constexpr (E::AUX_BYTES != 0) tma_prefetch_desc(&tma_aux);
    // wide: a stage is freed only when the consumers of BOTH CTAs are done with it, since the partner's producer
    // multicasts into this CTA's copy of the stage
    for (int s = 0; s < L::STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], NUM_EPI_WARPS * (wide ? CLUSTER : 1));
    }
    for (int b = 0; b < NUM_CONSUMER_WG * L::MAX_NBUF; ++b) mbar_init(&full_bar[2 * L::STAGES + b], 1);
    fence_barrier_init();
  }
  // wide: the partner's barriers must be initialised before anything is multicast or arrived on them
  if (wide) cluster_sync();
  else __syncthreads();

  if (warp < 4) {
    // ===================== TMA producer (one thread) =====================
    // the producer warpgroup hands its registers to the consumers (40 + 2 x 232 per thread fit the 64K register file)
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
    if (warp == 0 && lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int w = walker; w < num_work; w += walkers) {
        int mu, nt, ks;
        work_to_tile(w, m_units, n_tiles, mu, nt, ks);
        const int m0 = (wide ? 2 * mu + crank : mu) * BM, n0 = nt * bn;
        const int kb0 = ks * p.kb_per_split;
        const int kb1 = min(total_kb, kb0 + p.kb_per_split);
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * stage_bytes;
          uint8_t* sb = sa + L::A_BYTES;
          mbar_arrive_expect_tx(&full_bar[stage], stage_bytes);
          const int k0 = kb * BK;
          if constexpr (A_MN == 0) {
            tma_load_2d(sa, &tma_a, &full_bar[stage], k0, m0);             // box {64 k, 128 rows}
          } else {
#pragma unroll
            for (int i = 0; i < BM / 64; ++i)                               // boxes {64 mn, 64 k}
              tma_load_2d(sa + i * (BK * 128), &tma_a, &full_bar[stage], m0 + 64 * i, (int)map_rows(k0, p.ak_rpg, p.ak_gs, p.ak_go));
          }
          // this CTA's BN rows of B, at their place in the tile's B stage (the same in both layouts: K-major 8-row
          // groups and MN-major 64-wide chunks are both BN * 128 B per BN rows)
          uint8_t* sbp = sb + crank * L::B_PART_BYTES;
          const int nb0 = n0 + crank * BN;
          if constexpr (B_MN == 0) {
            if (wide) tma_load_2d_multicast(sbp, &tma_b, &full_bar[stage], k0, nb0, (1u << CLUSTER) - 1);
            else tma_load_2d(sbp, &tma_b, &full_bar[stage], k0, nb0);   // box {64 k, 128 rows}
          } else {
#pragma unroll
            for (int i = 0; i < BN / 64; ++i) {
              if (wide) tma_load_2d_multicast(sbp + i * (BK * 128), &tma_b, &full_bar[stage], nb0 + 64 * i, k0, (1u << CLUSTER) - 1);
              else tma_load_2d(sbp + i * (BK * 128), &tma_b, &full_bar[stage], nb0 + 64 * i, k0);
            }
          }
          if (++stage == L::STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===================== consumers: wgmma mainloop + fused epilogue =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
  const int wg = warp / 4 - 1;               // consumer warpgroup: accumulator rows [64 wg, 64 wg + 64) of the tile
  const int wl = warp & 3;                   // warp within the warpgroup
  const bool leader = (threadIdx.x & 127) == 0;   // issues the warpgroup's epilogue TMA stores and aux loads
  uint8_t* ebuf = smem + L::EPI_OFF + wg * L::EPI_BYTES_PER_WG;
  uint64_t* aux_bar = full_bar + 2 * L::STAGES + wg * L::MAX_NBUF;
  float gate_t = 1.0f;
  if constexpr (EPI == OFK_EPI_GATE_RESID_F32) {
    if (p.gate != nullptr) gate_t = tanhf(__ldg(p.gate));
  }
  // one copy of the consumer loop per tile shape, so that the narrow one carries none of the wide one's state
  auto consume = [&](auto wide_c) {
    constexpr bool WIDE = decltype(wide_c)::value;
    constexpr int TILE_N = WIDE ? BN_WIDE : BN;
    constexpr int STAGE_BYTES = WIDE ? L::WIDE_STAGE_BYTES : L::NARROW_STAGE_BYTES;
    constexpr int SUBN = E::SUBN, NBUF = E::NBUF, SUBT = TILE_N / SUBN;
    static_assert(E::BYTES <= L::EPI_BYTES_PER_WG && NBUF <= L::MAX_NBUF && NBUF - 1 < SUBT, "epilogue buffers");
    auto release = [&](int s) {
      if (lane != 0) return;
      if constexpr (WIDE) {
#pragma unroll
        for (int r = 0; r < CLUSTER; ++r) mbar_arrive_cluster(&empty_bar[s], r);
      } else {
        mbar_arrive(&empty_bar[s]);
      }
    };
    // This warpgroup's first row and the tile's first column for work item w.
    auto tile_origin = [&](int w, int& row0, int& col0) {
      int mu, nt, ks;
      work_to_tile(w, m_units, n_tiles, mu, nt, ks);
      row0 = (WIDE ? 2 * mu + crank : mu) * BM + wg * 64;
      col0 = nt * TILE_N;
    };
    // Leader only: TMA-load the aux box at (row0, col) for the q-th sub-tile of this warpgroup.
    auto load_aux = [&](uint32_t q, int row0, int col) {
      uint64_t* bar = &aux_bar[q % NBUF];
      mbar_arrive_expect_tx(bar, 64 * SUBN * E::AUX_BYTES);
      tma_load_2d(ebuf + (q % NBUF) * E::OUT_BUF_BYTES, &tma_aux, bar, col, row0);
    };
    // ... for sub-tile s of work item w, if there is one
    auto load_aux_of = [&](uint32_t q, int w, int s) {
      if (w >= num_work) return;
      int row0, col0;
      tile_origin(w, row0, col0);
      load_aux(q, row0, col0 + s * SUBN);
    };
    // Leader only: store the sub-tile at (row0, col).  A grouped output map is a 3-D map (columns, rows in group,
    // groups) whose box is p.out_chunk rows that never cross a group (see gemm_impl): the 64 rows go out in
    // 64 / out_chunk stores, each at non-negative coordinates, and those wholly past M are skipped.
    auto store_out = [&](const uint8_t* buf, const uint8_t* buf2, int row0, int col) {
      constexpr bool GROUPED = EPI == OFK_EPI_STORE_BF16 || EPI == OFK_EPI_BIAS_BF16 || EPI == OFK_EPI_STORE_F32;
      static_assert(!GROUPED || E::OUT_PITCH == 128, "a grouped store starts at any row: rows must be 128-byte aligned");
      const uint64_t policy = p.stream_out ? l2_policy_evict_first() : 0;
      if constexpr (EPI == OFK_EPI_ATOMIC_F32) {
        tma_reduce_add_3d(&tma_out, buf, col, row0, 0);
      } else if constexpr (GROUPED) {
        if (p.out_rpg == 0) {
          if (p.stream_out) tma_store_3d_hint(&tma_out, buf, col, row0, 0, policy);
          else tma_store_3d(&tma_out, buf, col, row0, 0);
        } else {
          for (int r = row0; r < row0 + 64 && r < p.M; r += p.out_chunk) {
            const uint8_t* src = buf + (r - row0) * E::OUT_PITCH;
            const int g = r / p.out_rpg;
            if (p.stream_out) tma_store_3d_hint(&tma_out, src, col, r - g * p.out_rpg, g, policy);
            else tma_store_3d(&tma_out, src, col, r - g * p.out_rpg, g);
          }
        }
      } else {
        if (p.stream_out) tma_store_3d_hint(&tma_out, buf, col, row0, 0, policy);
        else tma_store_3d(&tma_out, buf, col, row0, 0);
      }
      if constexpr (E::HAS_OUT2) {
        if (p.out2 != nullptr) {
          if (p.stream_out) tma_store_2d_hint(&tma_out2, buf2, col, row0, policy);
          else tma_store_2d(&tma_out2, buf2, col, row0);
        }
      }
      bulk_commit_group();
    };

    int stage = 0; uint32_t phase = 0;
    uint32_t q = 0;   // sub-tiles this warpgroup has finished
    if constexpr (E::AUX_BYTES != 0) {
      if (leader) {
#pragma unroll
        for (int s = 0; s < NBUF - 1; ++s) load_aux_of(s, walker, s);
      }
    }
    float d[TILE_N / 2];
    for (int w = walker; w < num_work; w += walkers) {
      int mu, nt, ks;
      work_to_tile(w, m_units, n_tiles, mu, nt, ks);
      const int kb0 = ks * p.kb_per_split;
      const int kb1 = min(total_kb, kb0 + p.kb_per_split);
      // The first k-step overwrites the accumulators (scale-d = 0), but wgmma still names them as inputs: zeroing them
      // here ends the previous tile's values at the epilogue instead of keeping all 128 live through it.
#pragma unroll
      for (int i = 0; i < TILE_N / 2; ++i) d[i] = 0.f;
      int prev_stage = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES);
        const uint32_t sb = sa + L::A_BYTES;
        // K-major : this warpgroup's 64 rows start 64 * 128 B in; 8-row groups 1024 B apart (SBO); advance 32 B per
        //           WGMMA_K inside the swizzle atom.
        // MN-major: 64-wide MN chunks BK * 128 B apart (LBO; this warpgroup's rows are chunk `wg`), 8-k groups 1024 B
        //           apart (SBO); advance 2 k-groups = 2048 B per WGMMA_K.
        auto adesc = [&](int k) {
          return A_MN ? make_wgmma_desc_sw128(sa + wg * (BK * 128) + k * 2048, BK * 128, 1024)
                      : make_wgmma_desc_sw128(sa + wg * (64 * 128) + k * 32, 16, 1024);
        };
        auto bdesc = [&](int k) {
          return B_MN ? make_wgmma_desc_sw128(sb + k * 2048, BK * 128, 1024) : make_wgmma_desc_sw128(sb + k * 32, 16, 1024);
        };
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / WGMMA_K; ++k) {
          if constexpr (WIDE) wgmma_m64n256k16_bf16<A_MN, B_MN>(d, adesc(k), bdesc(k), (kb > kb0 || k > 0) ? 1u : 0u);
          else wgmma_m64n128k16_bf16<A_MN, B_MN>(d, adesc(k), bdesc(k), (kb > kb0 || k > 0) ? 1u : 0u);
        }
        wgmma_commit();
        // keep one k-block of MMAs in flight; the one before it has retired, so its ring slot can be refilled
        wgmma_wait<1>();
        if (prev_stage >= 0) release(prev_stage);
        prev_stage = stage;
        if (++stage == L::STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      // every stage goes back to the producer before the epilogue, so the next tile's loads overlap it
      release(prev_stage);

      // Epilogue, one sub-tile of SUBN columns at a time, from the live fragments: thread t of the warpgroup holds
      // rows fr and fr + 8 of the 64, columns 8 j + fc and 8 j + fc + 1 of every 8 (wgmma_m64n128k16_bf16's layout).
      int row0, col0;
      tile_origin(w, row0, col0);
      const int fr = 16 * wl + lane / 4, fc = 2 * (lane % 4);
#pragma unroll
      for (int s = 0; s < SUBT; ++s) {
        const uint32_t qs = q + s;
        uint8_t* buf = ebuf + (qs % NBUF) * E::OUT_BUF_BYTES;
        uint8_t* buf2 = ebuf + E::OUT2_BASE + (qs % (E::NBUF2 > 0 ? E::NBUF2 : 1)) * E::OUT2_BUF_BYTES;
        const uint32_t sbuf = smem_u32(buf), sbuf2 = smem_u32(buf2);
        if constexpr (E::AUX_BYTES != 0) mbar_wait(&aux_bar[qs % NBUF], (qs / NBUF) & 1);
#pragma unroll
        for (int j = 0; j < SUBN / 8; ++j) {
          const int c = 8 * j + fc;
          const int i = 4 * (s * (SUBN / 8) + j);
          float b0 = 0.f, b1 = 0.f;
          if constexpr (E::HAS_BIAS) {
            // per-column bias: the four lanes of a row read 8 consecutive floats, every row the same (broadcast)
            if (col0 + s * SUBN + c < p.N) {
              const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + col0 + s * SUBN + c));
              b0 = b.x; b1 = b.y;
            }
          }
          epilogue_pair<EPI>(p, gate_t, sbuf, sbuf2, fr, c, E::HAS_BIAS ? d[i] + b0 : d[i],
                             E::HAS_BIAS ? d[i + 1] + b1 : d[i + 1]);
          epilogue_pair<EPI>(p, gate_t, sbuf, sbuf2, fr + 8, c, E::HAS_BIAS ? d[i + 2] + b0 : d[i + 2],
                             E::HAS_BIAS ? d[i + 3] + b1 : d[i + 3]);
        }
        // the TMA store (async proxy) must see these generic-proxy writes
        fence_proxy_async_smem();
        // the next sub-tile's buffers without an aux load to wait on are free once the stores that last read them have
        if constexpr (E::PRE_WAIT >= 0) {
          if (leader) bulk_wait_group_read<E::PRE_WAIT>();
        }
        named_bar_sync(1 + wg, 128);
        if (leader) {
          store_out(buf, buf2, row0, col0 + s * SUBN);
          if constexpr (E::AUX_BYTES != 0) {
            // the buffer of sub-tile qs - 1 is free once its store has read it: load sub-tile qs + NBUF - 1 into it
            bulk_wait_group_read<1>();
            if (s + NBUF - 1 < SUBT) load_aux(qs + NBUF - 1, row0, col0 + (s + NBUF - 1) * SUBN);
            else load_aux_of(qs + NBUF - 1, w + walkers, s + NBUF - 1 - SUBT);
          }
        }
      }
      q += SUBT;
    }
    // every bulk store must be complete before the CTA exits
    if (leader) bulk_wait_group_all();
    // wide: neither CTA may exit while its partner can still arrive on its barriers (everything multicast into this
    // CTA has been consumed by now).  The cluster barrier waits for non-exited threads only: the producer warpgroup
    // has left.  (A barrier in the producer's code as well made ptxas hold the consumers to 168 registers, and spill.)
    if constexpr (WIDE) cluster_sync();
  };
  if (wide) consume(std::true_type{});
  else consume(std::false_type{});
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
  const void* ptr; long long ld, gstride; int rows, cols, groups, box_inner, box_outer, box_groups, elem_bytes, swizzle;
  bool operator==(const MapKey& o) const {
    return ptr == o.ptr && ld == o.ld && gstride == o.gstride && rows == o.rows && cols == o.cols &&
           groups == o.groups && box_inner == o.box_inner && box_outer == o.box_outer && box_groups == o.box_groups &&
           elem_bytes == o.elem_bytes && swizzle == o.swizzle;
  }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    size_t h = reinterpret_cast<size_t>(k.ptr);
    h = h * 1000003u ^ (size_t)k.ld; h = h * 1000003u ^ (size_t)k.rows; h = h * 1000003u ^ (size_t)k.cols;
    h = h * 1000003u ^ (size_t)(k.box_inner * 1024 + k.box_outer);
    h = h * 1000003u ^ (size_t)k.gstride; h = h * 1000003u ^ (size_t)(k.groups * 512 + k.box_groups);
    h = h * 1000003u ^ (size_t)(k.elem_bytes * 1024 + k.swizzle);
    return h;
  }
};

// Row-major bf16 (elem_bytes 2) or fp32 (4) tensor [rows, cols] (cols contiguous, row stride ld elements), swizzled
// in spans of `swizzle` bytes (32, 64 or 128).  groups = 0: 2-D, box {box_inner, box_outer}.  groups >= 1: 3-D
// [groups, rows, cols] with a group stride of gstride elements, box {box_inner, box_outer, box_groups}.
static int get_tensor_map(const void* ptr, long long ld, int rows, int cols, int box_inner, int box_outer,
                          CUtensorMap* out, int elem_bytes = 2, int swizzle = 128, int groups = 0,
                          long long gstride = 0, int box_groups = 1) {
  static std::mutex mu;
  static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> cache;
  MapKey key{ptr, ld, gstride, rows, cols, groups, box_inner, box_outer, box_groups, elem_bytes, swizzle};
  {
    std::lock_guard<std::mutex> g(mu);
    auto it = cache.find(key);
    if (it != cache.end()) { *out = it->second; return 0; }
  }
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) return ofk_set_error(OFK_ERR_DRIVER, "cuTensorMapEncodeTiled entry point not found");
  const cuuint32_t rank = groups > 0 ? 3 : 2;
  cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)(groups > 0 ? groups : 1)};
  cuuint64_t strides[2] = {(cuuint64_t)ld * elem_bytes, (cuuint64_t)gstride * elem_bytes};
  cuuint32_t box[3] = {(cuuint32_t)box_inner, (cuuint32_t)box_outer, (cuuint32_t)box_groups};
  cuuint32_t estr[3] = {1, 1, 1};
  const CUtensorMapSwizzle sw = swizzle == 32 ? CU_TENSOR_MAP_SWIZZLE_32B
                                : swizzle == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B;
  CUtensorMap m;
  CUresult r = enc(&m, elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank,
                   const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[200];
    snprintf(buf, sizeof buf, "cuTensorMapEncodeTiled failed (%d) rows=%d cols=%d groups=%d ld=%lld box=%dx%d", (int)r,
             rows, cols, groups, ld, box_inner, box_outer);
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

// Persistent grid.  The wide shape is used when its work items fill every cluster slot at least once; below that,
// 256-wide tiles would leave SMs idle (at M of a few rows, half of them on a weight-read-bound problem), and the
// narrow shape runs.  Cluster slots come from the occupancy of this kernel's shared-memory size, since not every GPC
// can hold an even number of these CTAs, less the reserved SMs, in whole clusters.
template <int A_MN, int B_MN, int EPI>
static int launch(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& to, const CUtensorMap& to2,
                  const CUtensorMap& tx, GemmParams p, cudaStream_t stream) {
  auto kern = gemm_kernel<A_MN, B_MN, EPI>;
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute cluster_attr;
  cluster_attr.id = cudaLaunchAttributeClusterDimension;
  cluster_attr.val.clusterDim.x = CLUSTER;
  cluster_attr.val.clusterDim.y = 1;
  cluster_attr.val.clusterDim.z = 1;
  cfg.blockDim = dim3(NUM_THREADS);
  cfg.dynamicSmemBytes = SmemLayout::TOTAL;
  cfg.stream = stream;
  static int max_clusters = -1;
  if (max_clusters < 0) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SmemLayout::TOTAL);
    if (e != cudaSuccess) return ofk_set_error(OFK_ERR_CUDA, cudaGetErrorString(e));
    cfg.gridDim = dim3(CLUSTER * g_num_sms);
    cfg.attrs = &cluster_attr;
    cfg.numAttrs = 1;
    int n = 0;
    e = cudaOccupancyMaxActiveClusters(&n, kern, &cfg);
    if (e != cudaSuccess) return ofk_set_error(OFK_ERR_CUDA, cudaGetErrorString(e));
    max_clusters = n;
  }
  const int m_tiles = (p.M + BM - 1) / BM;
  const int cluster_slots = (CLUSTER * max_clusters - g_reserved_sms) / CLUSTER;
  const int wide_work = (m_tiles + 1) / 2 * ((p.N + BN_WIDE - 1) / BN_WIDE) * p.splits;
  const int last_split_kb = (p.K + BK - 1) / BK - (p.splits - 1) * p.kb_per_split;   // the shortest split
  p.wide = cluster_slots > 0 && wide_work >= cluster_slots && last_split_kb >= SmemLayout::STAGES;
  p.m_units = p.wide ? (m_tiles + 1) / 2 : m_tiles;
  p.n_tiles = (p.N + (p.wide ? BN_WIDE : BN) - 1) / (p.wide ? BN_WIDE : BN);
  p.num_work = p.m_units * p.n_tiles * p.splits;
  p.total_kb = (p.K + BK - 1) / BK;
  if (p.wide) {
    cfg.gridDim = dim3(CLUSTER * cluster_slots);
    cfg.attrs = &cluster_attr;
    cfg.numAttrs = 1;
  } else {
    const int work = m_tiles * ((p.N + BN - 1) / BN) * p.splits;
    const int avail = g_num_sms - g_reserved_sms;
    cfg.gridDim = dim3(work < avail ? work : avail);
    cfg.attrs = nullptr;
    cfg.numAttrs = 0;
  }
  cudaError_t e = cudaLaunchKernelEx(&cfg, kern, ta, tb, to, to2, tx, p);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) return ofk_set_error(OFK_ERR_CUDA, cudaGetErrorString(e));
  ofk_count_launch();
  return 0;
}

// The epilogue's tensor maps, boxes of 64 rows x SUBN columns: out as a 3-D map (columns, rows in group, groups; one
// group of M rows without a grouped row map), out2 and aux as 2-D maps.  Absent operands get a copy of out's map.
// A grouped out map's box never crosses a group, so every store is at non-negative coordinates:
//   rows_per_group % 64 == 0: {SUBN, 64, 1}, one store per 64 rows;
//   64 % rows_per_group == 0: {SUBN, rpg, 64 / rpg}, 64 / rpg whole groups in one store (decoding: rpg = 1);
//   otherwise               : {SUBN, h, 1} with h = gcd(rpg, 64), 64 / h stores per 64 rows (group starts are
//                             multiples of h, and so is every 64-row block).
template <int EPI>
static int dispatch_major(int a_mn, int b_mn, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p,
                          cudaStream_t s) {
  using E = EpiTraits<EPI>;
  CUtensorMap to, to2, tx;
  const int ob = E::OUT_BYTES;
  int rc;
  if (p.out_rpg > 0) {
    const int rpg = p.out_rpg;
    const int box_rows = rpg % 64 == 0 ? 64 : 64 % rpg == 0 ? rpg : p.out_chunk;
    const int box_groups = rpg % 64 != 0 && 64 % rpg == 0 ? 64 / rpg : 1;
    rc = get_tensor_map(static_cast<const uint8_t*>(p.out) + (long long)p.out_go * p.ldo * ob, p.ldo, rpg, p.N,
                        E::SUBN, box_rows, &to, ob, E::OUT_PITCH, p.M / rpg, (long long)p.out_gs * p.ldo, box_groups);
  } else
    rc = get_tensor_map(p.out, p.ldo, p.M, p.N, E::SUBN, 64, &to, ob, E::OUT_PITCH, 1, (long long)p.M * p.ldo);
  if (rc) return rc;
  to2 = tx = to;
  if (E::HAS_OUT2 && p.out2 != nullptr) {
    rc = get_tensor_map(p.out2, p.ldo2, p.M, p.N, E::SUBN, 64, &to2, 2, E::OUT2_PITCH);
    if (rc) return rc;
  }
  if (E::AUX_BYTES != 0) {
    rc = get_tensor_map(p.aux, p.ldaux, p.M, p.N, E::SUBN, 64, &tx, E::AUX_BYTES, E::SUBN * E::AUX_BYTES);
    if (rc) return rc;
  }
  if (a_mn == 0 && b_mn == 0) return launch<0, 0, EPI>(ta, tb, to, to2, tx, p, s);
  if (a_mn == 0 && b_mn == 1) return launch<0, 1, EPI>(ta, tb, to, to2, tx, p, s);
  if (a_mn == 1 && b_mn == 1) return launch<1, 1, EPI>(ta, tb, to, to2, tx, p, s);
  return launch<1, 0, EPI>(ta, tb, to, to2, tx, p, s);
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
  if (out_rpg > 0 && M % out_rpg != 0)   // the output map holds whole groups (M / rows_per_group of them)
    return ofk_set_error(OFK_ERR_ARG, "grouped output rows need M to be a multiple of rows_per_group");
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
  const bool has_bias = epi == OFK_EPI_BIAS_BF16 || epi == OFK_EPI_BIAS_QGELU_BF16 || epi == OFK_EPI_BIAS_RESID_F32 ||
                        epi == OFK_EPI_BIAS_GELU_BF16;
  if (has_bias && !bias) return ofk_set_error(OFK_ERR_ARG, "bias epilogue without bias");
  if ((epi == OFK_EPI_GATE_RESID_F32 || epi == OFK_EPI_BIAS_RESID_F32 || epi == OFK_EPI_DGELU_BF16) && !aux)
    return ofk_set_error(OFK_ERR_ARG, "epilogue needs aux operand");
  if (epi == OFK_EPI_GELU_DUAL && !out2) return ofk_set_error(OFK_ERR_ARG, "GELU_DUAL needs out2");
  // TMA needs 16-byte-aligned bases and row strides, for the operands and for the epilogue's out / out2 / aux maps
  // alike; the bias keeps the 16-byte alignment it has always been checked for.
  auto misaligned = [](const void* ptr, long long ld, int elem_bytes) {
    return (reinterpret_cast<uintptr_t>(ptr) & 15) != 0 || ((ld * elem_bytes) & 15) != 0;
  };
  const bool f32_out = epi == OFK_EPI_STORE_F32 || epi == OFK_EPI_ATOMIC_F32 || epi == OFK_EPI_GATE_RESID_F32 ||
                       epi == OFK_EPI_BIAS_RESID_F32;
  const bool uses_out2 = epi == OFK_EPI_GELU_DUAL || epi == OFK_EPI_GATE_RESID_F32 || epi == OFK_EPI_BIAS_RESID_F32;
  const int aux_bytes = (epi == OFK_EPI_GATE_RESID_F32 || epi == OFK_EPI_BIAS_RESID_F32) ? 4 : epi == OFK_EPI_DGELU_BF16 ? 2 : 0;
  if (misaligned(A, lda, 2) || misaligned(B, ldb, 2))
    return ofk_set_error(OFK_ERR_ALIGN, "GEMM operand must be 16-byte aligned with a 16-byte-multiple row stride");
  if (misaligned(out, ldo, f32_out ? 4 : 2) || (uses_out2 && out2 && misaligned(out2, ldo2, 2)) ||
      (aux_bytes && misaligned(aux, ldaux, aux_bytes)))
    return ofk_set_error(OFK_ERR_ALIGN, "GEMM out / out2 / aux must be 16-byte aligned with a 16-byte-multiple row stride");
  if (has_bias && (reinterpret_cast<uintptr_t>(bias) & 15))
    return ofk_set_error(OFK_ERR_ALIGN, "GEMM bias must be 16-byte aligned");
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
  p.out_chunk = 64;   // rows per grouped store (see dispatch_major)
  if (out_rpg > 0 && out_rpg % 64 != 0 && 64 % out_rpg != 0) {
    p.out_chunk = 1;
    while (out_rpg % (2 * p.out_chunk) == 0) p.out_chunk *= 2;   // gcd(rpg, 64): rpg is not a multiple of 64
  }
  p.wide = 0;   // chosen by launch()
  const int a_rows = ak_rpg > 0 ? (K / ak_rpg) * ak_gs : K;   // physical row count of an MN-major A
  {
    static int stream_mode = -1;   // OFK_GEMM_STREAM_OUT=0/1 overrides; default: stream when the outputs exceed ~32 MB
    if (stream_mode < 0) { const char* e = getenv("OFK_GEMM_STREAM_OUT"); stream_mode = e ? atoi(e) + 2 : 0; }
    if (stream_mode >= 2) p.stream_out = stream_mode - 2;
    else p.stream_out = ((long long)M * N >= (16LL << 20)) ? 1 : 0;
  }

  // K-major: tensor [rows, K], box {64 (k), 128 rows}. MN-major: tensor [K, rows], box {64 (rows), 64 (k)}.
  // A wide tile's B is two such 128-row boxes (K-major) or four 64-row ones, half of them loaded by each CTA.
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
