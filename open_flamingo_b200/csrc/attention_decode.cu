// Decode attention of the frozen LM's decoder blocks with a KV cache: one query row per (batch, head) against the
// first nk rows of a K/V cache, head_dim 64, 80 or 128, bf16 in/out, fp32 softmax and P.V.  Semantics are those of
// ofk_attn_dense_fwd at nq = 1:
//
//   S = scale * q K^T + slope[h] * key_index          (ALiBi; softmax is invariant to MPT's per-row constant)
//   S[key_mask[b, key] != 0] = "finfo.min"            (a fully masked row attends uniformly, like masked_fill)
//   o = softmax(S) V
//
// At nq = 1 the products are matrix-vector, so tensor cores do not help (MPT is plain multi-head attention) and the
// kernel is bound by reading K and V.  Each key row is read once, by head_dim / 8 threads with one 16-byte load
// each.  A key group is C lanes, head_dim / 8 rounded up to a power of two, so that a group is an aligned part of a
// warp and its dot product sums in a shuffle tree; at head_dim 80 (GPT-NeoX, 10 loads per row) lanes 10..15 of each
// 16-lane group load nothing and add zeros.  A CTA of 128 threads holds 128 / C key groups, and every group keeps
// UNROLL keys of K and V in flight.
// Split-KV ("flash-decoding"): the keys are cut into `nsplit` contiguous chunks, one CTA per (split, head, batch), so
// that a small batch x heads still fills the GPU.  Each CTA merges its groups' (max, sum, acc) in shared memory in a
// fixed order and writes one partial; a second kernel merges the partials in split order.  The split count is a pure
// function of (batch, heads, nk, SM count), and nothing is added with atomics, so the output is the same bits on
// every launch and does not depend on how many rows the cache holds beyond nk.
//
// ofk_attn_decode_dev reads nk from device memory, so that one captured CUDA graph serves every decode step: the same
// kernels evaluate split_count on the device (Params::nk_dev non-NULL), the grid holds the largest split count any
// nk <= nk_max can ask for, CTAs past the runtime count exit, and the combine kernel, always launched, returns when
// the runtime plan has one split.  Every CTA that does work computes exactly what ofk_attn_decode computes at that nk.
// ofk_kv_append writes one new K/V row per batch entry at a device-side position, for the same reason.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "ofk_internal.h"
#include "ofk_ptx.cuh"

namespace ofk {
namespace decode {

constexpr int THREADS = 128;
constexpr int UNROLL = 4;         // keys per group and iteration: 2 * UNROLL 16-byte loads in flight per thread
constexpr int MAX_SPLITS = 64;
constexpr int MIN_CHUNK = 64;     // fewest keys a split is given
constexpr int CHUNK_ALIGN = 32;
constexpr float LOG2E = 1.4426950408889634f;
constexpr float MASKED = -30000.0f;  // log2-domain stand-in for finfo.min, as in attention_dense.cu

struct Params {
  const __nv_bfloat16 *q, *k, *v;
  __nv_bfloat16* o;
  const unsigned char* mask;  // [batch, >= nk] bytes, nonzero = masked, or NULL
  const float* slopes;        // [heads] or NULL
  float* ws;                  // nsplit > 1: [batch, heads, nsplit, head_dim + 2] partials (max, sum, acc[head_dim])
  const int* nk_dev;          // NULL: nk, chunk and nsplit below are the plan; else the key count is
                              // min(*nk_dev, nk) and the plan is made on the device from num_sms
  long long q_bs, kv_bs, ldkv, o_bs, mask_bs;
  int heads, nk, chunk, nsplit, num_sms;
  float sl2;                  // scale * log2(e)
};

// Splits so that (splits x batch x heads) CTAs make about two per SM, each split at least MIN_CHUNK keys (rounded up
// to CHUNK_ALIGN), and no split empty.  Depends on nothing but its arguments; the host and the device call the same
// code, so both make the same plan.
__host__ __device__ __forceinline__ int split_count(long long bh, int nk, int num_sms, int* chunk) {
  int s = (nk + MIN_CHUNK - 1) / MIN_CHUNK;
  s = s < MAX_SPLITS ? s : MAX_SPLITS;
  const long long cap = (2LL * num_sms + bh - 1) / bh;
  s = (long long)s < cap ? s : (int)cap;
  s = s > 1 ? s : 1;
  int c = (nk + s - 1) / s;
  c = (c + CHUNK_ALIGN - 1) / CHUNK_ALIGN * CHUNK_ALIGN;
  *chunk = c;
  return (nk + c - 1) / c;
}

// An upper bound of split_count over every nk in [1, nk_max]: the split count before the chunk rounding, which is
// non-decreasing in nk and never below the rounded count.
static int max_split_count(long long bh, int nk_max, int num_sms) {
  int s = std::min(MAX_SPLITS, (nk_max + MIN_CHUNK - 1) / MIN_CHUNK);
  return (int)std::max(1LL, std::min((long long)s, (2LL * num_sms + bh - 1) / bh));
}

// The key count and split plan of this launch.  A device key count <= 0 gives one split over no keys: zeros.
__device__ __forceinline__ void plan(const Params& p, long long bh, int* nk, int* chunk, int* nsplit) {
  if (p.nk_dev == nullptr) {
    *nk = p.nk; *chunk = p.chunk; *nsplit = p.nsplit;
    return;
  }
  const int n = min(*p.nk_dev, p.nk);
  if (n <= 0) {
    *nk = 0; *chunk = 0; *nsplit = 1;
    return;
  }
  *nk = n;
  *nsplit = split_count(bh, n, p.num_sms, chunk);
}

__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  f[0] = bf16_lo(u.x); f[1] = bf16_hi(u.x); f[2] = bf16_lo(u.y); f[3] = bf16_hi(u.y);
  f[4] = bf16_lo(u.z); f[5] = bf16_hi(u.z); f[6] = bf16_lo(u.w); f[7] = bf16_hi(u.w);
}

template <int HD>
__global__ void __launch_bounds__(THREADS) kv_decode_split_kernel(const Params p) {
  constexpr int CV = HD / 8;                      // threads that load a key row
  constexpr int C = CV <= 8 ? 8 : 16;             // lanes per key group, a power of two
  static_assert(HD % 8 == 0 && CV <= C, "head_dim must be a multiple of 8 and at most 128");
  constexpr int NG = THREADS / C;     // key groups per CTA
  constexpr int STEP = NG * UNROLL;   // keys per CTA iteration
  __shared__ float s_m[NG], s_l[NG];
  __shared__ float s_acc[NG][HD];

  const int split = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int grp = threadIdx.x / C, c = threadIdx.x % C;
  const bool active = c < CV;         // lanes past the row's last 16-byte piece hold zeros
  int nk, chunk, nsplit;
  plan(p, (long long)gridDim.z * p.heads, &nk, &chunk, &nsplit);
  if (split >= nsplit) return;   // uniform over the CTA, before any barrier
  const int k0 = split * chunk, k1 = min(nk, k0 + chunk);

  float qf[8];
  unpack8(active ? *reinterpret_cast<const uint4*>(p.q + b * p.q_bs + h * HD + c * 8) : make_uint4(0u, 0u, 0u, 0u), qf);
  const __nv_bfloat16* kp = p.k + b * p.kv_bs + h * HD + c * 8;
  const __nv_bfloat16* vp = p.v + b * p.kv_bs + h * HD + c * 8;
  const unsigned char* mp = p.mask != nullptr ? p.mask + b * p.mask_bs : nullptr;
  const float slope2 = p.slopes != nullptr ? p.slopes[h] * LOG2E : 0.f;

  float m = -INFINITY, l = 0.f, acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;

  // the loop bound is uniform over the CTA, so every lane of a group takes part in its shuffles
  for (int base = k0; base < k1; base += STEP) {
    uint4 kr[UNROLL], vr[UNROLL];
    bool msk[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const int key = base + u * NG + grp;
      kr[u] = vr[u] = make_uint4(0u, 0u, 0u, 0u);
      msk[u] = false;
      if (key < k1) {
        if (active) {
          kr[u] = __ldg(reinterpret_cast<const uint4*>(kp + key * p.ldkv));
          vr[u] = __ldg(reinterpret_cast<const uint4*>(vp + key * p.ldkv));
        }
        if (mp != nullptr) msk[u] = mp[key] != 0;
      }
    }
    float s[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      float kf[8];
      unpack8(kr[u], kf);
      float d = qf[0] * kf[0];
#pragma unroll
      for (int i = 1; i < 8; ++i) d = fmaf(qf[i], kf[i], d);
#pragma unroll
      for (int o = C / 2; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);   // same sum on every lane
      const int key = base + u * NG + grp;
      s[u] = key < k1 ? (msk[u] ? MASKED : fmaf(d, p.sl2, slope2 * (float)key)) : -INFINITY;
    }
    float mx = m;
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) mx = fmaxf(mx, s[u]);
    const float sub = mx == -INFINITY ? 0.f : mx;
    const float corr = ex2_approx(m - sub);
    l *= corr;
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] *= corr;
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const float pu = ex2_approx(s[u] - sub);
      float vf[8];
      unpack8(vr[u], vf);
      l += pu;
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = fmaf(pu, vf[i], acc[i]);
    }
    m = mx;
  }

  // merge the key groups in group order
  if (c == 0) { s_m[grp] = m; s_l[grp] = l; }
  if (active) {
#pragma unroll
    for (int i = 0; i < 8; ++i) s_acc[grp][c * 8 + i] = acc[i];
  }
  __syncthreads();
  if (threadIdx.x < HD) {
    const int d = threadIdx.x;
    float M = -INFINITY;
#pragma unroll
    for (int g = 0; g < NG; ++g) M = fmaxf(M, s_m[g]);
    const float sub = M == -INFINITY ? 0.f : M;
    float L = 0.f, A = 0.f;
#pragma unroll
    for (int g = 0; g < NG; ++g) {
      const float w = ex2_approx(s_m[g] - sub);
      L = fmaf(s_l[g], w, L);
      A = fmaf(s_acc[g][d], w, A);
    }
    if (nsplit == 1) {
      p.o[b * p.o_bs + h * HD + d] = __float2bfloat16_rn(L > 0.f ? A * (1.f / L) : 0.f);
    } else {
      float* part = p.ws + (((long long)b * p.heads + h) * nsplit + split) * (HD + 2);
      part[2 + d] = A;
      if (d == 0) { part[0] = M; part[1] = L; }
    }
  }
}

// One CTA per (batch, head), one thread per output column; partials are merged in split order.
template <int HD>
__global__ void __launch_bounds__(HD) kv_decode_combine_kernel(const Params p) {
  const int bh = blockIdx.x, d = threadIdx.x;
  const int b = bh / p.heads, h = bh % p.heads;
  int nk, chunk, nsplit;
  plan(p, (long long)gridDim.x, &nk, &chunk, &nsplit);
  if (nsplit == 1) return;   // the split kernel wrote the output
  const float* part = p.ws + (long long)bh * nsplit * (HD + 2);
  float M = -INFINITY;
  for (int s = 0; s < nsplit; ++s) M = fmaxf(M, part[s * (HD + 2)]);
  float L = 0.f, A = 0.f;
  for (int s = 0; s < nsplit; ++s) {
    const float* ps = part + s * (HD + 2);
    const float w = ex2_approx(ps[0] - M);
    L = fmaf(ps[1], w, L);
    A = fmaf(ps[2 + d], w, A);
  }
  p.o[b * p.o_bs + h * HD + d] = __float2bfloat16_rn(L > 0.f ? A * (1.f / L) : 0.f);
}

// One CTA row per batch entry; each thread moves 16 bytes of the new row.  Thread 0 of the first CTA sets the key-mask
// byte.  The position is read on the device; outside [0, capacity) nothing is written.
constexpr int APPEND_THREADS = 128;

__global__ void __launch_bounds__(APPEND_THREADS) kv_append_kernel(const uint4* src, long long src_bs, uint4* cache,
                                                                   long long cache_bs, long long ld, int vecs,
                                                                   int capacity, const int* pos_dev,
                                                                   unsigned char* key_mask, long long mask_bs,
                                                                   const unsigned char* new_masked) {
  const int b = blockIdx.y;
  const int pos = *pos_dev;
  if (pos < 0 || pos >= capacity) return;
  const int i = blockIdx.x * APPEND_THREADS + threadIdx.x;
  // strides are in bf16 elements, multiples of 8: one uint4 is 8 elements
  if (i < vecs) cache[(b * cache_bs + pos * ld) / 8 + i] = src[b * src_bs / 8 + i];
  if (key_mask != nullptr && blockIdx.x == 0 && threadIdx.x == 0)
    key_mask[b * mask_bs + pos] = (new_masked != nullptr && new_masked[b] != 0) ? 1 : 0;
}

static bool misaligned(const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) != 0; }

// Argument checks shared by both decode entry points; nk is the key count (ofk_attn_decode) or nk_max.
static int check_decode_args(const void* q, long long q_bstride, const void* k, const void* v, long long kv_bstride,
                             long long ldkv, const void* o, long long o_bstride, int batch, int heads, int head_dim,
                             int nk, const unsigned char* key_mask, long long mask_bstride, const void* workspace) {
  if (!q || !k || !v || !o || !workspace) return ofk_set_error(OFK_ERR_ARG, "attention decode: null pointer");
  if (head_dim != 64 && head_dim != 80 && head_dim != 128)
    return ofk_set_error(OFK_ERR_ARG, "attention decode: head_dim must be 64, 80 or 128");
  if (batch < 1 || heads < 1 || nk < 1) return ofk_set_error(OFK_ERR_ARG, "attention decode: empty problem");
  if (batch > 65535 || heads > 65535) return ofk_set_error(OFK_ERR_ARG, "attention decode: batch/heads exceed grid limits");
  if (misaligned(q) || misaligned(k) || misaligned(v) || misaligned(o) || misaligned(workspace) ||
      (key_mask != nullptr && misaligned(key_mask)))
    return ofk_set_error(OFK_ERR_ALIGN, "attention decode: pointers must be 16-byte aligned");
  if ((q_bstride | kv_bstride | ldkv | o_bstride) % 8 != 0 || (key_mask != nullptr && mask_bstride % 8 != 0))
    return ofk_set_error(OFK_ERR_ALIGN, "attention decode: strides must be multiples of 8 elements");
  return 0;
}

static int device_sms(int* sms) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
      *sms <= 0) {
    cudaGetLastError();
    return ofk_set_error(OFK_ERR_CUDA, "attention decode: no CUDA device");
  }
  return 0;
}

static Params make_params(const void* q, long long q_bstride, const void* k, const void* v, long long kv_bstride,
                          long long ldkv, void* o, long long o_bstride, int heads, int nk, float scale,
                          const unsigned char* key_mask, long long mask_bstride, const float* slopes, void* workspace) {
  Params p{};
  p.q = (const __nv_bfloat16*)q; p.k = (const __nv_bfloat16*)k; p.v = (const __nv_bfloat16*)v; p.o = (__nv_bfloat16*)o;
  p.mask = key_mask; p.slopes = slopes; p.ws = (float*)workspace;
  p.q_bs = q_bstride; p.kv_bs = kv_bstride; p.ldkv = ldkv; p.o_bs = o_bstride; p.mask_bs = mask_bstride;
  p.heads = heads; p.nk = nk; p.sl2 = scale * LOG2E;
  return p;
}

// grid_splits: the split kernel's grid width (the plan's split count, or its upper bound for a device key count).
template <int HD>
static int launch_hd(const Params& p, int batch, int grid_splits, bool always_combine, cudaStream_t s) {
  kv_decode_split_kernel<HD><<<dim3(grid_splits, p.heads, batch), THREADS, 0, s>>>(p);
  OFK_CHECK_LAUNCH();
  if (always_combine || p.nsplit > 1) {
    kv_decode_combine_kernel<HD><<<(unsigned)((long long)batch * p.heads), HD, 0, s>>>(p);
    OFK_CHECK_LAUNCH();
  }
  return 0;
}

static int launch(int head_dim, const Params& p, int batch, int grid_splits, bool always_combine, cudaStream_t s) {
  if (head_dim == 64) return launch_hd<64>(p, batch, grid_splits, always_combine, s);
  if (head_dim == 80) return launch_hd<80>(p, batch, grid_splits, always_combine, s);
  return launch_hd<128>(p, batch, grid_splits, always_combine, s);
}

}  // namespace decode
}  // namespace ofk

extern "C" long long ofk_attn_decode_workspace_bytes(int batch, int heads, int head_dim, int nk) {
  using namespace ofk::decode;
  if ((head_dim != 64 && head_dim != 80 && head_dim != 128) || batch < 1 || heads < 1 || nk < 1) return OFK_ERR_ARG;
  const long long splits = std::min(MAX_SPLITS, (nk + MIN_CHUNK - 1) / MIN_CHUNK);
  return (long long)batch * heads * splits * (head_dim + 2) * (long long)sizeof(float);
}

extern "C" int ofk_attn_decode(const void* q, long long q_bstride, const void* k, const void* v, long long kv_bstride,
                               long long ldkv, void* o, long long o_bstride, int batch, int heads, int head_dim, int nk,
                               float scale, const unsigned char* key_mask, long long mask_bstride, const float* slopes,
                               void* workspace, void* stream) {
  using namespace ofk::decode;
  int rc = check_decode_args(q, q_bstride, k, v, kv_bstride, ldkv, o, o_bstride, batch, heads, head_dim, nk, key_mask,
                             mask_bstride, workspace);
  int sms = 0;
  if (rc != 0 || (rc = device_sms(&sms)) != 0) return rc;
  Params p = make_params(q, q_bstride, k, v, kv_bstride, ldkv, o, o_bstride, heads, nk, scale, key_mask, mask_bstride,
                         slopes, workspace);
  p.nsplit = split_count((long long)batch * heads, nk, sms, &p.chunk);
  cudaStream_t s = (cudaStream_t)stream;
  return launch(head_dim, p, batch, p.nsplit, false, s);
}

extern "C" int ofk_attn_decode_dev(const void* q, long long q_bstride, const void* k, const void* v,
                                   long long kv_bstride, long long ldkv, void* o, long long o_bstride, int batch,
                                   int heads, int head_dim, int nk_max, const int* nk_dev, float scale,
                                   const unsigned char* key_mask, long long mask_bstride, const float* slopes,
                                   void* workspace, void* stream) {
  using namespace ofk::decode;
  if (!nk_dev) return ofk_set_error(OFK_ERR_ARG, "attention decode: null pointer");
  int rc = check_decode_args(q, q_bstride, k, v, kv_bstride, ldkv, o, o_bstride, batch, heads, head_dim, nk_max,
                             key_mask, mask_bstride, workspace);
  if (rc != 0) return rc;
  if ((reinterpret_cast<uintptr_t>(nk_dev) & 3) != 0)
    return ofk_set_error(OFK_ERR_ALIGN, "attention decode: nk_dev must be 4-byte aligned");
  int sms = 0;
  if ((rc = device_sms(&sms)) != 0) return rc;
  Params p = make_params(q, q_bstride, k, v, kv_bstride, ldkv, o, o_bstride, heads, nk_max, scale, key_mask,
                         mask_bstride, slopes, workspace);
  p.nk_dev = nk_dev;
  p.num_sms = sms;
  const int grid = max_split_count((long long)batch * heads, nk_max, sms);
  cudaStream_t s = (cudaStream_t)stream;
  return launch(head_dim, p, batch, grid, true, s);
}

extern "C" int ofk_kv_append(const void* src, long long src_bstride, void* cache, long long cache_bstride,
                             long long ld, int batch, int width, int capacity, const int* pos_dev,
                             unsigned char* key_mask, long long mask_bstride, const unsigned char* new_masked,
                             void* stream) {
  using namespace ofk::decode;
  if (!src || !cache || !pos_dev) return ofk_set_error(OFK_ERR_ARG, "kv append: null pointer");
  if (batch < 1 || width < 1 || capacity < 1) return ofk_set_error(OFK_ERR_ARG, "kv append: empty problem");
  if (batch > 65535) return ofk_set_error(OFK_ERR_ARG, "kv append: batch exceeds grid limits");
  if (ld < width || (key_mask != nullptr && mask_bstride < capacity))
    return ofk_set_error(OFK_ERR_ARG, "kv append: row stride below the row width");
  if (misaligned(src) || misaligned(cache) || (reinterpret_cast<uintptr_t>(pos_dev) & 3) != 0)
    return ofk_set_error(OFK_ERR_ALIGN, "kv append: src and cache must be 16-byte aligned, pos_dev 4-byte aligned");
  if ((width | src_bstride | cache_bstride | ld) % 8 != 0)
    return ofk_set_error(OFK_ERR_ALIGN, "kv append: width and strides must be multiples of 8 elements");
  const int vecs = width / 8;
  dim3 grid((unsigned)((vecs + APPEND_THREADS - 1) / APPEND_THREADS), (unsigned)batch);
  kv_append_kernel<<<grid, APPEND_THREADS, 0, (cudaStream_t)stream>>>(
      (const uint4*)src, src_bstride, (uint4*)cache, cache_bstride, ld, vecs, capacity, pos_dev, key_mask, mask_bstride,
      new_masked);
  OFK_CHECK_LAUNCH();
  return 0;
}
