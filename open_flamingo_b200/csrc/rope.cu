// Rotary position embeddings of the GPT-NeoX decoder blocks (HF GPTNeoXAttention + apply_rotary_pos_emb), as a
// layout change around the attention core.
//
// GPT-NeoX's query_key_value Linear emits, per row, the heads one after another, each as (q | k | v) of head_dim
// columns.  ofk_rope_pack reads those rows, rotates the first `rot` columns of q and k in the rotate_half form
//
//   y[j] = x[j] * cos[j] + rotate_half(x)[j] * sin[j],  rotate_half(x) = (-x[rot/2 .. rot), x[0 .. rot/2))
//
// and writes q, k and v to three destinations of their own, each head `width` columns wide with columns
// [head_dim, width) zero.  The attention cores exist for head_dim 64 and 128 only; a head_dim-80 head padded with
// zero columns to 128 gives the same scores, softmax and output, since zero columns add exact zeros to every product.
// The products are rounded where autocast rounds them in HF's module: the bf16 inputs are multiplied by the fp32 cos
// and sin and added in fp32 (no fused multiply-add, as PyTorch's separate kernels do) and the sum is rounded to bf16
// once.  Columns at or past `rot` are copied bit for bit.
//
// With rot = 0 nothing is rotated and the kernel only re-lays heads out: the cached path uses that to pad the K/V rows
// of its cache (K columns, then V columns, head_dim per head) to the padded width.
//
// ofk_rope_append_dev is the one-token form for a captured decode step: it writes q unpadded and the rotated K and the
// V into the KV-cache row at a position read on the device (and that row's key-mask byte), so that one CUDA graph
// serves every position.  It rotates with the same device function as ofk_rope_pack, so the two agree bit for bit.
//
// ofk_rope_unpack_bwd is the adjoint: from the padded dq, dk, dv it writes the gradient of the interleaved rows,
// applying the transposed rotation  dx = dy * cos + rotate_half^T(dy * sin),  rotate_half^T(u) = (u[rot/2 .. rot),
// -u[0 .. rot/2)),  in fp32 with one bf16 rounding; the padding columns are not read.
//
// Each thread moves 8 columns (16 bytes) of one head; head_dim and the widths are multiples of 8, so such a piece is
// all data or all padding.  The rotation partner at distance rot/2 need not sit in the same piece and is read per
// element.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "ofk_internal.h"
#include "ofk_ptx.cuh"

namespace ofk {
namespace rope {

constexpr int THREADS = 128;

struct PackParams {
  const __nv_bfloat16* src[3];   // q, k, v sources (NULL: part not written)
  __nv_bfloat16* dst[3];
  long long src_bs, src_ld;
  long long dst_bs[3], dst_ld[3];
  const float *cos, *sin;
  long long cs_bs, cs_ld;
  int src_hs, rows, heads, hd, rot;
  int width[3];
};

struct UnpackParams {
  const __nv_bfloat16* d[3];     // dq, dk, dv, each head `width` columns
  __nv_bfloat16* out;            // [batch, rows, heads * 3 * hd] interleaved (q | k | v) per head
  long long d_bs[3], d_ld[3];
  long long out_bs, out_ld;
  const float *cos, *sin;
  long long cs_bs, cs_ld;
  int rows, heads, hd, rot, width;
};

struct AppendParams {
  const __nv_bfloat16* src;      // [batch, heads * 3 * hd] interleaved (q | k | v) per head
  __nv_bfloat16* q;              // [batch, heads * hd]
  __nv_bfloat16* cache;          // [batch, capacity, >= 2 * heads * hd]: K columns, then V columns
  const float *cos, *sin;        // [1 or batch, rot]
  const int* pos;
  unsigned char* key_mask;       // [batch, >= capacity] or NULL
  const unsigned char* new_masked;
  long long src_bs, q_bs, cache_bs, ld, cs_bs, mask_bs;
  int heads, hd, rot, capacity;
};

__device__ __forceinline__ float ld_bf16(const __nv_bfloat16* p) { return __bfloat162float(*p); }

__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  return make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
}

__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  f[0] = bf16_lo(u.x); f[1] = bf16_hi(u.x); f[2] = bf16_lo(u.y); f[3] = bf16_hi(u.y);
  f[4] = bf16_lo(u.z); f[5] = bf16_hi(u.z); f[6] = bf16_lo(u.w); f[7] = bf16_hi(u.w);
}

// Columns [j0, j0 + 8) of one head x (bf16, 16-byte aligned at j0) with the first `rot` columns rotated by the
// row's c, s: the one place where ofk_rope_pack and ofk_rope_append_dev round, so that they round alike.
__device__ __forceinline__ uint4 rotate8(const __nv_bfloat16* x, int j0, int rot, const float* c, const float* s) {
  uint4 out = *reinterpret_cast<const uint4*>(x + j0);
  if (j0 < rot) {
    const int half = rot / 2;
    float f[8];
    unpack8(out, f);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int j = j0 + e;
      if (j < rot) {
        const float partner = j < half ? -ld_bf16(x + j + half) : ld_bf16(x + j - half);
        f[e] = __fadd_rn(__fmul_rn(f[e], c[j]), __fmul_rn(partner, s[j]));
      }
    }
    out = pack8(f);   // the unrotated elements are bf16 values: packing them again is exact
  }
  return out;
}

// One CTA per (batch row, part); blockIdx.x = b * rows + t, blockIdx.y = part (0 q, 1 k, 2 v).
__global__ void __launch_bounds__(THREADS) rope_pack_kernel(const PackParams p) {
  const int part = blockIdx.y;
  const __nv_bfloat16* src = p.src[part];
  if (src == nullptr) return;
  const long long b = blockIdx.x / p.rows, t = blockIdx.x % p.rows;
  const int W = p.width[part];
  const bool rotate = part < 2 && p.rot > 0;
  src += b * p.src_bs + t * p.src_ld;
  __nv_bfloat16* dst = p.dst[part] + b * p.dst_bs[part] + t * p.dst_ld[part];
  const float* c = rotate ? p.cos + b * p.cs_bs + t * p.cs_ld : nullptr;
  const float* s = rotate ? p.sin + b * p.cs_bs + t * p.cs_ld : nullptr;
  const int pieces = p.heads * W / 8;
  for (int i = threadIdx.x; i < pieces; i += THREADS) {
    const int h = i * 8 / W, j0 = i * 8 % W;
    uint4 out = make_uint4(0u, 0u, 0u, 0u);
    if (j0 < p.hd) {
      const __nv_bfloat16* x = src + (long long)h * p.src_hs;
      out = rotate ? rotate8(x, j0, p.rot, c, s) : *reinterpret_cast<const uint4*>(x + j0);
    }
    *reinterpret_cast<uint4*>(dst + (long long)h * W + j0) = out;
  }
}

// One CTA per (batch row, part), blockIdx.x = b, blockIdx.y = part (0 q, 1 k, 2 v).  q goes to its own row; k and v go
// to cache row *pos of their batch entry (K columns, then V columns), and nowhere when *pos is outside [0, capacity).
// The k CTA also writes the row's key-mask byte, as ofk_kv_append does.
__global__ void __launch_bounds__(THREADS) rope_append_dev_kernel(const AppendParams p) {
  const int part = blockIdx.y;
  const long long b = blockIdx.x;
  const int D = p.heads * p.hd;
  __nv_bfloat16* dst;
  if (part == 0) {
    dst = p.q + b * p.q_bs;
  } else {
    const int pos = *p.pos;
    if (pos < 0 || pos >= p.capacity) return;
    dst = p.cache + b * p.cache_bs + pos * p.ld + (part - 1) * D;
    if (part == 1 && p.key_mask != nullptr && threadIdx.x == 0)
      p.key_mask[b * p.mask_bs + pos] = (p.new_masked != nullptr && p.new_masked[b] != 0) ? 1 : 0;
  }
  const __nv_bfloat16* src = p.src + b * p.src_bs + part * p.hd;
  const bool rotate = part < 2 && p.rot > 0;
  const float* c = rotate ? p.cos + b * p.cs_bs : nullptr;
  const float* s = rotate ? p.sin + b * p.cs_bs : nullptr;
  for (int i = threadIdx.x; i < D / 8; i += THREADS) {
    const int h = i * 8 / p.hd, j0 = i * 8 % p.hd;
    const __nv_bfloat16* x = src + (long long)h * 3 * p.hd;
    *reinterpret_cast<uint4*>(dst + h * p.hd + j0) =
        rotate ? rotate8(x, j0, p.rot, c, s) : *reinterpret_cast<const uint4*>(x + j0);
  }
}

// One CTA per batch row; each thread writes 8 columns of the interleaved gradient row.
__global__ void __launch_bounds__(THREADS) rope_unpack_bwd_kernel(const UnpackParams p) {
  const long long b = blockIdx.x / p.rows, t = blockIdx.x % p.rows;
  const int half = p.rot / 2;
  const float* c = p.rot > 0 ? p.cos + b * p.cs_bs + t * p.cs_ld : nullptr;
  const float* s = p.rot > 0 ? p.sin + b * p.cs_bs + t * p.cs_ld : nullptr;
  __nv_bfloat16* out = p.out + b * p.out_bs + t * p.out_ld;
  const int hw = 3 * p.hd;
  const int pieces = p.heads * hw / 8;
  for (int i = threadIdx.x; i < pieces; i += THREADS) {
    const int h = i * 8 / hw, r = i * 8 % hw;
    const int part = r / p.hd, j0 = r % p.hd;
    const __nv_bfloat16* g = p.d[part] + b * p.d_bs[part] + t * p.d_ld[part] + (long long)h * p.width;
    uint4 v = *reinterpret_cast<const uint4*>(g + j0);
    if (part < 2 && j0 < p.rot) {
      float f[8];
      unpack8(v, f);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int j = j0 + e;
        if (j < p.rot) {
          const float other = j < half ? ld_bf16(g + j + half) * s[j + half] : -(ld_bf16(g + j - half) * s[j - half]);
          f[e] = fmaf(f[e], c[j], other);
        }
      }
      v = pack8(f);
    }
    *reinterpret_cast<uint4*>(out + (long long)h * hw + part * p.hd + j0) = v;
  }
}

static bool misaligned(const void* ptr, unsigned bytes) { return (reinterpret_cast<uintptr_t>(ptr) & (bytes - 1)) != 0; }

// Checks shared by both entry points: the problem, the rotation and the cos/sin operands.
static int check_common(int batch, int rows, int heads, int head_dim, int rot, const float* cos, const float* sin,
                        long long cs_bstride, long long ld_cs) {
  if (batch < 1 || rows < 1 || heads < 1) return ofk_set_error(OFK_ERR_ARG, "rope: empty problem");
  if ((long long)batch * rows > 0x7fffffffLL) return ofk_set_error(OFK_ERR_ARG, "rope: batch * rows exceeds the grid");
  if (head_dim < 8 || head_dim % 8 != 0) return ofk_set_error(OFK_ERR_ARG, "rope: head_dim must be a positive multiple of 8");
  if (rot < 0 || rot % 2 != 0 || rot > head_dim)
    return ofk_set_error(OFK_ERR_ARG, "rope: rot must be even and in [0, head_dim]");
  if (rot > 0) {
    if (!cos || !sin) return ofk_set_error(OFK_ERR_ARG, "rope: rotation needs cos and sin");
    if (cs_bstride < 0 || ld_cs < rot) return ofk_set_error(OFK_ERR_ARG, "rope: cos/sin strides must be >= 0 and >= rot");
    if (misaligned(cos, 4) || misaligned(sin, 4)) return ofk_set_error(OFK_ERR_ALIGN, "rope: cos and sin must be 4-byte aligned");
  }
  return 0;
}

}  // namespace rope
}  // namespace ofk

using namespace ofk::rope;

extern "C" int ofk_rope_pack(const void* src_q, const void* src_k, const void* src_v, long long src_bstride,
                             long long ld_src, int src_head_stride, int batch, int rows, int heads, int head_dim,
                             int rot, const float* cos, const float* sin, long long cs_bstride, long long ld_cs,
                             void* q, long long q_bstride, long long ldq, int q_width, void* k, long long k_bstride,
                             long long ldk, int k_width, void* v, long long v_bstride, long long ldv, int v_width,
                             void* stream) {
  const void* srcs[3] = {src_q, src_k, src_v};
  void* dsts[3] = {q, k, v};
  const long long bss[3] = {q_bstride, k_bstride, v_bstride}, lds[3] = {ldq, ldk, ldv};
  const int widths[3] = {q_width, k_width, v_width};
  if (!src_q && !src_k && !src_v) return ofk_set_error(OFK_ERR_ARG, "rope_pack: no part to write");
  for (int i = 0; i < 3; ++i)
    if (srcs[i] && !dsts[i]) return ofk_set_error(OFK_ERR_ARG, "rope_pack: a part with a source needs a destination");
  int rc = check_common(batch, rows, heads, head_dim, rot, cos, sin, cs_bstride, ld_cs);
  if (rc != 0) return rc;
  if (src_head_stride < head_dim || src_bstride < 0 || ld_src < 0)
    return ofk_set_error(OFK_ERR_ARG, "rope_pack: source head stride below head_dim, or a negative stride");
  for (int i = 0; i < 3; ++i) {
    if (!srcs[i]) continue;
    if (widths[i] < head_dim || widths[i] % 8 != 0)
      return ofk_set_error(OFK_ERR_ARG, "rope_pack: each width must be >= head_dim and a multiple of 8");
    if (bss[i] < 0 || lds[i] < (long long)heads * widths[i])
      return ofk_set_error(OFK_ERR_ARG, "rope_pack: destination row stride below heads * width");
  }
  for (int i = 0; i < 3; ++i)
    if (srcs[i] && (misaligned(srcs[i], 16) || misaligned(dsts[i], 16)))
      return ofk_set_error(OFK_ERR_ALIGN, "rope_pack: sources and destinations must be 16-byte aligned");
  if ((src_bstride | ld_src | (long long)src_head_stride) % 8 != 0)
    return ofk_set_error(OFK_ERR_ALIGN, "rope_pack: source strides must be multiples of 8 elements");
  for (int i = 0; i < 3; ++i)
    if (srcs[i] && (bss[i] | lds[i]) % 8 != 0)
      return ofk_set_error(OFK_ERR_ALIGN, "rope_pack: destination strides must be multiples of 8 elements");
  PackParams p{};
  for (int i = 0; i < 3; ++i) {
    p.src[i] = (const __nv_bfloat16*)srcs[i];
    p.dst[i] = (__nv_bfloat16*)dsts[i];
    p.dst_bs[i] = bss[i]; p.dst_ld[i] = lds[i]; p.width[i] = widths[i];
  }
  p.src_bs = src_bstride; p.src_ld = ld_src; p.src_hs = src_head_stride;
  p.cos = cos; p.sin = sin; p.cs_bs = cs_bstride; p.cs_ld = ld_cs;
  p.rows = rows; p.heads = heads; p.hd = head_dim; p.rot = rot;
  rope_pack_kernel<<<dim3((unsigned)((long long)batch * rows), 3), THREADS, 0, (cudaStream_t)stream>>>(p);
  OFK_CHECK_LAUNCH();
  return 0;
}

extern "C" int ofk_rope_append_dev(const void* qkv, long long qkv_bstride, int batch, int heads, int head_dim, int rot,
                                   const float* cos, const float* sin, long long cs_bstride, void* q,
                                   long long q_bstride, void* cache, long long cache_bstride, long long ld, int capacity,
                                   const int* pos_dev, unsigned char* key_mask, long long mask_bstride,
                                   const unsigned char* new_masked, void* stream) {
  if (!qkv || !q || !cache || !pos_dev) return ofk_set_error(OFK_ERR_ARG, "rope_append_dev: null pointer");
  int rc = check_common(batch, 1, heads, head_dim, rot, cos, sin, cs_bstride, rot);
  if (rc != 0) return rc;
  if (capacity < 1) return ofk_set_error(OFK_ERR_ARG, "rope_append_dev: capacity must be >= 1");
  const long long D = (long long)heads * head_dim;
  if (qkv_bstride < 3 * D || q_bstride < D || ld < 2 * D || cache_bstride < capacity * ld ||
      (key_mask != nullptr && mask_bstride < capacity))
    return ofk_set_error(OFK_ERR_ARG, "rope_append_dev: a stride is below its row width");
  if (misaligned(qkv, 16) || misaligned(q, 16) || misaligned(cache, 16) || misaligned(pos_dev, 4))
    return ofk_set_error(OFK_ERR_ALIGN, "rope_append_dev: qkv, q and cache must be 16-byte aligned, pos_dev 4-byte");
  if ((qkv_bstride | q_bstride | cache_bstride | ld) % 8 != 0)
    return ofk_set_error(OFK_ERR_ALIGN, "rope_append_dev: strides must be multiples of 8 elements");
  AppendParams p{};
  p.src = (const __nv_bfloat16*)qkv; p.q = (__nv_bfloat16*)q; p.cache = (__nv_bfloat16*)cache;
  p.cos = cos; p.sin = sin; p.pos = pos_dev; p.key_mask = key_mask; p.new_masked = new_masked;
  p.src_bs = qkv_bstride; p.q_bs = q_bstride; p.cache_bs = cache_bstride; p.ld = ld; p.cs_bs = cs_bstride;
  p.mask_bs = mask_bstride;
  p.heads = heads; p.hd = head_dim; p.rot = rot; p.capacity = capacity;
  rope_append_dev_kernel<<<dim3((unsigned)batch, 3), THREADS, 0, (cudaStream_t)stream>>>(p);
  OFK_CHECK_LAUNCH();
  return 0;
}

extern "C" int ofk_rope_unpack_bwd(const void* dq, long long dq_bstride, long long lddq, const void* dk,
                                   long long dk_bstride, long long lddk, const void* dv, long long dv_bstride,
                                   long long lddv, int width, int batch, int rows, int heads, int head_dim, int rot,
                                   const float* cos, const float* sin, long long cs_bstride, long long ld_cs,
                                   void* dqkv, long long dqkv_bstride, long long lddqkv, void* stream) {
  if (!dq || !dk || !dv || !dqkv) return ofk_set_error(OFK_ERR_ARG, "rope_unpack_bwd: null pointer");
  int rc = check_common(batch, rows, heads, head_dim, rot, cos, sin, cs_bstride, ld_cs);
  if (rc != 0) return rc;
  if (width < head_dim || width % 8 != 0)
    return ofk_set_error(OFK_ERR_ARG, "rope_unpack_bwd: width must be >= head_dim and a multiple of 8");
  const long long bss[3] = {dq_bstride, dk_bstride, dv_bstride}, lds[3] = {lddq, lddk, lddv};
  for (int i = 0; i < 3; ++i)
    if (bss[i] < 0 || lds[i] < (long long)heads * width)
      return ofk_set_error(OFK_ERR_ARG, "rope_unpack_bwd: gradient row stride below heads * width");
  if (dqkv_bstride < 0 || lddqkv < 3LL * heads * head_dim)
    return ofk_set_error(OFK_ERR_ARG, "rope_unpack_bwd: output row stride below heads * 3 * head_dim");
  if (misaligned(dq, 16) || misaligned(dk, 16) || misaligned(dv, 16) || misaligned(dqkv, 16))
    return ofk_set_error(OFK_ERR_ALIGN, "rope_unpack_bwd: operands must be 16-byte aligned");
  if ((dq_bstride | lddq | dk_bstride | lddk | dv_bstride | lddv | dqkv_bstride | lddqkv) % 8 != 0)
    return ofk_set_error(OFK_ERR_ALIGN, "rope_unpack_bwd: strides must be multiples of 8 elements");
  UnpackParams p{};
  p.d[0] = (const __nv_bfloat16*)dq; p.d[1] = (const __nv_bfloat16*)dk; p.d[2] = (const __nv_bfloat16*)dv;
  for (int i = 0; i < 3; ++i) { p.d_bs[i] = bss[i]; p.d_ld[i] = lds[i]; }
  p.out = (__nv_bfloat16*)dqkv; p.out_bs = dqkv_bstride; p.out_ld = lddqkv;
  p.cos = cos; p.sin = sin; p.cs_bs = cs_bstride; p.cs_ld = ld_cs;
  p.rows = rows; p.heads = heads; p.hd = head_dim; p.rot = rot; p.width = width;
  rope_unpack_bwd_kernel<<<(unsigned)((long long)batch * rows), THREADS, 0, (cudaStream_t)stream>>>(p);
  OFK_CHECK_LAUNCH();
  return 0;
}
