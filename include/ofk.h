/*
 * ofk.h -- C ABI of libofk.so: the H100 (sm_90a) kernels behind the OpenFlamingo dense hot path.
 *
 * The reference (mlfoundations/open_flamingo) is pure eager PyTorch and has NO native interface; each
 * entry point below names the reference Python it replaces (paths relative to the reference repo root,
 * open_flamingo/src/...).  INTEGRATION.md shows the ctypes binding a maintainer would add.
 *
 * Conventions
 *  - All pointers are DEVICE pointers unless stated; no torch types cross this boundary.
 *  - `stream` is a cudaStream_t passed as void*.  Kernels are enqueued on it and never synchronise.
 *  - Nothing here allocates device memory: the caller owns outputs and workspaces.
 *  - Return value: 0 on success, negative OFK_ERR_* otherwise; ofk_last_error() gives the message.
 *    Nothing throws across the ABI.
 *  - bf16 tensors are raw uint16 storage (__nv_bfloat16); "f32" is IEEE float.
 *  - Row-major everywhere; `ld*` are row strides in ELEMENTS.
 */
#ifndef OFK_H_
#define OFK_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OFK_ABI_VERSION 4

enum {
  OFK_OK = 0,
  OFK_ERR_ARG = -1,    /* bad argument (shape / null / unsupported combination) */
  OFK_ERR_ALIGN = -2,  /* pointer or stride alignment violates the TMA / vector-access contract */
  OFK_ERR_CUDA = -3,   /* CUDA runtime error at launch */
  OFK_ERR_DRIVER = -4  /* driver entry point (tensor-map encode) unavailable or failed */
};

/* GEMM epilogues (fused into the wgmma kernel's register->global stage). */
enum {
  OFK_EPI_STORE_BF16 = 0,      /* out(bf16) = acc                                            nn.Linear, helpers.py:35-37,153-155 */
  OFK_EPI_STORE_F32 = 1,       /* out(f32)  = acc                                                                               */
  OFK_EPI_ATOMIC_F32 = 2,      /* out(f32) += acc  (red.global.add; wgrad / split-K / dmedia accumulation over layers)          */
  OFK_EPI_BIAS_BF16 = 3,       /* out(bf16) = acc + bias[n]                                  ViT in_proj / out_proj (open_clip) */
  OFK_EPI_BIAS_QGELU_BF16 = 4, /* out(bf16) = quick_gelu(acc + bias[n])                      ViT mlp.c_fc + QuickGELU           */
  OFK_EPI_GELU_DUAL = 5,       /* out(bf16) = z = acc ; out2(bf16) = gelu_erf(z)             FeedForward helpers.py:19-20        */
  OFK_EPI_GATE_RESID_F32 = 6,  /* out(f32) = bf16(acc)*tanh(*gate) + aux(f32); out2(bf16)=acc (optional; gate NULL => 1)
                                  helpers.py:267-277 (x = branch * gate.tanh() + x), helpers.py:130-131 (Perceiver residuals)   */
  OFK_EPI_DGELU_BF16 = 7,      /* out(bf16) = acc * gelu_erf'(aux(bf16) = z)                 autograd of helpers.py:20           */
  OFK_EPI_BIAS_RESID_F32 = 8,  /* out(f32) = bf16(acc + bias[n]) + aux(f32)  (out may alias aux)  ViT residual adds            */
  OFK_EPI_BIAS_GELU_BF16 = 9   /* out(bf16) = gelu_erf(acc + bias[n])                        ViT mlp.c_fc + nn.GELU (non-openai) */
};

const char* ofk_last_error(void);
int ofk_abi_version(void);
/* Number of kernels this library has launched since load (bench.py's `gpu_launches`). */
long long ofk_launch_count(void);

/* ------------------------------------------------------------------------------------------------
 * GEMM  out[m,n] = epi( sum_k A(m,k) * B(n,k) ), bf16 operands, fp32 accumulate in registers (wgmma).
 *   a_mn_major = 0: A stored [M,K] (K contiguous).  = 1: A stored [K,M] (M contiguous).
 *   b_mn_major = 0: B stored [N,K] (K contiguous).  = 1: B stored [K,N] (N contiguous).
 *   forward  y = x W^T       : A=x [R,in]  (0), B=W [out,in] (0)         nn.Linear (helpers.py:18-21,35-37,153-155)
 *   dgrad    dx = dy W       : A=dy [R,out](0), B=W [out,in] (1), K=out  autograd of the above
 *   wgrad    dW += dy^T x    : A=dy [R,out](1), B=x [R,in]   (1), K=R    autograd of the above (ATOMIC_F32)
 *   splits  : split-K factor (ATOMIC_F32 only).  block_n: 0, 128, 256 or 512 -- a tile-width hint, ignored: the
 *             sm_90a kernel picks 128 x 128 or 128 x 256 tiles from the problem's size, and both give the same bits.
 * Requirements: N % 16 == 0; operand base pointers 16-byte aligned, lda/ldb % 8 == 0.  The epilogue moves its
 *   operands in 16-byte pieces, so the same holds for every one it uses: `out` 16-byte aligned with ldo % 4 == 0
 *   (f32 out) or ldo % 8 == 0 (bf16 out); `out2` (bf16) with ldo2 % 8 == 0; `aux` with ldaux % 4 == 0 (f32, the
 *   RESID epilogues) or % 8 == 0 (bf16, DGELU); `bias` 16-byte aligned.  Violations return OFK_ERR_ALIGN, and every
 *   argument is checked before the first CUDA call.  K needs no alignment: past K the operands are read as zeros.
 */
int ofk_gemm_bf16(int epi, int a_mn_major, int b_mn_major, const void* A, long long lda, const void* B,
                  long long ldb, int M, int N, int K, int splits, int block_n, void* out, long long ldo,
                  void* out2, long long ldo2, const void* aux, long long ldaux, const float* bias,
                  const float* gate, void* stream);

/* Leave `n` SMs (rounded down to whole TPCs of two SMs, at most 64) out of every persistent GEMM grid launched from now
 * on; returns the previous value.  The data-parallel step uses it while gradient-chunk all-reduces are in flight
 * (train.GradBucket): a persistent grid that owns all 132 SMs lets NCCL's CTAs in only at kernel boundaries, which serialises the
 * "overlapped" reduction behind each GEMM.  0 restores the full grid. */
int ofk_gemm_reserve_sms(int n);

/* Same GEMM with grouped row maps (logical row r -> (r / rows_per_group) * group_stride + group_offset + r % rpg):
 *   out_*  : where the rows of `out` go inside a larger interleaved buffer (STORE_BF16 / BIAS_BF16 / STORE_F32;
 *            M must be a multiple of rows_per_group, else OFK_ERR_ARG);
 *   a_k_*  : which physical rows of an MN-major A form the reduction dimension (rows_per_group % 64 == 0).
 * Lets PerceiverAttention's k/v for the media tokens and for the latents (helpers.py:53-54: to_kv(cat(x, latents)))
 * be produced by two GEMMs that write straight into the concatenated [b*T, v+n, 2*inner] layout, and lets the
 * wgrads reduce over only the media (or only the latent) rows of the concatenated gradient.  0 = identity. */
int ofk_gemm_bf16_grouped(int epi, int a_mn_major, int b_mn_major, const void* A, long long lda, const void* B,
                          long long ldb, int M, int N, int K, int splits, int block_n, void* out, long long ldo,
                          const float* bias, int out_rows_per_group, int out_group_stride, int out_group_offset,
                          int a_k_rows_per_group, int a_k_group_stride, int a_k_group_offset, void* stream);

/* ------------------------------------------------------------------------------------------------
 * LayerNorm over the last dim (eps inside sqrt, affine), fp32 statistics.  nn.LayerNorm at
 * helpers.py:17,32-33,47-48,105,132,151,184.
 *   x: [rows, D] f32 (ldx).  y: bf16 (y_is_f32 = 0) or f32, written at
 *   row index  (r / rows_per_group) * group_stride + group_offset + r % rows_per_group  of y (ldy) --
 *   this lets two LayerNorms write the two halves of PerceiverAttention's cat((x, latents), -2)
 *   (helpers.py:53) in place (rows_per_group <= 0: identity mapping; otherwise 0 <= group_offset and
 *   group_offset + rows_per_group <= group_stride, OFK_ERR_ARG).  mean/rstd: [rows] f32 outputs (may be NULL).
 *   D % 4 == 0, D <= 4096.  ldx, ldy multiples of 4; x, gamma, beta and an f32 y 16-byte aligned, a bf16 y 8-byte
 *   aligned (OFK_ERR_ALIGN).  Every argument is checked before the first CUDA call.
 */
int ofk_layernorm_fwd(const float* x, long long ldx, const float* gamma, const float* beta,
                      float eps, int rows, int D, void* y, int y_is_f32, long long ldy, int rows_per_group,
                      int group_stride, int group_offset, float* mean, float* rstd, void* stream);

/* LayerNorm backward.  dy: [rows, D] bf16 or f32 (same row mapping as fwd via dy_* group args);
 * x: f32 [rows, D]; dx(f32) = LN'(dy) (+ dx_add if non-NULL; dx_add may alias dx); dx NULL = parameter
 * gradients only (PerceiverAttention.norm_media: its input, the frozen ViT features, needs no gradient).
 * dgamma/dbeta (f32 [D]) are ACCUMULATED (+=).  workspace: >= ofk_layernorm_bwd_workspace(rows, D) bytes.
 * Requirements: the group mapping, D and strides as in the forward; x, gamma, dx, dx_add, workspace and an f32 dy
 * 16-byte aligned, a bf16 dy 8-byte aligned (OFK_ERR_ALIGN), all checked before the first CUDA call. */
long long ofk_layernorm_bwd_workspace(int rows, int D);
int ofk_layernorm_bwd(const void* dy, int dy_is_f32, long long lddy, int rows_per_group, int group_stride,
                      int group_offset, const float* x, long long ldx, const float* gamma, const float* mean,
                      const float* rstd, int rows, int D, float* dx, long long lddx, const float* dx_add,
                      long long ldadd, float* dgamma, float* dbeta, void* workspace, void* stream);

/* ------------------------------------------------------------------------------------------------
 * RMSNorm of the LLaMA decoder blocks (HF LlamaRMSNorm), csrc/rmsnorm.cu.  One 256-thread block per row; fp32
 * statistics summed in a fixed order, so both directions give the same bits on every launch.
 * ofk_rmsnorm_fwd:  y(bf16) = bf16(gamma * (x * rstd)),  rstd = rsqrt(mean(x^2) + eps): LlamaRMSNorm's product order,
 *   rounded once where autocast rounds its fp32 output as the next Linear's operand.
 *   x: [rows, D] f32 (ldx); gamma: [D] f32; y: [rows, D] bf16 (ldy); rstd: [rows] f32 output, or NULL.
 * ofk_rmsnorm_bwd (input gradient only: the LM's norms are frozen):
 *   dx(f32) = rstd * (gamma * dy - xhat * mean(gamma * dy * xhat)) + dx_add,  xhat = x * rstd,
 *   dy: [rows, D] bf16 (lddy); x, gamma, rstd: those of the forward; dx: [rows, D] f32 (lddx); dx_add: [rows, D] f32
 *   (ldadd) or NULL, and may alias dx.
 * Requirements: x, gamma, y (fwd) and dy, x, gamma, rstd, dx (bwd) non-NULL, rows >= 1, D a positive multiple of 8
 *   and <= 8192, every row stride >= D (OFK_ERR_ARG); x, gamma, y, dy, dx and dx_add 16-byte aligned, rstd 4-byte,
 *   ldx, lddx and ldadd multiples of 4 and ldy, lddy multiples of 8 (OFK_ERR_ALIGN).  Every argument is checked
 *   before the first CUDA call.
 */
int ofk_rmsnorm_fwd(const float* x, long long ldx, const float* gamma, float eps, int rows, int D, void* y,
                    long long ldy, float* rstd, void* stream);
int ofk_rmsnorm_bwd(const void* dy, long long lddy, const float* x, long long ldx, const float* gamma,
                    const float* rstd, int rows, int D, float* dx, long long lddx, const float* dx_add,
                    long long ldadd, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Attention core  O = softmax(scale * Q K^T + mask) V  per (batch, head), head_dim = 64, bf16 in/out,
 * fp32 softmax, online (flash-style).  Warpgroup kernels whose QK^T / PV (and the backward's five products) are wgmma on
 * 128-byte-swizzled shared-memory tiles, P / dS fed from registers.
 *   q: [batch, nq, heads*64] (ldq row stride), k/v: [batch, nk, heads*64] (ldk/ldv), o like q (ldo).
 *   q_bstride/k_bstride...: batch strides in elements.  lse: [batch, heads, nq] f32 (log2 domain, for bwd).
 *   mask_mode: 0 = none                                              PerceiverAttention helpers.py:58-63, ViT MHA
 *              1 = media mask, text_time == block+1  (torch.eq)       MaskedCrossAttention helpers.py:196-229
 *              2 = media mask, text_time >= block+1  (torch.ge)       only_attend_immediate_media=False
 *   text_time: [batch, nq] int32 (cumsum of media_locations, helpers.py:199-208); keys are grouped in
 *   blocks of `keys_per_media` (the Perceiver's latent count: a multiple of 16 dividing nk).  Mode 1 rows with
 *   text_time == 0 produce exact zeros (helpers.py:223-229) and LSE 0; any other row with no allowed key attends
 *   uniformly over all nk keys and passes no gradient to q or k (masked_fill(-finfo.max) + softmax, helpers.py:218-221).
 * Requirements (both directions): batch, heads, nq, nk >= 1 and batch, heads <= 65535 (OFK_ERR_ARG); q, k, v, o (and
 *   d_o) 16-byte aligned with every batch and row stride a multiple of 8 elements; lse, delta and text_time 4-byte
 *   aligned; dq, dk, dv 4-byte aligned with even batch and row strides (OFK_ERR_ALIGN).  Every argument is checked
 *   before the first CUDA call.  Output rows are written whole; bytes outside them are never touched.
 */
int ofk_attn_fwd(const void* q, const void* k, const void* v, void* o, float* lse, int batch, int heads, int nq,
                 int nk, long long q_bstride, long long ldq, long long k_bstride, long long ldk,
                 long long v_bstride, long long ldv, long long o_bstride, long long ldo, float scale,
                 int mask_mode, const int* text_time, int keys_per_media, void* stream);

/* Backward of the above.  delta: [batch, heads, nq] f32 scratch.  dq like q; dk/dv like k/v (bf16).
 * dq/dk/dv are fully overwritten.  */
int ofk_attn_bwd(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                 float* delta, void* dq, void* dk, void* dv, int batch, int heads, int nq, int nk,
                 long long q_bstride, long long ldq, long long k_bstride, long long ldk, long long v_bstride,
                 long long ldv, long long o_bstride, long long ldo, long long dq_bstride, long long lddq,
                 long long dk_bstride, long long lddk, long long dv_bstride, long long lddv, float scale,
                 int mask_mode, const int* text_time, int keys_per_media, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Dense self-attention core of the frozen LM's decoder blocks (HF MptAttention; reached via
 * flamingo_lm.py:63-65 -- SURVEY.md section 8f rank 1).  head_dim 64 or 128.  Same wgmma warpgroup kernels as above,
 * on the same tile layer (csrc/attention_dense.cu, csrc/attention_tile.cuh).
 *   S = scale * Q K^T + slopes[h] * key_index  (ALiBi; slopes NULL = no bias)
 *   masked (mask[b, q, k] != 0, mask: [batch, nq, nk] bytes or NULL; and/or causal: key > query + nk - nq)
 *   scores take "finfo.min" exactly like masked_fill: a fully masked row attends uniformly.
 *   pure_causal_flag: optional DEVICE int; nonzero means "the mask is exactly the causal rule" (all-ones HF
 *   attention_mask): the kernel then ignores `mask`, applies the causal rule and skips key tiles above the
 *   diagonal -- a device-side decision, so no host synchronisation is needed to pick the fast path.
 *   lse: [batch, heads, nq] f32, log2 domain (consumed only by ofk_attn_dense_bwd).
 * Backward is dgrad only (the LM is frozen): dq/dk/dv bf16, fully overwritten.
 * Requirements: head_dim 64 or 128; batch, heads, nq, nk >= 1 and batch, heads <= 65535; causal != 0 or a non-NULL
 *   pure_causal_flag needs nq <= nk (OFK_ERR_ARG): the cache always holds the current chunk, and with nq > nk whole
 *   query blocks would have no allowed key.  q, k, v, o (and d_o) 16-byte aligned with every batch and row stride a
 *   multiple of 8 elements; lse, delta, slopes and pure_causal_flag 4-byte aligned; dq, dk, dv 4-byte aligned with
 *   even batch and row strides (OFK_ERR_ALIGN).  mask is read byte by byte.  Every argument is checked before the
 *   first CUDA call.
 */
int ofk_attn_dense_fwd(const void* q, const void* k, const void* v, void* o, float* lse, int batch, int heads,
                       int head_dim, int nq, int nk, long long q_bstride, long long ldq, long long k_bstride,
                       long long ldk, long long v_bstride, long long ldv, long long o_bstride, long long ldo,
                       float scale, int causal, const unsigned char* mask, const float* slopes,
                       const int* pure_causal_flag, void* stream);
int ofk_attn_dense_bwd(const void* q, const void* k, const void* v, const void* o, const void* d_o,
                       const float* lse, float* delta, void* dq, void* dk, void* dv, int batch, int heads,
                       int head_dim, int nq, int nk, long long q_bstride, long long ldq, long long k_bstride,
                       long long ldk, long long v_bstride, long long ldv, long long o_bstride, long long ldo,
                       long long dq_bstride, long long lddq, long long dk_bstride, long long lddk,
                       long long dv_bstride, long long lddv, float scale, int causal, const unsigned char* mask,
                       const float* slopes, const int* pure_causal_flag, void* stream);

/* Decode attention of the same blocks with a KV cache (HF MptAttention or GPTNeoXAttention with past_key_values, one new
 * token): split-KV ("flash-decoding") over the cache, csrc/attention_decode.cu.  Semantics are those of
 * ofk_attn_dense_fwd at nq = 1:
 *   S = scale * q K^T + slopes[h] * key_index  (slopes NULL = no bias); key_mask[b, key] != 0 sets the score to
 *   "finfo.min" (a fully masked row attends uniformly); softmax and P.V in fp32, o stored as bf16.
 *   q: [batch, heads*head_dim] rows (q_bstride), k/v: [batch, nk, heads*head_dim] (shared kv_bstride and row stride
 *   ldkv -- the K and V column slices of one cache buffer), o like q (o_bstride), key_mask: [batch, >= nk] bytes
 *   (mask_bstride) or NULL, slopes: [heads] f32 or NULL.
 *   workspace: caller-owned, >= ofk_attn_decode_workspace_bytes(batch, heads, head_dim, nk) bytes; needs no
 *   initialisation.  The workspace-size function returns OFK_ERR_ARG for arguments the kernel would reject.
 * The key split is a pure function of (batch, heads, head_dim, nk, SM count) and partials are merged in a fixed order
 * without atomics: the output is bitwise identical from launch to launch and does not depend on the cache's capacity.
 * head_dim 80 (GPT-NeoX, RedPajama-INCITE-3B) runs on the same kernel with 16 lanes per key row, 10 of them loading.
 * Requirements: head_dim 64, 80 or 128; batch, heads, nk >= 1 (OFK_ERR_ARG); q, k, v, o, key_mask and workspace 16-byte
 * aligned, every batch or row stride a multiple of 8 elements (OFK_ERR_ALIGN).  Every argument is checked before the
 * first CUDA call. */
long long ofk_attn_decode_workspace_bytes(int batch, int heads, int head_dim, int nk);
int ofk_attn_decode(const void* q, long long q_bstride, const void* k, const void* v, long long kv_bstride,
                    long long ldkv, void* o, long long o_bstride, int batch, int heads, int head_dim, int nk,
                    float scale, const unsigned char* key_mask, long long mask_bstride, const float* slopes,
                    void* workspace, void* stream);

/* The same decode attention with the key count in DEVICE memory, so that one captured CUDA graph serves every decode
 * step: nk = min(*nk_dev, nk_max), read by the kernels.  The split plan is made on the device by the function the host
 * uses for ofk_attn_decode, so the output at a given nk is bitwise identical to ofk_attn_decode at that nk, whatever
 * nk_max is.  k/v, key_mask and slopes are as above with room for nk_max rows; no row at or past nk is read.
 * *nk_dev <= 0 writes zeros.  workspace: >= ofk_attn_decode_workspace_bytes(batch, heads, head_dim, nk_max) bytes.
 * Requirements: those of ofk_attn_decode with nk_max in place of nk, plus nk_dev non-NULL (OFK_ERR_ARG) and 4-byte
 * aligned (OFK_ERR_ALIGN).  Every argument is checked before the first CUDA call. */
int ofk_attn_decode_dev(const void* q, long long q_bstride, const void* k, const void* v, long long kv_bstride,
                        long long ldkv, void* o, long long o_bstride, int batch, int heads, int head_dim, int nk_max,
                        const int* nk_dev, float scale, const unsigned char* key_mask, long long mask_bstride,
                        const float* slopes, void* workspace, void* stream);

/* Append one K/V row per batch entry at a DEVICE-side position (the companion of ofk_attn_decode_dev in a captured
 * decode step):  cache[b, *pos_dev, 0:width] = src[b, 0:width]  (bf16, 16-byte accesses), and, when key_mask is
 * non-NULL, key_mask[b, *pos_dev] = (new_masked != NULL && new_masked[b] != 0)  (1 = the new token is padding).
 *   src: [batch, width] rows (src_bstride); cache: [batch, capacity, >= width] (cache_bstride, row stride ld);
 *   key_mask: [batch, >= capacity] bytes (mask_bstride) or NULL; new_masked: [batch] bytes or NULL (= unmasked).
 * A position outside [0, capacity) writes nothing.
 * Requirements: src, cache, pos_dev non-NULL; batch, width, capacity >= 1, batch <= 65535; ld >= width and
 *   mask_bstride >= capacity (OFK_ERR_ARG); src and cache 16-byte aligned, pos_dev 4-byte aligned, width and every
 *   stride of src and cache a multiple of 8 elements (OFK_ERR_ALIGN).  Every argument is checked before the first CUDA
 *   call. */
int ofk_kv_append(const void* src, long long src_bstride, void* cache, long long cache_bstride, long long ld,
                  int batch, int width, int capacity, const int* pos_dev, unsigned char* key_mask,
                  long long mask_bstride, const unsigned char* new_masked, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Rotary q/k packing of the GPT-NeoX decoder blocks (HF GPTNeoXAttention: apply_rotary_pos_emb on the rotate_half
 * form), csrc/rope.cu.  The query_key_value Linear emits rows of `heads` heads, each (q | k | v) of head_dim columns.
 *
 * ofk_rope_pack: for each part p in (q, k, v) whose source is non-NULL, reads head h of row (b, t) at
 *   src_p + b * src_bstride + t * ld_src + h * src_head_stride  (head_dim columns; the three parts share the strides)
 * and writes it to  dst_p + b * p_bstride + t * ldp + h * p_width, columns [head_dim, p_width) zero.  For q and k the
 * first `rot` columns are rotated:  y[j] = x[j] * cos[j] + rotate_half(x)[j] * sin[j]  with the product and the sum in
 * fp32 (not fused) and one rounding to bf16, as autocast rounds HF's module; the other columns are bit copies.
 *   cos, sin: f32 at  b * cs_bstride + t * ld_cs + j  (cs_bstride 0 = one table for every batch entry).  rot = 0 turns
 *   the rotation off and cos/sin may be NULL: the kernel then only re-lays heads out (e.g. pads cached K/V rows, whose
 *   K and V are two sources with head stride head_dim).
 *   The interleaved QKV GEMM output is src_q = qkv, src_k = qkv + head_dim, src_v = qkv + 2 * head_dim with head
 *   stride 3 * head_dim.
 * ofk_rope_unpack_bwd: the adjoint.  From dq, dk, dv (heads of `width` columns, padding not read) writes the gradient
 *   of the interleaved rows  dqkv[b, t, h * 3 * head_dim + p * head_dim + j],  with the transposed rotation
 *   dx = dy * cos + rotate_half^T(dy * sin),  rotate_half^T(u) = (u[rot/2 .. rot), -u[0 .. rot/2)),  fp32, one rounding.
 * Requirements: batch, rows, heads >= 1, head_dim a positive multiple of 8, rot even in [0, head_dim], cos and sin
 *   non-NULL with cs_bstride >= 0 and ld_cs >= rot when rot > 0, every width >= head_dim and a multiple of 8, every
 *   destination row stride >= heads * width (dqkv: >= 3 * heads * head_dim), src_head_stride >= head_dim, at least one
 *   source and a destination for each (OFK_ERR_ARG); bf16 operands 16-byte aligned with every stride a multiple of 8
 *   elements, cos and sin 4-byte aligned (OFK_ERR_ALIGN).  Every argument is checked before the first CUDA call.
 */
int ofk_rope_pack(const void* src_q, const void* src_k, const void* src_v, long long src_bstride, long long ld_src,
                  int src_head_stride, int batch, int rows, int heads, int head_dim, int rot, const float* cos,
                  const float* sin, long long cs_bstride, long long ld_cs, void* q, long long q_bstride, long long ldq,
                  int q_width, void* k, long long k_bstride, long long ldk, int k_width, void* v, long long v_bstride,
                  long long ldv, int v_width, void* stream);

/* ofk_rope_append_dev: the one-token rotary packing of a captured decode step (the companion of ofk_attn_decode_dev,
 * in place of ofk_rope_pack + ofk_kv_append).  For each batch entry b, from the interleaved row qkv + b * qkv_bstride
 * (heads of (q | k | v), head_dim columns each) it writes
 *   q + b * q_bstride:  the rotated q, heads * head_dim columns (unpadded);
 *   cache + b * cache_bstride + (*pos_dev) * ld:  the rotated k in columns [0, heads * head_dim) and v in
 *     [heads * head_dim, 2 * heads * head_dim), the KV-cache row layout;
 *   key_mask[b * mask_bstride + *pos_dev] = (new_masked != NULL && new_masked[b] != 0), when key_mask is non-NULL.
 * The rotation is ofk_rope_pack's, bit for bit (the same device function), with cos, sin f32 at b * cs_bstride + j
 * (cs_bstride 0 = one table for every batch entry); rot = 0 turns it off and cos/sin may be NULL.  A position outside
 * [0, capacity) writes q only.
 * Requirements: qkv, q, cache, pos_dev non-NULL, batch and heads >= 1, head_dim a positive multiple of 8, rot even in
 *   [0, head_dim], cos and sin non-NULL with cs_bstride >= 0 when rot > 0, capacity >= 1, qkv_bstride >= 3 * heads *
 *   head_dim, q_bstride >= heads * head_dim, ld >= 2 * heads * head_dim, cache_bstride >= capacity * ld and, with a
 *   key_mask, mask_bstride >= capacity (OFK_ERR_ARG); qkv, q and cache 16-byte aligned with their strides multiples of
 *   8 elements, cos, sin and pos_dev 4-byte aligned (OFK_ERR_ALIGN).  Every argument is checked before the first CUDA
 *   call. */
int ofk_rope_append_dev(const void* qkv, long long qkv_bstride, int batch, int heads, int head_dim, int rot,
                        const float* cos, const float* sin, long long cs_bstride, void* q, long long q_bstride,
                        void* cache, long long cache_bstride, long long ld, int capacity, const int* pos_dev,
                        unsigned char* key_mask, long long mask_bstride, const unsigned char* new_masked,
                        void* stream);
int ofk_rope_unpack_bwd(const void* dq, long long dq_bstride, long long lddq, const void* dk, long long dk_bstride,
                        long long lddk, const void* dv, long long dv_bstride, long long lddv, int width, int batch,
                        int rows, int heads, int head_dim, int rot, const float* cos, const float* sin,
                        long long cs_bstride, long long ld_cs, void* dqkv, long long dqkv_bstride, long long lddqkv,
                        void* stream);

/* ------------------------------------------------------------------------------------------------
 * Small fused elementwise / reduction kernels.
 */
/* text_time[b, t] = inclusive cumsum over t of (ids[b,t] == media_id)   (helpers.py:208; flamingo.py:310)
 * or, cached-media mode, count_nonzero(media_locations[b,:]) broadcast (helpers.py:199-205). */
int ofk_text_time(const long long* input_ids, long long media_token_id, int batch, int t_txt, int n_loc,
                  const unsigned char* media_locations, int use_cached_media, int* text_time, void* stream);

/* Training labels on the device (train_utils.py:102-106 for image-text pairs, :126-149 for interleaved MMC4 rows):
 * labels = input_ids with pad_token_id and media_token_id replaced by -100; with interleaved != 0 also every token
 * before the row's first <image> and every token after an <|endofchunk|> up to the next <image> (the
 * <|endofchunk|> keeps its label).  Replaces the reference's per-row Python while-loops; int64 in / out,
 * row strides in elements, rows independent; bit-exact. */
int ofk_make_labels(const long long* input_ids, long long ld_ids, int batch, int t_txt, long long pad_token_id,
                    long long media_token_id, long long endofchunk_token_id, int interleaved, long long* labels,
                    long long ld_labels, void* stream);

/* dst(bf16) = src(f32), n elements (n % 8 == 0 fast path). */
int ofk_cast_f32_bf16(const float* src, void* dst, long long n, void* stream);

/* Grid-wide sums (dgate, sumsq) write one partial per block into a caller-owned float workspace of at least
 * ofk_reduce_workspace_bytes() bytes and add the partials in a fixed order, so their results are the same on every
 * run.  One workspace per stream; it needs no initialisation. */
long long ofk_reduce_workspace_bytes(void);

/* Gate backward (autograd of helpers.py:274,277):
 *   dbranch(bf16)[i] = dout(f32)[i] * tanh(*gate);  dgate[0] += (1 - tanh(*gate)^2) * sum_i dout[i]*branch(bf16)[i]
 * gate NULL => multiplier 1 and no dgate (plain residual branch, helpers.py:130-131).  workspace: see above (may be
 * NULL when no dgate is wanted).  n % 8 == 0 (OFK_ERR_ARG); dout, dbranch and (with a gate) branch 16-byte aligned
 * (OFK_ERR_ALIGN). */
int ofk_gate_bwd(const float* dout, const void* branch, const float* gate, void* dbranch, float* dgate,
                 long long n, float* workspace, void* stream);

/* h(bf16) = gelu_erf(z(bf16)), n elements, with the GELU of the BIAS_GELU_BF16 epilogue: a BIAS_BF16 GEMM followed by this
 * gives the bits of a BIAS_GELU_BF16 GEMM and keeps z for the DGELU_BF16 backward (HF GPTNeoXMLP under autocast).
 * n % 8 == 0 (OFK_ERR_ARG); z and h 16-byte aligned (OFK_ERR_ALIGN). */
int ofk_gelu_bf16(const void* z, void* h, long long n, void* stream);

/* SwiGLU of the LLaMA MLP (HF LlamaMLP: act_fn(gate_proj(x)) * up_proj(x), act_fn = SiLU) on gu = [g | u]: the
 * [rows, 2F] bf16 output (ldgu) of one GEMM against the concatenated gate|up weight, g = gu[:, :F], u = gu[:, F:].
 * ofk_swiglu_fwd:  h(bf16) [rows, F] (ldh) = bf16(bf16(silu(g)) * u), silu(g) = g / (1 + exp(-g)) in fp32: the two
 *   roundings autocast makes.
 * ofk_swiglu_bwd:  from dh(bf16) [rows, F] (lddh), writes dgu(bf16) [rows, 2F] (lddgu), the operand of one dgrad GEMM
 *   with the concatenated weight:  dgu[:, :F] = bf16(dh * u * silu'(g)) in fp32 with one rounding,
 *   silu'(g) = s (1 + g (1 - s)), s = sigmoid(g);  dgu[:, F:] = bf16(dh * bf16(silu(g))), the value the forward used.
 * Requirements: every pointer non-NULL, rows >= 1, F a positive multiple of 8, ldgu and lddgu >= 2F, ldh and lddh >= F
 *   (OFK_ERR_ARG); every pointer 16-byte aligned and every stride a multiple of 8 (OFK_ERR_ALIGN).  Every argument is
 *   checked before the first CUDA call. */
int ofk_swiglu_fwd(const void* gu, long long ldgu, int rows, int F, void* h, long long ldh, void* stream);
int ofk_swiglu_bwd(const void* dh, long long lddh, const void* gu, long long ldgu, int rows, int F, void* dgu,
                   long long lddgu, void* stream);

/* OPT decoder block (HF OPTDecoderLayer, pre-LN, under autocast; modeling_opt.py OPTAttention.forward and
 * OPTDecoderLayer.forward):
 * ofk_relu_bf16:      h(bf16) = relu(z(bf16)), n elements, exact (a NaN passes through); h may be z.
 * ofk_relu_bwd_bf16:  dz(bf16) = h <= 0 ? 0 : dh, from the relu output h (torch's threshold_backward); dz may be dh.
 *   n % 8 == 0 (OFK_ERR_ARG); every pointer 16-byte aligned (OFK_ERR_ALIGN).
 * ofk_scale_bf16:     y(bf16) = bf16(x * s) over [rows, cols] (ldx, ldy): OPTAttention's q_proj(x) * scaling on the bf16
 *   projection, and the same product for its gradient; y may be x.  rows >= 1, cols a positive multiple of 8,
 *   ldx and ldy >= cols (OFK_ERR_ARG); strides multiples of 8, x and y 16-byte aligned (OFK_ERR_ALIGN).
 * Every argument is checked before the first CUDA call. */
int ofk_relu_bf16(const void* z, void* h, long long n, void* stream);
int ofk_relu_bwd_bf16(const void* dh, const void* h, void* dz, long long n, void* stream);
int ofk_scale_bf16(const void* x, long long ldx, int rows, int cols, float s, void* y, long long ldy, void* stream);

/* Residual dropout (OPTDecoderLayer: residual + nn.functional.dropout(branch, p) in training, with the branch a bf16
 * Linear output and the residual the fp32 stream):
 * ofk_dropout_resid_fwd:  out(f32)[r, c] = kept(r, c) ? x[r, c] + bf16(branch(bf16)[r, c] * scale) : x[r, c]
 * ofk_dropout_resid_bwd:  dbranch(bf16)[r, c] = kept(r, c) ? bf16(bf16(dout(f32)[r, c]) * scale) : 0
 *   scale = float(1 / (double)float(1 - p)), torch's dropout scale.  kept(r, c): Philox-4x32-10 with key = seed and
 *   counter = (c / 4, r, offset low word, offset high word) gives four 32-bit words; word c % 4 >= floor(p * 2^32)
 *   keeps the element.  seed_offset: device int64 [2] = (seed, offset), read on the device (so a captured graph may
 *   advance it between replays); may be NULL when p == 0, which keeps everything (out = x + branch, the bits of a
 *   GATE_RESID_F32 epilogue without gate).  The backward regenerates the forward's mask from the same pair; no mask
 *   is stored.  out may be x.
 *   Requirements: x, branch, out (dout, dbranch) non-NULL, p in [0, 1), a seed pair when p > 0, rows >= 1, cols a
 *   positive multiple of 8, every stride >= cols (OFK_ERR_ARG); f32 strides multiples of 4, bf16 strides multiples
 *   of 8, seed_offset 8-byte aligned, the other pointers 16-byte aligned (OFK_ERR_ALIGN).  Every argument is checked
 *   before the first CUDA call. */
int ofk_dropout_resid_fwd(const float* x, long long ldx, const void* branch, long long ldb, int rows, int cols,
                          double p, const long long* seed_offset, float* out, long long ldo, void* stream);
int ofk_dropout_resid_bwd(const float* dout, long long ldd, int rows, int cols, double p,
                          const long long* seed_offset, void* dbranch, long long lddb, void* stream);

/* ------------------------------------------------------------------------------------------------
 * CLIP image preprocessing: open_clip's eval transform (image_transform(is_train=False), the image_processor that
 * create_model_and_transforms returns, factory.py:42) on decoded uint8 pixels:
 *   Resize(S, BICUBIC) + CenterCrop(S) + ToTensor + Normalize(mean, std)
 * bit for bit what torchvision + Pillow compute from the same PIL image in mode RGB (c = 3) or L (c = 1; resampled as
 * one channel and replicated to R = G = B after the crop, as open_clip's _convert_to_rgb runs after the crop).
 *   Resize: the shorter side becomes S, the longer int(S * long / short); Pillow's two-pass fixed-point bicubic
 *     (a = -0.5, int32 taps at 22 fractional bits, uint8 intermediate), horizontal pass first unless the image is more
 *     than 100 times taller than wide and its height shrinks (Image.resize's order).
 *   CenterCrop: top = round((H - S) / 2), left = round((W - S) / 2), half to even.  Only the crop window is computed.
 *   out = ((float)u8 / 255 - mean[c]) / std[c] in IEEE fp32.
 * shape: host int64 [n][4] = (h, w, c, row stride in bytes) per image; pixels are HWC uint8 rows.  Requirements: n in
 *   [1, 65535], S in [1, 4096], h, w >= 1, S * max(h, w) < 2^31, c in {1, 3}, row stride >= w * c (OFK_ERR_ARG).
 * ofk_image_plan_size: host only; writes the plan's size and the device workspace size (the plan's device copy plus
 *   the uint8 intermediates).
 * ofk_image_plan: host only; src: n device pointers (host array) to each image's pixel (0, 0); mean, std: 3 host floats
 *   each, finite, std nonzero; plan: caller-owned host buffer of exactly plan_bytes, 16-byte aligned (OFK_ERR_ALIGN).
 * ofk_clip_preprocess: checks the plan (every table and intermediate inside its bounds), copies it into `workspace`
 *   (device, >= the workspace size, 16-byte aligned) on `stream` and makes two launches for the whole batch, writing
 *   out[i] (f32 [3, S, S] at out + i * out_image_stride, stride >= 3 S^2, out 4-byte aligned).  A pageable plan may be
 *   reused when the call returns; a pinned one once the stream has passed the copy.  Every argument is checked before
 *   the first CUDA call. */
int ofk_image_plan_size(int n, const long long* shape, int S, long long* plan_bytes, long long* workspace_bytes);
int ofk_image_plan(int n, const void* const* src, const long long* shape, int S, const float* mean, const float* std_,
                   void* plan, long long plan_bytes);
int ofk_clip_preprocess(const void* plan, long long plan_bytes, void* workspace, long long workspace_bytes, float* out,
                        long long out_image_stride, void* stream);

/* dst(f32) += src(f32) */
int ofk_add_f32(float* dst, const float* src, long long n, void* stream);

/* ViT patch extraction: images [n, 3, H, W] f32 NCHW -> patches [n * (H/P)*(W/P), ldp] bf16 with the
 * (c, ph, pw) ordering of a conv weight [out, 3, P, P] flattened; columns >= 3*P*P are zero.  Replaces the
 * stride-P conv of open_clip VisionTransformer.conv1 (third party; call site flamingo.py:195). */
int ofk_patchify(const float* images, int n, int H, int W, int P, void* patches, long long ldp, void* stream);

/* tokens[n, 1 + g, D] f32 = cat(class_emb, patch_emb(bf16)[n, g, D]) + pos_emb[1+g, D]   (open_clip ViT)
 * g >= 0, D > 0 and D % 4 == 0 (OFK_ERR_ARG); patch_emb may be NULL when g == 0; patch_emb 8-byte aligned, class_emb, pos_emb, tokens 16-byte aligned
 * (OFK_ERR_ALIGN). */
int ofk_vit_assemble(const void* patch_emb, const float* class_emb, const float* pos_emb, int n, int g, int D,
                     float* tokens, void* stream);

/* Shifted causal-LM cross-entropy on the LM-head logits (the loss Flamingo.forward returns with labels,
 * flamingo.py:111-117 -> HF ForCausalLMLoss: float logits, labels shifted by one, mean over non-ignored).
 *   logits: [rows = B*T, vocab] bf16 or f32 (ld); labels: [B, T] int64 (host-unshifted when shift_labels = 1).
 *   fwd: lse[rows]; *loss_sum += sum(lse - logit[target]); *count += #non-ignored rows.  (caller zeroes them)
 *   bwd: dlogits = (softmax - onehot) * (*grad_scale) / max(*count, 1) for non-ignored rows, 0 otherwise.
 *   Targets outside [0, vocab) count as ignored.  bf16 rows are read 8 at a time when vocab, ld (and ldd) are
 *   multiples of 8 and logits (and dlogits) are 16-byte aligned, one at a time otherwise.
 *   Logits may be -inf (masked vocabulary entries). */
int ofk_ce_fwd(const void* logits, int logits_is_f32, long long ld, long long rows, int vocab,
               const long long* labels, int T, int shift_labels, long long ignore_index, float* lse,
               float* loss_sum, float* count, void* stream);
int ofk_ce_bwd(const void* logits, int logits_is_f32, long long ld, long long rows, int vocab,
               const long long* labels, int T, int shift_labels, long long ignore_index, const float* lse,
               const float* grad_scale, const float* count, void* dlogits, long long ldd, void* stream);

/* Fused AdamW over a flat f32 parameter / gradient buffer (train.py:392-415, train_utils.py:208-216):
 * grads are first scaled by clip_scale (global-norm clip), decoupled weight decay `wd`.
 * Also emits the bf16 operand copy for the next step's GEMMs (w_bf16 may be NULL).
 * step_dev / lr_dev (optional DEVICE floats) override bias_corr1/2 (= 1 - beta^step) and lr, so that a captured
 * CUDA graph of the training step stays valid as the step count and learning-rate schedule advance. */
int ofk_adamw(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, void* w_bf16, long long n,
              float lr, float beta1, float beta2, float eps, float wd, float bias_corr1, float bias_corr2,
              const float* clip_scale, const float* step_dev, const float* lr_dev, void* stream);

/* out[0] += sum_i x[i]^2   (global grad norm, train_utils.py:208); workspace: see ofk_reduce_workspace_bytes. */
int ofk_sumsq(const float* x, long long n, float* out, float* workspace, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* OFK_H_ */
