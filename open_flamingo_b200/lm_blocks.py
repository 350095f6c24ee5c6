"""Frozen-LM decoder blocks on the sm_90a kernels (SURVEY.md section 8f, rank 1): HF `MptBlock` (OF-3B, OF-9B),
HF `GPTNeoXLayer` (OF-4B; see the GPT-NeoX section below), HF `LlamaDecoderLayer` (OF-9B v1; see the LLaMA
section) and HF `OPTDecoderLayer` (see the OPT section).

The reference runs the frozen LM's decoder block as ordinary PyTorch (`self.decoder_layer(lang_x, ...)`,
flamingo_lm.py:63-65).  For the LM family named by BASELINE.json (MPT: HF `MptBlock` = LN -> Wqkv -> causal
ALiBi attention -> out_proj -> +res -> LN -> up_proj -> GELU(erf) -> down_proj -> +res, no biases) this module
evaluates the same block with the kernels already used by the gated blocks (wgmma GEMMs with fused
GELU / residual epilogues, LayerNorm, dense attention), forward plus the dgrad-only backward a frozen block
needs.

Decoding with a KV cache runs on the kernels too when the cache is a kv_cache.KVCache and no gradient is recorded
(`no_grad` / `inference_mode`): the K/V projection GEMM (GPT-NeoX: the rotary packing) writes the new rows straight
into the cache buffer, one new token attends through the split-KV decode kernel (ops.attn_decode) and a multi-token
chunk (prefill, or a chunk after a prefix) through the dense kernel over the cached keys.  Anything else -- other LM
families, HF's DynamicCache, dropout (but OPT's residual dropout, see the OPT section), clip_qkv, output_attentions (GPT-NeoX: also output_hidden_states, which HF
records with hooks on the layer modules) -- takes the block's own PyTorch forward, exactly as in the reference (a
block that declines still reads and extends a KVCache through HF's attention module and `KVCache.update`).

Numerics are those of the block under `torch.autocast(bfloat16)`: fp32 residual stream, fp32 LayerNorm/softmax,
bf16 GEMM operands, bf16 K/V cache.
"""
import weakref

import torch

from . import _lib as L
from . import ops
from .fused import padded_w16, w16
from .kv_cache import KVCache

bf16 = torch.bfloat16
f32 = torch.float32

ENABLED = True  # module-level switch (bench.py --lm eager turns it off to time the reference's PyTorch LM path)

_zero_bias = {}
# (weakref to HF's [B,1,T,nk] bool mask, its byte form for the kernels, (whether that is the decode form, whether True
# meant "attend")) -- converted once per forward and shared by every block
_mask_cache = [None, None, None]


def _zeros(n, device):
    key = (n, device)
    t = _zero_bias.get(key)
    if t is None:
        t = torch.zeros(n, device=device, dtype=f32)
        _zero_bias[key] = t
    return t


def _kernel_mask(m, B, T, nk, decode, true_attends=False):
    """HF's 4-D bool mask `m` [1 or B, 1, T, nk] as the kernels' bytes (nonzero = masked), or None if `m` is not such a
    mask.  decode: key padding only, [B, nk rounded up to 8] for the decode kernel; else [B, T, nk].  true_attends: True
    in `m` means "attend" (HF's sdpa mask for GPT-NeoX) rather than "masked" (MPT)."""
    if m.dtype != torch.bool or m.dim() != 4 or m.shape[0] not in (1, B) or m.shape[1] != 1 or m.shape[2] != T or \
            m.shape[3] != nk:
        return None
    ref = _mask_cache[0]
    if ref is not None and ref() is m and _mask_cache[1].shape[0] == B and _mask_cache[2] == (decode, true_attends):
        return _mask_cache[1]
    m_masked = ~m if true_attends else m
    if decode:   # key padding only, rows padded to a multiple of 8 bytes for the decode kernel
        mask = torch.zeros((B, -(-nk // 8) * 8), dtype=torch.uint8, device=m.device)
        mask[:, :nk].copy_(m_masked.expand(B, 1, 1, nk).reshape(B, nk))
    else:
        mask = m_masked.expand(B, 1, T, nk).reshape(B, T, nk).contiguous()
    _mask_cache[0], _mask_cache[1], _mask_cache[2] = weakref.ref(m), mask, (decode, true_attends)
    return mask


def _block_tail(x2d, o, eps, wout, n2_w, wup, wdown):
    """The block after its attention core: out-proj + residual -> LayerNorm -> up-proj GELU -> down-proj + residual.
    x2d: [R, D] f32 block input, o: [R, D] bf16 attention output.  Returns (out, x1, mean2, rstd2, z); the last four
    are what the backward needs."""
    R, D = x2d.shape
    x1 = ops.gemm(o, w16(wout), epi=L.EPI_GATE_RESID_F32, aux=x2d)                 # + residual
    x1n, mean2, rstd2 = ops.layernorm_fwd(x1, n2_w, _zeros(D, x2d.device), eps)
    z = torch.empty((R, wup.shape[0]), device=x2d.device, dtype=bf16)
    h = torch.empty((R, wup.shape[0]), device=x2d.device, dtype=bf16)
    ops.gemm(x1n, w16(wup), epi=L.EPI_GELU_DUAL, out=z, out2=h)
    del x1n
    out = ops.gemm(h, w16(wdown), epi=L.EPI_GATE_RESID_F32, aux=x1)                # + residual
    return out, x1, mean2, rstd2, z


def cached_block_forward(x, layer, mask, pure_flag, slopes, heads, eps, n1_w, wqkv, wout, n2_w, wup, wdown):
    """Inference forward of one block that appends its nq new tokens to `layer` (a kv_cache.KVCacheLayer) and attends
    over everything cached.  x: [B, nq, D] f32.  mask: nq == 1: [B, >= nk] bytes (key padding, row stride a multiple
    of 8); nq > 1: [B, nq, nk] bytes; None = causal only.  Returns [B, nq, D] f32."""
    B, nq, D = x.shape
    R = B * nq
    hd = D // heads
    x2d = x.reshape(R, D)
    if not x2d.is_contiguous():
        x2d = x2d.contiguous()
    xn, _, _ = ops.layernorm_fwd(x2d, n1_w, _zeros(D, x.device), eps, want_stats=False)
    w = w16(wqkv)
    q = ops.gemm(xn, w[:D])                                                         # [R, D]
    if not layer.is_initialized:
        layer.init_storage(B, heads, hd, bf16, x.device)
    past = layer.length
    buf = layer.reserve(nq)
    cap = buf.shape[1]
    # K and V rows land in cache rows [past, past + nq) of every batch entry: logical row b*nq + t -> b*cap + past + t
    ops.gemm_grouped(xn, w[D:], out=buf.view(B * cap, 2 * D), M=R, N=2 * D, K=D, out_map=(nq, cap, past))
    del xn
    layer.length = past + nq
    k, v = layer.kv_views()
    scale = float(hd ** -0.5)
    if nq == 1:
        o = ops.attn_decode(q, k, v, heads, hd, scale, key_mask=mask, slopes=slopes)
    else:
        o, _ = ops.attn_dense_fwd(q.view(B, nq, D), k, v, heads, hd, scale, causal=mask is None, mask=mask,
                                  slopes=slopes, pure_causal_flag=pure_flag, want_lse=False)
    return _block_tail(x2d, o.view(R, D), eps, wout, n2_w, wup, wdown)[0].view(B, nq, D)


def decode_step_block_forward(x, layer, pos_nk, key_mask, new_masked, workspace, slopes, heads, eps, n1_w, wqkv, wout,
                              n2_w, wup, wdown):
    """cached_block_forward for one new token with its position on the device, so that the step can be captured in a
    CUDA graph once and replayed at every position.  pos_nk: int32 [2] device tensor (cache row of the new token,
    key count = row + 1); key_mask: the cache's [B, >= capacity] padding bytes; new_masked: uint8 [B], 1 where the new
    token is padding; workspace: ops.decode_workspace at the layer's capacity.  The GEMMs have the shapes of the eager
    path (q with N = D, K/V with N = 2D) and only the K/V destination differs -- a staging row that ops.kv_append
    copies into the cache -- so the result is the eager path's, bit for bit.  x: [B, 1, D] f32; returns the same."""
    B, _, D = x.shape
    hd = D // heads
    x2d = x.reshape(B, D)
    if not x2d.is_contiguous():
        x2d = x2d.contiguous()
    xn, _, _ = ops.layernorm_fwd(x2d, n1_w, _zeros(D, x.device), eps, want_stats=False)
    w = w16(wqkv)
    q = ops.gemm(xn, w[:D])                                                         # [B, D]
    kv = ops.gemm(xn, w[D:])                                                        # [B, 2D]
    del xn
    buf = layer.buf
    ops.kv_append(kv, buf, pos_nk[0:1], key_mask=key_mask, new_masked=new_masked)
    o = ops.attn_decode_dev(q, buf[..., :D], buf[..., D:], heads, hd, float(hd ** -0.5), pos_nk[1:2],
                            key_mask=key_mask, slopes=slopes, workspace=workspace)
    return _block_tail(x2d, o, eps, wout, n2_w, wup, wdown)[0].view(B, 1, D)


class FrozenMptBlockFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, mask, pure_flag, slopes, heads, eps, n1_w, wqkv, wout, n2_w, wup, wdown):
        B, T, D = x.shape
        R = B * T
        hd = D // heads
        x2d = x.reshape(R, D)
        if not x2d.is_contiguous():
            x2d = x2d.contiguous()
        xn, mean1, rstd1 = ops.layernorm_fwd(x2d, n1_w, _zeros(D, x.device), eps)
        qkv = ops.gemm(xn, w16(wqkv))                                               # [R, 3D]
        del xn
        q3 = qkv.view(B, T, 3 * D)
        scale = float(hd ** -0.5)
        o, lse = ops.attn_dense_fwd(q3[..., :D], q3[..., D:2 * D], q3[..., 2 * D:], heads, hd, scale,
                                    causal=mask is None, mask=mask, slopes=slopes, pure_causal_flag=pure_flag)
        out, x1, mean2, rstd2, z = _block_tail(x2d, o.view(R, D), eps, wout, n2_w, wup, wdown)
        ctx.save_for_backward(x2d, mean1, rstd1, qkv, o, lse, x1, mean2, rstd2, z, n1_w, wqkv, wout, n2_w, wup,
                              wdown, slopes, mask if mask is not None else x2d.new_empty(0),
                              pure_flag if pure_flag is not None else x2d.new_empty(0))
        ctx.meta = (B, T, D, heads, hd, scale, mask is not None, pure_flag is not None)
        return out.view(B, T, D)

    @staticmethod
    def backward(ctx, dout):
        (x2d, mean1, rstd1, qkv, o, lse, x1, mean2, rstd2, z, n1_w, wqkv, wout, n2_w, wup, wdown, slopes,
         mask, pure_flag) = ctx.saved_tensors
        B, T, D, heads, hd, scale, has_mask, has_flag = ctx.meta
        if not has_mask:
            mask = None
        if not has_flag:
            pure_flag = None
        R = B * T
        d2 = dout.reshape(R, D)
        if not d2.is_contiguous():
            d2 = d2.contiguous()
        if d2.dtype != f32:
            d2 = d2.float()
        dbr = ops.gate_bwd(d2, None, None, None)                                    # bf16 cast
        dz = ops.gemm(dbr, w16(wdown), b_mn=True, epi=L.EPI_DGELU_BF16, aux=z)      # (d W_down) * gelu'(z)
        dx1n = ops.gemm(dz, w16(wup), b_mn=True)
        del dz, dbr
        dx1 = ops.layernorm_bwd(dx1n, x1, n2_w, mean2, rstd2, dx_add=d2)
        da = ops.gate_bwd(dx1, None, None, None)
        d_o = ops.gemm(da, w16(wout), b_mn=True)                                    # [R, D]
        del da
        q3 = qkv.view(B, T, 3 * D)
        dqkv = torch.empty_like(qkv)
        dq3 = dqkv.view(B, T, 3 * D)
        ops.attn_dense_bwd(q3[..., :D], q3[..., D:2 * D], q3[..., 2 * D:], o, d_o.view(B, T, D), lse, heads, hd, scale,
                           causal=mask is None, mask=mask, slopes=slopes, pure_causal_flag=pure_flag,
                           dq=dq3[..., :D], dk=dq3[..., D:2 * D], dv=dq3[..., 2 * D:])
        dxn = ops.gemm(dqkv, w16(wqkv), b_mn=True)
        dx = ops.layernorm_bwd(dxn, x2d, n1_w, mean1, rstd1, dx_add=dx1)
        return (dx.view(B, T, D),) + (None,) * 11


def _alibi_slopes(position_bias):
    """HF builds bias[h, 0, k] = slope_h * (k - (L-1)) (build_mpt_alibi_tensor); recover slope_h."""
    pb = position_bias
    if pb.dim() != 3 or pb.shape[-1] < 2:
        return None
    return (pb[:, 0, -1] - pb[:, 0, -2]).float().contiguous()


class FastMptBlock:
    """Callable with HF MptBlock.forward's signature; returns None when the fast path does not apply."""

    def __init__(self, block):
        self.block = block
        self._slopes = None

    def supported(self, hidden_states, position_bias, output_attentions):
        """The block and call are ones the kernels evaluate, whatever the cache."""
        b = self.block
        if not ENABLED or not hidden_states.is_cuda or output_attentions:
            return False
        a = b.attn
        if getattr(a, "clip_qkv", None) or (b.training and (a.attn_dropout_p > 0 or b.dropout_rate > 0 or
                                                            b.ffn.hidden_dropout > 0)):
            return False
        if a.head_dim not in (64, 128) or position_bias is None:
            return False
        if a.Wqkv.bias is not None or a.out_proj.bias is not None or b.ffn.up_proj.bias is not None or \
                b.ffn.down_proj.bias is not None or b.norm_1.bias is not None or b.norm_2.bias is not None:
            return False
        if any(p.requires_grad for p in b.parameters()):
            return False  # this path has no wgrad: frozen blocks only
        if not isinstance(b.ffn.act, torch.nn.GELU) or b.ffn.act.approximate != "none":
            return False
        if abs(a.softmax_scale - a.head_dim ** -0.5) > 1e-9:
            return False
        return True

    def weights(self):
        b = self.block
        a = b.attn
        return (b.norm_1.weight, a.Wqkv.weight, a.out_proj.weight, b.norm_2.weight, b.ffn.up_proj.weight,
                b.ffn.down_proj.weight)

    def slopes(self, device, position_bias=None):
        """The block's ALiBi slopes on `device`, from `position_bias` or, if None, from the model's own builder."""
        if self._slopes is None or self._slopes.device != device:
            if position_bias is None:
                from transformers.models.mpt.modeling_mpt import build_mpt_alibi_tensor
                a = self.block.attn   # what MptModel.forward builds
                position_bias = build_mpt_alibi_tensor(a.n_heads, a.max_seq_length, device=device)
            self._slopes = _alibi_slopes(position_bias)
        return self._slopes

    def decode_step(self, x, layer, pos_nk, key_mask, new_masked, workspace):
        """One captured decode step of this block (decode_step_block_forward)."""
        a = self.block.attn
        return decode_step_block_forward(x, layer, pos_nk, key_mask, new_masked, workspace, self.slopes(x.device),
                                         a.n_heads, self.block.norm_1.eps, *self.weights())

    def applicable(self, hidden_states, position_bias, attention_mask, layer_past, use_cache, output_attentions):
        """The uncached path (FrozenMptBlockFn, forward and backward)."""
        if layer_past is not None or use_cache:
            return False   # a cache other than KVCache, or a caller that wants a `present` back: the block's own forward
        return self.supported(hidden_states, position_bias, output_attentions)

    def cache_layer(self, hidden_states, position_bias, layer_past, output_attentions):
        """The KVCacheLayer the cached path appends to, or None when that path does not apply: it needs a KVCache whose
        layer is empty or holds bf16 storage on this device for this batch, and no gradient being recorded."""
        if not isinstance(layer_past, KVCache) or torch.is_grad_enabled():
            return None
        if not self.supported(hidden_states, position_bias, output_attentions):
            return None
        a = self.block.attn
        if a.layer_idx is None or not 0 <= a.layer_idx < len(layer_past.layers):
            return None
        layer = layer_past.layers[a.layer_idx]
        if layer.is_initialized and (layer.buf.dtype != bf16 or layer.buf.device != hidden_states.device or
                                     layer.buf.shape[0] != hidden_states.shape[0] or layer.heads != a.n_heads or
                                     layer.head_dim != a.head_dim):
            return None
        return layer

    def __call__(self, hidden_states, position_bias=None, attention_mask=None, layer_past=None, use_cache=False,
                 output_attentions=False, pure_causal_flag=None, **kwargs):
        layer = None
        if layer_past is not None or use_cache:
            layer = self.cache_layer(hidden_states, position_bias, layer_past, output_attentions)
            if layer is None:
                return None
        elif not self.applicable(hidden_states, position_bias, attention_mask, layer_past, use_cache,
                                 output_attentions):
            return None
        b = self.block
        a = b.attn
        B, T, D = hidden_states.shape
        if self.slopes(hidden_states.device, position_bias) is None:
            return None
        nk = T if layer is None else layer.length + T
        decode = layer is not None and T == 1
        mask = None
        if attention_mask is not None:
            mask = _kernel_mask(attention_mask, B, T, nk, decode)
            if mask is None:
                return None
        x = hidden_states if hidden_states.dtype == f32 else hidden_states.float()
        weights = self.weights()
        flag = pure_causal_flag if mask is not None else None
        if layer is not None:
            out = cached_block_forward(x, layer, mask, flag, self._slopes, a.n_heads, b.norm_1.eps, *weights)
        else:
            out = FrozenMptBlockFn.apply(x, mask, flag, self._slopes, a.n_heads, b.norm_1.eps, *weights)
        if out.dtype != hidden_states.dtype:
            out = out.to(hidden_states.dtype)
        return out, None


# ---- GPT-NeoX (HF GPTNeoXLayer: OpenFlamingo-4B's RedPajama-INCITE-3B) ------------------------------------------------
#
#   a = LN1(x);  qkv = a Wqkv^T + bqkv  (heads interleaved as (q | k | v));  q, k = rotary(q, k; cos, sin)
#   y = softmax(q k^T / sqrt(hd) + mask) v Wd^T + bd
#   sequential: x1 = y + x,  out = MLP(LN2(x1)) + x1;   parallel: out = MLP(LN2(x)) + y + x
#   MLP(u) = gelu_erf(u W1^T + b1) W2^T + b2
#
# The attention cores exist for head_dim 64 and 128.  Other head_dims (80 for RedPajama-INCITE-3B: D 2560, 32 heads) run
# on the 128 cores with every head zero-padded to 128 columns: ops.rope_pack writes the rotated q, k and v in that
# layout, zero columns add exact zeros to q k^T, to P v and to every backward product, so the result is the head_dim-80
# attention.  The attention output then has H * 128 columns; the out-projection reads it through a copy of Wd with the
# same zero columns (fused.padded_w16), and in the backward the dgrad GEMM with that copy yields the padded d_o directly.
# Decoding one token runs the decode kernel at head_dim 80 directly, on an unpadded KV cache; its graph-captured form
# (decode_step_neox_block_forward) writes the new K/V row with ops.rope_append_dev at a position read on the device.


def _neox_width(hd):
    """Head width the attention cores run a head_dim-hd head at."""
    return hd if hd in (64, 128) else 128


def _neox_tail(x2d, o, parallel, eps2, wout16, bd, n2_w, n2_b, w1, b1, w2, b2, keep_z):
    """The block after its attention core.  x2d: [R, D] f32 block input; o: [R, heads * width] bf16 attention output;
    wout16: the bf16 out-projection weight for that width.  Returns (out, x1, mean2, rstd2, z): x1 = bf16(y) + x, the
    LayerNorm-2 statistics (of x1, or of x in the parallel form) and the bf16 pre-activation z (None unless keep_z).

    The parallel form adds bf16(y) and bf16(mlp) to the fp32 stream one after the other; autocast adds them in bf16
    first, so this is the more precise of the two (by at most one bf16 rounding of y + mlp)."""
    x1 = ops.gemm(o, wout16, epi=L.EPI_BIAS_RESID_F32, bias=bd, aux=x2d)
    un, mean2, rstd2 = ops.layernorm_fwd(x2d if parallel else x1, n2_w, n2_b, eps2, want_stats=keep_z)
    if keep_z:   # z for the DGELU_BF16 backward; gelu_bf16 gives the bits BIAS_GELU_BF16 would
        z = ops.gemm(un, w16(w1), epi=L.EPI_BIAS_BF16, bias=b1)
        h = ops.gelu_bf16(z)
    else:
        z = None
        h = ops.gemm(un, w16(w1), epi=L.EPI_BIAS_GELU_BF16, bias=b1)
    del un
    out = ops.gemm(h, w16(w2), epi=L.EPI_BIAS_RESID_F32, bias=b2, aux=x1)
    return out, x1, mean2, rstd2, z


def _rows(x):
    B, T, D = x.shape
    x2d = x.reshape(B * T, D)
    return x2d if x2d.is_contiguous() else x2d.contiguous()


class FrozenNeoXBlockFn(torch.autograd.Function):
    """A frozen GPTNeoXLayer: forward, and the backward to its input only (the parameters take no gradient).
    x: [B, T, D] f32; mask: [B, T, T] bytes (nonzero = masked) or None for causal only; cos, sin: f32 [1 or B, T, rot]."""

    @staticmethod
    def forward(ctx, x, mask, pure_flag, cos, sin, heads, parallel, eps1, eps2, n1_w, n1_b, wqkv, bqkv, wd, bd, n2_w,
                n2_b, w1, b1, w2, b2):
        B, T, D = x.shape
        R = B * T
        hd = D // heads
        W = _neox_width(hd)
        x2d = _rows(x)
        xn, mean1, rstd1 = ops.layernorm_fwd(x2d, n1_w, n1_b, eps1)
        qkv = ops.gemm(xn, w16(wqkv), epi=L.EPI_BIAS_BF16, bias=bqkv)                # [R, 3D]
        del xn
        q, k, v = ops.rope_pack(qkv.view(B, T, 3 * D), heads, hd, cos, sin, q_width=W, kv_width=W)
        del qkv
        scale = float(hd ** -0.5)
        o, lse = ops.attn_dense_fwd(q, k, v, heads, W, scale, causal=mask is None, mask=mask,
                                    pure_causal_flag=pure_flag)
        out, x1, mean2, rstd2, z = _neox_tail(x2d, o.view(R, heads * W), parallel, eps2, padded_w16(wd, heads, hd, W),
                                              bd, n2_w, n2_b, w1, b1, w2, b2, keep_z=True)
        ctx.save_for_backward(x2d, mean1, rstd1, q, k, v, o, lse, x1, mean2, rstd2, z, cos, sin, n1_w, wqkv, wd, n2_w,
                              w1, w2, mask if mask is not None else x2d.new_empty(0),
                              pure_flag if pure_flag is not None else x2d.new_empty(0))
        ctx.meta = (B, T, D, heads, hd, W, scale, parallel, mask is not None, pure_flag is not None)
        return out.view(B, T, D)

    @staticmethod
    def backward(ctx, dout):
        (x2d, mean1, rstd1, q, k, v, o, lse, x1, mean2, rstd2, z, cos, sin, n1_w, wqkv, wd, n2_w, w1, w2, mask,
         pure_flag) = ctx.saved_tensors
        B, T, D, heads, hd, W, scale, parallel, has_mask, has_flag = ctx.meta
        mask = mask if has_mask else None
        pure_flag = pure_flag if has_flag else None
        R = B * T
        d2 = _rows(dout)
        if d2.dtype != f32:
            d2 = d2.float()
        dbr = ops.gate_bwd(d2, None, None, None)                                     # bf16 cast
        dz = ops.gemm(dbr, w16(w2), b_mn=True, epi=L.EPI_DGELU_BF16, aux=z)          # (d W2) * gelu'(z)
        du = ops.gemm(dz, w16(w1), b_mn=True)
        del dz
        # d/dx1 (sequential) or the MLP branch's share of d/dx (parallel), plus the straight-through d2
        dx1 = ops.layernorm_bwd(du, x2d if parallel else x1, n2_w, mean2, rstd2, dx_add=d2)
        del du
        dy = dbr if parallel else ops.gate_bwd(dx1, None, None, None)
        d_o = ops.gemm(dy, padded_w16(wd, heads, hd, W), b_mn=True)                 # [R, heads * W], padding zero
        del dy, dbr
        dq, dk, dv = ops.attn_dense_bwd(q, k, v, o, d_o.view(B, T, heads * W), lse, heads, W, scale,
                                        causal=mask is None, mask=mask, pure_causal_flag=pure_flag)
        del d_o
        dqkv = ops.rope_unpack_bwd(dq, dk, dv, heads, hd, cos, sin)                  # [B, T, 3D]
        del dq, dk, dv
        dxn = ops.gemm(dqkv.view(R, 3 * D), w16(wqkv), b_mn=True)
        dx = ops.layernorm_bwd(dxn, x2d, n1_w, mean1, rstd1, dx_add=dx1)
        return (dx.view(B, T, D),) + (None,) * 20


def cached_neox_block_forward(x, layer, mask, pure_flag, cos, sin, heads, parallel, eps1, eps2, n1_w, n1_b, wqkv, bqkv,
                              wd, bd, n2_w, n2_b, w1, b1, w2, b2):
    """Inference forward of one GPT-NeoX block that appends its nq new tokens to `layer` (a kv_cache.KVCacheLayer,
    unpadded head_dim rows, so HF's attention can extend it through KVCacheLayer.update) and attends over everything
    cached.  ops.rope_pack writes the rotated K and the V straight into cache rows [past, past + nq).
      nq == 1: q unpadded, the decode kernel at head_dim hd, the out-projection with Wd itself;
      nq > 1 : q and the cached K/V rows [0, nk) padded to the core's width, the dense kernel, the padded Wd.
    mask: as for cached_block_forward.  x: [B, nq, D] f32; returns the same."""
    B, nq, D = x.shape
    hd = D // heads
    x2d = _rows(x)
    xn, _, _ = ops.layernorm_fwd(x2d, n1_w, n1_b, eps1, want_stats=False)
    qkv = ops.gemm(xn, w16(wqkv), epi=L.EPI_BIAS_BF16, bias=bqkv).view(B, nq, 3 * D)
    del xn
    if not layer.is_initialized:
        layer.init_storage(B, heads, hd, bf16, x.device)
    past = layer.length
    rows = layer.reserve(nq)[:, past:past + nq]
    scale = float(hd ** -0.5)
    W = hd if nq == 1 else _neox_width(hd)
    q, _, _ = ops.rope_pack(qkv, heads, hd, cos, sin, q_width=W, k=rows[..., :D], v=rows[..., D:])
    del qkv
    layer.length = past + nq
    k, v = layer.kv_views()
    if nq == 1:
        o = ops.attn_decode(q.view(B, D), k, v, heads, hd, scale, key_mask=mask)
    else:
        if W != hd:
            _, k, v = ops.rope_pack(None, heads, hd, kv_src=(k, v), kv_width=W)
        o, _ = ops.attn_dense_fwd(q, k, v, heads, W, scale, causal=mask is None, mask=mask, pure_causal_flag=pure_flag,
                                  want_lse=False)
    return _neox_tail(x2d, o.view(B * nq, heads * W), parallel, eps2, padded_w16(wd, heads, hd, W), bd, n2_w, n2_b,
                      w1, b1, w2, b2, keep_z=False)[0].view(B, nq, D)


def decode_step_neox_block_forward(x, layer, pos_nk, key_mask, new_masked, workspace, cos, sin, heads, parallel, eps1,
                                   eps2, n1_w, n1_b, wqkv, bqkv, wd, bd, n2_w, n2_b, w1, b1, w2, b2):
    """cached_neox_block_forward for one new token with its position on the device, so that the step can be captured
    in a CUDA graph once and replayed at every position (the GPT-NeoX decode_step_block_forward).  pos_nk, key_mask,
    new_masked, workspace: as there; cos, sin: f32 [1 or B, 1, rot] of the new token's position.  The GEMMs, epilogues
    and shapes are the eager nq == 1 path's, and ops.rope_append_dev rotates as ops.rope_pack does while writing K and V
    into cache row pos_nk[0], so the result is the eager path's, bit for bit.  x: [B, 1, D] f32; returns the same."""
    B, _, D = x.shape
    hd = D // heads
    x2d = _rows(x)
    xn, _, _ = ops.layernorm_fwd(x2d, n1_w, n1_b, eps1, want_stats=False)
    qkv = ops.gemm(xn, w16(wqkv), epi=L.EPI_BIAS_BF16, bias=bqkv)                   # [B, 3D]
    del xn
    buf = layer.buf
    q = ops.rope_append_dev(qkv, heads, hd, cos, sin, buf, pos_nk[0:1], key_mask=key_mask, new_masked=new_masked)
    del qkv
    o = ops.attn_decode_dev(q, buf[..., :D], buf[..., D:], heads, hd, float(hd ** -0.5), pos_nk[1:2],
                            key_mask=key_mask, workspace=workspace)
    return _neox_tail(x2d, o, parallel, eps2, w16(wd), bd, n2_w, n2_b, w1, b1, w2, b2, keep_z=False)[0].view(B, 1, D)


class FastNeoXBlock:
    """Callable with HF GPTNeoXLayer.forward's signature; returns None when the fast path does not apply, and the
    block's output tensor otherwise."""

    def __init__(self, block):
        self.block = block

    def records_outputs(self, output_attentions=None, output_hidden_states=None):
        """Whether the caller asked HF to record this layer's hidden states or attention weights.  GPTNeoXModel
        records both with hooks on the GPTNeoXLayer and GPTNeoXAttention modules, which the fast path does not call,
        so such a call must run HF's layer.  An explicit keyword wins; without one the model config's default holds,
        as in HF's capture_outputs."""
        cfg = self.block.attention.config
        if output_attentions is None:
            output_attentions = getattr(cfg, "output_attentions", False)
        if output_hidden_states is None:
            output_hidden_states = getattr(cfg, "output_hidden_states", False)
        return bool(output_attentions or output_hidden_states)

    def supported(self, hidden_states, position_embeddings, record_outputs):
        """The block and call are ones the kernels evaluate, whatever the cache.  record_outputs: see
        records_outputs."""
        if position_embeddings is None or not self.block_supported(hidden_states, record_outputs):
            return False
        cos, sin = position_embeddings
        if cos.dtype != f32 or sin.dtype != f32 or cos.dim() != 3 or cos.shape != sin.shape or \
                cos.stride() != sin.stride() or cos.stride(2) != 1 or cos.shape[2] % 2 or \
                not 0 < cos.shape[2] <= self.block.attention.head_size:
            return False
        return True

    def block_supported(self, hidden_states, record_outputs):
        """The part of `supported` that does not read the rotary tables: what decode_graph can check before the model's
        rotary module has run."""
        b = self.block
        a = b.attention
        if not ENABLED or not hidden_states.is_cuda or record_outputs:
            return False
        hd = a.head_size
        if hd not in (64, 80, 128) or abs(a.scaling - hd ** -0.5) > 1e-9:
            return False
        if b.training and (a.attention_dropout > 0 or b.post_attention_dropout.p > 0 or b.post_mlp_dropout.p > 0):
            return False
        if getattr(a.config, "hidden_act", None) != "gelu":
            return False
        lins = (a.query_key_value, a.dense, b.mlp.dense_h_to_4h, b.mlp.dense_4h_to_h, b.input_layernorm,
                b.post_attention_layernorm)
        if any(m.bias is None for m in lins) or any(p.dtype != f32 for p in b.parameters()):
            return False
        if any(p.requires_grad for p in b.parameters()):
            return False   # this path has no wgrad: frozen blocks only
        return True

    def weights(self):
        b = self.block
        a = b.attention
        return (b.input_layernorm.weight, b.input_layernorm.bias, a.query_key_value.weight, a.query_key_value.bias,
                a.dense.weight, a.dense.bias, b.post_attention_layernorm.weight, b.post_attention_layernorm.bias,
                b.mlp.dense_h_to_4h.weight, b.mlp.dense_h_to_4h.bias, b.mlp.dense_4h_to_h.weight,
                b.mlp.dense_4h_to_h.bias)

    def step_args(self):
        """The head count, residual form and LayerNorm eps of the block, then its weights: the arguments after cos and
        sin of cached_neox_block_forward and decode_step_neox_block_forward."""
        b = self.block
        return (b.attention.config.num_attention_heads, bool(b.use_parallel_residual), b.input_layernorm.eps,
                b.post_attention_layernorm.eps) + self.weights()

    def decode_step(self, x, layer, pos_nk, key_mask, new_masked, workspace, position_embeddings):
        """One captured decode step of this block (decode_step_neox_block_forward); position_embeddings: the (cos, sin)
        of the new token's position."""
        cos, sin = position_embeddings
        return decode_step_neox_block_forward(x, layer, pos_nk, key_mask, new_masked, workspace, cos, sin,
                                              *self.step_args())

    def applicable(self, hidden_states, position_embeddings, layer_past, use_cache, record_outputs):
        """The uncached path (FrozenNeoXBlockFn, forward and backward)."""
        if layer_past is not None or use_cache:
            return False
        return self.supported(hidden_states, position_embeddings, record_outputs)

    def cache_layer(self, hidden_states, position_embeddings, layer_past, record_outputs):
        """The KVCacheLayer the cached path appends to, or None (see FastMptBlock.cache_layer)."""
        if not isinstance(layer_past, KVCache) or torch.is_grad_enabled():
            return None
        if not self.supported(hidden_states, position_embeddings, record_outputs):
            return None
        a = self.block.attention
        if a.layer_idx is None or not 0 <= a.layer_idx < len(layer_past.layers):
            return None
        layer = layer_past.layers[a.layer_idx]
        if layer.is_initialized and (layer.buf.dtype != bf16 or layer.buf.device != hidden_states.device or
                                     layer.buf.shape[0] != hidden_states.shape[0] or
                                     layer.heads != a.config.num_attention_heads or layer.head_dim != a.head_size):
            return None
        return layer

    def __call__(self, hidden_states, attention_mask=None, position_ids=None, use_cache=False, layer_past=None,
                 position_embeddings=None, output_attentions=None, output_hidden_states=None, pure_causal_flag=None,
                 **kwargs):
        record = self.records_outputs(output_attentions, output_hidden_states)
        layer = None
        if layer_past is not None or use_cache:
            layer = self.cache_layer(hidden_states, position_embeddings, layer_past, record)
            if layer is None:
                return None
        elif not self.applicable(hidden_states, position_embeddings, layer_past, use_cache, record):
            return None
        B, T, _ = hidden_states.shape
        cos, sin = position_embeddings
        if cos.shape[0] not in (1, B) or cos.shape[1] != T:
            return None
        nk = T if layer is None else layer.length + T
        mask = None
        if attention_mask is not None:   # HF's sdpa mask, True = attend; a float (eager) mask is declined here
            mask = _kernel_mask(attention_mask, B, T, nk, layer is not None and T == 1, true_attends=True)
            if mask is None:
                return None
        x = hidden_states if hidden_states.dtype == f32 else hidden_states.float()
        flag = pure_causal_flag if mask is not None else None
        rest = (cos, sin) + self.step_args()
        if layer is not None:
            out = cached_neox_block_forward(x, layer, mask, flag, *rest)
        else:
            out = FrozenNeoXBlockFn.apply(x, mask, flag, *rest)
        return out if out.dtype == hidden_states.dtype else out.to(hidden_states.dtype)


# ---- LLaMA (HF LlamaDecoderLayer: the LM of the OpenFlamingo-9B v1 checkpoint, LLaMA-7B) -------------------------------
#
#   a = rmsnorm1(x);  q, k, v = a Wq^T, a Wk^T, a Wv^T;  q, k = rotary(q, k; cos, sin)     (rotate_half, full head)
#   x1 = x + softmax(q k^T / sqrt(hd) + mask) v Wo^T
#   out = x1 + (silu(g) * u) Wd^T,   g, u = rmsnorm2(x1) Wg^T, rmsnorm2(x1) Wu^T             no biases anywhere
#
# Under autocast HF rounds to bf16 at: the RMSNorm outputs (as Linear operands), every Linear output, q and k after the
# rotation (as sdpa operands), silu(g) and silu(g) * u.  The kernels round at the same points: ofk_rmsnorm_fwd, the
# STORE_BF16 / GATE_RESID_F32 GEMM epilogues, ofk_rope_pack and ofk_swiglu_fwd.
#
# Q, K and V come from one GEMM against one bf16 copy of [Wq; Wk; Wv] whose rows are re-ordered per head as
# (q | k | v) -- the GPT-NeoX query_key_value layout -- so ofk_rope_pack splits and rotates its output and
# ofk_rope_unpack_bwd writes the gradient the dgrad GEMM with the same copy takes.  Likewise g and u come from one GEMM
# against a bf16 [Wg; Wu].  These packed copies are the only bf16 copies of those five weights.

_wpack_cache = {}


def _packed_w16(layout, params, fill):
    """The bf16 weight `fill(params)` builds from several fp32 parameters, kept until one of them changes.  `layout`
    names everything besides the parameters that `fill` reads (it is part of the cache key, so the same parameters
    packed another way get their own copy).  Refreshed by w16's rule -- weakly referenced parameters at the same
    version counters and addresses -- so `load_state_dict` or an in-place edit is seen."""
    key = (layout,) + tuple(id(p) for p in params)
    state = tuple((p._version, p.data_ptr()) for p in params)
    ent = _wpack_cache.get(key)
    if ent is not None and all(r() is p for r, p in zip(ent[0], params)) and ent[1] == state:
        return ent[2]
    t = fill(params)
    refs = tuple(weakref.ref(p, lambda _r, k=key: _wpack_cache.pop(k, None)) for p in params)
    _wpack_cache[key] = (refs, state, t)
    return t


def _qkv16(wq, wk, wv, heads):
    """bf16 [3D, D] copy of the q/k/v projections with rows in the per-head (q | k | v) order: packed row
    (h * 3 + p) * hd + j is row j of head h of part p (Wq, Wk, Wv)."""
    def fill(ps):
        D, K = ps[0].shape
        t = torch.empty((heads, 3, D // heads, K), device=ps[0].device, dtype=bf16)
        for i, p in enumerate(ps):
            t[:, i].copy_(p.detach().view(heads, D // heads, K))
        return t.view(3 * D, K)
    return _packed_w16(("qkv", heads), (wq, wk, wv), fill)


def _gu16(wg, wu):
    """bf16 [2F, D] copy of cat([Wg, Wu]): the gate|up GEMM writes gu = [g | u]."""
    def fill(ps):
        F, K = ps[0].shape
        t = torch.empty((2 * F, K), device=ps[0].device, dtype=bf16)
        t[:F].copy_(ps[0].detach())
        t[F:].copy_(ps[1].detach())
        return t
    return _packed_w16("gate|up", (wg, wu), fill)


def _llama_tail(x2d, o, eps2, wo, n2_w, wg, wu, wd, want_rstd):
    """The block after its attention core.  x2d: [R, D] f32 block input; o: [R, D] bf16 attention output.  Returns
    (out, x1, rstd2, gu): x1 = x + bf16(o Wo^T), the second RMSNorm's rstd (None unless want_rstd) and gu = [g | u]."""
    x1 = ops.gemm(o, w16(wo), epi=L.EPI_GATE_RESID_F32, aux=x2d)                   # + residual
    a2, rstd2 = ops.rmsnorm_fwd(x1, n2_w, eps2, want_rstd=want_rstd)
    gu = ops.gemm(a2, _gu16(wg, wu))                                                # [R, 2F]
    del a2
    h = ops.swiglu_fwd(gu)
    out = ops.gemm(h, w16(wd), epi=L.EPI_GATE_RESID_F32, aux=x1)                    # + residual
    return out, x1, rstd2, gu


class FrozenLlamaBlockFn(torch.autograd.Function):
    """A frozen LlamaDecoderLayer: forward, and the backward to its input only (the parameters take no gradient).
    x: [B, T, D] f32; mask: [B, T, T] bytes (nonzero = masked) or None for causal only; cos, sin: f32 [1 or B, T, rot]."""

    @staticmethod
    def forward(ctx, x, mask, pure_flag, cos, sin, heads, eps1, eps2, n1_w, wq, wk, wv, wo, n2_w, wg, wu, wd):
        B, T, D = x.shape
        R = B * T
        hd = D // heads
        x2d = _rows(x)
        a, rstd1 = ops.rmsnorm_fwd(x2d, n1_w, eps1)
        qkv = ops.gemm(a, _qkv16(wq, wk, wv, heads))                                # [R, 3D], heads as (q | k | v)
        del a
        q, k, v = ops.rope_pack(qkv.view(B, T, 3 * D), heads, hd, cos, sin)
        del qkv
        scale = float(hd ** -0.5)
        o, lse = ops.attn_dense_fwd(q, k, v, heads, hd, scale, causal=mask is None, mask=mask,
                                    pure_causal_flag=pure_flag)
        out, x1, rstd2, gu = _llama_tail(x2d, o.view(R, D), eps2, wo, n2_w, wg, wu, wd, want_rstd=True)
        ctx.save_for_backward(x2d, rstd1, q, k, v, o, lse, x1, rstd2, gu, cos, sin, n1_w, wq, wk, wv, wo, n2_w, wg, wu,
                              wd, mask if mask is not None else x2d.new_empty(0),
                              pure_flag if pure_flag is not None else x2d.new_empty(0))
        ctx.meta = (B, T, D, heads, hd, scale, mask is not None, pure_flag is not None)
        return out.view(B, T, D)

    @staticmethod
    def backward(ctx, dout):
        (x2d, rstd1, q, k, v, o, lse, x1, rstd2, gu, cos, sin, n1_w, wq, wk, wv, wo, n2_w, wg, wu, wd, mask,
         pure_flag) = ctx.saved_tensors
        B, T, D, heads, hd, scale, has_mask, has_flag = ctx.meta
        mask = mask if has_mask else None
        pure_flag = pure_flag if has_flag else None
        R = B * T
        d2 = _rows(dout)
        if d2.dtype != f32:
            d2 = d2.float()
        dbr = ops.gate_bwd(d2, None, None, None)                                     # bf16 cast
        dh = ops.gemm(dbr, w16(wd), b_mn=True)                                       # [R, F]
        del dbr
        dgu = ops.swiglu_bwd(dh, gu)                                                 # [R, 2F]
        del dh
        da2 = ops.gemm(dgu, _gu16(wg, wu), b_mn=True)
        del dgu
        dx1 = ops.rmsnorm_bwd(da2, x1, n2_w, rstd2, dx_add=d2)
        del da2
        dy = ops.gate_bwd(dx1, None, None, None)
        d_o = ops.gemm(dy, w16(wo), b_mn=True)                                       # [R, D]
        del dy
        dq, dk, dv = ops.attn_dense_bwd(q, k, v, o, d_o.view(B, T, D), lse, heads, hd, scale,
                                        causal=mask is None, mask=mask, pure_causal_flag=pure_flag)
        del d_o
        dqkv = ops.rope_unpack_bwd(dq, dk, dv, heads, hd, cos, sin)                  # [B, T, 3D]
        del dq, dk, dv
        da = ops.gemm(dqkv.view(R, 3 * D), _qkv16(wq, wk, wv, heads), b_mn=True)
        dx = ops.rmsnorm_bwd(da, x2d, n1_w, rstd1, dx_add=dx1)
        return (dx.view(B, T, D),) + (None,) * 16


def cached_llama_block_forward(x, layer, mask, pure_flag, cos, sin, heads, eps1, eps2, n1_w, wq, wk, wv, wo, n2_w, wg,
                               wu, wd):
    """Inference forward of one LLaMA block that appends its nq new tokens to `layer` (a kv_cache.KVCacheLayer) and
    attends over everything cached.  ops.rope_pack writes the rotated K and the V straight into cache rows
    [past, past + nq); one token attends through the decode kernel, a chunk through the dense kernel over the cached
    views.  mask: as for cached_block_forward.  x: [B, nq, D] f32; returns the same."""
    B, nq, D = x.shape
    hd = D // heads
    x2d = _rows(x)
    a, _ = ops.rmsnorm_fwd(x2d, n1_w, eps1, want_rstd=False)
    qkv = ops.gemm(a, _qkv16(wq, wk, wv, heads)).view(B, nq, 3 * D)
    del a
    if not layer.is_initialized:
        layer.init_storage(B, heads, hd, bf16, x.device)
    past = layer.length
    rows = layer.reserve(nq)[:, past:past + nq]
    q, _, _ = ops.rope_pack(qkv, heads, hd, cos, sin, k=rows[..., :D], v=rows[..., D:])
    del qkv
    layer.length = past + nq
    k, v = layer.kv_views()
    scale = float(hd ** -0.5)
    if nq == 1:
        o = ops.attn_decode(q.view(B, D), k, v, heads, hd, scale, key_mask=mask)
    else:
        o, _ = ops.attn_dense_fwd(q, k, v, heads, hd, scale, causal=mask is None, mask=mask, pure_causal_flag=pure_flag,
                                  want_lse=False)
    return _llama_tail(x2d, o.view(B * nq, D), eps2, wo, n2_w, wg, wu, wd, want_rstd=False)[0].view(B, nq, D)


class FastLlamaBlock:
    """Callable with HF LlamaDecoderLayer.forward's signature; returns None when the fast path does not apply, and the
    block's output tensor otherwise.

    Graph-replayed decoding does not cover LLaMA: decode_graph.eligible declines an LM that is neither GPT-NeoX nor
    has MPT's `transformer` / `norm_f`, so `generate(..., cache_implementation="static")` runs the eager cached path
    on the fixed-capacity KVCache, step by step.  Those steps are the ones a growing KVCache takes (the same kernels
    on the same rows; the decode kernel's split does not depend on the capacity), so they give the same bits."""

    def __init__(self, block):
        self.block = block

    def records_outputs(self, output_attentions=None, output_hidden_states=None):
        """Whether the caller asked HF to record this layer's hidden states or attention weights, which LlamaModel
        does with hooks on the modules the fast path does not call (see FastNeoXBlock.records_outputs)."""
        cfg = self.block.self_attn.config
        if output_attentions is None:
            output_attentions = getattr(cfg, "output_attentions", False)
        if output_hidden_states is None:
            output_hidden_states = getattr(cfg, "output_hidden_states", False)
        return bool(output_attentions or output_hidden_states)

    def supported(self, hidden_states, position_embeddings, record_outputs):
        """The block and call are ones the kernels evaluate, whatever the cache."""
        if position_embeddings is None or not self.block_supported(hidden_states, record_outputs):
            return False
        cos, sin = position_embeddings
        if cos.dtype != f32 or sin.dtype != f32 or cos.dim() != 3 or cos.shape != sin.shape or \
                cos.stride() != sin.stride() or cos.stride(2) != 1 or cos.shape[2] % 2 or \
                not 0 < cos.shape[2] <= self.block.self_attn.head_dim:
            return False
        return True

    def block_supported(self, hidden_states, record_outputs):
        """The part of `supported` that does not read the rotary tables."""
        b = self.block
        a = b.self_attn
        cfg = a.config
        if not ENABLED or not hidden_states.is_cuda or record_outputs:
            return False
        hd = a.head_dim
        if hd not in (64, 128) or abs(a.scaling - hd ** -0.5) > 1e-9:
            return False
        if cfg.num_key_value_heads != cfg.num_attention_heads or cfg.num_attention_heads * hd != cfg.hidden_size:
            return False   # grouped-query attention needs a K/V head map the cores do not have
        if getattr(cfg, "hidden_act", None) != "silu" or b.mlp.intermediate_size % 16:
            return False   # the GEMMs take N % 16 == 0, the down-projection's dgrad has N = intermediate_size
        if b.training and a.attention_dropout > 0:
            return False
        lins = (a.q_proj, a.k_proj, a.v_proj, a.o_proj, b.mlp.gate_proj, b.mlp.up_proj, b.mlp.down_proj)
        if any(m.bias is not None for m in lins) or any(p.dtype != f32 for p in b.parameters()):
            return False
        if any(p.requires_grad for p in b.parameters()):
            return False   # this path has no wgrad: frozen blocks only
        return True

    def weights(self):
        b = self.block
        a = b.self_attn
        m = b.mlp
        return (b.input_layernorm.weight, a.q_proj.weight, a.k_proj.weight, a.v_proj.weight, a.o_proj.weight,
                b.post_attention_layernorm.weight, m.gate_proj.weight, m.up_proj.weight, m.down_proj.weight)

    def step_args(self):
        """The head count and RMSNorm eps of the block, then its weights: the arguments after cos and sin of
        cached_llama_block_forward."""
        b = self.block
        return (b.self_attn.config.num_attention_heads, b.input_layernorm.variance_epsilon,
                b.post_attention_layernorm.variance_epsilon) + self.weights()

    def applicable(self, hidden_states, position_embeddings, past_key_values, use_cache, record_outputs):
        """The uncached path (FrozenLlamaBlockFn, forward and backward)."""
        if past_key_values is not None or use_cache:
            return False
        return self.supported(hidden_states, position_embeddings, record_outputs)

    def cache_layer(self, hidden_states, position_embeddings, past_key_values, record_outputs):
        """The KVCacheLayer the cached path appends to, or None (see FastMptBlock.cache_layer)."""
        if not isinstance(past_key_values, KVCache) or torch.is_grad_enabled():
            return None
        if not self.supported(hidden_states, position_embeddings, record_outputs):
            return None
        a = self.block.self_attn
        if a.layer_idx is None or not 0 <= a.layer_idx < len(past_key_values.layers):
            return None
        layer = past_key_values.layers[a.layer_idx]
        if layer.is_initialized and (layer.buf.dtype != bf16 or layer.buf.device != hidden_states.device or
                                     layer.buf.shape[0] != hidden_states.shape[0] or
                                     layer.heads != a.config.num_attention_heads or layer.head_dim != a.head_dim):
            return None
        return layer

    def __call__(self, hidden_states, attention_mask=None, position_ids=None, past_key_values=None, use_cache=False,
                 position_embeddings=None, output_attentions=None, output_hidden_states=None, pure_causal_flag=None,
                 **kwargs):
        record = self.records_outputs(output_attentions, output_hidden_states)
        layer = None
        if past_key_values is not None or use_cache:
            layer = self.cache_layer(hidden_states, position_embeddings, past_key_values, record)
            if layer is None:
                return None
        elif not self.applicable(hidden_states, position_embeddings, past_key_values, use_cache, record):
            return None
        B, T, _ = hidden_states.shape
        cos, sin = position_embeddings
        if cos.shape[0] not in (1, B) or cos.shape[1] != T:
            return None
        nk = T if layer is None else layer.length + T
        mask = None
        if attention_mask is not None:   # HF's sdpa mask, True = attend; a float (eager) mask is declined here
            mask = _kernel_mask(attention_mask, B, T, nk, layer is not None and T == 1, true_attends=True)
            if mask is None:
                return None
        x = hidden_states if hidden_states.dtype == f32 else hidden_states.float()
        flag = pure_causal_flag if mask is not None else None
        rest = (cos, sin) + self.step_args()
        if layer is not None:
            out = cached_llama_block_forward(x, layer, mask, flag, *rest)
        else:
            out = FrozenLlamaBlockFn.apply(x, mask, flag, *rest)
        return out if out.dtype == hidden_states.dtype else out.to(hidden_states.dtype)


# ---- OPT (HF OPTDecoderLayer, pre-LN: OPT-125m, 1.3B, 2.7B, 6.7B) ----------------------------------------------------
#
#   a = LN1(x);  q = bf16(bf16(a Wq^T + bq) * s), s = hd^-0.5;  k, v = a Wk^T + bk, a Wv^T + bv
#   x1 = x + dropout_p(bf16(softmax(q k^T + mask) v Wo^T + bo))          (OPTAttention scales q, attention at scale 1)
#   out = x1 + dropout_p(bf16(relu(bf16(LN2(x1) W1^T + b1)) W2^T + b2))
#
# Q, K and V come from one BIAS_BF16 GEMM against the packed per-head (q | k | v) copy of [Wq; Wk; Wv] (_qkv16, as for
# LLaMA) and the matching packed bias; ofk_rope_pack without rotation splits the heads (head_dim 80 zero-padded to 128,
# as for GPT-NeoX) and ofk_scale_bf16 then rounds q * s to bf16, the rounding HF makes (s is exact at head_dim 64 only).
# The backward applies the same product to dq before ofk_rope_unpack_bwd.
#
# The residual dropout (OPT configs set dropout = 0.1, and the frozen LM trains in train mode) runs as a BIAS_BF16 GEMM
# followed by ofk_dropout_resid_fwd; its backward regenerates the mask from the saved (seed, offset) pair.  With
# dropout off (eval, or p = 0) the residual adds are BIAS_RESID_F32 epilogues, the same bits in one pass.


class _DropoutRng:
    """Per-device dropout state: `state` = int64 device (seed, next offset).  Each dropout call takes the pair with
    capturable device ops (a clone, then the offset advanced in place), so a captured training step draws fresh masks
    at every replay.  The seed is drawn from torch's default CUDA generator; it is drawn again whenever that generator
    was re-seeded since (its initial seed changed, or its offset went back below where the draw left it), so
    `torch.manual_seed` reproduces a run.  Re-seeding is checked on eager calls only, never while a graph is captured."""

    def __init__(self, device):
        self.device = device
        self.state = torch.zeros(2, dtype=torch.int64, device=device)
        self.mark = None   # (initial seed, generator offset) right after the last draw

    def _reseed_if_needed(self):
        gen = torch.cuda.default_generators[self.device.index]
        if self.mark is not None and gen.initial_seed() == self.mark[0] and gen.get_offset() >= self.mark[1]:
            return
        seed = torch.empty(1, dtype=torch.int64, device=self.device).random_(generator=gen)
        self.state[0:1].copy_(seed)
        self.state[1:2].zero_()
        self.mark = (gen.initial_seed(), gen.get_offset())

    def take(self):
        """A fresh int64 (seed, offset) pair for one dropout call."""
        if not torch.cuda.is_current_stream_capturing():
            self._reseed_if_needed()
        pair = self.state.clone()
        self.state[1:2].add_(1)
        return pair


_dropout_rngs = {}


def dropout_rng(device):
    """The _DropoutRng of a CUDA device."""
    device = torch.device(device)
    if device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    rng = _dropout_rngs.get(device.index)
    if rng is None:
        rng = _dropout_rngs[device.index] = _DropoutRng(device)
    return rng


def _qkv_bias(bq, bk, bv, heads):
    """fp32 [3D] packed bias matching _qkv16's rows: element (h * 3 + p) * hd + j is element h * hd + j of part p."""
    def fill(ps):
        D = ps[0].shape[0]
        t = torch.empty((heads, 3, D // heads), device=ps[0].device, dtype=f32)
        for i, b in enumerate(ps):
            t[:, i].copy_(b.detach().view(heads, D // heads))
        return t.view(3 * D)
    return _packed_w16(("qkv bias", heads), (bq, bk, bv), fill)


def _opt_resid(branch_in, w16_, bias, x2d, p):
    """x2d + dropout_p(bf16(branch_in W^T + bias)): (sum, the (seed, offset) pair or None when dropout is off)."""
    if p > 0:
        so = dropout_rng(x2d.device).take()
        y = ops.gemm(branch_in, w16_, epi=L.EPI_BIAS_BF16, bias=bias)
        return ops.dropout_resid_fwd(x2d, y, p, so), so
    return ops.gemm(branch_in, w16_, epi=L.EPI_BIAS_RESID_F32, bias=bias, aux=x2d), None


def _opt_tail(x2d, o, p, eps2, wo16, bo, n2_w, n2_b, w1, b1, w2, b2, want_stats):
    """The block after its attention core.  x2d: [R, D] f32 block input; o: [R, heads * width] bf16 attention output;
    wo16: the bf16 out-projection weight for that width; p: the residual dropout probability (0 = off).  Returns
    (out, x1, mean2, rstd2, h, so1, so2): LayerNorm-2 statistics (None unless want_stats), h = relu(bf16(fc1)) and the
    two dropout pairs (None when off)."""
    x1, so1 = _opt_resid(o, wo16, bo, x2d, p)
    un, mean2, rstd2 = ops.layernorm_fwd(x1, n2_w, n2_b, eps2, want_stats=want_stats)
    h = ops.gemm(un, w16(w1), epi=L.EPI_BIAS_BF16, bias=b1)
    del un
    ops.relu_bf16(h, out=h)
    out, so2 = _opt_resid(h, w16(w2), b2, x1, p)
    return out, x1, mean2, rstd2, h, so1, so2


def _opt_qkv(xn, B, T, heads, wq, wk, wv, bq, bk, bv):
    return ops.gemm(xn, _qkv16(wq, wk, wv, heads), epi=L.EPI_BIAS_BF16,
                    bias=_qkv_bias(bq, bk, bv, heads)).view(B, T, 3 * heads * (wq.shape[0] // heads))


class FrozenOptBlockFn(torch.autograd.Function):
    """A frozen pre-LN OPTDecoderLayer: forward, and the backward to its input only (the parameters take no gradient).
    x: [B, T, D] f32; mask: [B, T, T] bytes (nonzero = masked) or None for causal only; p: residual dropout (0 = off)."""

    @staticmethod
    def forward(ctx, x, mask, pure_flag, heads, p, eps1, eps2, n1_w, n1_b, wq, wk, wv, bq, bk, bv, wo, bo, n2_w, n2_b,
                w1, b1, w2, b2):
        B, T, D = x.shape
        R = B * T
        hd = D // heads
        W = _neox_width(hd)
        s = float(hd ** -0.5)
        x2d = _rows(x)
        xn, mean1, rstd1 = ops.layernorm_fwd(x2d, n1_w, n1_b, eps1)
        qkv = _opt_qkv(xn, B, T, heads, wq, wk, wv, bq, bk, bv)
        del xn
        q, k, v = ops.rope_pack(qkv, heads, hd, q_width=W, kv_width=W)
        del qkv
        ops.scale_bf16(q, s, out=q)
        o, lse = ops.attn_dense_fwd(q, k, v, heads, W, 1.0, causal=mask is None, mask=mask, pure_causal_flag=pure_flag)
        out, x1, mean2, rstd2, h, so1, so2 = _opt_tail(x2d, o.view(R, heads * W), p, eps2, padded_w16(wo, heads, hd, W),
                                                       bo, n2_w, n2_b, w1, b1, w2, b2, want_stats=True)
        empty = x2d.new_empty(0)
        ctx.save_for_backward(x2d, mean1, rstd1, q, k, v, o, lse, x1, mean2, rstd2, h, n1_w, wq, wk, wv, wo, n2_w, w1, w2,
                              mask if mask is not None else empty, pure_flag if pure_flag is not None else empty,
                              so1 if so1 is not None else empty, so2 if so2 is not None else empty)
        ctx.meta = (B, T, D, heads, hd, W, s, p, mask is not None, pure_flag is not None)
        return out.view(B, T, D)

    @staticmethod
    def backward(ctx, dout):
        (x2d, mean1, rstd1, q, k, v, o, lse, x1, mean2, rstd2, h, n1_w, wq, wk, wv, wo, n2_w, w1, w2, mask, pure_flag,
         so1, so2) = ctx.saved_tensors
        B, T, D, heads, hd, W, s, p, has_mask, has_flag = ctx.meta
        mask = mask if has_mask else None
        pure_flag = pure_flag if has_flag else None
        R = B * T
        d2 = _rows(dout)
        if d2.dtype != f32:
            d2 = d2.float()
        dy2 = ops.dropout_resid_bwd(d2, p, so2) if p > 0 else ops.gate_bwd(d2, None, None, None)
        dh = ops.gemm(dy2, w16(w2), b_mn=True)                                       # [R, F]
        del dy2
        ops.relu_bwd_bf16(dh, h, out=dh)
        du = ops.gemm(dh, w16(w1), b_mn=True)
        del dh
        dx1 = ops.layernorm_bwd(du, x1, n2_w, mean2, rstd2, dx_add=d2)
        del du
        dy1 = ops.dropout_resid_bwd(dx1, p, so1) if p > 0 else ops.gate_bwd(dx1, None, None, None)
        d_o = ops.gemm(dy1, padded_w16(wo, heads, hd, W), b_mn=True)                # [R, heads * W], padding zero
        del dy1
        dq, dk, dv = ops.attn_dense_bwd(q, k, v, o, d_o.view(B, T, heads * W), lse, heads, W, 1.0,
                                        causal=mask is None, mask=mask, pure_causal_flag=pure_flag)
        del d_o
        ops.scale_bf16(dq, s, out=dq)                                                 # d(q_proj) = bf16(dq * s)
        dqkv = ops.rope_unpack_bwd(dq, dk, dv, heads, hd)                             # [B, T, 3D]
        del dq, dk, dv
        dxn = ops.gemm(dqkv.view(R, 3 * D), _qkv16(wq, wk, wv, heads), b_mn=True)
        dx = ops.layernorm_bwd(dxn, x2d, n1_w, mean1, rstd1, dx_add=dx1)
        return (dx.view(B, T, D),) + (None,) * 22


def cached_opt_block_forward(x, layer, mask, pure_flag, heads, p, eps1, eps2, n1_w, n1_b, wq, wk, wv, bq, bk, bv, wo, bo,
                             n2_w, n2_b, w1, b1, w2, b2):
    """Inference forward of one OPT block that appends its nq new tokens to `layer` (a kv_cache.KVCacheLayer, unpadded
    head_dim rows, so HF's attention can extend it through KVCacheLayer.update) and attends over everything cached.
    ops.rope_pack (no rotation) writes the K and V straight into cache rows [past, past + nq).
      nq == 1: q unpadded, the decode kernel at head_dim hd, the out-projection with Wo itself;
      nq > 1 : q and the cached K/V rows [0, nk) padded to the core's width, the dense kernel, the padded Wo.
    mask: as for cached_block_forward.  x: [B, nq, D] f32; returns the same."""
    B, nq, D = x.shape
    hd = D // heads
    x2d = _rows(x)
    xn, _, _ = ops.layernorm_fwd(x2d, n1_w, n1_b, eps1, want_stats=False)
    qkv = _opt_qkv(xn, B, nq, heads, wq, wk, wv, bq, bk, bv)
    del xn
    if not layer.is_initialized:
        layer.init_storage(B, heads, hd, bf16, x.device)
    past = layer.length
    rows = layer.reserve(nq)[:, past:past + nq]
    W = hd if nq == 1 else _neox_width(hd)
    q, _, _ = ops.rope_pack(qkv, heads, hd, q_width=W, k=rows[..., :D], v=rows[..., D:])
    del qkv
    ops.scale_bf16(q, float(hd ** -0.5), out=q)
    layer.length = past + nq
    k, v = layer.kv_views()
    if nq == 1:
        o = ops.attn_decode(q.view(B, D), k, v, heads, hd, 1.0, key_mask=mask)
    else:
        if W != hd:
            _, k, v = ops.rope_pack(None, heads, hd, kv_src=(k, v), kv_width=W)
        o, _ = ops.attn_dense_fwd(q, k, v, heads, W, 1.0, causal=mask is None, mask=mask, pure_causal_flag=pure_flag,
                                  want_lse=False)
    return _opt_tail(x2d, o.view(B * nq, heads * W), p, eps2, padded_w16(wo, heads, hd, W), bo, n2_w, n2_b, w1, b1,
                     w2, b2, want_stats=False)[0].view(B, nq, D)


class FastOptBlock:
    """Callable with HF OPTDecoderLayer.forward's signature; returns None when the fast path does not apply, and the
    block's output tensor otherwise.

    Graph-replayed decoding does not cover OPT: decode_graph.eligible declines an LM that is neither GPT-NeoX nor has
    MPT's `transformer` / `norm_f`, so `generate(..., cache_implementation="static")` runs the eager cached path on the
    fixed-capacity KVCache, step by step, with the bits of a growing KVCache (see FastLlamaBlock)."""

    def __init__(self, block):
        self.block = block

    def records_outputs(self, output_attentions=None, output_hidden_states=None):
        """Whether the caller asked HF to record this layer's hidden states or attention weights, which OPTDecoder
        does with hooks on the modules the fast path does not call (see FastNeoXBlock.records_outputs)."""
        cfg = self.block.self_attn.config
        if output_attentions is None:
            output_attentions = getattr(cfg, "output_attentions", False)
        if output_hidden_states is None:
            output_hidden_states = getattr(cfg, "output_hidden_states", False)
        return bool(output_attentions or output_hidden_states)

    def supported(self, hidden_states, record_outputs):
        """The block and call are ones the kernels evaluate, whatever the cache."""
        b = self.block
        a = b.self_attn
        if not ENABLED or not hidden_states.is_cuda or record_outputs:
            return False
        if not b.do_layer_norm_before or getattr(a.config, "activation_function", None) != "relu":
            return False   # post-LN (OPT-350m) and other activations are HF's
        hd = a.head_dim
        if hd not in (64, 80, 128) or abs(a.scaling - hd ** -0.5) > 1e-9 or a.embed_dim != a.num_heads * hd:
            return False
        if a.embed_dim > 4096 or b.fc1.out_features % 16:
            return False   # the LayerNorm kernels take D <= 4096; the fc2 dgrad GEMM has N = ffn_dim
        if b.training and a.dropout > 0:
            return False   # attention-probability dropout is not in the attention cores
        if not 0.0 <= self.dropout_p() < 1.0:
            return False
        lins = (a.q_proj, a.k_proj, a.v_proj, a.out_proj, b.fc1, b.fc2)
        norms = (b.self_attn_layer_norm, b.final_layer_norm)
        if any(m.bias is None for m in lins) or any(n.weight is None or n.bias is None for n in norms):
            return False
        if any(p.dtype != f32 for p in b.parameters()):
            return False
        if any(p.requires_grad for p in b.parameters()):
            return False   # this path has no wgrad: frozen blocks only
        return True

    def dropout_p(self):
        """The residual dropout probability this call applies: the layer's in training mode, else 0."""
        return float(self.block.dropout) if self.block.training else 0.0

    def weights(self):
        b = self.block
        a = b.self_attn
        return (b.self_attn_layer_norm.weight, b.self_attn_layer_norm.bias, a.q_proj.weight, a.k_proj.weight,
                a.v_proj.weight, a.q_proj.bias, a.k_proj.bias, a.v_proj.bias, a.out_proj.weight, a.out_proj.bias,
                b.final_layer_norm.weight, b.final_layer_norm.bias, b.fc1.weight, b.fc1.bias, b.fc2.weight, b.fc2.bias)

    def step_args(self):
        """The head count, dropout probability and LayerNorm eps of the block, then its weights: the arguments after
        pure_flag of FrozenOptBlockFn and cached_opt_block_forward."""
        b = self.block
        return (b.self_attn.num_heads, self.dropout_p(), b.self_attn_layer_norm.eps,
                b.final_layer_norm.eps) + self.weights()

    def applicable(self, hidden_states, past_key_values, use_cache, record_outputs):
        """The uncached path (FrozenOptBlockFn, forward and backward)."""
        if past_key_values is not None or use_cache:
            return False
        return self.supported(hidden_states, record_outputs)

    def cache_layer(self, hidden_states, past_key_values, record_outputs):
        """The KVCacheLayer the cached path appends to, or None (see FastMptBlock.cache_layer)."""
        if not isinstance(past_key_values, KVCache) or torch.is_grad_enabled():
            return None
        if not self.supported(hidden_states, record_outputs):
            return None
        a = self.block.self_attn
        if a.layer_idx is None or not 0 <= a.layer_idx < len(past_key_values.layers):
            return None
        layer = past_key_values.layers[a.layer_idx]
        if layer.is_initialized and (layer.buf.dtype != bf16 or layer.buf.device != hidden_states.device or
                                     layer.buf.shape[0] != hidden_states.shape[0] or
                                     layer.heads != a.num_heads or layer.head_dim != a.head_dim):
            return None
        return layer

    def __call__(self, hidden_states, attention_mask=None, past_key_values=None, use_cache=False, position_ids=None,
                 output_attentions=None, output_hidden_states=None, pure_causal_flag=None, **kwargs):
        record = self.records_outputs(output_attentions, output_hidden_states)
        layer = None
        if past_key_values is not None or use_cache:
            layer = self.cache_layer(hidden_states, past_key_values, record)
            if layer is None:
                return None
        elif not self.applicable(hidden_states, past_key_values, use_cache, record):
            return None
        B, T, _ = hidden_states.shape
        nk = T if layer is None else layer.length + T
        mask = None
        if attention_mask is not None:   # HF's sdpa mask, True = attend; a float (eager) mask is declined here
            mask = _kernel_mask(attention_mask, B, T, nk, layer is not None and T == 1, true_attends=True)
            if mask is None:
                return None
        x = hidden_states if hidden_states.dtype == f32 else hidden_states.float()
        flag = pure_causal_flag if mask is not None else None
        if layer is not None:
            out = cached_opt_block_forward(x, layer, mask, flag, *self.step_args())
        else:
            out = FrozenOptBlockFn.apply(x, mask, flag, *self.step_args())
        return out if out.dtype == hidden_states.dtype else out.to(hidden_states.dtype)


def accelerate(decoder_layer):
    """Return a fast evaluator for a recognised frozen decoder block (HF MptBlock, GPTNeoXLayer, LlamaDecoderLayer or
    OPTDecoderLayer), else None."""
    name = type(decoder_layer).__name__
    if name == "MptBlock" and hasattr(decoder_layer, "attn") and hasattr(decoder_layer, "ffn"):
        return FastMptBlock(decoder_layer)
    if name == "GPTNeoXLayer" and hasattr(decoder_layer, "attention") and hasattr(decoder_layer, "mlp"):
        return FastNeoXBlock(decoder_layer)
    if name == "LlamaDecoderLayer" and hasattr(decoder_layer, "self_attn") and hasattr(decoder_layer, "mlp"):
        return FastLlamaBlock(decoder_layer)
    if name == "OPTDecoderLayer" and hasattr(decoder_layer, "self_attn") and hasattr(decoder_layer, "fc1"):
        return FastOptBlock(decoder_layer)
    return None
