"""Frozen-LM decoder blocks on the sm_90a kernels (SURVEY.md section 8f, rank 1).

The reference runs the frozen LM's decoder block as ordinary PyTorch (`self.decoder_layer(lang_x, ...)`,
flamingo_lm.py:63-65).  For the LM family named by BASELINE.json (MPT: HF `MptBlock` = LN -> Wqkv -> causal
ALiBi attention -> out_proj -> +res -> LN -> up_proj -> GELU(erf) -> down_proj -> +res, no biases) this module
evaluates the same block with the kernels already used by the gated blocks (wgmma GEMMs with fused
GELU / residual epilogues, LayerNorm, dense attention), forward plus the dgrad-only backward a frozen block
needs.  Anything else -- other LM families, KV-cache decoding, dropout, clip_qkv, output_attentions -- takes the
block's own PyTorch forward, exactly as in the reference.

Numerics are those of the block under `torch.autocast(bfloat16)`: fp32 residual stream, fp32 LayerNorm/softmax,
bf16 GEMM operands.
"""
import weakref

import torch

from . import _lib as L
from . import ops
from .fused import w16

bf16 = torch.bfloat16
f32 = torch.float32

ENABLED = True  # module-level switch (bench.py --lm eager turns it off to time the reference's PyTorch LM path)

_zero_bias = {}
_mask_cache = [None, None]  # (weakref to HF's [B,1,T,T] bool mask, its contiguous [B,T,T] byte view) -- one per forward


def _zeros(n, device):
    key = (n, device)
    t = _zero_bias.get(key)
    if t is None:
        t = torch.zeros(n, device=device, dtype=f32)
        _zero_bias[key] = t
    return t


class FrozenMptBlockFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, mask, pure_flag, slopes, heads, eps, n1_w, wqkv, wout, n2_w, wup, wdown):
        B, T, D = x.shape
        R = B * T
        hd = D // heads
        x2d = x.reshape(R, D)
        if not x2d.is_contiguous():
            x2d = x2d.contiguous()
        zb = _zeros(D, x.device)
        xn, mean1, rstd1 = ops.layernorm_fwd(x2d, n1_w, zb, eps)
        qkv = ops.gemm(xn, w16(wqkv))                                               # [R, 3D]
        del xn
        q3 = qkv.view(B, T, 3 * D)
        scale = float(hd ** -0.5)
        o, lse = ops.attn_dense_fwd(q3[..., :D], q3[..., D:2 * D], q3[..., 2 * D:], heads, hd, scale,
                                    causal=mask is None, mask=mask, slopes=slopes, pure_causal_flag=pure_flag)
        x1 = ops.gemm(o.view(R, D), w16(wout), epi=L.EPI_GATE_RESID_F32, aux=x2d)   # + residual
        x1n, mean2, rstd2 = ops.layernorm_fwd(x1, n2_w, zb, eps)
        z = torch.empty((R, wup.shape[0]), device=x.device, dtype=bf16)
        h = torch.empty((R, wup.shape[0]), device=x.device, dtype=bf16)
        ops.gemm(x1n, w16(wup), epi=L.EPI_GELU_DUAL, out=z, out2=h)
        del x1n
        out = ops.gemm(h, w16(wdown), epi=L.EPI_GATE_RESID_F32, aux=x1)             # + residual
        del h
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

    def applicable(self, hidden_states, position_bias, attention_mask, layer_past, use_cache, output_attentions):
        b = self.block
        if not ENABLED or not hidden_states.is_cuda or layer_past is not None or output_attentions:
            return False
        if use_cache:
            return False   # a caller that wants a `present` back (tuple-cache HF versions) gets the block's own forward
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

    def __call__(self, hidden_states, position_bias=None, attention_mask=None, layer_past=None, use_cache=False,
                 output_attentions=False, pure_causal_flag=None, **kwargs):
        if not self.applicable(hidden_states, position_bias, attention_mask, layer_past, use_cache, output_attentions):
            return None
        b = self.block
        a = b.attn
        B, T, D = hidden_states.shape
        if self._slopes is None or self._slopes.device != hidden_states.device:
            self._slopes = _alibi_slopes(position_bias)
            if self._slopes is None:
                return None
        mask = None
        if attention_mask is not None:
            m = attention_mask
            if m.dtype != torch.bool or m.dim() != 4 or m.shape[1] != 1 or m.shape[2] != T or m.shape[3] != T:
                return None
            ref = _mask_cache[0]
            if ref is not None and ref() is m and _mask_cache[1].shape[0] == B:
                mask = _mask_cache[1]
            else:
                mask = m.expand(B, 1, T, T).reshape(B, T, T).contiguous()
                _mask_cache[0], _mask_cache[1] = weakref.ref(m), mask
        x = hidden_states if hidden_states.dtype == f32 else hidden_states.float()
        out = FrozenMptBlockFn.apply(x, mask, pure_causal_flag if mask is not None else None, self._slopes, a.n_heads, b.norm_1.eps, b.norm_1.weight, a.Wqkv.weight,
                                     a.out_proj.weight, b.norm_2.weight, b.ffn.up_proj.weight, b.ffn.down_proj.weight)
        if out.dtype != hidden_states.dtype:
            out = out.to(hidden_states.dtype)
        return out, None


def accelerate(decoder_layer):
    """Return a fast evaluator for a recognised frozen decoder block, else None."""
    if type(decoder_layer).__name__ == "MptBlock" and hasattr(decoder_layer, "attn") and hasattr(decoder_layer, "ffn"):
        return FastMptBlock(decoder_layer)
    return None
