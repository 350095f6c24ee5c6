"""Float64 restatement of HF GPTNeoXLayer as lm_blocks.FrozenNeoXBlockFn computes it (test code only), with the
rounding operators and the dense attention rules of rounded_reference.py placed at the kernels' rounding points:

  a = rb(LN1(x));  qkv = rb(a rf(Wqkv)^T + bqkv)            BIAS_BF16 epilogue, dgrad GEMM output bf16
  q, k = rb(rotate(q), rotate(k))                           ofk_rope_pack rounds once; the dense backward writes bf16 dq
                                                            and dk, ofk_rope_unpack_bwd rounds their transpose again
  o = rb(attention(q, k, v))                                dense rules: P unrounded forward, P and dS rounded backward
  y = rb(o rf(Wd)^T + bd);  x1 = x + y                      BIAS_RESID_F32 (bf16(acc + b) + fp32 residual)
  u = rb(LN2(x1 or x));  z = rb(u rf(W1)^T + b1);  h = rf(gb(gelu(z)))       BIAS_BF16, gelu_bf16, DGELU_BF16
  out = rb(h rf(W2)^T + b2) + x1

Padding the heads to 128 columns adds exact zeros only, so the restatement works at head_dim.  rotate() is HF's
rotate_half form on the first rot = cos.shape[-1] columns.  With rounding=False it is the plain float64 block.
"""
import torch
import torch.nn.functional as F

import rounded_reference as RR

NAMES = ("input_layernorm.weight", "input_layernorm.bias", "attention.query_key_value.weight",
         "attention.query_key_value.bias", "attention.dense.weight", "attention.dense.bias",
         "post_attention_layernorm.weight", "post_attention_layernorm.bias", "mlp.dense_h_to_4h.weight",
         "mlp.dense_h_to_4h.bias", "mlp.dense_4h_to_h.weight", "mlp.dense_4h_to_h.bias")


def rotate(t, cos, sin, heads):
    """HF apply_rotary_pos_emb on t [B, T, heads * hd] with cos/sin [1 or B, T, rot]."""
    B, T, D = t.shape
    th = t.reshape(B, T, heads, D // heads)
    rot = cos.shape[-1]
    x1, x2, rest = th[..., :rot // 2], th[..., rot // 2:rot], th[..., rot:]
    c, s = cos[:, :, None, :], sin[:, :, None, :]
    y = th[..., :rot] * c + torch.cat((-x2, x1), -1) * s
    return torch.cat((y, rest), -1).reshape(B, T, D)


def neox_block(x, w, heads, cos, sin, allowed, parallel, eps=1e-5, rounding=True):
    """x: [B, T, D] float64; w: dict NAMES -> float64 tensors; cos, sin: float64 [1 or B, T, rot];
    allowed: [B, T, T] bool (True = attend)."""
    r = RR.Rounder(rounding)
    B, T, D = x.shape
    hd = D // heads
    a = r.rb(F.layer_norm(x, (D,), w[NAMES[0]], w[NAMES[1]], eps))
    qkv = r.rb(a @ r.rf(w[NAMES[2]]).t() + w[NAMES[3]]).view(B, T, heads, 3, hd)
    q, k, v = (qkv[..., i, :].reshape(B, T, D) for i in range(3))
    q, k = r.rb(rotate(q, cos, sin, heads)), r.rb(rotate(k, cos, sin, heads))
    uniform = ~allowed.any(-1)
    o = r.rb(RR.attention(q, k, v, heads, hd ** -0.5, r, allowed=allowed, uniform=uniform, round_fwd_p=False))
    x1 = x + r.rb(o @ r.rf(w[NAMES[4]]).t() + w[NAMES[5]])
    u = r.rb(F.layer_norm(x if parallel else x1, (D,), w[NAMES[6]], w[NAMES[7]], eps))
    z = r.rb(u @ r.rf(w[NAMES[8]]).t() + w[NAMES[9]])
    h = r.rf(r.gb(F.gelu(z)))
    return r.rb(h @ r.rf(w[NAMES[10]]).t() + w[NAMES[11]]) + x1
