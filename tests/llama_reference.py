"""Float64 restatement of HF LlamaDecoderLayer as lm_blocks.FrozenLlamaBlockFn computes it (test code only), with the
rounding operators and the dense attention rules of rounded_reference.py placed at the kernels' rounding points:

  a = rb(rmsnorm1(x));  q, k, v = rb(a rf(Wq)^T), rb(a rf(Wk)^T), rb(a rf(Wv)^T)    ofk_rmsnorm_fwd, STORE_BF16; the
                                                                                    gradients are bf16 dgrad outputs
  q, k = rb(rotate(q)), rb(rotate(k))                                               ofk_rope_pack / ofk_rope_unpack_bwd
  o = rb(attention(q, k, v))                                                        dense rules, as for GPT-NeoX
  x1 = x + rb(o rf(Wo)^T)                                                           GATE_RESID_F32, bf16 cast of dx1
  a2 = rb(rmsnorm2(x1));  g, u = rb(a2 rf(Wg)^T), rb(a2 rf(Wu)^T)                    one [Wg; Wu] GEMM
  h = rb(rf(silu(g)) * u)                                                           ofk_swiglu_fwd / ofk_swiglu_bwd:
                                                                                    silu'(g) unrounded, d(silu) unrounded
  out = rb(h rf(Wd)^T) + x1

rmsnorm(x) = w * (x * rsqrt(mean(x^2) + eps)), LlamaRMSNorm's order.  With rounding=False it is the plain float64
block."""
import torch
import torch.nn.functional as F

import rounded_reference as RR
from neox_reference import rotate

NAMES = ("input_layernorm.weight", "self_attn.q_proj.weight", "self_attn.k_proj.weight", "self_attn.v_proj.weight",
         "self_attn.o_proj.weight", "post_attention_layernorm.weight", "mlp.gate_proj.weight", "mlp.up_proj.weight",
         "mlp.down_proj.weight")


def rmsnorm(x, w, eps):
    return w * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps))


def llama_block(x, w, heads, cos, sin, allowed, eps, rounding=True):
    """x: [B, T, D] float64; w: dict NAMES -> float64 tensors; cos, sin: float64 [1 or B, T, rot];
    allowed: [B, T, T] bool (True = attend)."""
    r = RR.Rounder(rounding)
    D = x.shape[-1]
    hd = D // heads
    n1, wq, wk, wv, wo, n2, wg, wu, wd = (w[n] for n in NAMES)
    a = r.rb(rmsnorm(x, n1, eps))
    q, k, v = (r.rb(a @ r.rf(m).t()) for m in (wq, wk, wv))
    q, k = r.rb(rotate(q, cos, sin, heads)), r.rb(rotate(k, cos, sin, heads))
    uniform = ~allowed.any(-1)
    o = r.rb(RR.attention(q, k, v, heads, hd ** -0.5, r, allowed=allowed, uniform=uniform, round_fwd_p=False))
    x1 = x + r.rb(o @ r.rf(wo).t())
    a2 = r.rb(rmsnorm(x1, n2, eps))
    g, u = r.rb(a2 @ r.rf(wg).t()), r.rb(a2 @ r.rf(wu).t())
    h = r.rb(r.rf(F.silu(g)) * u)
    return r.rb(h @ r.rf(wd).t()) + x1
