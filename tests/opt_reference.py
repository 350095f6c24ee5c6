"""Float64 restatement of HF OPTDecoderLayer (pre-LN) as lm_blocks.FrozenOptBlockFn computes it (test code only), with
the rounding operators and the dense attention rules of rounded_reference.py placed at the kernels' rounding points:

  a = rb(LN1(x));  q = rb(rb(a rf(Wq)^T + bq) * s);  k, v = rb(a rf(Wk)^T + bk), rb(a rf(Wv)^T + bv)
                                                    BIAS_BF16, ofk_scale_bf16 (forward and dq), bf16 dgrad outputs
  o = rb(attention(q, k, v)) at scale 1             dense rules, as for GPT-NeoX
  x1 = x + drop1(rb(o rf(Wo)^T + bo))               BIAS_RESID_F32, or BIAS_BF16 + ofk_dropout_resid_fwd / _bwd
  u = rb(LN2(x1));  z = rb(u rf(W1)^T + b1);  h = gb(relu(z))                relu exact, dh a bf16 dgrad output
  out = x1 + drop2(rb(h rf(W2)^T + b2))

drop(y) = gb(m * rb(y * scale)) with m the 0/1 keep mask and scale torch's float32 dropout scale (identity when m is
None): the forward keeps bf16(y * scale), the backward gives bf16(bf16(dout) * scale) where kept.  With rounding=False
it is the plain float64 block."""
import torch
import torch.nn.functional as F

import rounded_reference as RR

NAMES = ("self_attn_layer_norm.weight", "self_attn_layer_norm.bias", "self_attn.q_proj.weight",
         "self_attn.q_proj.bias", "self_attn.k_proj.weight", "self_attn.k_proj.bias", "self_attn.v_proj.weight",
         "self_attn.v_proj.bias", "self_attn.out_proj.weight", "self_attn.out_proj.bias", "final_layer_norm.weight",
         "final_layer_norm.bias", "fc1.weight", "fc1.bias", "fc2.weight", "fc2.bias")


def dropout_scale(p):
    """torch's dropout scale as a float32 value: 1 / float32(1 - p), divided in double."""
    return float(torch.tensor(1.0 / float(torch.tensor(1.0 - p, dtype=torch.float32)), dtype=torch.float32))


def opt_block(x, w, heads, allowed, masks=None, p=0.0, relu_on=None, eps=1e-5, rounding=True):
    """x: [B, T, D] float64; w: dict NAMES -> float64 tensors; allowed: [B, T, T] bool (True = attend);
    masks: None, or the (attention-residual, MLP-residual) keep masks [B, T, D] (0/1) of a dropout p call;
    relu_on: None, or the [B, T, F] bool where the kernels' ReLU passed z.  A pre-activation within the GEMMs'
    accumulation error of 0 can take the other sign in float64, and the ReLU derivative then differs by a whole dh
    element, so the restatement of a kernel run takes the kernels' ReLU decisions."""
    r = RR.Rounder(rounding)
    B, T, D = x.shape
    hd = D // heads
    n1w, n1b, wq, bq, wk, bk, wv, bv, wo, bo, n2w, n2b, w1, b1, w2, b2 = (w[n] for n in NAMES)
    s = float(torch.tensor(hd ** -0.5, dtype=torch.float32))
    scale = dropout_scale(p)

    def drop(y, m):
        return y if m is None else r.gb(m * r.rb(y * scale))

    m1, m2 = masks if masks is not None else (None, None)
    a = r.rb(F.layer_norm(x, (D,), n1w, n1b, eps))
    q = r.rb(r.rb(a @ r.rf(wq).t() + bq) * s)
    k, v = r.rb(a @ r.rf(wk).t() + bk), r.rb(a @ r.rf(wv).t() + bv)
    uniform = ~allowed.any(-1)
    o = r.rb(RR.attention(q, k, v, heads, 1.0, r, allowed=allowed, uniform=uniform, round_fwd_p=False))
    x1 = x + drop(r.rb(o @ r.rf(wo).t() + bo), m1)
    u = r.rb(F.layer_norm(x1, (D,), n2w, n2b, eps))
    z = r.rb(u @ r.rf(w1).t() + b1)
    h = r.gb(torch.relu(z) if relu_on is None else torch.where(relu_on, z, torch.zeros_like(z)))
    return x1 + drop(r.rb(h @ r.rf(w2).t() + b2), m2)
