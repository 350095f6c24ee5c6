"""Float64 restatements of the fused blocks that round to bf16 exactly where the kernels round (test code only).

`fused.py` and `lm_blocks.FrozenMptBlockFn` compose GEMM, LayerNorm, attention and elementwise kernels and write
every backward by hand.  Each function here restates one of those blocks with float64 autograd on top of
`oracle/flamingo_oracle.py` (the Flamingo blocks) and HF `MptBlock` semantics (the frozen LM block), with three
rounding operators placed at the kernels' rounding points (DESIGN §2; `gemm.cu` epilogues, the attention rules):

  rf(t)  value rounded to bf16, gradient passed through   (bf16 operand copies whose gradient is an fp32 store)
  rb(t)  value and incoming gradient rounded to bf16       (bf16 activations whose gradient is a bf16 GEMM output)
  gb(t)  identity forward, gradient rounded to bf16

Rounding points, gated block and FFN:
  xn = rb(LN(x)) (its gradient is the bf16 dgrad GEMM output); weights rf(W); q, kv = rb(.) (the attention backward
  writes bf16 dq / dk / dv); media enters as rf(media) (dmedia is an fp32 store).
  Media attention (MediaRules): the forward rounds exp2(s - m) to bf16 for P.V, with m the running row maximum after
  each 64-key tile and the row sum l over the unrounded values; o = rb(acc / l).  The backward recomputes P from the
  LSE, rounds it for dV = P^T dO, rounds dS = P (dP - delta) scale for dQ and dK, and forms delta from the bf16 o.
  branch = rb(o Wout^T) (the gate backward writes bf16 dbranch = tanh(g) dout), x1 = x + tanh(g) branch in fp64.
  z = rb(xn2 W1^T), h = gelu(z) with gb between: the DGELU epilogue computes dz = bf16(bf16(dh) gelu'(z)).
Perceiver, unfolded (PerceiverLayerFn): kv_in = rb(cat(LN_media(x), LN_latents(latents))) and the compact latn for
  to_q is a second rb(LN_latents(latents)): two dgrad GEMMs, two roundings.
Perceiver, folded (PerceiverFoldedLayerFn, fused.py:392-415): media rows of kv = rb(rf(x_hat) rf(W_kv o gamma)^T +
  W_kv beta), the bias added in fp32 before the bf16 store; latent rows as unfolded.  x carries no gradient there.
FinalNormFn rounds nothing.
MPT block (FrozenMptBlockFn): as above with the dense rules: ALiBi scores, byte mask with finfo.min semantics, and P
  fed to P.V as hi + lo, so the forward does not round P; the backward rounds P and dS as the media rules do.

With rounding=False every operator is the identity and each function is the plain float64 block:
tests/test_rounded_reference_cpu.py pins that against the oracle and HF to 1e-12, forward and every gradient.
"""
import math

import torch
import torch.nn.functional as F

from oracle import flamingo_oracle as O

bf16 = torch.bfloat16
BKV = 64   # keys per attention tile: the running maximum of the online softmax is updated once per tile


def to_bf16(t):
    return t.to(bf16).to(t.dtype)


class _RF(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        return to_bf16(x)

    @staticmethod
    def backward(ctx, g):
        return g


class _RB(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        return to_bf16(x)

    @staticmethod
    def backward(ctx, g):
        return to_bf16(g)


class _GB(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        return x.clone()

    @staticmethod
    def backward(ctx, g):
        return to_bf16(g)


rf, rb, gb = _RF.apply, _RB.apply, _GB.apply


def _identity(t):
    return t


class Rounder:
    """The three rounding operators, or identities when rounding is off."""

    def __init__(self, rounding):
        self.on = bool(rounding)
        self.rf, self.rb, self.gb = (rf, rb, gb) if self.on else (_identity, _identity, _identity)


# ---------------------------------------------------------------------------------------------- attention
class _Attention(torch.autograd.Function):
    """softmax(scale Q K^T + bias) V per head with the kernels' row rules and rounding.

    q [B, nq, H*hd], k / v [B, nk, H*hd]; allowed [B, nq, nk] bool; uniform [B, nq]: rows that attend uniformly over
    all keys with no gradient to q or k; zero [B, nq]: rows that output 0; bias [H, nk] or None (ALiBi, slope * key)."""

    @staticmethod
    def forward(ctx, q, k, v, allowed, uniform, zero, bias, heads, scale, round_fwd_p, rounding):
        Q, K, V = (O._split_heads(t, heads) for t in (q, k, v))                 # [B, H, n, hd]
        B, H, nq, _ = Q.shape
        nk = K.shape[2]
        S = scale * Q @ K.transpose(-1, -2)
        if bias is not None:
            S = S + bias.view(1, H, 1, nk)
        live = (allowed & ~(uniform | zero)[..., None])[:, None].expand(B, H, nq, nk)
        unif = uniform[:, None, :, None].expand(B, H, nq, nk)
        Sm = torch.where(live, S, torch.full_like(S, -math.inf))
        Sm = torch.where(unif, torch.zeros_like(S), Sm)                            # uniform rows: every score 0
        m = Sm.amax(-1, keepdim=True)
        m = torch.where(torch.isfinite(m), m, torch.zeros_like(m))
        E = torch.exp(Sm - m)
        lsum = E.sum(-1, keepdim=True)
        P = E / torch.where(lsum > 0, lsum, torch.ones_like(lsum))
        if rounding and round_fwd_p:
            # per 64-key tile: bf16(exp(s - m_t)) with m_t the running maximum after the tile, rescaled in fp32
            nt = -(-nk // BKV)
            pad = nt * BKV - nk
            St = F.pad(Sm, (0, pad), value=-math.inf).view(B, H, nq, nt, BKV)
            mt = torch.cummax(St.amax(-1), dim=-1).values                          # [B, H, nq, nt]
            mt_f = torch.where(torch.isfinite(mt), mt, torch.zeros_like(mt))
            pt = to_bf16(torch.exp(St - mt_f[..., None]))
            rescale = torch.where(torch.isfinite(mt), torch.exp(mt_f - m), torch.zeros_like(mt))
            pt = pt * rescale[..., None]
            Pf = pt.view(B, H, nq, nt * BKV)[..., :nk] / torch.where(lsum > 0, lsum, torch.ones_like(lsum))
        else:
            Pf = P
        Oh = Pf @ V
        ctx.save_for_backward(Q, K, V, P, live, Oh)
        ctx.meta = (heads, scale, bool(rounding))
        return O._merge_heads(Oh)

    @staticmethod
    def backward(ctx, do):
        Q, K, V, P, live, Oh = ctx.saved_tensors
        heads, scale, rounding = ctx.meta
        dO = O._split_heads(do, heads)
        Ov = to_bf16(Oh) if rounding else Oh                                       # delta from the stored bf16 o
        dP = dO @ V.transpose(-1, -2)
        delta = (dO * Ov).sum(-1, keepdim=True)
        dS = torch.where(live, P * (dP - delta) * scale, torch.zeros_like(P))
        Pv = P
        if rounding:
            dS, Pv = to_bf16(dS), to_bf16(P)
        dq = O._merge_heads(dS @ K)
        dk = O._merge_heads(dS.transpose(-1, -2) @ Q)
        dv = O._merge_heads(Pv.transpose(-1, -2) @ dO)
        return dq, dk, dv, None, None, None, None, None, None, None, None


def attention(q, k, v, heads, scale, r, allowed=None, uniform=None, zero=None, bias=None, round_fwd_p=True):
    B, nq, nk = q.shape[0], q.shape[1], k.shape[1]
    dev = q.device
    if allowed is None:
        allowed = torch.ones(B, nq, nk, dtype=torch.bool, device=dev)
    if uniform is None:
        uniform = torch.zeros(B, nq, dtype=torch.bool, device=dev)
    if zero is None:
        zero = torch.zeros(B, nq, dtype=torch.bool, device=dev)
    return _Attention.apply(q, k, v, allowed, uniform, zero, bias, heads, scale, round_fwd_p, r.on)


def media_rows(media_locations, use_cached_media, t_txt, T_img, n, immediate):
    """(allowed [B, T, T_img*n], uniform [B, T], zero [B, T]) of the media mask (helpers.py:196-229)."""
    tt = O.text_time_of(media_locations, use_cached_media, t_txt)
    key_time = (torch.arange(T_img * n, device=tt.device) // n + 1)
    t = tt[:, :, None]
    allowed = (t == key_time) if immediate else (t >= key_time)
    zero = (tt == 0) if immediate else torch.zeros_like(tt, dtype=torch.bool)
    uniform = ~allowed.any(-1) & ~zero
    return allowed, uniform, zero


# ---------------------------------------------------------------------------------------------- Flamingo blocks
def _w(sd, name, r):
    return r.rf(sd[name])


def feed_forward(x, sd, prefix, r):
    """helpers.py:15-22: the FFN branch (before its gate), rounded as the GELU_DUAL / DGELU epilogues round."""
    xn = r.rb(O._ln(x, sd, prefix + ".0"))
    z = r.rb(xn @ _w(sd, prefix + ".1.weight", r).t())
    h = r.rf(r.gb(F.gelu(z)))
    return r.rb(h @ _w(sd, prefix + ".3.weight", r).t())


def masked_cross_attention(x, media, sd, prefix, media_locations=None, use_cached_media=False, heads=8,
                           only_attend_immediate_media=True, r=None):
    """helpers.py:160-233 -> the attention branch (before its gate).  media: (B, T_img, n, Dv)."""
    B, T_txt, _ = x.shape
    _, T_img, n, Dv = media.shape
    xn = r.rb(O._ln(x, sd, prefix + ".norm"))
    q = r.rb(xn @ _w(sd, prefix + ".to_q.weight", r).t())
    kv = r.rb(r.rf(media.reshape(B, T_img * n, Dv)) @ _w(sd, prefix + ".to_kv.weight", r).t())
    k, v = kv.chunk(2, dim=-1)
    mask = {}
    if media_locations is not None:
        allowed, uniform, zero = media_rows(media_locations, use_cached_media, T_txt, T_img, n,
                                            only_attend_immediate_media)
        mask = dict(allowed=allowed, uniform=uniform, zero=zero)
    o = r.rb(attention(q, k, v, heads, (q.shape[-1] // heads) ** -0.5, r, **mask))
    return r.rb(o @ _w(sd, prefix + ".to_out.weight", r).t())


def gated_cross_attention_block(x, media, sd, prefix="", media_locations=None, use_cached_media=False, heads=8,
                                only_attend_immediate_media=True, rounding=True, trace=None):
    """helpers.py:260-279 as GatedXattnBlockFn computes it.  trace: optional dict that receives the two branches and
    the block's midpoint x1 (what the gate gradients are dot products of)."""
    r = Rounder(rounding)
    p = prefix + "." if prefix else ""
    a = masked_cross_attention(x, media, sd, p + "attn", media_locations, use_cached_media, heads,
                               only_attend_immediate_media, r)
    x1 = a * sd[p + "attn_gate"].tanh() + x
    f = feed_forward(x1, sd, p + "ff", r)
    if trace is not None:
        trace.update(attn_branch=a, x1=x1, ff_branch=f)
    return f * sd[p + "ff_gate"].tanh() + x1


def perceiver_attention(x, latents, sd, prefix, heads, r):
    """helpers.py:39-65 as PerceiverLayerFn computes it.  x: (U, v, D), latents: (U, n, D)."""
    kv_in = r.rb(torch.cat((O._ln(x, sd, prefix + ".norm_media"), O._ln(latents, sd, prefix + ".norm_latents")), -2))
    latn = r.rb(O._ln(latents, sd, prefix + ".norm_latents"))
    q = r.rb(latn @ _w(sd, prefix + ".to_q.weight", r).t())
    k, v = r.rb(kv_in @ _w(sd, prefix + ".to_kv.weight", r).t()).chunk(2, dim=-1)
    o = r.rb(attention(q, k, v, heads, (q.shape[-1] // heads) ** -0.5, r))
    return r.rb(o @ _w(sd, prefix + ".to_out.weight", r).t())


def perceiver_attention_folded(x, latents, sd, prefix, heads, r, eps=1e-5):
    """helpers.py:39-65 as PerceiverFoldedLayerFn computes it: LN_media(x) W^T = x_hat (W o gamma)^T + W beta."""
    W, gamma, beta = sd[prefix + ".to_kv.weight"], sd[prefix + ".norm_media.weight"], sd[prefix + ".norm_media.bias"]
    x_hat = r.rf(F.layer_norm(x, (x.shape[-1],), eps=eps))
    kv_media = r.rb(x_hat @ r.rf(W * gamma[None, :]).t() + W @ beta)
    latn_kv = r.rb(O._ln(latents, sd, prefix + ".norm_latents"))
    kv_lat = r.rb(latn_kv @ r.rf(W).t())
    latn = r.rb(O._ln(latents, sd, prefix + ".norm_latents"))
    q = r.rb(latn @ _w(sd, prefix + ".to_q.weight", r).t())
    k, v = torch.cat((kv_media, kv_lat), -2).chunk(2, dim=-1)
    o = r.rb(attention(q, k, v, heads, (q.shape[-1] // heads) ** -0.5, r))
    return r.rb(o @ _w(sd, prefix + ".to_out.weight", r).t())


def perceiver_resampler(x, sd, prefix="", depth=None, heads=8, folded=False, rounding=True):
    """helpers.py:107-132 as PerceiverResampler runs it: frame / media-time embeddings, depth x (attention layer,
    FFN) on the latents broadcast over U = b*T, FinalNormFn.  x: (b, T, F, v, D)."""
    r = Rounder(rounding)
    b, T, Fr, v, D = x.shape
    if prefix + "frame_embs" in sd:
        x = x + sd[prefix + "frame_embs"][:Fr].view(1, 1, Fr, 1, D)
    x = x.reshape(b, T, Fr * v, D)
    if prefix + "media_time_embs" in sd:
        x = x + sd[prefix + "media_time_embs"][:T]
    U = b * T
    x = x.reshape(U, Fr * v, D)
    lat = sd[prefix + "latents"]
    latents = lat.unsqueeze(0).expand(U, *lat.shape)
    if depth is None:
        depth = 1 + max(int(k[len(prefix) + 7:].split(".")[0]) for k in sd if k.startswith(prefix + "layers."))
    attn = perceiver_attention_folded if folded else perceiver_attention
    for i in range(depth):
        latents = attn(x, latents, sd, f"{prefix}layers.{i}.0", heads, r) + latents
        latents = feed_forward(latents, sd, f"{prefix}layers.{i}.1", r) + latents
    return O._ln(latents, sd, prefix + "norm").view(b, T, *lat.shape)


# ---------------------------------------------------------------------------------------------- MPT block
def mpt_block(x, w, heads, slopes, mask=None, eps=1e-5, rounding=True):
    """HF MptBlock.forward (no biases, GELU(erf), ALiBi) as FrozenMptBlockFn computes it.

    w: dict with norm_1, Wqkv, out_proj, norm_2, up_proj, down_proj (HF weight tensors); slopes [H];
    mask: [B, T, T] bool, True = masked (HF's attention_mask), or None = causal."""
    r = Rounder(rounding)
    B, T, D = x.shape
    hd = D // heads
    xn = r.rb(F.layer_norm(x, (D,), w["norm_1"], None, eps))
    qkv = r.rb(xn @ r.rf(w["Wqkv"]).t())
    q, k, v = qkv.chunk(3, dim=-1)
    if mask is None:
        mask = torch.ones(T, T, dtype=torch.bool, device=x.device).triu(1).expand(B, T, T)
    allowed = ~mask
    uniform = ~allowed.any(-1)
    bias = slopes.to(x.dtype)[:, None] * torch.arange(T, device=x.device, dtype=x.dtype)
    o = r.rb(attention(q, k, v, heads, hd ** -0.5, r, allowed=allowed, uniform=uniform, bias=bias,
                       round_fwd_p=False))
    x1 = x + r.rb(o @ r.rf(w["out_proj"]).t())
    x1n = r.rb(F.layer_norm(x1, (D,), w["norm_2"], None, eps))
    z = r.rb(x1n @ r.rf(w["up_proj"]).t())
    h = r.rf(r.gb(F.gelu(z)))
    return x1 + r.rb(h @ r.rf(w["down_proj"]).t())
