"""Fused forward/backward of the OpenFlamingo hot-path blocks on top of the libofk.so kernels.

Each block is ONE torch.autograd.Function whose forward and backward are explicit kernel sequences
(no autograd graph inside, no torch math on the hot path):

  gated_xattn_block   <->  GatedCrossAttentionBlock.forward   (helpers.py:260-279)
                            = MaskedCrossAttention (helpers.py:160-233) * tanh(attn_gate) + x,
                              FeedForward (helpers.py:15-22)       * tanh(ff_gate)   + x
  perceiver_layer     <->  one `latents = attn(x, latents) + latents; latents = ff(latents) + latents`
                            step of PerceiverResampler.forward (helpers.py:129-131)
  final_norm          <->  PerceiverResampler.norm (helpers.py:132)

Numerics follow the reference under `torch.autocast(bfloat16)` (train_utils.py:34-43): fp32 master weights and
fp32 residual stream; LayerNorm / softmax in fp32; GEMM operands rounded to bf16 at the same points where
autocast rounds them; fp32 accumulation.

Weight gradients: if a parameter carries `_ofk_grad` (an fp32 buffer, normally a view into the flat DDP
bucket -- see train.FlatTrainer) the wgrad GEMM accumulates straight into it and autograd receives None;
otherwise a fresh fp32 gradient tensor is returned and autograd/DDP handle it as usual.
"""
import weakref

import torch

from . import _lib as L
from . import ops

bf16 = torch.bfloat16
f32 = torch.float32

_w16_cache = {}

# set by train.GradBucket: called with a block's parameter tuple (gated block, resampler layer, final norm) once its
# backward kernels are enqueued
block_backward_hook = None


def w16(param):
    """bf16 operand copy of an fp32 master weight, refreshed when the parameter changes.

    The cache entry holds a weak reference to the parameter and is only trusted if it still points at THIS object
    (ids, versions and device addresses are all recycled once a parameter is freed)."""
    cached = getattr(param, "_ofk_w16", None)
    if cached is not None:
        # Maintained by the fused AdamW kernel (train.FlatTrainer), which writes parameter and copy through raw
        # pointers and so never bumps the version counter.  Anything else that changes the fp32 master --
        # model.load_state_dict(...) after the trainer was built (the reference's resume path, train.py:297-308), a
        # manual edit under no_grad -- does bump it: re-cast into the trainer's buffer before the GEMMs read it.
        if getattr(param, "_ofk_w16_version", None) != param._version:
            ops.cast_bf16(param.detach(), out=cached)
            param._ofk_w16_version = param._version
        return cached
    key = id(param)
    ent = _w16_cache.get(key)
    ver = param._version
    if ent is not None and ent[0]() is param and ent[1] == ver and ent[2] == param.data_ptr():
        return ent[3]
    t = ops.cast_bf16(param.detach())
    _w16_cache[key] = (weakref.ref(param, lambda _r, k=key: _w16_cache.pop(k, None)), ver, param.data_ptr(), t)
    return t


class _GradSink:
    """Where a parameter's gradient goes: its `_ofk_grad` bucket view (accumulate, return None) or a fresh tensor."""

    def __init__(self, param, needs):
        self.param = param
        self.direct = getattr(param, "_ofk_grad", None) if needs else None
        self.needs = needs
        self.buf = None

    def buffer(self):
        if not self.needs:
            return None
        if self.direct is not None:
            return self.direct
        if self.buf is None:
            self.buf = torch.zeros(self.param.shape, device=self.param.device, dtype=f32)
        return self.buf

    def result(self):
        return None if (not self.needs or self.direct is not None) else self.buffer()


def _wgrad(dy16, x16, sink):
    """sink += dy^T x   (dy: [R, out], x: [R, in], both bf16, reduction over R; accumulating epilogue).  No split-K:
    split-K partials would land in the gradient in whatever order the CTAs finish, so the gradient would change from
    run to run in its last bits (and through Adam, by far more at near-zero entries)."""
    buf = sink.buffer()
    if buf is None:
        return
    out_f, in_f = dy16.shape[1], x16.shape[1]
    ops.gemm(dy16, x16, a_mn=True, b_mn=True, epi=L.EPI_ATOMIC_F32, out=buf.view(out_f, in_f))


# ------------------------------------------------------------------------------------------ FeedForward
def _ffn_forward(x2d, ln_w, ln_b, w1, w2, gate):
    """x2d fp32 [R, D] -> x2d + tanh(gate) * W2 gelu(W1 LN(x2d))   (helpers.py:15-22, :277)."""
    R, D = x2d.shape
    xn, mean, rstd = ops.layernorm_fwd(x2d, ln_w, ln_b)
    inner = w1.shape[0]
    z = torch.empty((R, inner), device=x2d.device, dtype=bf16)
    h = torch.empty((R, inner), device=x2d.device, dtype=bf16)
    ops.gemm(xn, w16(w1), epi=L.EPI_GELU_DUAL, out=z, out2=h)
    branch = torch.empty((R, D), device=x2d.device, dtype=bf16) if gate is not None else None
    out = ops.gemm(h, w16(w2), epi=L.EPI_GATE_RESID_F32, aux=x2d, gate=gate, out2=branch)
    return out, (xn, mean, rstd, z, h, branch)


def _ffn_backward(dout, x2d, saved, ln_w, w1, w2, gate, sinks):
    """Returns d(x2d).  sinks: dict name -> _GradSink for ln_w, ln_b, w1, w2, gate."""
    xn, mean, rstd, z, h, branch = saved
    dgate = sinks["gate"].buffer() if gate is not None else None
    dbr = ops.gate_bwd(dout, branch, gate, dgate)                       # [R, D] bf16
    _wgrad(dbr, h, sinks["w2"])                                         # dW2 += dbr^T h
    dz = ops.gemm(dbr, w16(w2), b_mn=True, epi=L.EPI_DGELU_BF16, aux=z)  # (dbr W2) * gelu'(z)
    del dbr
    _wgrad(dz, xn, sinks["w1"])                                         # dW1 += dz^T LN(x)
    dxn = ops.gemm(dz, w16(w1), b_mn=True)                              # [R, D] bf16
    del dz
    return ops.layernorm_bwd(dxn, x2d, ln_w, mean, rstd, dgamma=sinks["ln_w"].buffer(), dbeta=sinks["ln_b"].buffer(),
                             dx_add=dout)


# ------------------------------------------------------------------------------------------ gated xattn block
class GatedXattnBlockFn(torch.autograd.Function):
    """x fp32 [B, T, D]; media fp32 [B, T_img*n, Dv] with its bf16 copy `media16` (cast once per forward for all
    layers); text_time int32 [B, T] (computed once per forward for all layers, cf. helpers.py:196-218 which the
    reference rebuilds in every layer)."""

    @staticmethod
    def forward(ctx, x, media, media16, text_time, mask_mode, heads, n_latents, norm_w, norm_b, wq, wkv, wout,
                attn_gate, ff_ln_w, ff_ln_b, ff_w1, ff_w2, ff_gate, kv_cache=None):
        B, T, D = x.shape
        R = B * T
        inner = wq.shape[0]
        x2d = x.reshape(R, D)
        if not x2d.is_contiguous():
            x2d = x2d.contiguous()
        M = media16.shape[0] * media16.shape[1]
        m2d = media16.view(M, media16.shape[2])
        # --- masked cross attention (helpers.py:184-233)
        xn, mean, rstd = ops.layernorm_fwd(x2d, norm_w, norm_b)
        q = ops.gemm(xn, w16(wq))                                            # [R, inner]
        # K/V of the media are recomputed by the reference in every layer on every decode step
        # (helpers.py:187-189); in no-grad mode they are computed once per (media, layer) and reused.
        kv_key = (id(wkv), wkv._version)
        kv = kv_cache.get(kv_key) if kv_cache is not None else None
        if kv is None:
            kv = ops.gemm(m2d, w16(wkv))                                     # [M, 2*inner]
            if kv_cache is not None:
                kv_cache[kv_key] = kv
        kv3 = kv.view(B, M // B, 2 * inner)
        o, lse = ops.attn_fwd(q.view(B, T, inner), kv3[..., :inner], kv3[..., inner:], heads,
                              float((inner // heads) ** -0.5), mask_mode=mask_mode, text_time=text_time,
                              keys_per_media=n_latents)
        a_branch = torch.empty((R, D), device=x.device, dtype=bf16)
        x1 = ops.gemm(o.view(R, inner), w16(wout), epi=L.EPI_GATE_RESID_F32, aux=x2d, gate=attn_gate, out2=a_branch)
        # --- gated feed forward (helpers.py:277)
        out, ff_saved = _ffn_forward(x1, ff_ln_w, ff_ln_b, ff_w1, ff_w2, ff_gate)
        ctx.save_for_backward(x2d, m2d, text_time, xn, mean, rstd, q, kv, o, lse, a_branch, x1, *ff_saved,
                              norm_w, wq, wkv, wout, attn_gate, ff_ln_w, ff_w1, ff_w2, ff_gate)
        ctx.meta = (B, T, D, M, inner, heads, n_latents, mask_mode)
        ctx.params = (norm_w, norm_b, wq, wkv, wout, attn_gate, ff_ln_w, ff_ln_b, ff_w1, ff_w2, ff_gate)
        ctx.media_shape = media.shape
        return out.view(B, T, D)

    @staticmethod
    def backward(ctx, dout):
        (x2d, m2d, text_time, xn, mean, rstd, q, kv, o, lse, a_branch, x1, f_xn, f_mean, f_rstd, f_z, f_h, f_branch,
         norm_w, wq, wkv, wout, attn_gate, ff_ln_w, ff_w1, ff_w2, ff_gate) = ctx.saved_tensors
        B, T, D, M, inner, heads, n_latents, mask_mode = ctx.meta
        R = B * T
        needs = ctx.needs_input_grad
        names = ("norm_w", "norm_b", "wq", "wkv", "wout", "attn_gate", "ff_ln_w", "ff_ln_b", "ff_w1", "ff_w2", "ff_gate")
        sinks = {n: _GradSink(p, needs[7 + i]) for i, (n, p) in enumerate(zip(names, ctx.params))}
        dout2d = dout.reshape(R, D)
        if not dout2d.is_contiguous():
            dout2d = dout2d.contiguous()
        if dout2d.dtype != f32:
            dout2d = dout2d.float()
        # --- feed forward
        dx1 = _ffn_backward(dout2d, x1, (f_xn, f_mean, f_rstd, f_z, f_h, f_branch), ff_ln_w, ff_w1, ff_w2, ff_gate,
                            {"ln_w": sinks["ff_ln_w"], "ln_b": sinks["ff_ln_b"], "w1": sinks["ff_w1"],
                             "w2": sinks["ff_w2"], "gate": sinks["ff_gate"]})
        # --- attention output projection + gate
        da = ops.gate_bwd(dx1, a_branch, attn_gate, sinks["attn_gate"].buffer())      # [R, D] bf16
        _wgrad(da, o.view(R, inner), sinks["wout"])
        d_o = ops.gemm(da, w16(wout), b_mn=True)                                      # [R, inner]
        del da
        # --- attention core
        kv3 = kv.view(B, M // B, 2 * inner)
        dkv = torch.empty_like(kv)
        dkv3 = dkv.view(B, M // B, 2 * inner)
        dq, _, _ = ops.attn_bwd(q.view(B, T, inner), kv3[..., :inner], kv3[..., inner:], o, d_o.view(B, T, inner), lse,
                                heads, float((inner // heads) ** -0.5), mask_mode=mask_mode, text_time=text_time,
                                keys_per_media=n_latents, dk=dkv3[..., :inner], dv=dkv3[..., inner:])
        dq2 = dq.view(R, inner)
        # --- projections
        _wgrad(dq2, xn, sinks["wq"])
        _wgrad(dkv, m2d, sinks["wkv"])
        dxn = ops.gemm(dq2, w16(wq), b_mn=True)                                       # [R, D] bf16
        dx = ops.layernorm_bwd(dxn, x2d, norm_w, mean, rstd, dgamma=sinks["norm_w"].buffer(),
                               dbeta=sinks["norm_b"].buffer(), dx_add=dx1)
        dmedia = None
        if needs[1]:
            dmedia = ops.gemm(dkv, w16(wkv), b_mn=True, epi=L.EPI_STORE_F32).view(ctx.media_shape)
        grads = [sinks[n].result() for n in names]
        if block_backward_hook is not None:
            block_backward_hook(ctx.params)
        return (dx.view(B, T, D) if needs[0] else None, dmedia, None, None, None, None, None, *grads, None)


# ------------------------------------------------------------------------------------------ perceiver layer
class PerceiverLayerFn(torch.autograd.Function):
    """x fp32 [U, v, Dv] (frozen ViT features, no grad); latents fp32 [U, n, Dv]."""

    @staticmethod
    def forward(ctx, x, latents, heads, nm_w, nm_b, nl_w, nl_b, wq, wkv, wout, ff_ln_w, ff_ln_b, ff_w1, ff_w2):
        U, v, Dv = x.shape
        n = latents.shape[1]
        inner = wq.shape[0]
        x2d = x.reshape(U * v, Dv)
        lat2d = latents.reshape(U * n, Dv)
        if not lat2d.is_contiguous():
            lat2d = lat2d.contiguous()
        # kv_input = cat((LN_media(x), LN_latents(latents)), -2), written in place by the two LayerNorms
        kv_in = torch.empty((U * (v + n), Dv), device=x.device, dtype=bf16)
        _, xm_mean, xm_rstd = ops.layernorm_fwd(x2d, nm_w, nm_b, out=kv_in, rows_per_group=v, group_stride=v + n,
                                                group_offset=0)
        ops.layernorm_fwd(lat2d, nl_w, nl_b, out=kv_in, rows_per_group=n, group_stride=v + n, group_offset=v,
                          want_stats=False)
        latn, l_mean, l_rstd = ops.layernorm_fwd(lat2d, nl_w, nl_b)                  # compact copy: A operand of to_q
        q = ops.gemm(latn, w16(wq))                                                  # [U*n, inner]
        kv = ops.gemm(kv_in, w16(wkv))                                               # [U*(v+n), 2*inner]
        kv3 = kv.view(U, v + n, 2 * inner)
        o, lse = ops.attn_fwd(q.view(U, n, inner), kv3[..., :inner], kv3[..., inner:], heads,
                              float((inner // heads) ** -0.5))
        lat1 = ops.gemm(o.view(U * n, inner), w16(wout), epi=L.EPI_GATE_RESID_F32, aux=lat2d)
        out, ff_saved = _ffn_forward(lat1, ff_ln_w, ff_ln_b, ff_w1, ff_w2, None)
        ctx.save_for_backward(x2d, lat2d, kv_in, xm_mean, xm_rstd, latn, l_mean, l_rstd, q, kv, o, lse, lat1,
                              *ff_saved[:5], nm_w, nl_w, wq, wkv, wout, ff_ln_w, ff_w1, ff_w2)
        ctx.meta = (U, v, n, Dv, inner, heads)
        ctx.params = (nm_w, nm_b, nl_w, nl_b, wq, wkv, wout, ff_ln_w, ff_ln_b, ff_w1, ff_w2)
        return out.view(U, n, Dv)

    @staticmethod
    def backward(ctx, dout):
        (x2d, lat2d, kv_in, xm_mean, xm_rstd, latn, l_mean, l_rstd, q, kv, o, lse, lat1, f_xn, f_mean, f_rstd, f_z,
         f_h, nm_w, nl_w, wq, wkv, wout, ff_ln_w, ff_w1, ff_w2) = ctx.saved_tensors
        U, v, n, Dv, inner, heads = ctx.meta
        needs = ctx.needs_input_grad
        names = ("nm_w", "nm_b", "nl_w", "nl_b", "wq", "wkv", "wout", "ff_ln_w", "ff_ln_b", "ff_w1", "ff_w2")
        sinks = {nm: _GradSink(p, needs[3 + i]) for i, (nm, p) in enumerate(zip(names, ctx.params))}
        sinks["gate"] = _GradSink(None, False)
        dout2d = dout.reshape(U * n, Dv)
        if not dout2d.is_contiguous():
            dout2d = dout2d.contiguous()
        if dout2d.dtype != f32:
            dout2d = dout2d.float()
        dlat1 = _ffn_backward(dout2d, lat1, (f_xn, f_mean, f_rstd, f_z, f_h, None), ff_ln_w, ff_w1, ff_w2, None,
                              {"ln_w": sinks["ff_ln_w"], "ln_b": sinks["ff_ln_b"], "w1": sinks["ff_w1"],
                               "w2": sinks["ff_w2"], "gate": sinks["gate"]})
        da = ops.gate_bwd(dlat1, None, None, None)                                   # bf16 cast of the residual-branch grad
        _wgrad(da, o.view(U * n, inner), sinks["wout"])
        d_o = ops.gemm(da, w16(wout), b_mn=True)
        del da
        kv3 = kv.view(U, v + n, 2 * inner)
        dkv = torch.empty_like(kv)
        dkv3 = dkv.view(U, v + n, 2 * inner)
        dq, _, _ = ops.attn_bwd(q.view(U, n, inner), kv3[..., :inner], kv3[..., inner:], o, d_o.view(U, n, inner), lse,
                                heads, float((inner // heads) ** -0.5), dk=dkv3[..., :inner], dv=dkv3[..., inner:])
        dq2 = dq.view(U * n, inner)
        _wgrad(dq2, latn, sinks["wq"])
        _wgrad(dkv, kv_in, sinks["wkv"])
        # d(kv_input): media rows feed only norm_media's affine grads (x itself is frozen), latent rows feed
        # norm_latents.
        dkv_in = ops.gemm(dkv, w16(wkv), b_mn=True)                                  # [U*(v+n), Dv] bf16
        dx_media = None
        if sinks["nm_w"].needs or sinks["nm_b"].needs or needs[0]:
            # needs[0]: the media tokens carry a gradient only when trainable frame / media-time embeddings were
            # added to them (helpers.py:118-125); the frozen ViT features themselves never do (flamingo.py:194).
            dx_media = ops.layernorm_bwd(dkv_in, x2d, nm_w, xm_mean, xm_rstd, dgamma=sinks["nm_w"].buffer(),
                                         dbeta=sinks["nm_b"].buffer(), want_dx=bool(needs[0]), rows_per_group=v,
                                         group_stride=v + n, group_offset=0)
        dlatn_q = ops.gemm(dq2, w16(wq), b_mn=True)                                  # [U*n, Dv] bf16
        dlat = ops.layernorm_bwd(dlatn_q, lat2d, nl_w, l_mean, l_rstd, dgamma=sinks["nl_w"].buffer(),
                                 dbeta=sinks["nl_b"].buffer(), dx_add=dlat1)
        dlat = ops.layernorm_bwd(dkv_in, lat2d, nl_w, l_mean, l_rstd, dgamma=sinks["nl_w"].buffer(),
                                 dbeta=sinks["nl_b"].buffer(), dx=dlat, dx_add=dlat, rows_per_group=n,
                                 group_stride=v + n, group_offset=v)
        grads = [sinks[nm].result() for nm in names]
        if block_backward_hook is not None:
            block_backward_hook(ctx.params)
        return (dx_media.view(U, v, Dv) if (needs[0] and dx_media is not None) else None,
                dlat.view(U, n, Dv) if needs[1] else None, None, *grads)


class FinalNormFn(torch.autograd.Function):
    """fp32 -> fp32 LayerNorm (PerceiverResampler.norm, helpers.py:132)."""

    @staticmethod
    def forward(ctx, x, w, b):
        shp = x.shape
        x2d = x.reshape(-1, shp[-1])
        if not x2d.is_contiguous():
            x2d = x2d.contiguous()
        y, mean, rstd = ops.layernorm_fwd(x2d, w, b, out_f32=True)
        ctx.save_for_backward(x2d, w, mean, rstd)
        ctx.params = (w, b)
        return y.view(shp)

    @staticmethod
    def backward(ctx, dy):
        x2d, w, mean, rstd = ctx.saved_tensors
        sw = _GradSink(ctx.params[0], ctx.needs_input_grad[1])
        sb = _GradSink(ctx.params[1], ctx.needs_input_grad[2])
        dy2d = dy.reshape(x2d.shape)
        if not dy2d.is_contiguous():
            dy2d = dy2d.contiguous()
        if dy2d.dtype != f32:
            dy2d = dy2d.float()
        dx = ops.layernorm_bwd(dy2d, x2d, w, mean, rstd, dgamma=sw.buffer(), dbeta=sb.buffer(),
                               want_dx=ctx.needs_input_grad[0])
        if block_backward_hook is not None:
            block_backward_hook(ctx.params)
        return (dx.view(dy.shape) if dx is not None else None), sw.result(), sb.result()


# ------------------------------------------------------------------------------------------ causal-LM loss
class CausalLMLossFn(torch.autograd.Function):
    """Shifted cross-entropy over [B, T, V] logits (HF ForCausalLMLoss semantics), fused fwd / bwd kernels."""

    @staticmethod
    def forward(ctx, logits, labels, ignore_index):
        B, T, V = logits.shape
        lg = logits.reshape(B * T, V)
        if lg.stride(1) != 1:
            lg = lg.contiguous()
        labels = labels.to(torch.int64).contiguous()
        lse = torch.empty(B * T, device=logits.device, dtype=f32)
        acc = torch.zeros(2, device=logits.device, dtype=f32)          # [loss_sum, count]
        L.check(L.lib().ofk_ce_fwd(lg.data_ptr(), int(lg.dtype == f32), lg.stride(0), B * T, V, labels.data_ptr(), T, 1,
                                   int(ignore_index), lse.data_ptr(), acc[0:1].data_ptr(), acc[1:2].data_ptr(),
                                   L.stream_ptr()))
        ctx.save_for_backward(lg, labels, lse, acc)
        ctx.meta = (B, T, V, int(ignore_index))
        return acc[0] / acc[1]     # mean over non-ignored targets (nan when there are none, like F.cross_entropy)

    @staticmethod
    def backward(ctx, g):
        lg, labels, lse, acc = ctx.saved_tensors
        B, T, V, ignore_index = ctx.meta
        d = torch.empty((B * T, V), device=lg.device, dtype=lg.dtype)
        gs = g.reshape(1).to(f32).contiguous()
        L.check(L.lib().ofk_ce_bwd(lg.data_ptr(), int(lg.dtype == f32), lg.stride(0), B * T, V, labels.data_ptr(), T, 1,
                                   ignore_index, lse.data_ptr(), gs.data_ptr(), acc[1:2].data_ptr(), d.data_ptr(),
                                   d.stride(0), L.stream_ptr()))
        return d.view(B, T, V), None, None


def causal_lm_loss(logits, labels, vocab_size=None, num_items_in_batch=None, ignore_index=-100, shift_labels=None,
                   **kwargs):
    """Drop-in for transformers' ForCausalLMLoss (`model.loss_function`).  Anything outside the plain training
    call (pre-shifted labels, num_items_in_batch, CPU tensors, exotic dtypes) defers to the HF implementation."""
    plain = (shift_labels is None and num_items_in_batch is None and logits.is_cuda and logits.dim() == 3 and
             logits.dtype in (bf16, f32) and labels.shape == logits.shape[:2])
    if not plain:
        from transformers.loss.loss_utils import ForCausalLMLoss
        return ForCausalLMLoss(logits, labels, vocab_size, num_items_in_batch=num_items_in_batch,
                               ignore_index=ignore_index, shift_labels=shift_labels, **kwargs)
    return CausalLMLossFn.apply(logits, labels.to(logits.device), ignore_index)


# ------------------------------------------------------------------------------------------ perceiver layer, folded
AUG = 16  # extra columns appended to the normalised media tokens: [1, 0, ..., 0] (column sums through the wgrad GEMM)


def normalise_media(x2d, eps=1e-5):
    """x_hat = (x - mean) / std as bf16 [rows, D + AUG] with column D == 1: computed ONCE per resampler forward --
    the media tokens are the same for all six layers (helpers.py:129-131 only updates the latents)."""
    rows, D = x2d.shape
    xa = torch.empty((rows, D + AUG), device=x2d.device, dtype=bf16)
    ones = torch.ones(D, device=x2d.device, dtype=f32)
    zeros = torch.zeros(D, device=x2d.device, dtype=f32)
    ops.layernorm_fwd(x2d, ones, zeros, eps, out=xa, want_stats=False)
    xa[:, D:] = 0
    xa[:, D] = 1
    return xa


class PerceiverFoldedLayerFn(torch.autograd.Function):
    """Same math as PerceiverLayerFn with norm_media folded into to_kv:
         to_kv(LN_media(x)) = x_hat (W_kv * gamma)^T + W_kv beta
    so a layer touches the media tokens with exactly one GEMM forward (no LayerNorm pass, no concat copy) and one
    wgrad GEMM backward (no media-row dgrad: x carries no gradient, flamingo.py:194), and the affine gradients
    are recovered from the [2*inner, D] wgrad:  dW_kv += dW_eff * gamma + colsum(dkv_media) beta^T,
    dgamma = sum_c dW_eff * W_kv,
    dbeta = W_kv^T colsum(dkv_media) (the column sums ride along as the extra ones-column of x_hat).
    Requires v % 64 == 0 (reduction k-blocks must not straddle images)."""

    @staticmethod
    def forward(ctx, xa, latents, heads, v, nm_w, nm_b, nl_w, nl_b, wq, wkv, wout, ff_ln_w, ff_ln_b, ff_w1, ff_w2):
        U, n, Dv = latents.shape
        inner = wq.shape[0]
        lat2d = latents.reshape(U * n, Dv)
        if not lat2d.is_contiguous():
            lat2d = lat2d.contiguous()
        latn, l_mean, l_rstd = ops.layernorm_fwd(lat2d, nl_w, nl_b)
        q = ops.gemm(latn, w16(wq))
        w_eff = (wkv.detach() * nm_w.detach().unsqueeze(0)).to(bf16)             # [2*inner, Dv]
        with torch.autocast("cuda", enabled=False):   # autocast would hand back a bf16 vector; the epilogue reads f32
            b_eff = torch.mv(wkv.detach(), nm_b.detach())                        # [2*inner] f32
        kv = torch.empty((U * (v + n), 2 * inner), device=latents.device, dtype=bf16)
        ops.gemm_grouped(xa[:, :Dv], w_eff, epi=L.EPI_BIAS_BF16, bias=b_eff, out=kv, M=U * v, N=2 * inner, K=Dv,
                         out_map=(v, v + n, 0))
        ops.gemm_grouped(latn, w16(wkv), epi=L.EPI_STORE_BF16, out=kv, M=U * n, N=2 * inner, K=Dv,
                         out_map=(n, v + n, v))
        kv3 = kv.view(U, v + n, 2 * inner)
        o, lse = ops.attn_fwd(q.view(U, n, inner), kv3[..., :inner], kv3[..., inner:], heads,
                              float((inner // heads) ** -0.5))
        lat1 = ops.gemm(o.view(U * n, inner), w16(wout), epi=L.EPI_GATE_RESID_F32, aux=lat2d)
        out, ff_saved = _ffn_forward(lat1, ff_ln_w, ff_ln_b, ff_w1, ff_w2, None)
        ctx.save_for_backward(xa, lat2d, latn, l_mean, l_rstd, q, kv, o, lse, lat1, *ff_saved[:5], nm_w, nl_w, wq, wkv,
                              wout, ff_ln_w, ff_w1, ff_w2)
        ctx.meta = (U, v, n, Dv, inner, heads)
        ctx.params = (nm_w, nm_b, nl_w, nl_b, wq, wkv, wout, ff_ln_w, ff_ln_b, ff_w1, ff_w2)
        return out.view(U, n, Dv)

    @staticmethod
    def backward(ctx, dout):
        (xa, lat2d, latn, l_mean, l_rstd, q, kv, o, lse, lat1, f_xn, f_mean, f_rstd, f_z, f_h, nm_w, nl_w, wq, wkv, wout,
         ff_ln_w, ff_w1, ff_w2) = ctx.saved_tensors
        U, v, n, Dv, inner, heads = ctx.meta
        needs = ctx.needs_input_grad
        names = ("nm_w", "nm_b", "nl_w", "nl_b", "wq", "wkv", "wout", "ff_ln_w", "ff_ln_b", "ff_w1", "ff_w2")
        sinks = {nm: _GradSink(p, needs[4 + i]) for i, (nm, p) in enumerate(zip(names, ctx.params))}
        sinks["gate"] = _GradSink(None, False)
        dout2d = dout.reshape(U * n, Dv)
        if not dout2d.is_contiguous():
            dout2d = dout2d.contiguous()
        if dout2d.dtype != f32:
            dout2d = dout2d.float()
        dlat1 = _ffn_backward(dout2d, lat1, (f_xn, f_mean, f_rstd, f_z, f_h, None), ff_ln_w, ff_w1, ff_w2, None,
                              {"ln_w": sinks["ff_ln_w"], "ln_b": sinks["ff_ln_b"], "w1": sinks["ff_w1"],
                               "w2": sinks["ff_w2"], "gate": sinks["gate"]})
        da = ops.gate_bwd(dlat1, None, None, None)
        _wgrad(da, o.view(U * n, inner), sinks["wout"])
        d_o = ops.gemm(da, w16(wout), b_mn=True)
        del da
        kv3 = kv.view(U, v + n, 2 * inner)
        dkv = torch.empty_like(kv)
        dkv3 = dkv.view(U, v + n, 2 * inner)
        dq, _, _ = ops.attn_bwd(q.view(U, n, inner), kv3[..., :inner], kv3[..., inner:], o, d_o.view(U, n, inner), lse,
                                heads, float((inner // heads) ** -0.5), dk=dkv3[..., :inner], dv=dkv3[..., inner:])
        dq2 = dq.view(U * n, inner)
        _wgrad(dq2, latn, sinks["wq"])
        # latent rows: ordinary wgrad / dgrad on a compact copy (U*n rows -- small)
        dkv_lat = dkv3[:, v:, :].reshape(U * n, 2 * inner)
        _wgrad(dkv_lat, latn, sinks["wkv"])
        # media rows: ONE wgrad over only the media rows of the concatenated gradient, against [x_hat | 1]
        if sinks["wkv"].needs or sinks["nm_w"].needs or sinks["nm_b"].needs:
            dweff = torch.zeros((2 * inner, Dv + AUG), device=kv.device, dtype=f32)
            ops.gemm_grouped(dkv, xa, a_mn=True, b_mn=True, epi=L.EPI_ATOMIC_F32, out=dweff, M=2 * inner, N=Dv + AUG,
                             K=U * v, ak_map=(v, v + n, 0))
            dw = dweff[:, :Dv]
            if sinks["wkv"].needs:   # d/dW[c, j] of sum_j W[c, j] (x_hat_j gamma_j + beta_j)
                sinks["wkv"].buffer().addcmul_(dw, nm_w.detach().unsqueeze(0))
                sinks["wkv"].buffer().addr_(dweff[:, Dv], ctx.params[1].detach())
            if sinks["nm_w"].needs:
                sinks["nm_w"].buffer().add_((dw * wkv.detach()).sum(0))
            if sinks["nm_b"].needs:
                with torch.autocast("cuda", enabled=False):
                    sinks["nm_b"].buffer().add_(torch.mv(wkv.detach().t(), dweff[:, Dv]))
        dlatn_q = ops.gemm(dq2, w16(wq), b_mn=True)
        dlat = ops.layernorm_bwd(dlatn_q, lat2d, nl_w, l_mean, l_rstd, dgamma=sinks["nl_w"].buffer(),
                                 dbeta=sinks["nl_b"].buffer(), dx_add=dlat1)
        dlatn_kv = ops.gemm(dkv_lat, w16(wkv), b_mn=True)
        dlat = ops.layernorm_bwd(dlatn_kv, lat2d, nl_w, l_mean, l_rstd, dgamma=sinks["nl_w"].buffer(),
                                 dbeta=sinks["nl_b"].buffer(), dx=dlat, dx_add=dlat)
        grads = [sinks[nm].result() for nm in names]
        if block_backward_hook is not None:
            block_backward_hook(ctx.params)
        return (None, dlat.view(U, n, Dv) if needs[1] else None, None, None, *grads)
