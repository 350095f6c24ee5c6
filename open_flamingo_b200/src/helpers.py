"""Drop-in replacements for the modules of the reference's open_flamingo/src/helpers.py, backed by the sm_90a
kernels in libofk.so.

Same class names, constructor signatures, parameter names/shapes (state-dict compatible with released
OpenFlamingo checkpoints, `load_state_dict(strict=False)`, README.md:125-126) and forward signatures as
  FeedForward (helpers.py:15-22), PerceiverAttention (:25-65), PerceiverResampler (:68-132),
  MaskedCrossAttention (:136-233), GatedCrossAttentionBlock (:236-279).
The nn.LayerNorm / nn.Linear children exist only to OWN the parameters under the reference's names; their own
forward() is never called -- all arithmetic runs in fused.* (CUDA only; there is no CPU fallback).
"""
import weakref

import torch
from torch import nn

from .. import _lib as L
from .. import fused, ops


def exists(val):
    return val is not None


def FeedForward(dim, mult=4):
    """Parameter container with the reference's Sequential layout: 0=LayerNorm, 1=Linear, 2=GELU, 3=Linear."""
    inner_dim = int(dim * mult)
    return nn.Sequential(
        nn.LayerNorm(dim),
        nn.Linear(dim, inner_dim, bias=False),
        nn.GELU(),
        nn.Linear(inner_dim, dim, bias=False),
    )


def _check_heads(dim_head, heads):
    if dim_head != 64:
        raise ValueError("the sm_90a attention kernels are specialised for dim_head=64 (the reference default)")
    if heads < 1:
        raise ValueError("heads must be >= 1")


class PerceiverAttention(nn.Module):
    """Parameter holder for one Perceiver attention (helpers.py:25-38); computed inside PerceiverResampler."""

    def __init__(self, *, dim, dim_head=64, heads=8):
        super().__init__()
        _check_heads(dim_head, heads)
        self.scale = dim_head ** -0.5
        self.heads = heads
        inner_dim = dim_head * heads
        self.norm_media = nn.LayerNorm(dim)
        self.norm_latents = nn.LayerNorm(dim)
        self.to_q = nn.Linear(dim, inner_dim, bias=False)
        self.to_kv = nn.Linear(dim, inner_dim * 2, bias=False)
        self.to_out = nn.Linear(inner_dim, dim, bias=False)

    def forward(self, x, latents):  # pragma: no cover - the fused layer owns the math
        raise RuntimeError("PerceiverAttention is evaluated by PerceiverResampler's fused layer kernel sequence")


class PerceiverResampler(nn.Module):
    def __init__(self, *, dim, depth=6, dim_head=64, heads=8, num_latents=64, max_num_media=None,
                 max_num_frames=None, ff_mult=4):
        super().__init__()
        _check_heads(dim_head, heads)
        if num_latents % 16 != 0:
            raise ValueError("num_latents must be a multiple of 16 (media-mask granularity of the xattn kernel)")
        self.latents = nn.Parameter(torch.randn(num_latents, dim))
        self.frame_embs = nn.Parameter(torch.randn(max_num_frames, dim)) if exists(max_num_frames) else None
        self.media_time_embs = nn.Parameter(torch.randn(max_num_media, 1, dim)) if exists(max_num_media) else None
        self.layers = nn.ModuleList([])
        for _ in range(depth):
            self.layers.append(nn.ModuleList([
                PerceiverAttention(dim=dim, dim_head=dim_head, heads=heads),
                FeedForward(dim=dim, mult=ff_mult),
            ]))
        self.norm = nn.LayerNorm(dim)

    def forward(self, x):
        """x: (b, T, F, v, D) -> (b, T, n, D)   (helpers.py:107-132)."""
        if x.dim() != 5:
            raise ValueError(f"PerceiverResampler expects (b, T, F, v, D), got {tuple(x.shape)}")
        L.require_cuda(x)
        b, T, F, v, D = x.shape
        x = x.float()
        if exists(self.frame_embs):  # helpers.py:118-120
            x = x + self.frame_embs[:F].view(1, 1, F, 1, D)
        x = x.reshape(b, T, F * v, D)
        if exists(self.media_time_embs):  # helpers.py:124-125
            x = x + self.media_time_embs[:T]
        U = b * T
        x3 = x.reshape(U, F * v, D).contiguous()
        n = self.latents.shape[0]
        latents = self.latents.unsqueeze(0).expand(U, n, D)  # broadcast view; grads reduce back over U
        vtok = F * v
        if vtok % 64 == 0 and D % 64 == 0 and not x3.requires_grad:
            # the media tokens never change across layers: normalise them once and fold each layer's norm_media
            # affine into its to_kv weights (fused.PerceiverFoldedLayerFn).  With trainable frame / media-time
            # embeddings (helpers.py:118-125) the media tokens DO need a gradient: the unfolded layer returns it.
            xa = fused.normalise_media(x3.view(U * vtok, D), self.layers[0][0].norm_media.eps)
            for attn, ff in self.layers:
                latents = fused.PerceiverFoldedLayerFn.apply(
                    xa, latents, attn.heads, vtok, attn.norm_media.weight, attn.norm_media.bias,
                    attn.norm_latents.weight, attn.norm_latents.bias, attn.to_q.weight, attn.to_kv.weight,
                    attn.to_out.weight, ff[0].weight, ff[0].bias, ff[1].weight, ff[3].weight)
        else:
            for attn, ff in self.layers:
                latents = fused.PerceiverLayerFn.apply(
                    x3, latents, attn.heads, attn.norm_media.weight, attn.norm_media.bias, attn.norm_latents.weight,
                    attn.norm_latents.bias, attn.to_q.weight, attn.to_kv.weight, attn.to_out.weight,
                    ff[0].weight, ff[0].bias, ff[1].weight, ff[3].weight)
        out = fused.FinalNormFn.apply(latents, self.norm.weight, self.norm.bias)
        return out.view(b, T, n, D)


class MaskedCrossAttention(nn.Module):
    """Parameter holder (helpers.py:136-158); evaluated inside GatedCrossAttentionBlock's fused sequence."""

    def __init__(self, *, dim, dim_visual, dim_head=64, heads=8, only_attend_immediate_media=True):
        super().__init__()
        _check_heads(dim_head, heads)
        self.scale = dim_head ** -0.5
        self.heads = heads
        inner_dim = dim_head * heads
        self.norm = nn.LayerNorm(dim)
        self.to_q = nn.Linear(dim, inner_dim, bias=False)
        self.to_kv = nn.Linear(dim_visual, inner_dim * 2, bias=False)
        self.to_out = nn.Linear(inner_dim, dim, bias=False)
        self.only_attend_immediate_media = only_attend_immediate_media

    def forward(self, x, media, media_locations=None, use_cached_media=False):  # pragma: no cover
        raise RuntimeError("MaskedCrossAttention is evaluated by GatedCrossAttentionBlock's fused kernel sequence")


class MediaContext:
    """Per-forward quantities shared by every gated block: the bf16 copy of the media latents and the
    text_time prefix sum (the reference recomputes both in each of its 24 layers, helpers.py:187-218)."""

    __slots__ = ("media_ref", "media_version", "loc_ref", "cached", "t_txt", "media16", "text_time", "kv")

    def matches(self, media, media_locations, use_cached_media, t_txt):
        if self.media_ref() is not media or self.media_version != media._version:
            return False
        if (self.loc_ref is None) != (media_locations is None):
            return False
        if self.loc_ref is not None and self.loc_ref() is not media_locations:
            return False
        return self.cached == bool(use_cached_media) and self.t_txt == t_txt


_shared_media_ctx = None  # one entry: all gated blocks of a forward pass see the same (media, media_locations) objects


def get_media_context(media, media_locations, use_cached_media, t_txt):
    """media: (B, T_img, n, Dv) fp32; media_locations: (B, T) bool or None."""
    global _shared_media_ctx
    ctx = _shared_media_ctx
    if ctx is not None and ctx.matches(media, media_locations, use_cached_media, t_txt):
        return ctx
    ctx = MediaContext()
    B, T_img, n, Dv = media.shape
    ctx.media_ref = weakref.ref(media)
    ctx.media_version = media._version
    ctx.loc_ref = None if media_locations is None else weakref.ref(media_locations)
    ctx.cached = bool(use_cached_media)
    ctx.t_txt = t_txt
    ctx.media16 = None
    ctx.text_time = None
    # per-layer media K/V for inference: survives across decode steps of one generate() call because the media
    # tensor object (and hence media16) is unchanged while only (media_locations, t_txt) vary
    prev = _shared_media_ctx
    same_media = prev is not None and prev.media_ref() is media and prev.media_version == media._version
    ctx.kv = prev.kv if same_media else {}
    if same_media:
        ctx.media16 = prev.media16
    if ctx.media16 is None:
        ctx.media16 = ops.cast_bf16(media.detach().reshape(B, T_img * n, Dv).float())
    if media_locations is not None:
        ctx.text_time = ops.text_time(media_locations=media_locations, use_cached_media=bool(use_cached_media),
                                      t_txt=t_txt)
    _shared_media_ctx = ctx
    return ctx


class GatedCrossAttentionBlock(nn.Module):
    def __init__(self, *, dim, dim_visual, dim_head=64, heads=8, ff_mult=4, only_attend_immediate_media=True):
        super().__init__()
        self.attn = MaskedCrossAttention(dim=dim, dim_visual=dim_visual, dim_head=dim_head, heads=heads,
                                         only_attend_immediate_media=only_attend_immediate_media)
        self.attn_gate = nn.Parameter(torch.tensor([0.0]))
        self.ff = FeedForward(dim, mult=ff_mult)
        self.ff_gate = nn.Parameter(torch.tensor([0.0]))

    def forward(self, x, media, media_locations=None, use_cached_media=False):
        """x: (B, T_txt, D); media: (B, T_img, n, Dv); media_locations: (B, T_txt) bool (helpers.py:260-279)."""
        L.require_cuda(x, media)
        if x.dim() != 3 or media.dim() != 4:
            raise ValueError("expected x (B, T_txt, D) and media (B, T_img, n, Dv)")
        if not use_cached_media:  # helpers.py:175-178 (the reference dereferences media_locations here)
            if not exists(media_locations):
                raise AttributeError("media_locations is required unless use_cached_media=True")
            assert media_locations.shape[1] == x.shape[1], (
                f"media_location.shape is {media_locations.shape} but x.shape is {x.shape}")
        B, T_txt, _ = x.shape
        _, T_img, n, Dv = media.shape
        ctx = get_media_context(media, media_locations, use_cached_media, T_txt)
        a = self.attn
        if not exists(media_locations):
            mask_mode = L.MASK_NONE  # helpers.py:196: no mask without media_locations
        else:
            mask_mode = L.MASK_MEDIA_EQ if a.only_attend_immediate_media else L.MASK_MEDIA_GE
        out_dtype = x.dtype
        out = fused.GatedXattnBlockFn.apply(
            x.float(), media.reshape(B, T_img * n, Dv).float(), ctx.media16, ctx.text_time, mask_mode, a.heads, n,
            a.norm.weight, a.norm.bias, a.to_q.weight, a.to_kv.weight, a.to_out.weight, self.attn_gate,
            self.ff[0].weight, self.ff[0].bias, self.ff[1].weight, self.ff[3].weight, self.ff_gate,
            None if torch.is_grad_enabled() else ctx.kv)
        return out if out_dtype == torch.float32 else out.to(out_dtype)
