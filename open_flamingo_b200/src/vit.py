"""CLIP ViT (ViT-L/14 et al.) forward pass on the sm_90a kernels -- the frozen vision encoder of Flamingo.

The reference takes this from open_clip (`open_clip.create_model_and_transforms`, factory.py:42-48; called at
flamingo.py:195 as `self.vision_encoder(x)[1]` under torch.no_grad).  open_clip is a third-party dependency
(`open_clip_torch>=2.16.0`, requirements.txt:6) that is neither vendored in the reference nor installed here, so
this restates its published VisionTransformer algorithm:
    conv1 (stride-P patch embed, no bias) -> [class_embedding ; patches] + positional_embedding -> ln_pre
    -> resblocks x L: x += out_proj(MHA(ln_1(x)));  x += c_proj(act(c_fc(ln_2(x))))   (act = QuickGELU for
       the OpenAI weights, exact GELU otherwise)
    -> with output_tokens=True returns (pooled, tokens): pooled = ln_post(x[:, 0]) @ proj, tokens = x[:, 1:]
       (patch tokens WITHOUT ln_post -- open_clip 2.16-2.20 behaviour, which is what Flamingo was trained with).
Parameter names follow open_clip's `visual.*` state dict so pretrained CLIP weights load unchanged.
Forward only (Flamingo never back-propagates into the ViT, flamingo.py:194).

Head width 64 (ViT-B, ViT-L) runs the media attention core on the in_proj output's q/k/v column blocks.  Other head
widths (ViT-H 80, ViT-g 88, ViT-bigG 104: any multiple of 8 in (64, 128]) have no core of their own: ops.rope_pack
copies each head into 128 zero-padded columns, the head_dim-128 dense core runs non-causal and unmasked on them, and
out_proj reads the padded output through fused.padded_w16 -- the path the GPT-NeoX blocks take at head_dim 80.
"""
import math

import torch
from torch import nn

from .. import _lib as L
from .. import ops
from ..fused import padded_w16, w16

bf16 = torch.bfloat16


class _Attn(nn.Module):
    def __init__(self, width):
        super().__init__()
        self.in_proj_weight = nn.Parameter(torch.empty(3 * width, width))
        self.in_proj_bias = nn.Parameter(torch.zeros(3 * width))
        self.out_proj = nn.Linear(width, width)


class _Mlp(nn.Module):
    def __init__(self, width, hidden):
        super().__init__()
        self.c_fc = nn.Linear(width, hidden)
        self.c_proj = nn.Linear(hidden, width)


class _ResBlock(nn.Module):
    def __init__(self, width, hidden):
        super().__init__()
        self.ln_1 = nn.LayerNorm(width)
        self.attn = _Attn(width)
        self.ln_2 = nn.LayerNorm(width)
        self.mlp = _Mlp(width, hidden)


class _Transformer(nn.Module):
    def __init__(self, width, layers, hidden):
        super().__init__()
        self.resblocks = nn.ModuleList([_ResBlock(width, hidden) for _ in range(layers)])


class VisionTransformer(nn.Module):
    """open_clip-compatible `visual` tower.  forward(images) -> (pooled, tokens) if output_tokens else pooled."""

    def __init__(self, image_size=224, patch_size=14, width=1024, layers=24, heads=16, mlp_ratio=4.0,
                 output_dim=768, quick_gelu=True, output_tokens=False):
        super().__init__()
        hd = width // heads if heads > 0 and width % heads == 0 else None
        if hd is None or not (hd == 64 or (64 < hd <= 128 and hd % 8 == 0)):
            raise ValueError(f"width {width} over {heads} heads: the sm_90a attention supports head widths 64 "
                             "(ViT-B, ViT-L) and multiples of 8 in (64, 128] on zero-padded heads (ViT-H 80, ViT-g 88, "
                             "ViT-bigG 104)")
        self.image_size, self.patch_size, self.width, self.heads = image_size, patch_size, width, heads
        self.grid = image_size // patch_size
        self.output_dim = output_dim
        self.quick_gelu = quick_gelu
        self.output_tokens = output_tokens
        scale = width ** -0.5
        self.conv1 = nn.Conv2d(3, width, kernel_size=patch_size, stride=patch_size, bias=False)
        self.class_embedding = nn.Parameter(scale * torch.randn(width))
        self.positional_embedding = nn.Parameter(scale * torch.randn(self.grid ** 2 + 1, width))
        self.ln_pre = nn.LayerNorm(width)
        self.transformer = _Transformer(width, layers, int(width * mlp_ratio))
        self.ln_post = nn.LayerNorm(width)
        self.proj = nn.Parameter(scale * torch.randn(width, output_dim))
        for blk in self.transformer.resblocks:
            nn.init.normal_(blk.attn.in_proj_weight, std=scale)
        self._pe_w16 = None

    def _patch_weight(self):
        """conv1.weight [width, 3, P, P] -> bf16 [width, Kp] with K = 3*P*P zero-padded to a multiple of 64."""
        w = self.conv1.weight
        k = w[0].numel()
        kp = ((k + 63) // 64) * 64
        c = self._pe_w16
        if c is None or c[0] != w._version or c[1].device != w.device:
            buf = torch.zeros((w.shape[0], kp), device=w.device, dtype=bf16)
            buf[:, :k] = w.detach().reshape(w.shape[0], k).to(bf16)
            self._pe_w16 = (w._version, buf)
            c = self._pe_w16
        return c[1], kp

    @torch.no_grad()
    def forward(self, x):
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError(f"expected images (N, 3, H, W), got {tuple(x.shape)}")
        L.require_cuda(x)
        N, _, H, W = x.shape
        P, D = self.patch_size, self.width
        if H % P or W % P or (H // P) * (W // P) + 1 != self.positional_embedding.shape[0]:
            raise ValueError("image size does not match the positional embedding")
        g = (H // P) * (W // P)
        S = g + 1
        wpe, kp = self._patch_weight()
        patches = ops.patchify(x.float(), P, kp)                                    # [N*g, kp] bf16
        pe = ops.gemm(patches, wpe)                                                 # [N*g, D] bf16
        tok = ops.vit_assemble(pe, self.class_embedding, self.positional_embedding, N, g, D)   # fp32 [N*S, D]
        xs, _, _ = ops.layernorm_fwd(tok, self.ln_pre.weight, self.ln_pre.bias, out_f32=True, want_stats=False)
        act = L.EPI_BIAS_QGELU_BF16 if self.quick_gelu else L.EPI_BIAS_GELU_BF16
        heads = self.heads
        hd = D // heads
        scale = 1.0 / math.sqrt(hd)
        for blk in self.transformer.resblocks:
            h, _, _ = ops.layernorm_fwd(xs, blk.ln_1.weight, blk.ln_1.bias, want_stats=False)
            qkv = ops.gemm(h, w16(blk.attn.in_proj_weight), epi=L.EPI_BIAS_BF16, bias=blk.attn.in_proj_bias)
            qkv3 = qkv.view(N, S, 3 * D)
            if hd == 64:
                o, _ = ops.attn_fwd(qkv3[..., :D], qkv3[..., D:2 * D], qkv3[..., 2 * D:], heads, scale,
                                    want_lse=False)
                wo = w16(blk.attn.out_proj.weight)
            else:
                # no core at this head_dim: every head zero-padded to 128 columns runs the head_dim-128 dense core,
                # whose zero columns add exact zeros, and out_proj reads the padded output through zero weight columns
                q, k, v = ops.rope_pack(qkv3, heads, hd, q_width=128, kv_width=128, blocks=True)
                o, _ = ops.attn_dense_fwd(q, k, v, heads, 128, scale, causal=False, mask=None, want_lse=False)
                wo = padded_w16(blk.attn.out_proj.weight, heads, hd, 128)
            ops.gemm(o.view(N * S, o.shape[-1]), wo, epi=L.EPI_BIAS_RESID_F32,
                     bias=blk.attn.out_proj.bias, aux=xs, out=xs)                   # x += out_proj(attn)  (in place)
            h, _, _ = ops.layernorm_fwd(xs, blk.ln_2.weight, blk.ln_2.bias, want_stats=False)
            f = ops.gemm(h, w16(blk.mlp.c_fc.weight), epi=act, bias=blk.mlp.c_fc.bias)
            ops.gemm(f, w16(blk.mlp.c_proj.weight), epi=L.EPI_BIAS_RESID_F32, bias=blk.mlp.c_proj.bias, aux=xs, out=xs)
        x3 = xs.view(N, S, D)
        tokens = x3[:, 1:]
        cls = torch.nn.functional.layer_norm(x3[:, 0], (D,), self.ln_post.weight, self.ln_post.bias)
        pooled = cls @ self.proj
        return (pooled, tokens) if self.output_tokens else pooled


class CLIPVisionStandIn(nn.Module):
    """Minimal stand-in for the open_clip CLIP object: Flamingo only ever touches `.visual` (flamingo.py:47)."""

    def __init__(self, visual):
        super().__init__()
        self.visual = visual
