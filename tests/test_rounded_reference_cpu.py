"""CPU: pins tests/rounded_reference.py, the rounding-faithful float64 restatement the fused-block contract tests
compare the kernels with.  With rounding off, every restated block equals the oracle (and HF MptBlock) in float64 to
1e-12 of each tensor's largest value, forward and every gradient; the rounding operators and the tiled P rounding of
the media attention do what the module docstring says."""
import math
from unittest import mock

import pytest
import torch

import rounded_reference as RR
from oracle import flamingo_oracle as O

f64 = torch.float64
TOL = 1e-12


def close(got, ref, what):
    scale = ref.abs().max().item()
    err = (got - ref).abs().max().item()
    assert err <= TOL * max(scale, 1e-300), f"{what}: max |err| {err:.3e} against max |ref| {scale:.3e}"


def params_like(shapes, seed):
    """float64 parameters with every LayerNorm weight / bias and gate drawn at random (none at its init value)."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shp in shapes.items():
        t = torch.randn(shp, generator=g, dtype=f64)
        if k.endswith("_gate"):
            t = 0.5 * t
        elif len(shp) == 2:
            t = t * shp[1] ** -0.5
        elif "norm" in k or k.startswith("ff.0") or ".1.0." in k:
            t = (1.0 + 0.3 * t) if k.endswith("weight") else 0.3 * t
        sd[k] = t
    return sd


def grads_of(fn, sd, inputs, seed):
    sd = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    ins = [t.clone().requires_grad_(True) for t in inputs]
    y = fn(sd, *ins)
    w = torch.randn(y.shape, generator=torch.Generator().manual_seed(seed), dtype=f64)
    (y * w).sum().backward()
    return y.detach(), {k: v.grad for k, v in sd.items()}, [t.grad for t in ins]


def compare(fn_a, fn_b, sd, inputs, what):
    ya, ga, ia = grads_of(fn_a, sd, inputs, 7)
    yb, gb, ib = grads_of(fn_b, sd, inputs, 7)
    close(ya, yb, f"{what} output")
    for k in sd:
        assert (ga[k] is None) == (gb[k] is None), f"{what} d{k}: gradient present on one side only"
        if ga[k] is not None:
            close(ga[k], gb[k], f"{what} d{k}")
    for i, (a, b) in enumerate(zip(ia, ib)):
        close(a, b, f"{what} d(input {i})")


# ------------------------------------------------------------------ the rounding operators
def test_rounding_operators():
    x = torch.tensor([1.0 + 2.0 ** -9, 1.0 + 3 * 2.0 ** -9, 1.0 / 3.0, -2.5e-40, 70000.0], dtype=f64,
                     requires_grad=True)
    g = torch.tensor([1.0 + 2.0 ** -9, -1.0 / 3.0, 3.0, 1.0 + 2.0 ** -7, 1e-3], dtype=f64)
    want = x.detach().to(torch.bfloat16).to(f64)
    assert want[0] == 1.0 and want[1] == 1.0 + 2.0 ** -7          # ties round to even
    for op, rounds_value, rounds_grad in ((RR.rf, True, False), (RR.rb, True, True), (RR.gb, False, True)):
        x.grad = None
        y = op(x)
        assert torch.equal(y.detach(), want if rounds_value else x.detach())
        y.backward(g)
        assert torch.equal(x.grad, g.to(torch.bfloat16).to(f64) if rounds_grad else g)
    r = RR.Rounder(False)
    assert r.rf(x) is x and r.rb(x) is x and r.gb(x) is x


def test_tiled_p_rounding_matches_an_online_softmax_loop():
    """The media forward's P rounding restated as the kernel's loop: per 64-key tile, the running max is updated,
    exp(s - m) is rounded to bf16 for P.V and l and the accumulator are rescaled."""
    g = torch.Generator().manual_seed(3)
    B, H, hd, nq, nk = 1, 2, 8, 5, 150
    q, k, v = (torch.randn(B, n, H * hd, generator=g, dtype=f64) for n in (nq, nk, nk))
    k[:, 100:] *= 3.0                        # later tiles raise the running max
    allowed = torch.rand(B, nq, nk, generator=g) > 0.3
    allowed[0, 1, :70] = False               # a row whose first tile is fully masked
    got = RR.attention(q, k, v, H, 0.5, RR.Rounder(True), allowed=allowed)
    Q, K, V = (O._split_heads(t, H) for t in (q, k, v))
    want = torch.zeros(B, H, nq, hd, dtype=f64)
    for h in range(H):
        for i in range(nq):
            m, l, acc = -math.inf, 0.0, torch.zeros(hd, dtype=f64)
            for t0 in range(0, nk, RR.BKV):
                s = 0.5 * (K[0, h, t0:t0 + RR.BKV] @ Q[0, h, i])
                s = torch.where(allowed[0, i, t0:t0 + RR.BKV], s, torch.full_like(s, -math.inf))
                mn = max(m, s.max().item())
                if mn == -math.inf:
                    continue
                corr = math.exp(m - mn) if m != -math.inf else 0.0
                p = torch.exp(s - mn)
                l = l * corr + p.sum().item()
                acc = acc * corr + RR.to_bf16(p) @ V[0, h, t0:t0 + RR.BKV]
                m = mn
            want[0, h, i] = acc / l
    close(got, O._merge_heads(want), "tiled P rounding")
    unrounded = RR.attention(q, k, v, H, 0.5, RR.Rounder(False), allowed=allowed)
    assert (got - unrounded).abs().max() > 1e-4, "the rounding of P must be visible"


# ------------------------------------------------------------------ gated cross-attention block
XATTN_SHAPES = {"attn.norm.weight": (48,), "attn.norm.bias": (48,), "attn.to_q.weight": (32, 48),
                "attn.to_kv.weight": (64, 40), "attn.to_out.weight": (48, 32), "attn_gate": (1,),
                "ff.0.weight": (48,), "ff.0.bias": (48,), "ff.1.weight": (192, 48), "ff.3.weight": (48, 192),
                "ff_gate": (1,)}


def xattn_locations(B, T, pattern):
    loc = torch.zeros(B, T, dtype=torch.bool)
    if pattern == "late":              # rows before the first <image>, then steps
        loc[0, [3, 7]] = True
        loc[1, [5]] = True
    elif pattern == "surplus":         # more <image> tokens than media: rows with no allowed key
        loc[0, [0, 2, 4, 6]] = True
        loc[1, [1]] = True
    return loc


@pytest.mark.parametrize("immediate", [True, False])
@pytest.mark.parametrize("cached,pattern", [(False, "late"), (False, "surplus"), (True, "late"), (True, "surplus"),
                                            (True, "none")])
def test_gated_block_unrounded_equals_oracle(immediate, cached, pattern):
    B, T, T_img, n = 2, 9, 2, 3
    loc = None if pattern == "none" else xattn_locations(B, T, pattern)
    sd = params_like(XATTN_SHAPES, 11)
    g = torch.Generator().manual_seed(12)
    x = torch.randn(B, T, 48, generator=g, dtype=f64)
    media = torch.randn(B, T_img, n, 40, generator=g, dtype=f64)
    compare(lambda s, xx, mm: RR.gated_cross_attention_block(xx, mm, s, "", loc, cached, 2, immediate, rounding=False),
            lambda s, xx, mm: O.gated_cross_attention_block(xx, mm, s, "", loc, cached, 2, immediate),
            sd, [x, media], f"gated block [{pattern}, cached={cached}, immediate={immediate}]")


def test_gated_block_rounding_moves_every_gradient():
    """With rounding on, the output and every gradient move (by about the bf16 rounding), so none of the rounding
    points is dead code."""
    B, T, T_img, n = 2, 9, 2, 3
    loc = xattn_locations(B, T, "late")
    sd = params_like(XATTN_SHAPES, 11)
    g = torch.Generator().manual_seed(12)
    x = torch.randn(B, T, 48, generator=g, dtype=f64)
    media = torch.randn(B, T_img, n, 40, generator=g, dtype=f64)
    ya, ga, ia = grads_of(lambda s, xx, mm: RR.gated_cross_attention_block(xx, mm, s, "", loc, False, 2), sd,
                          [x, media], 7)
    yb, gb_, ib = grads_of(lambda s, xx, mm: RR.gated_cross_attention_block(xx, mm, s, "", loc, False, 2,
                                                                            rounding=False), sd, [x, media], 7)
    for what, a, b in [("y", ya, yb)] + [(k, ga[k], gb_[k]) for k in sd] + [("dx", ia[0], ib[0]),
                                                                           ("dmedia", ia[1], ib[1])]:
        rel = ((a - b).norm() / b.norm()).item()
        top = math.inf if what.endswith("_gate") else 5e-2      # the gate gradients cancel (DESIGN §2)
        assert 1e-5 < rel < top, f"{what}: rounding moved it by {rel:.2e} of its norm"


# ------------------------------------------------------------------ Perceiver
def perceiver_shapes(D, inner, depth, n, embs):
    s = {"latents": (n, D), "norm.weight": (D,), "norm.bias": (D,)}
    if embs:
        s["frame_embs"] = (2, D)
        s["media_time_embs"] = (3, 1, D)
    for i in range(depth):
        p = f"layers.{i}"
        s.update({f"{p}.0.norm_media.weight": (D,), f"{p}.0.norm_media.bias": (D,),
                  f"{p}.0.norm_latents.weight": (D,), f"{p}.0.norm_latents.bias": (D,),
                  f"{p}.0.to_q.weight": (inner, D), f"{p}.0.to_kv.weight": (2 * inner, D),
                  f"{p}.0.to_out.weight": (D, inner), f"{p}.1.0.weight": (D,), f"{p}.1.0.bias": (D,),
                  f"{p}.1.1.weight": (4 * D, D), f"{p}.1.3.weight": (D, 4 * D)})
    return s


@pytest.mark.parametrize("folded,embs", [(False, False), (False, True), (True, False)])
def test_perceiver_unrounded_equals_oracle(folded, embs):
    D, inner, depth, n = 32, 16, 2, 4
    sd = params_like(perceiver_shapes(D, inner, depth, n, embs), 21)
    sd["latents"] = torch.randn(n, D, generator=torch.Generator().manual_seed(22), dtype=f64)
    x = 1.5 * torch.randn(2, 2, 2, 5, D, generator=torch.Generator().manual_seed(23), dtype=f64) + 0.3
    compare(lambda s, xx: RR.perceiver_resampler(xx, s, heads=2, folded=folded, rounding=False),
            lambda s, xx: O.perceiver_resampler(xx, s, heads=2), sd, [x], f"perceiver [folded={folded}, embs={embs}]")


# ------------------------------------------------------------------ MPT block
def hf_block(D, heads, seed):
    from transformers import MptConfig
    from transformers.models.mpt.modeling_mpt import MptBlock, build_mpt_alibi_tensor
    cfg = MptConfig(d_model=D, n_heads=heads, n_layers=1, vocab_size=32, max_seq_len=64, expansion_ratio=4)
    blk = MptBlock(cfg, 0).to(f64).eval().requires_grad_(False)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for _, p in blk.named_parameters():
            if p.dim() == 1:
                p.copy_(1.0 + 0.3 * torch.randn(p.shape, generator=g, dtype=f64))
            else:
                p.copy_(torch.randn(p.shape, generator=g, dtype=f64) * p.shape[1] ** -0.5)
    alibi = build_mpt_alibi_tensor(heads, cfg.max_seq_len).to(f64)
    return blk, alibi


def mpt_weights(blk):
    return {"norm_1": blk.norm_1.weight, "Wqkv": blk.attn.Wqkv.weight, "out_proj": blk.attn.out_proj.weight,
            "norm_2": blk.norm_2.weight, "up_proj": blk.ffn.up_proj.weight, "down_proj": blk.ffn.down_proj.weight}


@pytest.mark.parametrize("kind", ["none", "causal", "right_pad", "left_pad"])
def test_mpt_block_unrounded_equals_hf(kind):
    D, heads, B, T = 32, 2, 2, 11
    blk, alibi = hf_block(D, heads, 5)
    causal = torch.ones(T, T, dtype=torch.bool).triu(1)
    att = torch.ones(B, T, dtype=torch.bool)
    if kind == "right_pad":
        att[0, T - 4:] = False
    elif kind == "left_pad":
        att[1, :3] = False                  # rows 0-2 of batch 1 see no key at all: uniform rows
    mask = causal.expand(B, T, T) | ~att[:, None, :]
    slopes = (alibi[:, 0, -1] - alibi[:, 0, -2])
    x = torch.randn(B, T, D, generator=torch.Generator().manual_seed(6), dtype=f64)
    w = torch.randn(B, T, D, generator=torch.Generator().manual_seed(7), dtype=f64)
    xr = x.clone().requires_grad_(True)
    # HF takes the softmax of `scores.float()`: keep it in float64 for the comparison
    with mock.patch.object(torch.Tensor, "float", lambda self: self):
        ref, _ = blk(xr, position_bias=alibi, attention_mask=None if kind == "none" else mask[:, None])
    (ref * w).sum().backward()
    xo = x.clone().requires_grad_(True)
    got = RR.mpt_block(xo, mpt_weights(blk), heads, slopes, None if kind == "none" else mask, blk.norm_1.eps,
                       rounding=False)
    (got * w).sum().backward()
    if kind == "none":   # HF without a mask attends to every key; the restatement's None means causal
        got2 = RR.mpt_block(x, mpt_weights(blk), heads, slopes, causal.expand(B, T, T), blk.norm_1.eps, rounding=False)
        close(got.detach(), got2, "mask None == causal mask")
        return
    close(got.detach(), ref.detach(), f"mpt [{kind}] output")
    close(xo.grad, xr.grad, f"mpt [{kind}] dx")
