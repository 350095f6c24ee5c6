"""GPU: decoding with a KV cache on the kernels.

- ofk_attn_decode (ops.attn_decode) against float64 on the same bf16 inputs, at tile and split edges, with ALiBi and
  padding masks, reading q and K/V as strided views whose neighbours are NaN; bitwise reproducibility.
- The cached fast path of the frozen MPT block (prefill, a 3-token chunk, then single tokens) against the uncached
  kernel path and against HF in fp32 / under autocast.
- Flamingo.generate and the cached-prefix forward under autocast(bf16): the new path runs, HF's MptAttention does not,
  and the results hold against the reference's own numerics.

Rule for bf16 paths (DESIGN section 2): err(ours, fp32) <= 2 * err(HF under autocast, fp32) per step, plus a floor for
steps where autocast happens to be nearly exact."""
import contextlib

import pytest
import torch

pytestmark = pytest.mark.gpu
OUT_TOL = 2e-2
bf16 = torch.bfloat16


# --------------------------------------------------------------------------------------------- kernel contract
def _case(B, H, hd, nk, slopes_on, mask_kind, cap, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    D = H * hd
    qkv = torch.full((B, 3 * D), float("nan"), device="cuda", dtype=bf16)
    qkv[:, :D] = torch.randn(B, D, device="cuda", generator=g).to(bf16)
    k = torch.randn(B, nk, D, device="cuda", generator=g).to(bf16)
    v = torch.randn(B, nk, D, device="cuda", generator=g).to(bf16)
    slopes = (torch.rand(H, device="cuda", generator=g) * 0.5) if slopes_on else None
    mask = None
    if mask_kind != "none":
        nk8 = -(-nk // 8) * 8
        mask = torch.randint(0, 2, (B, nk8), device="cuda", generator=g, dtype=torch.uint8)   # junk past nk
        pad = torch.randint(0, nk, (B,), device="cuda", generator=g)
        mask[:, :nk] = (torch.arange(nk, device="cuda")[None] < pad[:, None]).to(torch.uint8)
        if mask_kind == "full":
            mask[0, :nk] = 1
    return qkv, k, v, slopes, mask


def _in_cache(k, v, cap):
    """K/V copied into a NaN-filled cache of `cap` rows with NaN columns around each slice; returns the views."""
    B, nk, D = k.shape
    buf = torch.full((B, cap, 2 * D + 24), float("nan"), device="cuda", dtype=bf16)
    buf[:, :nk, 8:8 + D] = k
    buf[:, :nk, D + 16:2 * D + 16] = v
    return buf[:, :nk, 8:8 + D], buf[:, :nk, D + 16:2 * D + 16]


def _reference(q, k, v, H, hd, scale, slopes, mask):
    B, nk, D = k.shape
    qd = q.double().view(B, H, hd)
    kd, vd = k.double().view(B, nk, H, hd), v.double().view(B, nk, H, hd)
    s = torch.einsum("bhd,bkhd->bhk", qd, kd) * scale
    if slopes is not None:
        s = s + slopes.double().view(1, H, 1) * torch.arange(nk, device="cuda", dtype=torch.float64).view(1, 1, nk)
    if mask is not None:
        s = s.masked_fill(mask[:, None, :nk].bool(), torch.finfo(torch.float64).min)
    p = torch.softmax(s, -1)
    return torch.einsum("bhk,bkhd->bhd", p, vd)


def _check_rows(got, ref, what):
    got = got.double().view_as(ref)
    err = (got - ref).abs().amax(-1)
    bound = ref.abs().amax(-1) * 2.0 ** -8 + 1e-6
    bad = err > bound
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    assert not bad.any(), f"{what}: {int(bad.sum())} rows over bound, worst err {err.max().item():.3e}"


@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("B,H", [(1, 2), (1, 16), (3, 32), (24, 16)])
@pytest.mark.parametrize("nk", [1, 63, 64, 65, 300, 2049, 4097])
def test_decode_kernel_contract(hd, B, H, nk):
    from open_flamingo_b200 import ops
    scale = hd ** -0.5
    for i, (slopes_on, mask_kind) in enumerate([(False, "none"), (True, "none"), (True, "pad"), (False, "pad"),
                                                (True, "full")]):
        qkv, k, v, slopes, mask = _case(B, H, hd, nk, slopes_on, mask_kind, nk + 40, 100 * nk + 7 * i + B)
        q = qkv[:, :hd * H]
        kc, vc = _in_cache(k, v, nk + 40)
        what = f"B{B} H{H} hd{hd} nk{nk} slopes={slopes_on} mask={mask_kind}"
        o = ops.attn_decode(q, kc, vc, H, hd, scale, key_mask=mask, slopes=slopes)
        ref = _reference(q, k, v, H, hd, scale, slopes, mask)
        _check_rows(o, ref, what)
        dm = None if mask is None else mask[:, :nk].reshape(B, 1, nk).contiguous()
        od, _ = ops.attn_dense_fwd(qkv.view(B, 1, 3 * H * hd)[..., :H * hd], kc, vc, H, hd, scale, mask=dm,
                                   slopes=slopes, want_lse=False)
        _check_rows(od.view(B, -1), ref, what + " (dense kernel)")
        # each is within one bf16 rounding of the exact value, so the two may differ by twice that
        err = (o.double() - od.view(B, -1).double()).view_as(ref).abs().amax(-1)
        assert (err <= 2 * (ref.abs().amax(-1) * 2.0 ** -8 + 1e-6)).all(), f"{what}: decode vs dense"
        # bitwise: repeated launches and a cache of another capacity
        assert torch.equal(o, ops.attn_decode(q, kc, vc, H, hd, scale, key_mask=mask, slopes=slopes)), what
        kc2, vc2 = _in_cache(k, v, 2 * nk + 123)
        assert torch.equal(o, ops.attn_decode(q, kc2, vc2, H, hd, scale, key_mask=mask, slopes=slopes)), what


def test_decode_rejects_bad_views():
    from open_flamingo_b200 import ops
    q = torch.randn(2, 256, device="cuda").to(bf16)
    k = torch.randn(2, 10, 256, device="cuda").to(bf16)
    with pytest.raises(ValueError):
        ops.attn_decode(q, k, k.float(), 2, 128, 0.1)
    with pytest.raises(ValueError):
        ops.attn_decode(q, k, k.clone()[:, :, :128], 2, 128, 0.1)
    with pytest.raises(ValueError):
        ops.attn_decode(q, k, torch.randn(2, 10, 512, device="cuda").to(bf16)[..., :256], 2, 128, 0.1)  # strides differ


# --------------------------------------------------------------------------------------------- block level
def _make_lm(d_model, n_heads, seed, n_layers=2, vocab=64):
    from transformers import MptConfig, MptForCausalLM
    from open_flamingo_b200 import lm_blocks
    torch.manual_seed(seed)
    cfg = MptConfig(d_model=d_model, n_heads=n_heads, n_layers=n_layers, vocab_size=vocab, max_seq_len=256,
                    expansion_ratio=4)
    lm = MptForCausalLM(cfg).cuda().eval().requires_grad_(False)
    with torch.no_grad():
        for p in lm.parameters():
            if p.dim() == 1:
                p.copy_(1.0 + 0.1 * torch.randn_like(p))
            else:
                p.copy_(torch.randn_like(p) * p.shape[1] ** -0.5)
    for blk in lm.transformer.blocks:   # route every block through the fast path, as FlamingoLayer does
        fast, orig = lm_blocks.accelerate(blk), blk.forward

        def fwd(hidden_states, *a, _fast=fast, _orig=orig, **kw):
            r = _fast(hidden_states, *a, **kw)
            return r if r is not None else _orig(hidden_states, *a, **kw)
        blk.forward = fwd
    return lm


@contextlib.contextmanager
def _fast_lm(on):
    from open_flamingo_b200 import lm_blocks
    prev = lm_blocks.ENABLED
    lm_blocks.ENABLED = on
    try:
        yield
    finally:
        lm_blocks.ENABLED = prev


@contextlib.contextmanager
def _count_calls():
    """Counts ops.attn_decode calls and HF MptAttention.forward calls."""
    from transformers.models.mpt import modeling_mpt
    from open_flamingo_b200 import ops
    n = {"decode": 0, "hf_attn": 0}
    dec, hf = ops.attn_decode, modeling_mpt.MptAttention.forward

    def dec_w(*a, **k):
        n["decode"] += 1
        return dec(*a, **k)

    def hf_w(self, *a, **k):
        n["hf_attn"] += 1
        return hf(self, *a, **k)
    ops.attn_decode, modeling_mpt.MptAttention.forward = dec_w, hf_w
    try:
        yield n
    finally:
        ops.attn_decode, modeling_mpt.MptAttention.forward = dec, hf


def _incremental(lm, ids, att, cache, steps):
    """Feed `steps` (list of widths) of ids through the LM with `cache`; returns the logits of each chunk."""
    out, pos = [], 0
    for w in steps:
        o = lm(input_ids=ids[:, pos:pos + w], attention_mask=att[:, :pos + w], past_key_values=cache,
               use_cache=True).logits
        out.append(o.float())
        pos += w
    return out


def _err(a, b, valid):
    return ((a - b).abs() * valid).max().item()


@pytest.mark.parametrize("d_model,n_heads", [(2048, 16), (4096, 32), (256, 4)])
def test_cached_block_path_matches_uncached_and_hf(d_model, n_heads):
    from transformers import DynamicCache
    from open_flamingo_b200.kv_cache import KVCache
    lm = _make_lm(d_model, n_heads, 11)
    B, T = 3, 40
    steps = [T, 3] + [1] * 8
    n = sum(steps)
    g = torch.Generator().manual_seed(12)
    ids = torch.randint(0, 64, (B, n), generator=g).cuda()
    att = torch.ones(B, n, dtype=torch.long, device="cuda")
    att[1, :5] = 0
    att[2, :11] = 0
    with torch.inference_mode():
        with _fast_lm(False):
            ref = lm(input_ids=ids, attention_mask=att).logits.float()                # HF fp32, full sequence
        with torch.autocast("cuda", dtype=bf16):
            with _fast_lm(True):
                full = lm(input_ids=ids, attention_mask=att).logits.float()           # uncached kernel path
                with _count_calls() as calls:
                    ours = _incremental(lm, ids, att, KVCache(2), steps)
            with _fast_lm(False):
                amp = _incremental(lm, ids, att, DynamicCache(), steps)
    assert calls["hf_attn"] == 0 and calls["decode"] == 2 * 8, calls
    scale = ref.abs().max().item()
    pos = 0
    for i, w in enumerate(steps):
        sl = slice(pos, pos + w)
        valid = att[:, sl, None].float()                # padded query rows attend uniformly in every arm; skip them
        e_full = _err(ours[i], full[:, sl], valid)
        assert e_full <= OUT_TOL * scale, f"step {i}: cached vs uncached kernel path {e_full:.3e} (max {scale:.3e})"
        e_ours, e_amp = _err(ours[i], ref[:, sl], valid), _err(amp[i], ref[:, sl], valid)
        assert e_ours <= 2 * e_amp + 5e-3 * scale, f"step {i}: err vs fp32 {e_ours:.3e}, amp {e_amp:.3e}"
        pos += w


# --------------------------------------------------------------------------------------------- model level
VIT = dict(image_size=56, patch_size=14, width=128, layers=2, heads=2, output_dim=128)
MPT = dict(d_model=256, n_heads=2, n_layers=4, vocab_size=97, max_seq_len=256, expansion_ratio=4)


def _model(every):
    from open_flamingo_b200.testing import build_flamingo
    model, _, tok = build_flamingo(VIT, MPT, cross_attn_every_n_layers=every, device="cuda", gate_init=1.0, seed=21)
    with torch.no_grad():
        # HF's near-zero init leaves every token almost tied.  Unit-variance (tied) embeddings make the logits decisive:
        # the residual stream keeps the current token's embedding, whose self-product (~d_model) leads the others by
        # far more than any bf16 error, so greedy and best-beam tokens are stable while every block still contributes.
        for name, p in model.lang_encoder.named_parameters():
            if "gated_cross_attn" in name or not name.startswith("transformer") or p.dim() != 2:
                continue
            p.copy_(torch.randn_like(p) * p.shape[1] ** -0.5)
        model.lang_encoder.get_input_embeddings().weight.normal_()
    media = tok.encode("<image>")[-1]
    g = torch.Generator().manual_seed(22)
    vision_x = torch.randn(3, 1, 1, 3, 56, 56, generator=g).cuda()
    lang_x = torch.randint(0, 90, (3, 24), generator=g)
    att = torch.ones_like(lang_x)
    att[0, :6] = 0
    att[2, :3] = 0
    lang_x = lang_x.masked_fill(att == 0, 0)
    for b, first in enumerate((6, 0, 3)):
        lang_x[b, first] = media
    return model, vision_x, lang_x.cuda(), att.cuda()


def _generate(model, vision_x, lang_x, att, mode, **kw):
    amp = torch.autocast("cuda", dtype=bf16) if mode != "fp32" else contextlib.nullcontext()
    with torch.inference_mode(), amp, _fast_lm(mode != "amp"):
        return model.generate(vision_x=vision_x, lang_x=lang_x, attention_mask=att, max_new_tokens=8, use_cache=True,
                              output_scores=True, return_dict_in_generate=True, pad_token_id=0, eos_token_id=None, **kw)


@pytest.mark.parametrize("every", [1, 2])
def test_generate_greedy_runs_on_kernels(every):
    model, vision_x, lang_x, att = _model(every)
    ref = _generate(model, vision_x, lang_x, att, "fp32")
    amp = _generate(model, vision_x, lang_x, att, "amp")
    with _count_calls() as calls:
        ours = _generate(model, vision_x, lang_x, att, "ours")
    assert calls["hf_attn"] == 0 and calls["decode"] == MPT["n_layers"] * 7, calls
    again = _generate(model, vision_x, lang_x, att, "ours")
    assert all(torch.equal(a, b) for a, b in zip(ours.scores, again.scores)), "two generate runs differ"
    # precondition of the token check: every step's fp32 top-2 margin exceeds 4x the measured autocast error
    assert torch.equal(ref.sequences, amp.sequences), "fp32 and autocast HF paths disagree: pick another seed"
    for i, (r, a, o) in enumerate(zip(ref.scores, amp.scores, ours.scores)):
        r, a, o = r.float(), a.float(), o.float()
        e_amp, e_ours = (a - r).abs().max().item(), (o - r).abs().max().item()
        top2 = r.topk(2, -1).values
        assert (top2[:, 0] - top2[:, 1]).min().item() > 4 * e_amp, f"step {i}: margin below 4x amp error"
        assert e_ours <= 2 * e_amp + 5e-3 * r.abs().max().item(), f"step {i}: err {e_ours:.3e} vs amp {e_amp:.3e}"
    assert torch.equal(ours.sequences, amp.sequences)
    # fp32: HF's path, HF's cache
    with _count_calls() as calls:
        _generate(model, vision_x, lang_x, att, "fp32")
    assert calls["decode"] == 0 and calls["hf_attn"] > 0


def test_generate_beam_search_matches_amp():
    model, vision_x, lang_x, att = _model(1)
    kw = dict(num_beams=3, length_penalty=0.0)
    amp = _generate(model, vision_x, lang_x, att, "amp", **kw)
    with _count_calls() as calls:
        ours = _generate(model, vision_x, lang_x, att, "ours", **kw)
    assert calls["hf_attn"] == 0 and calls["decode"] == MPT["n_layers"] * 7, calls
    assert torch.equal(ours.sequences, amp.sequences)


def test_rank_classification_sequence_matches_uncached_forward():
    """cache_media -> use_cache=True prefix -> one-token forwards with past_key_values, as the reference's evaluation
    scores class names; the logits match one uncached forward over the concatenation."""
    model, vision_x, lang_x, att = _model(1)
    cont = torch.randint(0, 90, (3, 4), generator=torch.Generator().manual_seed(5)).cuda()
    full = torch.cat([lang_x, cont], 1)
    full_att = torch.cat([att, torch.ones_like(cont)], 1)
    with torch.inference_mode(), torch.autocast("cuda", dtype=bf16):
        ref = model(vision_x=vision_x, lang_x=full, attention_mask=full_att).logits.float()
        with _count_calls() as calls:
            model.cache_media(input_ids=lang_x, vision_x=vision_x)
            out = model(vision_x=None, lang_x=lang_x, attention_mask=att, clear_conditioned_layers=False, use_cache=True)
            pkv, got = out.past_key_values, [out.logits.float()]
            for t in range(cont.shape[1]):
                out = model(vision_x=None, lang_x=cont[:, t:t + 1], attention_mask=full_att[:, :lang_x.shape[1] + t + 1],
                            clear_conditioned_layers=False, past_key_values=pkv, use_cache=True)
                got.append(out.logits.float())
            model.uncache_media()
    from open_flamingo_b200.kv_cache import KVCache
    assert isinstance(pkv, KVCache) and calls["hf_attn"] == 0 and calls["decode"] == MPT["n_layers"] * 4, calls
    got = torch.cat(got, 1)
    valid = full_att[:, :, None].float()
    scale = ref.abs().max().item()
    assert _err(got, ref, valid) <= OUT_TOL * scale


def test_declining_block_and_grad_mode_use_hf_attention():
    model, vision_x, lang_x, att = _model(1)
    blocks = model.lang_encoder.old_decoder_blocks
    with torch.inference_mode(), torch.autocast("cuda", dtype=bf16):
        base = model(vision_x=vision_x, lang_x=lang_x, attention_mask=att).logits.float()
    blocks[1].attn.clip_qkv = 1e6          # never clips, but makes block 1 decline the fast path
    try:
        with _count_calls() as calls:
            out = _generate(model, vision_x, lang_x, att, "ours")
        assert calls["hf_attn"] == 8 and calls["decode"] == (MPT["n_layers"] - 1) * 7, calls
        assert torch.isfinite(out.scores[-1]).all()
        with torch.inference_mode(), torch.autocast("cuda", dtype=bf16):
            model.cache_media(input_ids=lang_x, vision_x=vision_x)
            o = model(vision_x=None, lang_x=lang_x, attention_mask=att, clear_conditioned_layers=False, use_cache=True)
            model.uncache_media()
        assert _err(o.logits.float(), base, att[:, :, None].float()) <= OUT_TOL * base.abs().max().item()
    finally:
        blocks[1].attn.clip_qkv = None
    with torch.autocast("cuda", dtype=bf16), _count_calls() as calls:   # grad enabled: HF's path throughout
        model.cache_media(input_ids=lang_x, vision_x=vision_x)
        model(vision_x=None, lang_x=lang_x, attention_mask=att, clear_conditioned_layers=False, use_cache=True)
        model.uncache_media()
    assert calls["decode"] == 0 and calls["hf_attn"] == MPT["n_layers"], calls


def test_golden_every1_greedy_under_autocast():
    from helpers_golden import load, seeded_tensor
    from test_blocks_gpu import build_product_model
    fx = load("flamingo_every1")
    model = build_product_model(fx, 1)
    vision_x = seeded_tensor("flamingo/vision_x", fx["vision_x_shape"], 33).cuda()
    lang_x = fx["lang_x"].cuda()[:, :12]
    with torch.inference_mode(), torch.autocast("cuda", dtype=bf16), _count_calls() as calls:
        gen = model.generate(vision_x=vision_x, lang_x=lang_x, attention_mask=torch.ones_like(lang_x),
                             max_new_tokens=6, do_sample=False, pad_token_id=0, use_cache=True)
    assert calls["decode"] > 0 and calls["hf_attn"] == 0, calls
    assert torch.equal(gen.cpu(), fx["generated"])
