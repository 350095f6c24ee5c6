"""GPU: the frozen LLaMA block (lm_blocks.FastLlamaBlock / FrozenLlamaBlockFn) and its cached decoding path.

Block, forward and input gradient, at head_dim 64 and 128, with HF's default rotary tables and with llama3 frequency
scaling, T = 77 (not a multiple of 64) and a left-padded row with per-row positions:
  (a) against tests/llama_reference.py, the float64 restatement that rounds where the kernels round:
      ||ours - ref_r||_2 <= L2 ||ref_r - ref_64||_2 and, per row, max |ours - ref_r| <= ROW 2^-8 max |ref_r|;
  (b) against HF's LlamaDecoderLayer: err(ours, fp32) <= 2 err(autocast, fp32) + a floor of 5e-3 of the largest value.
Only rows of real tokens are compared; padding query rows must be finite.

Cached path (kv_cache.KVCache under autocast): prefill + a 3-token chunk + single tokens against the uncached kernel
path and HF's DynamicCache; greedy generate token-identical to HF autocast; beam search; the rank-classification loop;
a fixed-capacity cache equal to the growing one bit for bit with no decode graph captured; a declined call
(output_attentions) in the middle of decoding continuing on the same KVCache.  HF's LlamaAttention.forward is counted
and never runs on the product side."""
import contextlib

import pytest
import torch

import llama_reference as LR

pytestmark = pytest.mark.gpu
bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64
L2, ROW = 1.0, 4.0
OUT_TOL = 2e-2
LLAMA3 = dict(rope_type="llama3", rope_theta=500000.0, factor=8.0, low_freq_factor=1.0, high_freq_factor=4.0,
              original_max_position_embeddings=32)


def _config(hd, heads, rope, **kw):
    from transformers import LlamaConfig
    args = dict(hidden_size=hd * heads, num_attention_heads=heads, num_key_value_heads=heads, num_hidden_layers=1,
                intermediate_size=3 * hd * heads, vocab_size=32, max_position_embeddings=512, rms_norm_eps=1e-6,
                attn_implementation="sdpa")
    args.update(kw)
    if rope == "llama3":
        args["rope_parameters"] = dict(LLAMA3)
    return LlamaConfig(**args)


def _block(hd, heads, rope, seed):
    from transformers.models.llama.modeling_llama import LlamaDecoderLayer, LlamaRotaryEmbedding
    torch.manual_seed(seed)
    cfg = _config(hd, heads, rope)
    blk = LlamaDecoderLayer(cfg, 0).cuda().eval().requires_grad_(False)
    with torch.no_grad():
        for name, p in blk.named_parameters():
            if "layernorm" in name:
                p.copy_(1.0 + 0.1 * torch.randn_like(p))
            else:
                p.copy_(torch.randn_like(p) * p.shape[1] ** -0.5)
    return blk, LlamaRotaryEmbedding(cfg).cuda()


def _inputs(blk, rope, B, T, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    D = blk.input_layernorm.weight.shape[0]
    x = torch.randn(B, T, D, device="cuda", generator=g)
    att = torch.ones(B, T, dtype=torch.long, device="cuda")
    att[1, :9] = 0                                                     # left padding, as generate() pads
    pos = (att.cumsum(-1) - 1).masked_fill(att == 0, 1)
    cos, sin = rope(x, pos)
    causal = torch.ones(T, T, dtype=torch.bool, device="cuda").tril()
    allowed = causal[None] & att.bool()[:, None, :]
    allowed |= torch.eye(T, dtype=torch.bool, device="cuda")[None]   # no empty row: HF's sdpa would return NaN there
    return x, att, cos, sin, allowed


def _valid(att):
    return att.bool()[..., None].float()


def _check_restatement(what, got, ref_r, ref_64, valid):
    got, ref_r, ref_64 = (t.double() * valid for t in (got, ref_r, ref_64))
    e, rnd = (got - ref_r).norm().item(), (ref_r - ref_64).norm().item()
    row = ((got - ref_r).abs().amax(-1) / (ref_r.abs().amax(-1) * 2.0 ** -8 + 1e-30)).max().item()
    assert e <= L2 * rnd, f"{what}: L2 {e:.3e} vs rounding effect {rnd:.3e} (ratio {e / max(rnd, 1e-30):.2f})"
    assert row <= ROW, f"{what}: row error {row:.2f} x 2^-8 of the row maximum"


def _check_hf(what, got, amp, ref, valid):
    e_ours = ((got.float() - ref) * valid).abs().max().item()
    e_amp = ((amp.float() - ref) * valid).abs().max().item()
    scale = (ref * valid).abs().max().item()
    assert e_ours <= 2 * e_amp + 5e-3 * scale, f"{what}: err vs fp32 {e_ours:.3e}, autocast {e_amp:.3e}"


@contextlib.contextmanager
def _count_calls():
    """Counts ops.attn_decode calls and HF LlamaAttention.forward calls."""
    from transformers.models.llama import modeling_llama as M
    from open_flamingo_b200 import ops
    n = {"decode": 0, "hf_attn": 0}
    dec, hf = ops.attn_decode, M.LlamaAttention.forward

    def dec_w(*a, **k):
        n["decode"] += 1
        return dec(*a, **k)

    def hf_w(self, *a, **k):
        n["hf_attn"] += 1
        return hf(self, *a, **k)
    ops.attn_decode, M.LlamaAttention.forward = dec_w, hf_w
    try:
        yield n
    finally:
        ops.attn_decode, M.LlamaAttention.forward = dec, hf


@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("rope", ["default", "llama3"])
def test_frozen_llama_block_forward_and_input_gradient(hd, rope):
    from open_flamingo_b200 import lm_blocks
    heads, B, T = 4, 2, 77
    blk, rope_emb = _block(hd, heads, rope, 7 + hd)
    fast = lm_blocks.accelerate(blk)
    assert isinstance(fast, lm_blocks.FastLlamaBlock)
    x, att, cos, sin, allowed = _inputs(blk, rope_emb, B, T, 8)
    m4 = allowed[:, None]
    valid = _valid(att)
    w_out = torch.randn(B, T, x.shape[-1], device="cuda", generator=torch.Generator(device="cuda").manual_seed(9))
    w_out = w_out * valid

    xg = x.clone().requires_grad_(True)
    with _count_calls() as calls:
        got = fast(xg, attention_mask=m4, position_embeddings=(cos, sin))
        assert got is not None and got.dtype == f32, "fast path declined"
        (got * w_out).sum().backward()
    assert calls["hf_attn"] == 0
    assert torch.isfinite(got).all(), "padding rows must be finite"

    res = {}
    for mode in ("fp32", "amp"):
        xr = x.clone().requires_grad_(True)
        ctx = torch.autocast("cuda", dtype=bf16) if mode == "amp" else contextlib.nullcontext()
        with ctx:
            out = blk(xr, attention_mask=m4, position_embeddings=(cos, sin))
        (out.float() * w_out).sum().backward()
        res[mode] = (out.float().detach(), xr.grad)
    what = f"hd{hd} rope={rope}"
    _check_hf(what + " out", got.detach(), res["amp"][0], res["fp32"][0], valid)
    _check_hf(what + " dx", xg.grad, res["amp"][1], res["fp32"][1], valid)

    sd = {n: p.detach().double() for n, p in blk.named_parameters()}
    refs = {}
    for rounding in (True, False):
        xd = x.double().requires_grad_(True)
        o = LR.llama_block(xd, sd, heads, cos.double(), sin.double(), allowed, 1e-6, rounding=rounding)
        (o * w_out.double()).sum().backward()
        refs[rounding] = (o.detach(), xd.grad)
    _check_restatement(what + " out", got.detach(), refs[True][0], refs[False][0], valid)
    _check_restatement(what + " dx", xg.grad, refs[True][1], refs[False][1], valid)

    again = fast(x, attention_mask=m4, position_embeddings=(cos, sin))
    assert torch.equal(again, got.detach()), "not bitwise repeatable"


def test_packed_weights_follow_load_state_dict():
    from open_flamingo_b200 import lm_blocks
    blk, rope = _block(64, 4, "default", 3)
    fast = lm_blocks.accelerate(blk)
    x, att, cos, sin, allowed = _inputs(blk, rope, 2, 40, 4)
    m4 = allowed[:, None]
    before = fast(x, attention_mask=m4, position_embeddings=(cos, sin))
    sd = blk.state_dict()
    sd["self_attn.k_proj.weight"] = -2 * sd["self_attn.k_proj.weight"]
    sd["mlp.up_proj.weight"] = 0.5 * sd["mlp.up_proj.weight"]
    blk.load_state_dict(sd)
    after = fast(x, attention_mask=m4, position_embeddings=(cos, sin))
    with torch.autocast("cuda", dtype=bf16):
        amp = blk(x, attention_mask=m4, position_embeddings=(cos, sin)).float()
    ref = blk(x, attention_mask=m4, position_embeddings=(cos, sin))
    assert not torch.equal(before, after)
    _check_hf("after load_state_dict", after, amp, ref, _valid(att))


# --------------------------------------------------------------------------------------------- cached path
@contextlib.contextmanager
def _fast_lm(on):
    from open_flamingo_b200 import lm_blocks
    prev = lm_blocks.ENABLED
    lm_blocks.ENABLED = on
    try:
        yield
    finally:
        lm_blocks.ENABLED = prev


def _make_lm(hd, heads, seed, n_layers=2, vocab=64):
    from open_flamingo_b200 import lm_blocks
    from open_flamingo_b200.testing import build_llama
    lm = build_llama(dict(hidden_size=hd * heads, num_attention_heads=heads, num_hidden_layers=n_layers,
                          intermediate_size=3 * hd * heads, vocab_size=vocab, max_position_embeddings=512),
                     device="cuda", seed=seed)
    lm.requires_grad_(False)
    with torch.no_grad():
        for name, p in lm.named_parameters():
            if p.dim() == 2 and "embed" not in name:
                p.copy_(torch.randn_like(p) * p.shape[1] ** -0.5)
    for blk in lm.model.layers:   # route every block through the fast path, as FlamingoLayer does
        fast, orig = lm_blocks.accelerate(blk), blk.forward

        def fwd(hidden_states, *a, _fast=fast, _orig=orig, **kw):
            r = _fast(hidden_states, *a, **kw)
            return r if r is not None else _orig(hidden_states, *a, **kw)
        blk.forward = fwd
    return lm


def _incremental(lm, ids, att, cache, steps, declined_at=None):
    out, pos = [], 0
    for i, w in enumerate(steps):
        kw = dict(output_attentions=True) if i == declined_at else {}
        o = lm(input_ids=ids[:, pos:pos + w], attention_mask=att[:, :pos + w], past_key_values=cache, use_cache=True,
               **kw)
        out.append(o.logits.float())
        pos += w
    return out


@pytest.mark.parametrize("hd", [64, 128])
def test_cached_path_matches_uncached_and_hf(hd):
    from transformers import DynamicCache
    from open_flamingo_b200.kv_cache import KVCache
    lm = _make_lm(hd, 4, 11)
    B, T = 3, 40
    steps = [T, 3] + [1] * 8
    n = sum(steps)
    ids = torch.randint(0, 64, (B, n), generator=torch.Generator().manual_seed(12)).cuda()
    att = torch.ones(B, n, dtype=torch.long, device="cuda")
    att[1, :5] = 0
    att[2, :11] = 0
    with torch.inference_mode():
        with _fast_lm(False):
            ref = lm(input_ids=ids, attention_mask=att).logits.float()
        with torch.autocast("cuda", dtype=bf16):
            with _fast_lm(True):
                full = lm(input_ids=ids, attention_mask=att).logits.float()
                with _count_calls() as calls:
                    ours = _incremental(lm, ids, att, KVCache(2), steps)
                with _count_calls() as declined_calls:
                    declined = _incremental(lm, ids, att, KVCache(2), steps, declined_at=5)
            with _fast_lm(False):
                amp = _incremental(lm, ids, att, DynamicCache(), steps)
    assert calls["hf_attn"] == 0 and calls["decode"] == 2 * 8, calls
    # step 5 (a single token) asked for attention weights: both blocks ran HF's layer on the same KVCache
    assert declined_calls["hf_attn"] == 2 and declined_calls["decode"] == 2 * 7, declined_calls
    scale = ref.abs().max().item()
    pos = 0
    for i, w in enumerate(steps):
        sl = slice(pos, pos + w)
        valid = att[:, sl, None].float()
        for got, what in ((ours[i], "cached"), (declined[i], "cached, step 5 declined")):
            assert torch.isfinite(got).all()
            e_full = ((got - full[:, sl]).abs() * valid).max().item()
            assert e_full <= OUT_TOL * scale, f"{what} step {i}: vs uncached kernel path {e_full:.3e} (max {scale:.3e})"
            e_ours = ((got - ref[:, sl]).abs() * valid).max().item()
            e_amp = ((amp[i] - ref[:, sl]).abs() * valid).max().item()
            assert e_ours <= 2 * e_amp + 5e-3 * scale, f"{what} step {i}: err vs fp32 {e_ours:.3e}, amp {e_amp:.3e}"
        pos += w


# --------------------------------------------------------------------------------------------- model level
VIT = dict(image_size=56, patch_size=14, width=128, layers=2, heads=2, output_dim=128)
LLAMA = dict(hidden_size=256, num_attention_heads=4, num_hidden_layers=4, intermediate_size=704, vocab_size=97,
             max_position_embeddings=256)


def _model(every):
    from open_flamingo_b200.testing import build_flamingo
    model, _, tok = build_flamingo(VIT, None, llama_kw=LLAMA, cross_attn_every_n_layers=every, device="cuda",
                                   gate_init=1.0, seed=21)
    with torch.no_grad():
        # unit-variance tied-like embeddings make greedy and best-beam tokens decisive (as in test_kv_decode_gpu)
        for name, p in model.lang_encoder.named_parameters():
            if "gated_cross_attn" in name or not name.startswith("model.layers") or p.dim() != 2:
                continue
            p.copy_(torch.randn_like(p) * p.shape[1] ** -0.5)
        model.lang_encoder.get_input_embeddings().weight.normal_()
        model.lang_encoder.get_output_embeddings().weight.copy_(model.lang_encoder.get_input_embeddings().weight)
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


def test_generate_greedy_beams_and_static_cache_run_on_kernels():
    model, vision_x, lang_x, att = _model(2)
    layers = LLAMA["num_hidden_layers"]
    ref = _generate(model, vision_x, lang_x, att, "fp32")
    amp = _generate(model, vision_x, lang_x, att, "amp")
    with _count_calls() as calls:
        ours = _generate(model, vision_x, lang_x, att, "ours")
    assert calls["hf_attn"] == 0 and calls["decode"] == layers * 7, calls
    again = _generate(model, vision_x, lang_x, att, "ours")
    assert all(torch.equal(a, b) for a, b in zip(ours.scores, again.scores)), "two generate runs differ"
    assert torch.equal(ref.sequences, amp.sequences), "fp32 and autocast HF paths disagree: pick another seed"
    for i, (r, a, o) in enumerate(zip(ref.scores, amp.scores, ours.scores)):
        r, a, o = r.float(), a.float(), o.float()
        e_amp, e_ours = (a - r).abs().max().item(), (o - r).abs().max().item()
        top2 = r.topk(2, -1).values
        assert (top2[:, 0] - top2[:, 1]).min().item() > 4 * e_amp, f"step {i}: margin below 4x amp error"
        assert e_ours <= 2 * e_amp + 5e-3 * r.abs().max().item(), f"step {i}: err {e_ours:.3e} vs amp {e_amp:.3e}"
    assert torch.equal(ours.sequences, amp.sequences)
    # a fixed-capacity cache: decode_graph declines a LLaMA LM, so every step runs eagerly on the fixed buffers and
    # computes the growing cache's bits
    lm = model.lang_encoder
    with _count_calls() as calls:
        static = _generate(model, vision_x, lang_x, att, "ours", cache_implementation="static")
    assert lm.decode_graphs.captures == 0 and calls["hf_attn"] == 0 and calls["decode"] == layers * 7, calls
    assert all(torch.equal(a, b) for a, b in zip(ours.scores, static.scores)), "static cache differs from growing"
    # beam search with 3 beams runs on the kernels and finds autocast's best beams
    kw = dict(num_beams=3, length_penalty=0.0)
    amp_b = _generate(model, vision_x, lang_x, att, "amp", **kw)
    with _count_calls() as calls:
        ours_b = _generate(model, vision_x, lang_x, att, "ours", **kw)
    assert calls["hf_attn"] == 0 and calls["decode"] == layers * 7, calls
    assert torch.equal(ours_b.sequences, amp_b.sequences)


def test_rank_classification_sequence_matches_uncached_forward():
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
    assert isinstance(pkv, KVCache) and calls["hf_attn"] == 0 and calls["decode"] == LLAMA["num_hidden_layers"] * 4
    got = torch.cat(got, 1)
    valid = full_att[:, :, None].float()
    assert ((got - ref).abs() * valid).max().item() <= OUT_TOL * ref.abs().max().item()


def test_training_step_uses_the_kernel_block():
    """Flamingo.forward + backward with a frozen LLaMA LM: the blocks run FrozenLlamaBlockFn, not HF's attention, and
    the loss and a trainable gradient agree with lm_blocks.ENABLED = False under autocast."""
    from open_flamingo_b200.testing import synthetic_batch
    model = _model(2)[0]
    batch = synthetic_batch(2, 2, 40, model.media_token_id, model.eoc_token_id, 90, image_size=56, seed=5)
    batch = {k: v.cuda() for k, v in batch.items()}
    res = {}
    for on in (True, False):
        model.zero_grad(set_to_none=True)
        with _fast_lm(on), _count_calls() as calls, torch.autocast("cuda", dtype=bf16):
            out = model(vision_x=batch["vision_x"], lang_x=batch["lang_x"], attention_mask=batch["attention_mask"],
                        labels=batch["labels"])
        out.loss.backward()
        g = next(p.grad for n, p in model.named_parameters() if n.endswith("attn.to_q.weight"))
        res[on] = (out.loss.item(), g.clone(), dict(calls))
    assert res[True][2]["hf_attn"] == 0 and res[False][2]["hf_attn"] == LLAMA["num_hidden_layers"]
    assert abs(res[True][0] - res[False][0]) <= 2e-2 * abs(res[False][0])
    ga, gb = res[True][1].flatten(), res[False][1].flatten()
    assert torch.nn.functional.cosine_similarity(ga, gb, dim=0).item() >= 0.99
