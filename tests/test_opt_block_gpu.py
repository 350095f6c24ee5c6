"""GPU: the frozen OPT block (lm_blocks.FastOptBlock / FrozenOptBlockFn) and its cached decoding path.

Block, forward and input gradient, at head_dim 64, 80 (run on the 128 cores, heads zero-padded) and 128, T = 77 and a
left-padded row:
  (a) against tests/opt_reference.py, the float64 restatement that rounds where the kernels round:
      ||ours - ref_r||_2 <= L2 ||ref_r - ref_64||_2 and, per row, max |ours - ref_r| <= ROW 2^-8 max |ref_r|;
  (b) against HF's OPTDecoderLayer: err(ours, fp32) <= 2 err(autocast, fp32) + a floor of 5e-3 of the largest value.
In training mode with dropout 0.1 the block is checked against the same restatement given the kernel's own keep masks,
recovered by running the dropout forward on the saved (seed, offset) pairs with x = 0 and branch = 1.

Cached path (kv_cache.KVCache under autocast): prefill + a 3-token chunk + single tokens against the uncached kernel
path and HF's DynamicCache; greedy generate token-identical to HF autocast; beam search; the rank-classification loop;
a fixed-capacity cache equal to the growing one bit for bit; a declined call (output_attentions) in the middle of
decoding continuing on the same KVCache.  HF's OPTAttention.forward is counted and never runs on the product side."""
import contextlib

import pytest
import torch

import opt_reference as OR
from test_llama_block_gpu import _check_hf, _check_restatement, _fast_lm, _incremental, _valid

pytestmark = pytest.mark.gpu
bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64
OUT_TOL = 2e-2


def _block(hd, heads, seed, dropout=0.0):
    from transformers import OPTConfig
    from transformers.models.opt.modeling_opt import OPTDecoderLayer
    torch.manual_seed(seed)
    D = hd * heads
    cfg = OPTConfig(hidden_size=D, num_attention_heads=heads, num_hidden_layers=1, ffn_dim=4 * D, vocab_size=32,
                    word_embed_proj_dim=D, max_position_embeddings=512, dropout=dropout, attention_dropout=0.0,
                    attn_implementation="sdpa")
    blk = OPTDecoderLayer(cfg, 0).cuda().eval().requires_grad_(False)
    with torch.no_grad():
        for name, p in blk.named_parameters():
            if "layer_norm" in name:
                p.copy_((1.0 if name.endswith("weight") else 0.0) + 0.1 * torch.randn_like(p))
            elif name.endswith("bias"):
                p.copy_(0.1 * torch.randn_like(p))
            else:
                p.copy_(torch.randn_like(p) * p.shape[1] ** -0.5)
    return blk


def _inputs(D, B, T, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, T, D, device="cuda", generator=g)
    att = torch.ones(B, T, dtype=torch.long, device="cuda")
    att[1, :9] = 0
    causal = torch.ones(T, T, dtype=torch.bool, device="cuda").tril()
    allowed = causal[None] & att.bool()[:, None, :]
    allowed |= torch.eye(T, dtype=torch.bool, device="cuda")[None]   # no empty row: HF's sdpa would return NaN there
    w_out = torch.randn(B, T, D, device="cuda", generator=g) * _valid(att)
    return x, att, allowed, w_out


@contextlib.contextmanager
def _count_calls():
    """Counts ops.attn_decode calls and HF OPTAttention.forward calls; records the (p, seed/offset) of every dropout
    forward and where every ReLU passed its input."""
    from transformers.models.opt import modeling_opt as M
    from open_flamingo_b200 import ops
    n = {"decode": 0, "hf_attn": 0, "dropout": [], "relu_on": []}
    dec, hf, drop, relu = ops.attn_decode, M.OPTAttention.forward, ops.dropout_resid_fwd, ops.relu_bf16

    def dec_w(*a, **k):
        n["decode"] += 1
        return dec(*a, **k)

    def hf_w(self, *a, **k):
        n["hf_attn"] += 1
        return hf(self, *a, **k)

    def drop_w(x, branch, p, so, out=None):
        n["dropout"].append((p, so))
        return drop(x, branch, p, so, out=out)

    def relu_w(z, out=None):
        h = relu(z, out=out)
        n["relu_on"].append(h > 0)
        return h
    ops.attn_decode, M.OPTAttention.forward, ops.dropout_resid_fwd, ops.relu_bf16 = dec_w, hf_w, drop_w, relu_w
    try:
        yield n
    finally:
        ops.attn_decode, M.OPTAttention.forward, ops.dropout_resid_fwd, ops.relu_bf16 = dec, hf, drop, relu


def _restatement(x, blk, heads, allowed, w_out, relu_on, masks=None, p=0.0):
    """(rounded, float64) restatements, the rounded one with the kernels' ReLU decisions `relu_on` [B * T, F]."""
    sd = {n: p_.detach().double() for n, p_ in blk.named_parameters()}
    refs = {}
    for rounding in (True, False):
        xd = x.double().requires_grad_(True)
        on = relu_on.view(x.shape[0], x.shape[1], -1) if rounding else None
        o = OR.opt_block(xd, sd, heads, allowed, masks=masks, p=p, relu_on=on, rounding=rounding)
        (o * w_out.double()).sum().backward()
        refs[rounding] = (o.detach(), xd.grad)
    return refs


@pytest.mark.parametrize("hd", [64, 80, 128])
def test_frozen_opt_block_forward_and_input_gradient(hd):
    from open_flamingo_b200 import lm_blocks
    heads, B, T = 4, 2, 77
    blk = _block(hd, heads, 7 + hd)
    fast = lm_blocks.accelerate(blk)
    assert isinstance(fast, lm_blocks.FastOptBlock)
    x, att, allowed, w_out = _inputs(hd * heads, B, T, 8)
    m4 = allowed[:, None]
    valid = _valid(att)
    xg = x.clone().requires_grad_(True)
    with _count_calls() as calls:
        got = fast(xg, attention_mask=m4)
        assert got is not None and got.dtype == f32, "fast path declined"
        (got * w_out).sum().backward()
    assert calls["hf_attn"] == 0 and not calls["dropout"]
    assert torch.isfinite(got).all(), "padding rows must be finite"
    res = {}
    for mode in ("fp32", "amp"):
        xr = x.clone().requires_grad_(True)
        ctx = torch.autocast("cuda", dtype=bf16) if mode == "amp" else contextlib.nullcontext()
        with ctx:
            out = blk(xr, attention_mask=m4)
        (out.float() * w_out).sum().backward()
        res[mode] = (out.float().detach(), xr.grad)
    what = f"hd{hd}"
    _check_hf(what + " out", got.detach(), res["amp"][0], res["fp32"][0], valid)
    _check_hf(what + " dx", xg.grad, res["amp"][1], res["fp32"][1], valid)
    assert len(calls["relu_on"]) == 1
    refs = _restatement(x, blk, heads, allowed, w_out, calls["relu_on"][0])
    _check_restatement(what + " out", got.detach(), refs[True][0], refs[False][0], valid)
    _check_restatement(what + " dx", xg.grad, refs[True][1], refs[False][1], valid)
    assert torch.equal(fast(x, attention_mask=m4), got.detach()), "not bitwise repeatable"


@pytest.mark.parametrize("hd", [64, 80])
def test_training_mode_dropout_against_the_restatement_with_the_kernel_masks(hd):
    from open_flamingo_b200 import lm_blocks, ops
    heads, B, T, p = 4, 2, 77, 0.1
    blk = _block(hd, heads, 3 + hd, dropout=p).train()
    fast = lm_blocks.accelerate(blk)
    D = hd * heads
    x, att, allowed, w_out = _inputs(D, B, T, 9)
    m4 = allowed[:, None]
    valid = _valid(att)
    xg = x.clone().requires_grad_(True)
    with _count_calls() as calls:
        got = fast(xg, attention_mask=m4)
        (got * w_out).sum().backward()
    assert calls["hf_attn"] == 0 and len(calls["dropout"]) == 2 and all(q == p for q, _ in calls["dropout"])
    masks = []
    for _, so in calls["dropout"]:
        keep = ops.dropout_resid_fwd(torch.zeros(B * T, D, device="cuda"), torch.ones(B * T, D, device="cuda",
                                                                                       dtype=bf16), p, so)
        masks.append((keep != 0).view(B, T, D).double())
    kept = torch.cat(masks).mean().item()
    assert abs(kept - (1 - p)) < 0.02, kept
    refs = _restatement(x, blk, heads, allowed, w_out, calls["relu_on"][0], masks=masks, p=p)
    _check_restatement(f"hd{hd} dropout out", got.detach(), refs[True][0], refs[False][0], valid)
    _check_restatement(f"hd{hd} dropout dx", xg.grad, refs[True][1], refs[False][1], valid)
    # the next call draws other masks; eval mode none
    again = fast(x, attention_mask=m4)
    assert not torch.equal(again, got.detach())
    blk.eval()
    ev = fast(x, attention_mask=m4)
    with torch.autocast("cuda", dtype=bf16):
        amp = blk(x, attention_mask=m4).float()
    _check_hf(f"hd{hd} eval", ev, amp, blk(x, attention_mask=m4), valid)


def test_packed_weights_follow_load_state_dict():
    from open_flamingo_b200 import lm_blocks
    blk = _block(64, 4, 3)
    fast = lm_blocks.accelerate(blk)
    x, att, allowed, _ = _inputs(256, 2, 40, 4)
    m4 = allowed[:, None]
    before = fast(x, attention_mask=m4)
    sd = blk.state_dict()
    sd["self_attn.k_proj.weight"] = -2 * sd["self_attn.k_proj.weight"]
    sd["self_attn.v_proj.bias"] = sd["self_attn.v_proj.bias"] + 0.5
    sd["fc1.weight"] = 0.5 * sd["fc1.weight"]
    blk.load_state_dict(sd)
    after = fast(x, attention_mask=m4)
    with torch.autocast("cuda", dtype=bf16):
        amp = blk(x, attention_mask=m4).float()
    ref = blk(x, attention_mask=m4)
    assert not torch.equal(before, after)
    _check_hf("after load_state_dict", after, amp, ref, _valid(att))


# --------------------------------------------------------------------------------------------- cached path
def _make_lm(hd, heads, seed, n_layers=2, vocab=64):
    from open_flamingo_b200 import lm_blocks
    from open_flamingo_b200.testing import build_opt
    D = hd * heads
    lm = build_opt(dict(hidden_size=D, num_attention_heads=heads, num_hidden_layers=n_layers, ffn_dim=4 * D,
                        word_embed_proj_dim=D, vocab_size=vocab, max_position_embeddings=512, dropout=0.1),
                   device="cuda", seed=seed)
    lm.requires_grad_(False)
    with torch.no_grad():
        for name, p in lm.named_parameters():
            if p.dim() == 2 and "embed" not in name:
                p.copy_(torch.randn_like(p) * p.shape[1] ** -0.5)
    for blk in lm.model.decoder.layers:   # route every block through the fast path, as FlamingoLayer does
        fast, orig = lm_blocks.accelerate(blk), blk.forward

        def fwd(hidden_states, *a, _fast=fast, _orig=orig, **kw):
            r = _fast(hidden_states, *a, **kw)
            return r if r is not None else _orig(hidden_states, *a, **kw)
        blk.forward = fwd
    return lm


@pytest.mark.parametrize("hd", [64, 80, 128])
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
    assert calls["hf_attn"] == 0 and calls["decode"] == 2 * 8 and not calls["dropout"], calls
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
OPT = dict(hidden_size=320, num_attention_heads=4, num_hidden_layers=4, ffn_dim=1280, word_embed_proj_dim=320,
           vocab_size=97, max_position_embeddings=256, dropout=0.1)   # head_dim 80


def _model(every):
    from open_flamingo_b200.testing import build_flamingo
    model, _, tok = build_flamingo(VIT, None, opt_kw=OPT, cross_attn_every_n_layers=every, device="cuda",
                                   gate_init=1.0, seed=21)
    with torch.no_grad():
        for name, p in model.lang_encoder.named_parameters():
            if "gated_cross_attn" in name or not name.startswith("model.decoder.layers") or p.dim() != 2:
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
    layers = OPT["num_hidden_layers"]
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
    lm = model.lang_encoder
    with _count_calls() as calls:
        static = _generate(model, vision_x, lang_x, att, "ours", cache_implementation="static")
    assert lm.decode_graphs.captures == 0 and calls["hf_attn"] == 0 and calls["decode"] == layers * 7, calls
    assert all(torch.equal(a, b) for a, b in zip(ours.scores, static.scores)), "static cache differs from growing"
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
    assert isinstance(pkv, KVCache) and calls["hf_attn"] == 0 and calls["decode"] == OPT["num_hidden_layers"] * 4
    got = torch.cat(got, 1)
    valid = full_att[:, :, None].float()
    assert ((got - ref).abs() * valid).max().item() <= OUT_TOL * ref.abs().max().item()


def test_training_step_uses_the_kernel_block():
    """Flamingo.forward + backward with a frozen OPT LM in train mode: the blocks run FrozenOptBlockFn with residual
    dropout, not HF's attention.  With the LM's blocks in eval mode (no dropout) the loss and a trainable gradient agree
    with lm_blocks.ENABLED = False under autocast."""
    from open_flamingo_b200.testing import synthetic_batch
    model = _model(2)[0]
    model.train()
    batch = synthetic_batch(2, 2, 40, model.media_token_id, model.eoc_token_id, 90, image_size=56, seed=5)
    batch = {k: v.cuda() for k, v in batch.items()}

    def run(on):
        model.zero_grad(set_to_none=True)
        with _fast_lm(on), _count_calls() as calls, torch.autocast("cuda", dtype=bf16):
            out = model(vision_x=batch["vision_x"], lang_x=batch["lang_x"], attention_mask=batch["attention_mask"],
                        labels=batch["labels"])
        out.loss.backward()
        g = next(p.grad for n, p in model.named_parameters() if n.endswith("attn.to_q.weight"))
        return out.loss.item(), g.clone(), calls

    loss_d, g_d, calls = run(True)
    layers = OPT["num_hidden_layers"]
    assert calls["hf_attn"] == 0 and len(calls["dropout"]) == 2 * layers and torch.isfinite(g_d).all()
    for blk in model.lang_encoder.old_decoder_blocks:
        blk.eval()
    res = {on: run(on) for on in (True, False)}
    assert res[True][2]["hf_attn"] == 0 and not res[True][2]["dropout"]
    assert res[False][2]["hf_attn"] == layers
    assert abs(res[True][0] - res[False][0]) <= 2e-2 * abs(res[False][0])
    ga, gb = res[True][1].flatten(), res[False][1].flatten()
    assert torch.nn.functional.cosine_similarity(ga, gb, dim=0).item() >= 0.99
    assert loss_d != res[True][0]
