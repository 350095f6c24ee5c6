"""CPU: kv_cache.KVCache follows HF's cache protocol exactly.

A tiny HF MptForCausalLM in fp32 decodes a left-padded batch of unequal prompts once with HF's DynamicCache and once
with KVCache passed as `past_key_values`.  Greedy decoding, seeded sampling and beam search must give the same sequences
and bitwise-identical scores: KVCache.update returns what DynamicCache returns, so any difference is a protocol error
(a wrong length, mask size, beam reorder or crop)."""
import pytest
import torch

from open_flamingo_b200.kv_cache import KVCache, KVCacheLayer

N_LAYERS = 2


@pytest.fixture(scope="module")
def lm():
    from transformers import MptConfig, MptForCausalLM
    torch.manual_seed(0)
    cfg = MptConfig(d_model=64, n_heads=4, n_layers=N_LAYERS, vocab_size=97, max_seq_len=256, expansion_ratio=2)
    model = MptForCausalLM(cfg).eval()
    with torch.no_grad():
        for p in model.parameters():   # HF's init is near zero; make the logits decisive enough to be interesting
            p.normal_(0.0, 0.5 if p.dim() > 1 else 0.1).add_(1.0 if p.dim() == 1 else 0.0)
    return model


def prompts():
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(3, 97, (3, 11), generator=g)
    att = torch.ones_like(ids)
    att[0, :4] = 0      # left padding: prompts of 7, 11 and 9 tokens
    att[2, :2] = 0
    ids = ids.masked_fill(att == 0, 0)
    return ids, att


def run(lm, cache, **kw):
    ids, att = prompts()
    with torch.no_grad():
        if kw.get("do_sample"):
            torch.manual_seed(7)
        return lm.generate(ids, attention_mask=att, past_key_values=cache, use_cache=True, output_scores=True,
                           return_dict_in_generate=True, pad_token_id=0, eos_token_id=None, **kw)


def same(a, b):
    assert torch.equal(a.sequences, b.sequences), (a.sequences, b.sequences)
    assert len(a.scores) == len(b.scores)
    for i, (x, y) in enumerate(zip(a.scores, b.scores)):
        assert torch.equal(x, y), f"step {i}: scores differ by {(x - y).abs().max().item()}"


@pytest.mark.parametrize("mode", ["greedy", "sample", "beam"])
def test_generate_matches_dynamic_cache_bitwise(lm, mode):
    kw = {"greedy": dict(do_sample=False), "sample": dict(do_sample=True, top_k=20),
          "beam": dict(do_sample=False, num_beams=3, length_penalty=0.0)}[mode]
    from transformers import DynamicCache
    cache = KVCache(N_LAYERS)
    got = run(lm, cache, max_new_tokens=12, **kw)
    ref = run(lm, DynamicCache(), max_new_tokens=12, **kw)
    same(got, ref)
    assert cache.get_seq_length() == got.sequences.shape[1] - 1   # the last token is sampled, never fed back


def test_long_run_crosses_two_capacity_growths(lm):
    from transformers import DynamicCache
    cache = KVCache(N_LAYERS)
    caps = []
    orig = KVCacheLayer.reserve

    def spy(self, n):
        buf = orig(self, n)
        if self is cache.layers[0] and (not caps or caps[-1] != buf.shape[1]):
            caps.append(buf.shape[1])
        return buf

    KVCacheLayer.reserve = spy
    try:
        got = run(lm, cache, max_new_tokens=40, do_sample=False)
    finally:
        KVCacheLayer.reserve = orig
    assert len(caps) >= 3, f"capacities seen: {caps}"   # the first allocation and at least two growths
    same(got, run(lm, DynamicCache(), max_new_tokens=40, do_sample=False))


def _step(lm, cache, ids, att):
    with torch.no_grad():
        return lm(input_ids=ids, attention_mask=att, past_key_values=cache, use_cache=True).logits


def test_crop_then_redecode(lm):
    """Decode 6 tokens one at a time, crop the cache back by 3, re-feed those 3 tokens: the logits are the same as the
    first time, for KVCache exactly as for DynamicCache."""
    from transformers import DynamicCache
    ids, att = prompts()
    g = torch.Generator().manual_seed(2)
    new = torch.randint(3, 97, (ids.shape[0], 6), generator=g)
    out = {}
    for name, cache in (("ours", KVCache(N_LAYERS)), ("hf", DynamicCache())):
        logits = [_step(lm, cache, ids, att)[:, -1]]
        a = att
        for t in range(6):
            a = torch.cat([a, torch.ones_like(a[:, :1])], 1)
            logits.append(_step(lm, cache, new[:, t:t + 1], a)[:, -1])
        cache.crop(cache.get_seq_length() - 3)
        assert cache.get_seq_length() == ids.shape[1] + 3
        a = a[:, :-3]
        redo = []
        for t in range(3, 6):
            a = torch.cat([a, torch.ones_like(a[:, :1])], 1)
            redo.append(_step(lm, cache, new[:, t:t + 1], a)[:, -1])
        for t in range(3):
            assert torch.equal(redo[t], logits[4 + t]), f"{name}: re-decoded step {t} differs"
        out[name] = logits
    for x, y in zip(out["ours"], out["hf"]):
        assert torch.equal(x, y)


def test_mask_sizes_agree_with_dynamic_cache(lm):
    from transformers import DynamicCache
    ids, att = prompts()
    ours, hf = KVCache(N_LAYERS), DynamicCache()
    for c in (ours, hf):
        _step(lm, c, ids, att)
    a = att
    for t in range(5):
        for q in (1, 3):
            for layer in range(N_LAYERS):
                assert ours.get_mask_sizes(q, layer) == hf.get_mask_sizes(q, layer)
        assert ours.get_seq_length() == hf.get_seq_length()
        assert ours.get_max_cache_shape() == hf.get_max_cache_shape() == -1
        a = torch.cat([a, torch.ones_like(a[:, :1])], 1)
        tok = ids[:, -1:]
        for c in (ours, hf):
            _step(lm, c, tok, a)
    ours.reset()
    assert ours.get_seq_length() == 0 and ours.get_mask_sizes(4, 0) == (4, 0)
