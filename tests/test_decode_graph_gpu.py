"""GPU: graph-replayed decoding is the eager cached decode, bit for bit.

1. ofk_attn_decode_dev equals ofk_attn_decode at the same nk, whatever nk_max, with rows past nk and the workspace
   NaN-filled; *nk_dev = 0 gives zeros and *nk_dev > nk_max the nk_max result.
2. ofk_kv_append changes exactly one row and one mask byte per batch entry, and nothing for a position past capacity.
3. One CUDA graph of (append + decode) replayed at positions p .. p + 40 equals the eager launches at each position.
4. generate(cache_implementation="static") against the eager KVCache path: same sequences, bit-identical logits at every
   step, every decode step replayed and no eager decode attention -- greedy, seeded sampling, beam search, a left-padded
   batch, at several LM widths.
5. The rank-classification loop with make_kv_cache(capacity=...) gives the eager loop's logits bit for bit.
6. A graph is reused across calls of one shape key without stale inputs, captured anew for another batch, and
   re-captured after load_state_dict.
   Calls alternating between inference_mode and no_grad each match eager, and a cache cropped back to its prefix
   after new weights were loaded in place reads the new weights.
7. Steps the graph does not serve run eagerly with the same results; a cache overflow raises before any launch; the
   capacity follows a generation_config passed to generate."""
import contextlib

import pytest
import torch

from test_kv_decode_gpu import MPT, VIT, _count_calls, _fast_lm

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16


# --------------------------------------------------------------------------------------------- kernels
def _decode_inputs(B, H, hd, nk, nk_max, slopes_on, mask_kind, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    D = H * hd
    q = torch.randn(B, D, device="cuda", generator=g).to(bf16)
    # 64 NaN rows past nk_max: a read beyond nk_max would show as a NaN output instead of going out of bounds
    buf = torch.full((B, nk_max + 64, 2 * D), float("nan"), device="cuda", dtype=bf16)
    buf[:, :nk] = torch.randn(B, nk, 2 * D, device="cuda", generator=g).to(bf16)
    slopes = torch.rand(H, device="cuda", generator=g) * 0.5 if slopes_on else None
    mask = None
    if mask_kind != "none":
        mask = torch.randint(0, 256, (B, -(-nk_max // 8) * 8), device="cuda", generator=g).to(torch.uint8)  # junk
        pad = torch.randint(0, nk, (B,), device="cuda", generator=g)
        mask[:, :nk] = (torch.arange(nk, device="cuda")[None] < pad[:, None]).to(torch.uint8)
        if mask_kind == "full":
            mask[0, :nk] = 1
    return q, buf, slopes, mask


def _nan_ws(B, H, hd, nk_max):
    from open_flamingo_b200 import ops
    return ops.decode_workspace(torch.device("cuda"), B, H, hd, nk_max).fill_(float("nan"))


@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("B,H", [(1, 2), (1, 16), (3, 32), (24, 16)])
@pytest.mark.parametrize("nk", [1, 63, 64, 65, 300, 2049, 4097])
def test_decode_dev_bitwise_equals_decode(hd, B, H, nk):
    from open_flamingo_b200 import ops
    D = H * hd
    scale = hd ** -0.5
    for nk_max in (nk, 8192):
        for i, (slopes_on, mask_kind) in enumerate([(False, "none"), (True, "none"), (True, "pad"), (False, "pad"),
                                                    (True, "full")]):
            q, buf, slopes, mask = _decode_inputs(B, H, hd, nk, nk_max, slopes_on, mask_kind, 31 * nk + 7 * i + B)
            what = f"B{B} H{H} hd{hd} nk{nk} nk_max{nk_max} slopes={slopes_on} mask={mask_kind}"
            ref = ops.attn_decode(q, buf[:, :nk, :D], buf[:, :nk, D:], H, hd, scale, key_mask=mask, slopes=slopes)
            nk_dev = torch.tensor([nk], device="cuda", dtype=torch.int32)
            got = ops.attn_decode_dev(q, buf[:, :nk_max, :D], buf[:, :nk_max, D:], H, hd, scale, nk_dev, key_mask=mask,
                                      slopes=slopes, workspace=_nan_ws(B, H, hd, nk_max))
            assert torch.equal(got, ref), what
            nk_dev.zero_()
            zero = ops.attn_decode_dev(q, buf[:, :nk_max, :D], buf[:, :nk_max, D:], H, hd, scale, nk_dev, key_mask=mask,
                                       slopes=slopes, workspace=_nan_ws(B, H, hd, nk_max))
            assert torch.equal(zero, torch.zeros_like(zero)), what + " (nk_dev = 0)"
            if nk_max == nk:   # past nk_max: the nk_max result, and no row of the NaN tail read
                nk_dev.fill_(nk_max + 1000)
                over = ops.attn_decode_dev(q, buf[:, :nk_max, :D], buf[:, :nk_max, D:], H, hd, scale, nk_dev, key_mask=mask,
                                           slopes=slopes, workspace=_nan_ws(B, H, hd, nk_max))
                assert torch.equal(over, ref), what + " (nk_dev > nk_max)"


def test_kv_append_writes_one_row_and_one_mask_byte():
    from open_flamingo_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(3)
    B, cap, W = 3, 70, 512
    src = torch.randn(B, W, device="cuda", generator=g).to(bf16)
    cache = torch.randn(B, cap, W + 16, device="cuda", generator=g).to(bf16)   # canary columns past W
    mask = torch.randint(0, 256, (B, 80), device="cuda", generator=g).to(torch.uint8)
    new_masked = torch.tensor([0, 7, 1], device="cuda", dtype=torch.uint8)
    for pos in (0, 5, cap - 1):
        c0, m0 = cache.clone(), mask.clone()
        ops.kv_append(src, cache[:, :, :W], torch.tensor([pos], device="cuda", dtype=torch.int32), key_mask=mask,
                      new_masked=new_masked)
        exp, mexp = c0.clone(), m0.clone()
        exp[:, pos, :W] = src
        mexp[:, pos] = torch.tensor([0, 1, 1], device="cuda", dtype=torch.uint8)
        assert torch.equal(cache.view(torch.int16), exp.view(torch.int16)), pos
        assert torch.equal(mask, mexp), pos
        ops.kv_append(src, cache[:, :, :W], torch.tensor([pos], device="cuda", dtype=torch.int32), key_mask=mask)
        mexp[:, pos] = 0
        assert torch.equal(mask, mexp), f"{pos}: NULL new_masked means unmasked"
    for pos in (cap, cap + 100, -1):
        c0, m0 = cache.clone(), mask.clone()
        ops.kv_append(src, cache[:, :, :W], torch.tensor([pos], device="cuda", dtype=torch.int32), key_mask=mask,
                      new_masked=new_masked)
        assert torch.equal(cache.view(torch.int16), c0.view(torch.int16)) and torch.equal(mask, m0), pos


def test_replayed_append_and_decode_match_eager_launches():
    from open_flamingo_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(4)
    B, H, hd, cap, p0 = 3, 16, 128, 256, 150
    D = H * hd
    buf = torch.full((B, cap, 2 * D), float("nan"), device="cuda", dtype=bf16)
    buf[:, :p0] = torch.randn(B, p0, 2 * D, device="cuda", generator=g).to(bf16)
    mask = torch.zeros(B, cap, device="cuda", dtype=torch.uint8)
    mask[1, :9] = 1
    ref_buf, ref_mask = buf.clone(), mask.clone()
    slopes = torch.rand(H, device="cuda", generator=g) * 0.5
    q, src = torch.empty(B, D, device="cuda", dtype=bf16), torch.empty(B, 2 * D, device="cuda", dtype=bf16)
    new_masked = torch.zeros(B, device="cuda", dtype=torch.uint8)
    pos_nk = torch.zeros(2, device="cuda", dtype=torch.int32)
    ws = ops.decode_workspace(torch.device("cuda"), B, H, hd, cap)
    out = torch.empty(B, D, device="cuda", dtype=bf16)

    def step():
        ops.kv_append(src, buf, pos_nk[0:1], key_mask=mask, new_masked=new_masked)
        ops.attn_decode_dev(q, buf[..., :D], buf[..., D:], H, hd, hd ** -0.5, pos_nk[1:2], key_mask=mask,
                            slopes=slopes, out=out, workspace=ws)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    pos_nk.copy_(torch.tensor([p0, p0 + 1]))
    q.copy_(torch.randn(B, D, device="cuda", generator=g))
    src.copy_(torch.randn(B, 2 * D, device="cuda", generator=g))
    with torch.cuda.stream(s):
        step()   # warm-up at p0: the replay below writes the same row again
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        step()
    for p in range(p0, p0 + 41):
        if p > p0:
            q.copy_(torch.randn(B, D, device="cuda", generator=g))
            src.copy_(torch.randn(B, 2 * D, device="cuda", generator=g))
        new_masked.copy_(torch.tensor([0, 0, p % 3 == 0], dtype=torch.uint8))
        pos_nk[0:1].fill_(p)
        pos_nk[1:2].fill_(p + 1)
        graph.replay()
        ref_buf[:, p] = src
        ref_mask[:, p] = new_masked
        ref = ops.attn_decode(q, ref_buf[:, :p + 1, :D], ref_buf[:, :p + 1, D:], H, hd, hd ** -0.5,
                              key_mask=ref_mask, slopes=slopes)
        assert torch.equal(out, ref), p
        assert torch.equal(buf[:, :p + 1].view(torch.int16), ref_buf[:, :p + 1].view(torch.int16)), p
        assert torch.equal(mask, ref_mask), p


# --------------------------------------------------------------------------------------------- model level
CONFIGS = {"every1": (1, {}), "every2": (2, {}), "mpt1b-width": (1, dict(d_model=2048, n_heads=16)),
           "hd64": (1, dict(d_model=256, n_heads=4))}


def _model(config, seed=21):
    """test_kv_decode_gpu's _model at other LM widths: decisive logits, a left-padded batch of three prompts."""
    from open_flamingo_b200.testing import build_flamingo
    every, over = CONFIGS[config]
    model, _, tok = build_flamingo(VIT, dict(MPT, **over), cross_attn_every_n_layers=every, device="cuda",
                                   gate_init=1.0, seed=seed)
    with torch.no_grad():
        for name, p in model.lang_encoder.named_parameters():
            if "gated_cross_attn" in name or not name.startswith("transformer") or p.dim() != 2:
                continue
            p.copy_(torch.randn_like(p) * p.shape[1] ** -0.5)
        model.lang_encoder.get_input_embeddings().weight.normal_()
    return model, tok.encode("<image>")[-1]


def _inputs(media, seed, B=3, T=24):
    g = torch.Generator().manual_seed(seed)
    vision_x = torch.randn(B, 1, 1, 3, 56, 56, generator=g).cuda()
    lang_x = torch.randint(0, 90, (B, T), generator=g)
    att = torch.ones_like(lang_x)
    for b in range(B):
        pad = [6, 0, 3][b % 3]
        att[b, :pad] = 0
        lang_x[b, :pad] = 0
        lang_x[b, pad] = media
    return vision_x, lang_x.cuda(), att.cuda()


MODES = {"greedy": dict(do_sample=False), "sample": dict(do_sample=True, top_k=20),
         "beam": dict(do_sample=False, num_beams=3, length_penalty=0.0)}
NEW = 8


def _gen(model, inputs, mode, static, grad_off=torch.inference_mode):
    vision_x, lang_x, att = inputs
    kw = dict(MODES[mode])
    if static:
        kw["cache_implementation"] = "static"
    with grad_off(), torch.autocast("cuda", dtype=bf16):
        torch.manual_seed(123)
        return model.generate(vision_x=vision_x, lang_x=lang_x, attention_mask=att, max_new_tokens=NEW,
                              min_new_tokens=NEW, use_cache=True, output_logits=True, return_dict_in_generate=True,
                              pad_token_id=0, eos_token_id=None, **kw)


def _same(got, ref):
    assert torch.equal(got.sequences, ref.sequences), (got.sequences, ref.sequences)
    assert len(got.logits) == len(ref.logits) == NEW
    for i, (a, b) in enumerate(zip(got.logits, ref.logits)):
        assert torch.equal(a, b), f"step {i}: logits differ by {(a.float() - b.float()).abs().max().item():.3e}"


@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("config", sorted(CONFIGS))
def test_static_generate_replays_and_matches_eager(config, mode):
    model, media = _model(config)
    inputs = _inputs(media, 22)
    ref = _gen(model, inputs, mode, static=False)
    graphs = model.lang_encoder.decode_graphs
    r0 = graphs.replays
    with _count_calls() as calls:
        got = _gen(model, inputs, mode, static=True)
    assert graphs.error is None, repr(graphs.error)
    assert graphs.replays - r0 == NEW - 1, "every decode step after the prompt is a replay"
    assert calls["decode"] == 0 and calls["hf_attn"] == 0, calls
    _same(got, ref)
    cache = got.past_key_values
    assert cache.capacity == 64 and cache.layers[0].buf.shape[0] == 3 * MODES[mode].get("num_beams", 1)


def _rank_loop(model, inputs, cont, capacity):
    vision_x, lang_x, att = inputs
    full_att = torch.cat([att, torch.ones_like(cont)], 1)
    with torch.inference_mode(), torch.autocast("cuda", dtype=bf16):
        model.cache_media(input_ids=lang_x, vision_x=vision_x)
        cache = model.lang_encoder.make_kv_cache(capacity=capacity)
        out = model(vision_x=None, lang_x=lang_x, attention_mask=att, clear_conditioned_layers=False,
                    past_key_values=cache, use_cache=True)
        got = [out.logits]
        for t in range(cont.shape[1]):
            out = model(vision_x=None, lang_x=cont[:, t:t + 1], attention_mask=full_att[:, :lang_x.shape[1] + t + 1],
                        clear_conditioned_layers=False, past_key_values=out.past_key_values, use_cache=True)
            got.append(out.logits)
        model.uncache_media()
    return got


def test_rank_classification_loop_matches_eager_bitwise():
    model, media = _model("every1")
    inputs = _inputs(media, 22)
    cont = torch.randint(0, 90, (3, 6), generator=torch.Generator().manual_seed(5)).cuda()
    ref = _rank_loop(model, inputs, cont, None)
    graphs = model.lang_encoder.decode_graphs
    r0 = graphs.replays
    with _count_calls() as calls:
        got = _rank_loop(model, inputs, cont, 30)
    assert graphs.replays - r0 == cont.shape[1] and calls["decode"] == 0, calls
    for i, (a, b) in enumerate(zip(got, ref)):
        assert torch.equal(a, b), f"forward {i}"


def test_graph_reuse_new_batch_and_reload():
    model, media = _model("every1")
    graphs = model.lang_encoder.decode_graphs
    a, b = _inputs(media, 40), _inputs(media, 41)
    assert not torch.equal(a[1], b[1]) and not torch.equal(a[0], b[0])
    outs = [_gen(model, x, "greedy", static=True) for x in (a, b)]
    assert graphs.captures == 1, graphs.captures
    for x, o in zip((a, b), outs):   # the second call read its own media K/V, text_time, mask and cache rows
        _same(o, _gen(model, x, "greedy", static=False))
    # the first output's cache still holds its own rows after the second call took over the graph's buffers
    assert outs[0].past_key_values.layers[0].buf.data_ptr() != outs[1].past_key_values.layers[0].buf.data_ptr()
    small = tuple(t[:2] for t in a)
    _same(_gen(model, small, "greedy", static=True), _gen(model, small, "greedy", static=False))
    assert graphs.captures == 2, "another batch is another shape key"
    other, _ = _model("every1", seed=77)
    model.load_state_dict(other.state_dict())
    del other
    got = _gen(model, a, "greedy", static=True)
    assert graphs.captures == 3, "new weights re-capture"
    ref = _gen(model, a, "greedy", static=False)
    _same(got, ref)
    assert not torch.equal(torch.stack(got.logits), torch.stack(outs[0].logits)), "the new weights were used"


def test_inference_mode_and_no_grad_calls_alternate():
    """Buffers made under inference_mode cannot be written in place under no_grad: each mode has its own graph."""
    model, media = _model("every1")
    graphs = model.lang_encoder.decode_graphs
    a, b = _inputs(media, 50), _inputs(media, 51)
    for x, grad_off in ((a, torch.inference_mode), (b, torch.no_grad), (a, torch.no_grad), (b, torch.inference_mode)):
        r0 = graphs.replays
        got = _gen(model, x, "greedy", static=True, grad_off=grad_off)
        assert graphs.error is None and graphs.replays - r0 == NEW - 1, (grad_off, graphs.error)
        _same(got, _gen(model, x, "greedy", static=False, grad_off=grad_off))
    assert graphs.captures == 2, graphs.captures


def test_reused_cache_after_crop_reads_reloaded_weights():
    """The scoring pattern: one prefix in a fixed-capacity cache, cropped back to it for every continuation.  New
    weights loaded in place between two continuations: the crop starts a new call, so the parameter snapshot is
    checked and the graph re-captured, and the second continuation reads the new weights everywhere."""
    model, media = _model("every1")
    graphs = model.lang_encoder.decode_graphs
    vision_x, lang_x, att = _inputs(media, 22)
    T = lang_x.shape[1]
    cont = torch.randint(0, 90, (3, 4), generator=torch.Generator().manual_seed(8)).cuda()
    full_att = torch.cat([att, torch.ones_like(cont)], 1)

    def prefix(cache):
        with torch.inference_mode(), torch.autocast("cuda", dtype=bf16):
            model(vision_x=None, lang_x=lang_x, attention_mask=att, clear_conditioned_layers=False,
                  past_key_values=cache, use_cache=True)

    def steps(cache):
        got = []
        with torch.inference_mode(), torch.autocast("cuda", dtype=bf16):
            for t in range(cont.shape[1]):
                got.append(model(vision_x=None, lang_x=cont[:, t:t + 1], attention_mask=full_att[:, :T + t + 1],
                                 clear_conditioned_layers=False, past_key_values=cache, use_cache=True).logits)
        return got
    with torch.inference_mode(), torch.autocast("cuda", dtype=bf16):
        model.cache_media(input_ids=lang_x, vision_x=vision_x)
        ref_cache = model.lang_encoder.make_kv_cache()
        cache = model.lang_encoder.make_kv_cache(capacity=30)
    prefix(ref_cache)   # eager, growing cache: the reference continues from here under the new weights
    prefix(cache)
    first = steps(cache)
    assert graphs.captures == 1
    other, _ = _model("every1", seed=78)
    model.load_state_dict(other.state_dict())
    del other
    cache.crop(T)
    r0 = graphs.replays
    second = steps(cache)
    assert graphs.replays - r0 == cont.shape[1] and graphs.captures == 2
    ref = steps(ref_cache)
    model.uncache_media()
    for i, (x, y) in enumerate(zip(second, ref)):
        assert torch.equal(x, y), f"step {i}"
    assert not torch.equal(second[-1], first[-1]), "the new weights were used"


def test_static_capacity_follows_generation_config():
    from transformers import GenerationConfig
    model, media = _model("every1")
    vision_x, lang_x, att = _inputs(media, 22)
    gc = GenerationConfig(max_new_tokens=50, min_new_tokens=50, do_sample=False, pad_token_id=0)
    outs = []
    for static in (True, False):
        kw = dict(cache_implementation="static") if static else {}
        with torch.inference_mode(), torch.autocast("cuda", dtype=bf16):
            outs.append(model.generate(vision_x=vision_x, lang_x=lang_x, attention_mask=att, generation_config=gc,
                                       eos_token_id=None, use_cache=True, return_dict_in_generate=True,
                                       output_logits=True, **kw))
    got, ref = outs
    assert got.past_key_values.capacity == 128   # 24 + 50 rows: not the model's default max_length of 20
    assert torch.equal(got.sequences, ref.sequences) and got.sequences.shape[1] == 24 + 50
    assert all(torch.equal(x, y) for x, y in zip(got.logits, ref.logits))


@contextlib.contextmanager
def _clip_qkv(model):
    blk = model.lang_encoder.old_decoder_blocks[1]
    blk.attn.clip_qkv = 1e6   # never clips, but makes the block decline the kernels
    try:
        yield
    finally:
        blk.attn.clip_qkv = None


def test_ineligible_steps_run_eagerly_with_the_same_results():
    model, media = _model("every1")
    graphs = model.lang_encoder.decode_graphs
    inputs = _inputs(media, 22)
    with _clip_qkv(model):
        r0 = graphs.replays
        got = _gen(model, inputs, "greedy", static=True)
        assert graphs.replays == r0
        _same(got, _gen(model, inputs, "greedy", static=False))
    cont = torch.randint(0, 90, (3, 4), generator=torch.Generator().manual_seed(6)).cuda()
    vision_x, lang_x, att = inputs
    full_att = torch.cat([att, torch.ones_like(cont)], 1)

    def loop(capacity, grad=False, enabled=True, hidden=False):
        ctx = torch.enable_grad() if grad else torch.inference_mode()
        with ctx, torch.autocast("cuda", dtype=bf16):
            model.cache_media(input_ids=lang_x, vision_x=vision_x)
            cache = model.lang_encoder.make_kv_cache(capacity=capacity)
            out = model(vision_x=None, lang_x=lang_x, attention_mask=att, clear_conditioned_layers=False,
                        past_key_values=cache, use_cache=True)
            res = [out.logits.detach()]
            with _fast_lm(enabled):
                for t in range(cont.shape[1]):
                    kw = dict(output_hidden_states=True) if hidden else {}
                    out = model.lang_encoder(input_ids=cont[:, t:t + 1],
                                             attention_mask=full_att[:, :lang_x.shape[1] + t + 1],
                                             past_key_values=out.past_key_values, use_cache=True, **kw)
                    res.append(out.logits.detach())
            model.uncache_media()
        return res
    for kw in (dict(enabled=False), dict(hidden=True), dict(grad=True)):
        r0 = graphs.replays
        got, ref = loop(30, **kw), loop(None, **kw)
        assert graphs.replays == r0, kw
        assert all(torch.equal(x, y) for x, y in zip(got, ref)), kw


def test_overflow_raises_before_any_launch():
    from open_flamingo_b200 import _lib
    model, media = _model("every1")
    vision_x, lang_x, att = _inputs(media, 22)
    with torch.inference_mode(), torch.autocast("cuda", dtype=bf16):
        model.cache_media(input_ids=lang_x, vision_x=vision_x)
        cache = model.lang_encoder.make_kv_cache(capacity=lang_x.shape[1])   # 64 rows
        out = model(vision_x=None, lang_x=lang_x, attention_mask=att, clear_conditioned_layers=False,
                    past_key_values=cache, use_cache=True)
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        big = torch.zeros(3, 41, dtype=torch.long, device="cuda")
        with pytest.raises(ValueError):
            model(vision_x=None, lang_x=big, attention_mask=torch.ones(3, 65, dtype=torch.long, device="cuda"),
                  clear_conditioned_layers=False, past_key_values=out.past_key_values, use_cache=True)
        assert _lib.launch_count() == n0
        model.uncache_media()
