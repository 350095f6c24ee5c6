"""GPU: graph-replayed decoding of GPT-NeoX LMs (OF-4B) is the eager cached decode, bit for bit.

1. ofk_rope_append_dev equals ofk_rope_pack into the cache row plus ofk_kv_append's mask byte, bit for bit (head_dim
   64, 80 and 128, full and partial rotary, shared and per-row cos/sin, positions 0, mid and capacity - 1), with NaN
   canary rows and columns; a position outside [0, capacity) writes q only.
2. ofk_attn_decode_dev at head_dim 80 equals ofk_attn_decode at the same nk, whatever nk_max.
3. One CUDA graph of (rope_append_dev + attn_decode_dev) replayed at positions p .. p + 40 equals the eager launches.
4. generate(cache_implementation="static") against the growing-KVCache eager path: every one-token step replayed, no
   eager decode attention or rotary packing during it, the same sequences and bit-identical logits at every step --
   greedy, seeded sampling, 3 beams, a left-padded batch of three, at head_dim 64, 80 and 128, quarter rotary and the
   parallel residual.
5. The rank-classification loop with make_kv_cache(capacity=...) gives the eager loop's logits bit for bit.
6. A graph is reused across calls of one shape key, captured anew for another batch and after load_state_dict; calls
   alternating between inference_mode and no_grad each match eager.
7. Calls the graph declines (output_hidden_states, a dynamic rope type) run eagerly with the eager results.
8. At OF-4B's LM dims (32 layers, D 2560, 32 heads of 80, a gated block before every 2nd layer), greedy B = 1: the
   graph equals eager bit for bit."""
import contextlib

import pytest
import torch

from test_decode_graph_gpu import _decode_inputs, _nan_ws
from test_neox_block_gpu import VIT, _fast_lm

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
i16 = torch.int16


# --------------------------------------------------------------------------------------------- kernels
def _tables(rows, rot, g):
    ang = torch.rand(rows, 1, rot, device="cuda", generator=g) * 12 - 6
    return ang.cos(), ang.sin()


@pytest.mark.parametrize("hd,rot", [(64, 64), (80, 80), (80, 20), (128, 128), (128, 32)])
@pytest.mark.parametrize("per_row", [False, True])
def test_rope_append_dev_equals_rope_pack_into_the_row(hd, rot, per_row):
    from open_flamingo_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(hd + rot + per_row)
    B, H, cap = 3, 4, 70
    D = H * hd
    qkv = torch.randn(B, 3 * D, device="cuda", generator=g).to(bf16)
    cos, sin = _tables(B if per_row else 1, rot, g)
    # NaN canaries: every row but the written one, and 16 columns past each row
    buf = torch.full((B, cap, 2 * D + 16), float("nan"), device="cuda", dtype=bf16)
    cache = buf[:, :, :2 * D]
    mask = torch.randint(0, 256, (B, 72), device="cuda", generator=g).to(torch.uint8)
    new_masked = torch.tensor([0, 7, 1], device="cuda", dtype=torch.uint8)
    exp_q, _, _ = ops.rope_pack(qkv.view(B, 1, 3 * D), H, hd, cos, sin)
    for pos in (0, cap // 2, cap - 1):
        b0, m0 = buf.clone(), mask.clone()
        q = ops.rope_append_dev(qkv, H, hd, cos, sin, cache, torch.tensor([pos], device="cuda", dtype=torch.int32),
                                key_mask=mask, new_masked=new_masked)
        exp = b0.clone()
        row = exp[:, pos:pos + 1, :2 * D]
        ops.rope_pack(qkv.view(B, 1, 3 * D), H, hd, cos, sin, q_width=hd, k=row[..., :D], v=row[..., D:])
        mexp = m0.clone()
        mexp[:, pos] = torch.tensor([0, 1, 1], device="cuda", dtype=torch.uint8)
        assert torch.equal(q.view(i16), exp_q.view(B, D).view(i16)), pos
        assert torch.equal(buf.view(i16), exp.view(i16)), pos
        assert torch.equal(mask, mexp), pos
        ops.rope_append_dev(qkv, H, hd, cos, sin, cache, torch.tensor([pos], device="cuda", dtype=torch.int32),
                            key_mask=mask)
        mexp[:, pos] = 0
        assert torch.equal(mask, mexp) and torch.equal(buf.view(i16), exp.view(i16)), f"{pos}: NULL new_masked"
    for pos in (cap, cap + 100, -1):
        b0, m0 = buf.clone(), mask.clone()
        q = ops.rope_append_dev(qkv, H, hd, cos, sin, cache, torch.tensor([pos], device="cuda", dtype=torch.int32),
                                key_mask=mask, new_masked=new_masked)
        assert torch.equal(q.view(i16), exp_q.view(B, D).view(i16)), pos
        assert torch.equal(buf.view(i16), b0.view(i16)) and torch.equal(mask, m0), pos


@pytest.mark.parametrize("B,H", [(1, 32), (3, 32), (24, 32)])
@pytest.mark.parametrize("nk", [1, 63, 65, 300, 2049, 4097])
def test_decode_dev_bitwise_equals_decode_head_dim_80(B, H, nk):
    from open_flamingo_b200 import ops
    hd = 80
    D = H * hd
    for nk_max in (nk, 8192):
        for i, mask_kind in enumerate(("none", "pad", "full")):
            q, buf, _, mask = _decode_inputs(B, H, hd, nk, nk_max, False, mask_kind, 31 * nk + 7 * i + B)
            ref = ops.attn_decode(q, buf[:, :nk, :D], buf[:, :nk, D:], H, hd, hd ** -0.5, key_mask=mask)
            nk_dev = torch.tensor([nk], device="cuda", dtype=torch.int32)
            got = ops.attn_decode_dev(q, buf[:, :nk_max, :D], buf[:, :nk_max, D:], H, hd, hd ** -0.5, nk_dev,
                                      key_mask=mask, workspace=_nan_ws(B, H, hd, nk_max))
            assert torch.equal(got, ref), f"B{B} H{H} nk{nk} nk_max{nk_max} mask={mask_kind}"


def test_replayed_rope_append_and_decode_match_eager_launches():
    from open_flamingo_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(5)
    B, H, hd, rot, cap, p0 = 3, 32, 80, 80, 256, 150
    D = H * hd
    buf = torch.full((B, cap, 2 * D), float("nan"), device="cuda", dtype=bf16)
    buf[:, :p0] = torch.randn(B, p0, 2 * D, device="cuda", generator=g).to(bf16)
    mask = torch.zeros(B, cap, device="cuda", dtype=torch.uint8)
    mask[1, :9] = 1
    ref_buf, ref_mask = buf.clone(), mask.clone()
    qkv = torch.empty(B, 3 * D, device="cuda", dtype=bf16)
    cos, sin = torch.empty(1, 1, rot, device="cuda"), torch.empty(1, 1, rot, device="cuda")
    new_masked = torch.zeros(B, device="cuda", dtype=torch.uint8)
    pos_nk = torch.zeros(2, device="cuda", dtype=torch.int32)
    ws = ops.decode_workspace(torch.device("cuda"), B, H, hd, cap)
    q, out = torch.empty(B, D, device="cuda", dtype=bf16), torch.empty(B, D, device="cuda", dtype=bf16)

    def step():
        ops.rope_append_dev(qkv, H, hd, cos, sin, buf, pos_nk[0:1], key_mask=mask, new_masked=new_masked, q=q)
        ops.attn_decode_dev(q, buf[..., :D], buf[..., D:], H, hd, hd ** -0.5, pos_nk[1:2], key_mask=mask, out=out,
                            workspace=ws)

    def new_inputs(p):
        qkv.copy_(torch.randn(B, 3 * D, device="cuda", generator=g))
        c, s = _tables(1, rot, g)
        cos.copy_(c)
        sin.copy_(s)
        new_masked.copy_(torch.tensor([0, 0, p % 3 == 0], dtype=torch.uint8))
        pos_nk.copy_(torch.tensor([p, p + 1], dtype=torch.int32))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    new_inputs(p0)
    with torch.cuda.stream(s):
        step()   # warm-up at p0: the replay below writes the same row again
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        step()
    for p in range(p0, p0 + 41):
        if p > p0:
            new_inputs(p)
        graph.replay()
        rq, _, _ = ops.rope_pack(qkv.view(B, 1, 3 * D), H, hd, cos, sin, k=ref_buf[:, p:p + 1, :D],
                                 v=ref_buf[:, p:p + 1, D:])
        ref_mask[:, p] = new_masked
        ref = ops.attn_decode(rq.view(B, D), ref_buf[:, :p + 1, :D], ref_buf[:, :p + 1, D:], H, hd, hd ** -0.5,
                              key_mask=ref_mask)
        assert torch.equal(q, rq.view(B, D)) and torch.equal(out, ref), p
        assert torch.equal(buf[:, :p + 1].view(i16), ref_buf[:, :p + 1].view(i16)), p
        assert torch.equal(mask, ref_mask), p


# --------------------------------------------------------------------------------------------- model level
BASE = dict(hidden_size=320, num_attention_heads=4, num_hidden_layers=4, intermediate_size=1280, vocab_size=97,
            max_position_embeddings=256)
CONFIGS = {"hd80": (2, {}),
           "hd64-quarter-rot": (1, dict(hidden_size=256, intermediate_size=1024, rotary_pct=0.25)),
           "hd128-parallel": (2, dict(hidden_size=256, num_attention_heads=2, intermediate_size=1024,
                                      use_parallel_residual=True, rotary_pct=0.5))}


def _model(config="hd80", seed=21, **over):
    """test_neox_block_gpu._model at other LM shapes: decisive logits, media before every row's text."""
    from open_flamingo_b200.testing import build_flamingo
    every, kw = CONFIGS[config]
    model, _, tok = build_flamingo(VIT, None, neox_kw=dict(BASE, **kw, **over), cross_attn_every_n_layers=every,
                                   device="cuda", gate_init=1.0, seed=seed)
    with torch.no_grad():
        for name, p in model.lang_encoder.named_parameters():
            if "gated_cross_attn" in name or not name.startswith("gpt_neox.layers") or p.dim() != 2:
                continue
            p.copy_(torch.randn_like(p) * p.shape[1] ** -0.5)
        model.lang_encoder.get_input_embeddings().weight.normal_()
        model.lang_encoder.get_output_embeddings().weight.copy_(model.lang_encoder.get_input_embeddings().weight)
    return model, tok.encode("<image>")[-1]


def _inputs(media, seed, B=3, T=24):
    """A left-padded batch (pads 6, 0, 3, as test_neox_block_gpu._model) with <image> first in every row."""
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


def _gen(model, inputs, mode, static, grad_off=torch.inference_mode, new=NEW, **extra):
    vision_x, lang_x, att = inputs
    kw = dict(MODES[mode], **extra)
    if static:
        kw["cache_implementation"] = "static"
    with grad_off(), torch.autocast("cuda", dtype=bf16):
        torch.manual_seed(123)
        return model.generate(vision_x=vision_x, lang_x=lang_x, attention_mask=att, max_new_tokens=new,
                              min_new_tokens=new, use_cache=True, output_logits=True, return_dict_in_generate=True,
                              pad_token_id=0, eos_token_id=None, **kw)


def _same(got, ref, new=NEW):
    assert torch.equal(got.sequences, ref.sequences), (got.sequences, ref.sequences)
    assert len(got.logits) == len(ref.logits) == new
    for i, (a, b) in enumerate(zip(got.logits, ref.logits)):
        assert torch.equal(a, b), f"step {i}: logits differ by {(a.float() - b.float()).abs().max().item():.3e}"


@contextlib.contextmanager
def _count_calls():
    """Counts eager ops.attn_decode and ops.rope_pack calls and HF GPTNeoXAttention.forward calls."""
    from transformers.models.gpt_neox import modeling_gpt_neox as M
    from open_flamingo_b200 import ops
    n = {"decode": 0, "rope_pack": 0, "hf_attn": 0}
    saved = ops.attn_decode, ops.rope_pack, M.GPTNeoXAttention.forward

    def counted(key, fn):
        def w(*a, **k):
            n[key] += 1
            return fn(*a, **k)
        return w
    ops.attn_decode, ops.rope_pack = counted("decode", saved[0]), counted("rope_pack", saved[1])
    M.GPTNeoXAttention.forward = counted("hf_attn", saved[2])
    try:
        yield n
    finally:
        ops.attn_decode, ops.rope_pack, M.GPTNeoXAttention.forward = saved


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
    # the prompt is the only eager step: per block one rope_pack (two at head_dim 80, whose cached rows the prompt's
    # dense attention reads padded), no decode attention, no HF attention
    kw = dict(BASE, **CONFIGS[config][1])
    per_block = 1 if kw["hidden_size"] // kw["num_attention_heads"] in (64, 128) else 2
    assert calls == {"decode": 0, "rope_pack": per_block * kw["num_hidden_layers"], "hf_attn": 0}, calls
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
    model, media = _model("hd80")
    inputs = _inputs(media, 22)
    cont = torch.randint(0, 90, (3, 6), generator=torch.Generator().manual_seed(5)).cuda()
    ref = _rank_loop(model, inputs, cont, None)
    graphs = model.lang_encoder.decode_graphs
    r0 = graphs.replays
    with _count_calls() as calls:
        got = _rank_loop(model, inputs, cont, 30)
    assert graphs.error is None and graphs.replays - r0 == cont.shape[1] and calls["decode"] == 0, calls
    for i, (a, b) in enumerate(zip(got, ref)):
        assert torch.equal(a, b), f"forward {i}"


def test_graph_reuse_new_batch_and_reload():
    model, media = _model("hd80")
    graphs = model.lang_encoder.decode_graphs
    a, b = _inputs(media, 40), _inputs(media, 41)
    outs = [_gen(model, x, "greedy", static=True) for x in (a, b)]
    assert graphs.captures == 1, graphs.captures
    for x, o in zip((a, b), outs):   # the second call read its own media K/V, text_time, mask, positions and rows
        _same(o, _gen(model, x, "greedy", static=False))
    small = tuple(t[:2] for t in a)
    _same(_gen(model, small, "greedy", static=True), _gen(model, small, "greedy", static=False))
    assert graphs.captures == 2, "another batch is another shape key"
    other, _ = _model("hd80", seed=77)
    model.load_state_dict(other.state_dict())
    del other
    got = _gen(model, a, "greedy", static=True)
    assert graphs.captures == 3, "new weights re-capture"
    _same(got, _gen(model, a, "greedy", static=False))
    assert not torch.equal(torch.stack(got.logits), torch.stack(outs[0].logits)), "the new weights were used"


def test_inference_mode_and_no_grad_calls_alternate():
    model, media = _model("hd80")
    graphs = model.lang_encoder.decode_graphs
    a, b = _inputs(media, 50), _inputs(media, 51)
    for x, grad_off in ((a, torch.inference_mode), (b, torch.no_grad), (a, torch.no_grad), (b, torch.inference_mode)):
        r0 = graphs.replays
        got = _gen(model, x, "greedy", static=True, grad_off=grad_off)
        assert graphs.error is None and graphs.replays - r0 == NEW - 1, (grad_off, graphs.error)
        _same(got, _gen(model, x, "greedy", static=False, grad_off=grad_off))
    assert graphs.captures == 2, graphs.captures


def test_declined_calls_run_eagerly_with_unchanged_results():
    model, media = _model("hd80")
    graphs = model.lang_encoder.decode_graphs
    inputs = _inputs(media, 22)
    r0 = graphs.replays
    got = _gen(model, inputs, "greedy", static=True, output_hidden_states=True)
    assert graphs.replays == r0 and graphs.captures == 0
    ref = _gen(model, inputs, "greedy", static=False, output_hidden_states=True)
    _same(got, ref)
    assert len(got.hidden_states) == NEW
    # a dynamic rope type recomputes its tables from a host-side length: such a model always decodes eagerly
    dyn, media = _model("hd80", rope_parameters=dict(rope_type="dynamic", factor=2.0, rope_theta=10000.0))
    assert dyn.lang_encoder.gpt_neox.rotary_emb.rope_type == "dynamic"
    with _count_calls() as calls:
        got = _gen(dyn, inputs, "greedy", static=True)
    g = dyn.lang_encoder.decode_graphs
    assert g.replays == 0 and g.captures == 0 and g.error is None
    assert calls["decode"] == BASE["num_hidden_layers"] * (NEW - 1) and calls["hf_attn"] == 0, calls
    _same(got, _gen(dyn, inputs, "greedy", static=False))


def test_of4b_dims_greedy_graph_equals_eager():
    from open_flamingo_b200.testing import NEOX_3B, build_flamingo
    model, _, tok = build_flamingo(VIT, None, neox_kw=NEOX_3B, cross_attn_every_n_layers=2, device="cuda",
                                   gate_init=1.0, seed=4)
    model.eval()
    assert sum(layer is not None for layer in model.lang_encoder.gated_cross_attn_layers) == 16
    media = tok.encode("<image>")[-1]
    vision_x, lang_x, att = _inputs(media, 30, B=1, T=20)
    graphs = model.lang_encoder.decode_graphs
    with _fast_lm(True):
        ref = _gen(model, (vision_x, lang_x, att), "greedy", static=False, new=5)
        got = _gen(model, (vision_x, lang_x, att), "greedy", static=True, new=5)
    assert graphs.error is None and graphs.replays == 4, (graphs.replays, graphs.error)
    _same(got, ref, new=5)
