"""CPU: graph-replayed decoding of GPT-NeoX LMs (OF-4B), without a GPU.

- ofk_rope_append_dev rejects bad arguments with the documented error code before it touches a device (as in
  test_rope_args_cpu.py: a child process with no CUDA device and made-up device addresses; a call whose arguments pass
  validation reaches the launch and returns OFK_ERR_CUDA, -3), and its kernel keeps everything in registers.
- decode_graph.eligible on CPU-built GPT-NeoX Flamingo LMs: a one-token step on a fixed-capacity cache is eligible, and
  each GPT-NeoX-specific reason to run the eager step instead declines it.  No kernel runs: eligible reads only
  `is_cuda`, the shapes and the device of the ids, which a stand-in provides.
- HF's generate does not pass position_ids to a Flamingo LM's one-token steps."""
import contextlib
import json
import os
import subprocess
import sys
import types

import pytest
import torch

from test_abi_cpu import _sass_by_kernel

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ARG, ALIGN, NO_DEVICE = -1, -2, -3
QKV, COS, SIN, Q, CACHE, POS, MASK, NEWM = (k << 32 for k in range(1, 9))
B, H, HD, ROT, CAP = 3, 4, 80, 80, 128
D = H * HD


def append_args(**kw):
    a = dict(qkv=QKV, qkv_bs=3 * D, batch=B, heads=H, head_dim=HD, rot=ROT, cos=COS, sin=SIN, cs_bs=0, q=Q, q_bs=D,
             cache=CACHE, cache_bs=CAP * 2 * D, ld=2 * D, capacity=CAP, pos=POS, mask=MASK, mask_bs=CAP,
             new_masked=NEWM, stream=0)
    a.update(kw)
    return list(a.values())


def _cases():
    c = {
        "valid": (append_args(), NO_DEVICE),
        "valid-partial-rot": (append_args(rot=20), NO_DEVICE),
        "valid-no-rotation": (append_args(rot=0, cos=0, sin=0), NO_DEVICE),
        "valid-per-row-cos": (append_args(cs_bs=ROT), NO_DEVICE),
        "valid-hd64": (append_args(head_dim=64, rot=64, qkv_bs=3 * H * 64, q_bs=H * 64, ld=2 * H * 64,
                                   cache_bs=CAP * 2 * H * 64), NO_DEVICE),
        "valid-hd128": (append_args(head_dim=128, rot=32, qkv_bs=3 * H * 128, q_bs=H * 128, ld=2 * H * 128,
                                    cache_bs=CAP * 2 * H * 128), NO_DEVICE),
        "valid-no-mask": (append_args(mask=0, mask_bs=0, new_masked=0), NO_DEVICE),
        "valid-no-new-masked": (append_args(new_masked=0), NO_DEVICE),
        "valid-odd-mask": (append_args(mask=MASK + 3, mask_bs=CAP + 1), NO_DEVICE),   # bytes: no alignment
        "valid-capacity1": (append_args(capacity=1, cache_bs=2 * D, mask_bs=8), NO_DEVICE),
        "valid-wide-rows": (append_args(qkv_bs=4 * D, q_bs=2 * D, ld=3 * D, cache_bs=CAP * 3 * D), NO_DEVICE),
        "rot-odd": (append_args(rot=21), ARG),
        "rot-gt-hd": (append_args(rot=HD + 2), ARG),
        "rot-neg": (append_args(rot=-2), ARG),
        "cos-missing": (append_args(cos=0), ARG),
        "sin-missing": (append_args(sin=0), ARG),
        "cs_bs-neg": (append_args(cs_bs=-ROT), ARG),
        "capacity0": (append_args(capacity=0), ARG),
        "capacity-neg": (append_args(capacity=-1), ARG),
        "hd-not-8": (append_args(head_dim=84, rot=84), ARG),
        "batch0": (append_args(batch=0), ARG),
        "heads0": (append_args(heads=0), ARG),
        "qkv-null": (append_args(qkv=0), ARG),
        "q-null": (append_args(q=0), ARG),
        "cache-null": (append_args(cache=0), ARG),
        "pos-null": (append_args(pos=0), ARG),
        "qkv_bs-short": (append_args(qkv_bs=3 * D - 8), ARG),
        "q_bs-short": (append_args(q_bs=D - 8), ARG),
        "ld-short": (append_args(ld=2 * D - 8, cache_bs=CAP * (2 * D - 8)), ARG),
        "cache_bs-short": (append_args(cache_bs=(CAP - 1) * 2 * D), ARG),
        "mask_bs-short": (append_args(mask_bs=CAP - 1), ARG),
        "pos+2B": (append_args(pos=POS + 2), ALIGN),
        "cos+2B": (append_args(cos=COS + 2), ALIGN),
        "sin+2B": (append_args(sin=SIN + 2), ALIGN),
    }
    for name, ptr in (("qkv", QKV), ("q", Q), ("cache", CACHE)):
        for off in (2, 8):
            c[f"{name}+{off}B"] = (append_args(**{name: ptr + off}), ALIGN)
    for name, base in (("qkv_bs", 3 * D), ("q_bs", D), ("cache_bs", CAP * 2 * D + 8)):
        c[f"{name}+4"] = (append_args(**{name: base + 4}), ALIGN)
    c["ld+4"] = (append_args(ld=2 * D + 4, cache_bs=CAP * (2 * D + 8)), ALIGN)
    return c


CASES = _cases()

CHILD = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
from open_flamingo_b200 import _lib
cases = json.load(sys.stdin)
lib = _lib.lib()
print(json.dumps({n: lib.ofk_rope_append_dev(*args) for n, (args, _) in cases.items()}))
"""


@pytest.fixture(scope="module")
def results():
    import __graft_entry__ as g
    g.build()
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", CHILD, ROOT]
    r = subprocess.run(cmd, input=json.dumps(CASES), capture_output=True, text=True, env=env, timeout=600)
    assert r.returncode == 0, r.stderr
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("case", sorted(CASES))
def test_rope_append_dev_return_code(results, case):
    got, want = results[case], CASES[case][1]
    assert got == want, f"{case}: returned {got}, expected {want} (-3 = the check ran after the launch or not at all)"


def test_rope_append_dev_kernel_uses_no_local_memory(results):
    kernels = _sass_by_kernel()
    names = [k for k in kernels if "rope_append_dev_kernel" in k]
    assert len(names) == 1, sorted(kernels)
    assert not kernels[names[0]] & {"LDL", "STL"}, f"{names[0]}: local-memory traffic"


# --------------------------------------------------------------------------------------------- eligibility
VIT = dict(image_size=56, patch_size=14, width=128, layers=1, heads=2, output_dim=128)
NEOX = dict(hidden_size=160, num_attention_heads=2, num_hidden_layers=2, intermediate_size=320, vocab_size=97,
            max_position_embeddings=256)
STEP_B, PAST = 3, 20


def _lm(every=2, **neox_over):
    from open_flamingo_b200.testing import build_flamingo
    model, _, _ = build_flamingo(VIT, None, neox_kw=dict(NEOX, **neox_over), cross_attn_every_n_layers=every,
                                 device="cpu", seed=3)
    return model.lang_encoder


def _step(lm):
    """A one-token step after a PAST-row prefill on a fixed-capacity cache, with the media conditioned."""
    from open_flamingo_b200.kv_cache import KVCache
    layers = lm._get_decoder_layers()
    a = layers[0].decoder_layer.attention
    cache = KVCache(len(layers), capacity=64)
    for cl in cache.layers:
        cl.init_storage(STEP_B, a.config.num_attention_heads, a.head_size, torch.bfloat16, "cpu")
        cl.length = PAST
    cache.ensure_key_mask(STEP_B, "cpu")
    for layer in layers:
        layer.condition_vis_x(torch.zeros(STEP_B, 1, 4, VIT["output_dim"]))
        layer.condition_media_locations(torch.zeros(STEP_B, PAST, dtype=torch.bool))
    ids = types.SimpleNamespace(is_cuda=True, shape=(STEP_B, 1), device=torch.device("cpu"), dim=lambda: 2)
    att = torch.ones(STEP_B, PAST + 1, dtype=torch.long)
    return ids, att, cache, dict(past_key_values=cache, use_cache=True, return_dict=True)


@contextlib.contextmanager
def _bf16_autocast_flags():
    """The state torch.autocast("cuda", dtype=torch.bfloat16) sets, without a device to check it against."""
    prev = torch.is_autocast_enabled("cuda"), torch.get_autocast_dtype("cuda")
    torch.set_autocast_enabled("cuda", True)
    torch.set_autocast_dtype("cuda", torch.bfloat16)
    try:
        yield
    finally:
        torch.set_autocast_enabled("cuda", prev[0])
        torch.set_autocast_dtype("cuda", prev[1])


def _eligible(lm, **kw_over):
    from open_flamingo_b200 import decode_graph
    ids, att, cache, kw = _step(lm)
    kw.update(kw_over)
    with torch.no_grad(), _bf16_autocast_flags():
        return decode_graph.eligible(lm, ids, att, cache, True, kw)


@pytest.fixture(scope="module")
def neox_lm():
    return _lm()


def test_one_token_neox_step_is_eligible(neox_lm):
    from open_flamingo_b200 import decode_graph, lm_blocks
    assert decode_graph._is_neox(neox_lm)
    layers = neox_lm._get_decoder_layers()
    assert all(isinstance(layer._fast_block, lm_blocks.FastNeoXBlock) for layer in layers)
    assert [layer.gated_cross_attn_layer is not None for layer in layers] == [False, True]
    assert _eligible(neox_lm)
    assert decode_graph._heads(layers[0]._fast_block) == (2, 80)


@pytest.mark.parametrize("case", ["position_ids", "output_hidden_states", "output_attentions",
                                  "config_output_hidden_states", "emb_dropout_training", "block_requires_grad",
                                  "block_dropout_training", "kernels_disabled", "wrong_head_layout"])
def test_neox_declines(neox_lm, case):
    from open_flamingo_b200 import lm_blocks
    lm = neox_lm
    kw = {}
    undo = []
    blk = lm._get_decoder_layers()[1].decoder_layer
    if case == "position_ids":
        kw["position_ids"] = torch.full((1, 1), PAST)
    elif case in ("output_hidden_states", "output_attentions"):
        kw[case] = True
    elif case == "config_output_hidden_states":
        lm.config.output_hidden_states = True
        undo.append(lambda: setattr(lm.config, "output_hidden_states", False))
    elif case == "emb_dropout_training":
        drop = lm.gpt_neox.emb_dropout
        drop.train()
        drop.p = 0.1
        undo.append(lambda: (drop.eval(), setattr(drop, "p", 0.0)))
    elif case == "block_requires_grad":
        blk.mlp.dense_h_to_4h.weight.requires_grad_(True)
        undo.append(lambda: blk.mlp.dense_h_to_4h.weight.requires_grad_(False))
    elif case == "block_dropout_training":
        blk.train()
        blk.attention.attention_dropout = 0.1
        undo.append(lambda: (blk.eval(), setattr(blk.attention, "attention_dropout", 0.0)))
    elif case == "kernels_disabled":
        lm_blocks.ENABLED = False
        undo.append(lambda: setattr(lm_blocks, "ENABLED", True))
    try:
        if case == "wrong_head_layout":
            ids, att, cache, kwargs = _step(lm)
            for cl in cache.layers:
                cl.init_storage(STEP_B, 4, 40, torch.bfloat16, "cpu")   # same width, other heads
                cl.length = PAST
            from open_flamingo_b200 import decode_graph
            with torch.no_grad(), _bf16_autocast_flags():
                assert not decode_graph.eligible(lm, ids, att, cache, True, kwargs)
        else:
            assert not _eligible(lm, **kw), case
    finally:
        for f in undo:
            f()
    assert _eligible(lm), f"{case}: not undone"


def test_emb_dropout_of_zero_in_training_mode_stays_eligible(neox_lm):
    drop = neox_lm.gpt_neox.emb_dropout
    assert drop.p == 0.0
    drop.train()
    try:
        assert _eligible(neox_lm)
    finally:
        drop.eval()


def test_non_default_rope_type_declines():
    lm = _lm(rope_parameters=dict(rope_type="dynamic", factor=2.0, rope_theta=10000.0))
    assert lm.config.rope_parameters["rope_type"] == "dynamic" and lm.gpt_neox.rotary_emb.rope_type == "dynamic"
    assert not _eligible(lm)


def test_generate_passes_no_position_ids_to_one_token_steps():
    """GenerationMixin adds position_ids only when the model's forward names them; FlamingoLMMixin.forward does not,
    so a one-token step carries only keywords decode_graph accepts."""
    import inspect
    from open_flamingo_b200 import decode_graph
    from open_flamingo_b200.kv_cache import KVCache
    lm = _lm(every=3)   # no gated layer: HF's blocks run on the CPU without media
    assert "position_ids" not in inspect.signature(lm.forward).parameters
    seen = []
    handle = lm.register_forward_pre_hook(lambda mod, args, kwargs: seen.append((args, dict(kwargs))), with_kwargs=True)
    try:
        ids = torch.randint(0, 90, (2, 7), generator=torch.Generator().manual_seed(1))
        att = torch.ones_like(ids)
        att[0, :2] = 0
        with torch.no_grad():
            lm.generate(input_ids=ids, attention_mask=att, past_key_values=KVCache(2, capacity=16), use_cache=True,
                        max_new_tokens=4, min_new_tokens=4, do_sample=False, pad_token_id=0, eos_token_id=None)
    finally:
        handle.remove()
    steps = [kw for _, kw in seen if kw["input_ids"].shape[1] == 1]
    assert len(steps) == 3, len(seen)
    for kw in steps:
        assert "position_ids" not in kw, sorted(kw)
        assert set(kw) - {"input_ids", "attention_mask"} <= decode_graph._STEP_KWARGS, sorted(kw)
