"""CPU: the host logic of lm_blocks.FastNeoXBlock -- accelerate() returns it for a GPTNeoXLayer, it declines every
call the kernels do not evaluate (the block's own PyTorch forward runs instead), and HF's sdpa mask (True = attend) is
turned into the kernels' bytes (nonzero = masked).  No kernel runs here: `supported` reads only hidden_states.is_cuda,
so a stand-in with is_cuda = True reaches every other check."""
import types

import pytest
import torch

CUDA_LIKE = types.SimpleNamespace(is_cuda=True)


def _layer(hd=80, heads=2, rot_pct=1.0, parallel=False, act="gelu", bias=True):
    from transformers import GPTNeoXConfig
    from transformers.models.gpt_neox.modeling_gpt_neox import GPTNeoXLayer
    cfg = GPTNeoXConfig(hidden_size=hd * heads, num_attention_heads=heads, num_hidden_layers=1,
                        intermediate_size=4 * hd * heads, vocab_size=32, use_parallel_residual=parallel,
                        hidden_act=act, attention_bias=bias)
    cfg.rope_parameters["partial_rotary_factor"] = rot_pct
    return GPTNeoXLayer(cfg, 0).eval().requires_grad_(False)


def _pe(T=5, rot=80, B=1, dtype=torch.float32):
    return torch.zeros(B, T, rot, dtype=dtype), torch.zeros(B, T, rot, dtype=dtype)


def test_accelerate_returns_the_neox_block():
    from open_flamingo_b200 import lm_blocks
    layer = _layer()
    fast = lm_blocks.accelerate(layer)
    assert isinstance(fast, lm_blocks.FastNeoXBlock) and fast.block is layer
    assert fast.supported(CUDA_LIKE, _pe(), False)
    assert fast.applicable(CUDA_LIKE, _pe(), None, False, False)
    assert fast.supported(CUDA_LIKE, _pe(rot=20), False)          # partial rotary
    assert lm_blocks.FastNeoXBlock(_layer(hd=64)).supported(CUDA_LIKE, _pe(rot=64), False)
    assert lm_blocks.FastNeoXBlock(_layer(hd=128)).supported(CUDA_LIKE, _pe(rot=32), False)
    assert lm_blocks.FastNeoXBlock(_layer(parallel=True)).supported(CUDA_LIKE, _pe(), False)


@pytest.mark.parametrize("case", ["cpu", "disabled", "output_attentions", "no_position_embeddings", "bf16_cos",
                                  "odd_rot", "rot_gt_hd", "head_dim_96", "hidden_act", "no_bias", "requires_grad",
                                  "dropout_training", "bad_scale", "bf16_weights"])
def test_declines(case):
    from open_flamingo_b200 import lm_blocks
    hd = 96 if case == "head_dim_96" else 80
    layer = _layer(hd=hd, act="gelu_new" if case == "hidden_act" else "gelu", bias=case != "no_bias")
    fast = lm_blocks.FastNeoXBlock(layer)
    hs, pe, oa = CUDA_LIKE, _pe(rot=hd), False
    prev = lm_blocks.ENABLED
    try:
        if case == "cpu":
            hs = torch.zeros(1, 5, 2 * hd)
        elif case == "disabled":
            lm_blocks.ENABLED = False
        elif case == "output_attentions":
            oa = True
        elif case == "no_position_embeddings":
            pe = None
        elif case == "bf16_cos":
            pe = _pe(dtype=torch.bfloat16)
        elif case == "odd_rot":
            pe = _pe(rot=21)
        elif case == "rot_gt_hd":
            pe = _pe(rot=hd + 2)
        elif case == "requires_grad":
            layer.mlp.dense_h_to_4h.weight.requires_grad_(True)   # not frozen: needs a wgrad this path lacks
        elif case == "dropout_training":
            layer.train()
            layer.attention.attention_dropout = 0.1
        elif case == "bad_scale":
            layer.attention.scaling = 128 ** -0.5
        elif case == "bf16_weights":
            layer.to(torch.bfloat16)
        assert not fast.supported(hs, pe, oa), case
        assert not fast.applicable(hs, pe, None, False, oa), case
        if case == "cpu":
            assert fast(hs, position_embeddings=pe) is None
    finally:
        lm_blocks.ENABLED = prev


def test_training_without_dropout_is_supported():
    from open_flamingo_b200 import lm_blocks
    layer = _layer().train()
    assert lm_blocks.FastNeoXBlock(layer).supported(CUDA_LIKE, _pe(), False)


def test_caches_other_than_kvcache_and_grad_mode_decline():
    from transformers import DynamicCache
    from open_flamingo_b200 import lm_blocks
    from open_flamingo_b200.kv_cache import KVCache
    fast = lm_blocks.FastNeoXBlock(_layer())
    assert not fast.applicable(CUDA_LIKE, _pe(), DynamicCache(), True, False)
    with torch.no_grad():
        assert fast.cache_layer(CUDA_LIKE, _pe(), DynamicCache(), False) is None
        assert fast.cache_layer(CUDA_LIKE, _pe(), KVCache(1), False) is not None
        assert fast.cache_layer(CUDA_LIKE, _pe(), KVCache(1), True) is None
    assert fast.cache_layer(CUDA_LIKE, _pe(), KVCache(1), False) is None   # gradient recorded


def test_sdpa_mask_polarity_and_decline_of_float_masks():
    from open_flamingo_b200 import lm_blocks
    B, T = 2, 6
    attend = torch.ones(T, T, dtype=torch.bool).tril().view(1, 1, T, T).expand(B, 1, T, T).clone()
    attend[1, :, :, :2] = False
    got = lm_blocks._kernel_mask(attend, B, T, T, False, true_attends=True)
    assert torch.equal(got.bool(), ~attend.view(B, T, T))
    step = attend[:, :, -1:, :]
    got = lm_blocks._kernel_mask(step, B, 1, T, True, true_attends=True)
    assert got.shape == (B, 8) and torch.equal(got[:, :T].bool(), ~step.view(B, T)) and not got[:, T:].any()
    assert lm_blocks._kernel_mask(torch.zeros(B, 1, T, T), B, T, T, False, true_attends=True) is None   # eager
    assert lm_blocks._kernel_mask(attend, B, T, T + 1, False, true_attends=True) is None


@pytest.mark.parametrize("case", ["kwarg_hidden_states", "kwarg_attentions", "config_hidden_states",
                                  "config_attentions"])
def test_declines_when_hf_records_layer_outputs(case):
    """GPTNeoXModel collects output_hidden_states / output_attentions with hooks on the GPTNeoXLayer and
    GPTNeoXAttention modules, which the fast path bypasses: such calls must run HF's layer, whether the request comes
    as a keyword or as the model config's default."""
    from open_flamingo_b200 import lm_blocks
    layer = _layer()
    fast = lm_blocks.FastNeoXBlock(layer)
    kw = {}
    if case.startswith("kwarg"):
        kw["output_" + case[len("kwarg_"):]] = True
    else:
        setattr(layer.attention.config, "output_" + case[len("config_"):], True)
    assert fast.records_outputs(kw.get("output_attentions"), kw.get("output_hidden_states"))
    assert fast(CUDA_LIKE, position_embeddings=_pe(), **kw) is None
    with torch.no_grad():
        from open_flamingo_b200.kv_cache import KVCache
        assert fast(CUDA_LIKE, position_embeddings=_pe(), layer_past=KVCache(1), use_cache=True, **kw) is None
    if case.startswith("config"):   # an explicit False overrides the config's default, as in HF's capture_outputs
        assert not fast.records_outputs(False, False)
        assert fast.supported(CUDA_LIKE, _pe(), fast.records_outputs(False, False))


def test_no_record_request_keeps_the_fast_path():
    from open_flamingo_b200 import lm_blocks
    fast = lm_blocks.FastNeoXBlock(_layer())
    assert not fast.records_outputs()
    assert fast.supported(CUDA_LIKE, _pe(), fast.records_outputs())
