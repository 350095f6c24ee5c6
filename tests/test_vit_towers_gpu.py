"""GPU: the LaION vision towers on the kernels -- head widths 80 (ViT-H/14), 88 (ViT-g/14) and 104 (ViT-bigG/14) run the
head_dim-128 dense core on zero-padded heads (vit.py).

  * each tower at full depth, 4 images at 224 px (257 tokens), against the oracle's vit_forward (flamingo.py:195 call
    site) under the rule of test_fullsize_parity_gpu.test_vit_l14_full_depth_257_tokens;
  * small towers at head_dim 80, 88, 104 and 128 at 224, 336 and 378 px (257, 577 and 730 tokens, so the last key tile
    is partial), against float64 and autocast restatements, with sharp attention so that a wrong scale or a padding
    column that is not zero would show;
  * dispatch: head_dim 64 keeps the media core, any other head_dim packs once and runs the dense core once per layer,
    and no torch attention runs; two forwards give the same bits;
  * Flamingo end to end with a ViT-H/14-width tower and with a ViT-bigG/14-width one (the Perceiver and the gated
    blocks' to_kv at Dv = 1280 and 1664): logits, loss and every trainable gradient under the three-way rule of
    test_fullsize_parity_gpu.py;
  * create_model_and_transforms with each tower name builds a model whose training step and generate run.
Tolerances, err = ||x - ref||_2 / ||ref||_2: err(ours, ref) <= 2 err(amp, ref) + 1e-3 and cosine >= 0.999."""
import contextlib

import pytest
import torch

from test_fullsize_parity_gpu import _NoTF32, _batch, _compare, _cos, _oracle_of, _rel, _three_ways

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16


def _cfg(name):
    from open_flamingo_b200 import testing as T
    return {"ViT-H-14": T.VIT_H14, "ViT-g-14": T.VIT_G14, "ViT-bigG-14": T.VIT_BIGG14}[name]


def _check(tag, ours, amp, ref):
    e_ours, e_amp, cos = _rel(ours, ref), _rel(amp.float(), ref), _cos(ours, ref)
    print(f"[{tag}] err ours {e_ours:.3e} / amp {e_amp:.3e}; cos {cos:.6f}")
    assert e_ours <= 2.0 * e_amp + 1e-3 and cos >= 0.999, (tag, e_ours, e_amp, cos)


@pytest.mark.parametrize("name,layers", [("ViT-H-14", 32), ("ViT-g-14", 40), ("ViT-bigG-14", 48)])
def test_laion_tower_full_depth_257_tokens(name, layers):
    from open_flamingo_b200.src.vit import VisionTransformer
    from oracle import flamingo_oracle as O
    cfg = _cfg(name)
    assert cfg["layers"] == layers and cfg["quick_gelu"] is False
    torch.manual_seed(2)
    with torch.device("cuda"):
        vit = VisionTransformer(**cfg, output_tokens=True)
    x = torch.randn(4, 3, 224, 224, device="cuda")
    sd = {k: v.detach().float() for k, v in vit.state_dict().items()}
    with torch.no_grad(), _NoTF32():
        pooled_ref, tok_ref = O.vit_forward(x, sd, "", heads=16, patch=14, quick_gelu=False)
        with torch.autocast("cuda", dtype=bf16):
            pooled_amp, tok_amp = O.vit_forward(x, sd, "", heads=16, patch=14, quick_gelu=False)
        pooled, tok = vit(x)
    assert tok.shape == (4, 256, cfg["width"]) and pooled.shape == (4, cfg["output_dim"])
    _check(f"{name} tokens", tok, tok_amp, tok_ref)
    _check(f"{name} pooled", pooled, pooled_amp, pooled_ref)
    del vit, sd
    torch.cuda.empty_cache()


def _small_tower(hd, image_size, heads=4, layers=2, seed=0):
    """A tower of `heads` heads of width hd whose in_proj is scaled up so that the attention is sharp."""
    from open_flamingo_b200.src.vit import VisionTransformer
    torch.manual_seed(seed)
    with torch.device("cuda"):
        vit = VisionTransformer(image_size=image_size, patch_size=14, width=heads * hd, layers=layers, heads=heads,
                                output_dim=64, quick_gelu=False, output_tokens=True)
    with torch.no_grad():
        for blk in vit.transformer.resblocks:
            blk.attn.in_proj_weight.mul_(2.0)
            blk.attn.in_proj_bias.normal_(0.0, 0.5)
            blk.attn.out_proj.bias.normal_(0.0, 0.5)
    return vit


@pytest.mark.parametrize("image_size", [224, 336, 378])
@pytest.mark.parametrize("hd", [80, 88, 104, 128])
def test_small_towers_against_float64(hd, image_size):
    from oracle import flamingo_oracle as O
    vit = _small_tower(hd, image_size)
    x = torch.randn(2, 3, image_size, image_size, device="cuda")
    sd = {k: v.detach().float() for k, v in vit.state_dict().items()}
    sd64 = {k: v.double() for k, v in sd.items()}
    with torch.no_grad():
        pooled_ref, tok_ref = O.vit_forward(x.double(), sd64, "", heads=4, patch=14, quick_gelu=False)
        with torch.autocast("cuda", dtype=bf16):
            pooled_amp, tok_amp = O.vit_forward(x, sd, "", heads=4, patch=14, quick_gelu=False)
        pooled, tok = vit(x)
    g = (image_size // 14) ** 2
    assert tok.shape == (2, g, 4 * hd)
    _check(f"hd {hd} {g + 1} tokens", tok, tok_amp, tok_ref)
    _check(f"hd {hd} {g + 1} pooled", pooled, pooled_amp, pooled_ref)


@contextlib.contextmanager
def _count_calls():
    """Counts ops.attn_fwd, ops.attn_dense_fwd and ops.rope_pack calls and torch's scaled_dot_product_attention."""
    from open_flamingo_b200 import ops
    F = torch.nn.functional
    n = {"attn_fwd": 0, "attn_dense_fwd": 0, "rope_pack": 0, "sdpa": 0}
    saved = ops.attn_fwd, ops.attn_dense_fwd, ops.rope_pack, F.scaled_dot_product_attention

    def counted(key, fn):
        def w(*a, **k):
            n[key] += 1
            return fn(*a, **k)
        return w
    ops.attn_fwd, ops.attn_dense_fwd, ops.rope_pack = (counted("attn_fwd", saved[0]),
                                                      counted("attn_dense_fwd", saved[1]),
                                                      counted("rope_pack", saved[2]))
    F.scaled_dot_product_attention = counted("sdpa", saved[3])
    try:
        yield n
    finally:
        ops.attn_fwd, ops.attn_dense_fwd, ops.rope_pack, F.scaled_dot_product_attention = saved


@pytest.mark.parametrize("hd", [64, 80, 104])
def test_dispatch_and_repeatability(hd):
    layers = 3
    vit = _small_tower(hd, 224, layers=layers)
    x = torch.randn(3, 3, 224, 224, device="cuda")
    with _count_calls() as calls, torch.autocast("cuda", dtype=bf16):
        pooled, tok = vit(x)
        pooled2, tok2 = vit(x)
    per_forward = {k: v // 2 for k, v in calls.items()}
    if hd == 64:
        assert per_forward == {"attn_fwd": layers, "attn_dense_fwd": 0, "rope_pack": 0, "sdpa": 0}, calls
    else:
        assert per_forward == {"attn_fwd": 0, "attn_dense_fwd": layers, "rope_pack": layers, "sdpa": 0}, calls
    assert torch.equal(tok, tok2) and torch.equal(pooled, pooled2), "two forwards differ"


@pytest.mark.parametrize("tower", ["ViT-H-14", "ViT-bigG-14"])
def test_flamingo_with_wide_tower_three_way(tower):
    from open_flamingo_b200.testing import MPT_1B, build_flamingo
    vit_cfg = dict(_cfg(tower), layers=4)
    model, _, tok = build_flamingo(vit_cfg, MPT_1B, cross_attn_every_n_layers=1, device="cuda", gate_init=1.0, seed=0)
    model.train()
    assert model.perceiver.latents.shape[-1] == vit_cfg["width"]
    orc, sd, trainable = _oracle_of(model, 1)
    orc.quick_gelu = False
    assert any(k.startswith("perceiver.") for k in trainable)
    assert any(".to_kv." in k and k.startswith("lang_encoder.gated_cross_attn_layers.") for k in trainable)
    runs = (_three_ways(model, orc, sd, trainable, _batch(tok, 2, 2, 64, MPT_1B["vocab_size"], seed=s))
            for s in (3, 13))
    _compare(f"Flamingo {tower}-width tower 2x(2 img, 64 tok)", runs, trainable)
    del model, orc, sd
    torch.cuda.empty_cache()


@pytest.mark.parametrize("name", ["ViT-H-14", "ViT-g-14", "ViT-bigG-14"])
def test_create_model_and_transforms_runs(name):
    from open_flamingo_b200.src.factory import create_model_and_transforms
    from open_flamingo_b200.testing import SimpleTokenizer, build_mpt, synthetic_batch
    mpt_kw = dict(d_model=256, n_heads=4, n_layers=2, vocab_size=101, max_seq_len=128, expansion_ratio=4)
    lm = build_mpt(mpt_kw, device="cuda", seed=1)
    with torch.device("cuda"):
        model, _, tok = create_model_and_transforms(name, None, lm, SimpleTokenizer(101),
                                                    cross_attn_every_n_layers=1)
    model = model.cuda()
    media_id, eoc_id = tok.encode("<image>")[-1], tok.encode("<|endofchunk|>")[-1]
    b = {k: v.cuda() for k, v in synthetic_batch(2, 1, 16, media_id, eoc_id, 101, seed=4).items()}
    visual = model.vision_encoder
    in_tower = dict.fromkeys(("attn_fwd", "attn_dense_fwd", "rope_pack", "sdpa"), 0)
    with _count_calls() as calls:
        # count only inside the tower: the Perceiver, the gated blocks and the LM run attention of their own
        before = {}
        hooks = (visual.register_forward_pre_hook(lambda m, a: before.update(calls)),
                 visual.register_forward_hook(
                     lambda m, a, o: in_tower.update({k: in_tower[k] + calls[k] - before[k] for k in in_tower})))
        model.train()
        with torch.autocast("cuda", dtype=bf16):
            out = model(vision_x=b["vision_x"], lang_x=b["lang_x"], attention_mask=b["attention_mask"],
                        labels=b["labels"])
        out.loss.backward()
        assert torch.isfinite(out.loss)
        grads = [p.grad for p in model.perceiver.parameters() if p.requires_grad]
        assert grads and all(g is not None and torch.isfinite(g).all() for g in grads)
        model.eval()
        with torch.no_grad(), torch.autocast("cuda", dtype=bf16):
            gen = model.generate(vision_x=b["vision_x"], lang_x=b["lang_x"][:, :8],
                                 attention_mask=b["attention_mask"][:, :8], max_new_tokens=3, do_sample=False,
                                 pad_token_id=0)
    for h in hooks:
        h.remove()
    assert gen.shape[1] >= 9
    # the tower ran twice (training step, generate), each time one pack and one dense call per layer
    n = 2 * len(visual.transformer.resblocks)
    assert in_tower == {"attn_fwd": 0, "attn_dense_fwd": n, "rope_pack": n, "sdpa": 0}, in_tower
    del model, lm
    torch.cuda.empty_cache()
