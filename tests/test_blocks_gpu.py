"""GPU parity of the kernel-backed modules against (a) the golden fixtures produced by the real reference and
(b) the fp32 oracle on the same seeded inputs.

Tolerances (bf16 GEMM operands, fp32 accumulate/softmax/LayerNorm/residual -- the reference's own amp_bf16
numerics, train_utils.py:34-43): outputs within 2e-2 of the tensor's max, gradients within 4e-2 of the
gradient's max and cosine similarity >= 0.999 against the fp32 reference."""
import pytest
import torch

from helpers_golden import (build_mpt, flamingo_state, greedy_generate, load, seeded_state_dict, seeded_tensor)

pytestmark = pytest.mark.gpu
OUT_TOL, GRAD_TOL, COS = 2e-2, 4e-2, 0.999


def cmp(got, ref, tol, what):
    got, ref = got.detach().float().cpu(), ref.detach().float().cpu()
    err = (got - ref).abs().max().item()
    scale = ref.abs().max().item() + 1e-9
    cos = torch.nn.functional.cosine_similarity(got.flatten(), ref.flatten(), dim=0).item() if ref.abs().sum() > 0 else 1.0
    assert err <= tol * scale and cos >= COS, f"{what}: err {err:.3e} / max {scale:.3e}, cos {cos:.5f}"


def check_gate_grads(what, blk, sd_cpu, x, media, loc, cached, immediate, w, g_ref):
    """The two tanh gates (helpers.py:255-258) get d gate = (1 - tanh^2 g) <dOut, branch>: one scalar that is a sum of
    B*T*D products of mixed sign.  Its error against the fp32 oracle is the projection of the branch's bf16-GEMM rounding
    noise (relative size eps ~ 5e-3 per element at D = 2048) onto dOut, i.e.
    of order eps * (1 - tanh^2) * ||dOut|| * ||branch|| / sqrt(N) whatever the value of the gradient itself -- so the
    check is against that noise scale (6 sigma, eps = 8e-3) plus 2e-2 of the value, not a percentage of a quantity that
    can cancel to nearly zero.  A second, well-conditioned check follows in the caller (loss = |y|^2 / 2)."""
    import math
    from oracle import flamingo_oracle as O
    with torch.no_grad():
        a = O.masked_cross_attention(x, media, sd_cpu, "attn", loc, cached, only_attend_immediate_media=immediate)
        x1 = a * sd_cpu["attn_gate"].tanh() + x
        f = O.feed_forward(x1, sd_cpu, "ff")
    n = x.numel()
    for name, branch, dout_norm in (("attn_gate", a, 2.0 * w.norm().item()), ("ff_gate", f, w.norm().item())):
        t = math.tanh(sd_cpu[name].item())
        noise = 6.0 * 8e-3 * (1 - t * t) * dout_norm * branch.norm().item() / math.sqrt(n)
        got, ref = dict(blk.named_parameters())[name].grad.item(), g_ref[name].item()
        assert abs(got - ref) <= noise + 2e-2 * abs(ref), \
            f"{what} grad {name}: {got:.5f} vs {ref:.5f} (|err| {abs(got - ref):.3e} > noise scale {noise:.3e} + 2%)"


def check_gate_grads_conditioned(what, blk, run_ours, run_oracle):
    """Well-conditioned gate-gradient check: with loss = |y|^2 / 2 the upstream gradient is y itself, which contains
    tanh(g) * branch, so <dOut, branch> has a large coherent part and the relative error is of the order of the bf16
    rounding (3e-2 allowed) -- this is the check that would catch a wrong formula or a wrong operand."""
    blk.zero_grad(set_to_none=True)
    y = run_ours()
    (0.5 * y.float().pow(2).sum()).backward()
    ref = run_oracle()
    for name in ("attn_gate", "ff_gate"):
        got, want = dict(blk.named_parameters())[name].grad.item(), ref[name].item()
        assert abs(got - want) <= 3e-2 * abs(want) + 1e-6, f"{what} conditioned grad {name}: {got:.6f} vs {want:.6f}"


def oracle_grads(fn, sd_cpu, *inputs):
    """Run the fp32 oracle on CPU, return (output, grads of sd, grads of inputs)."""
    from oracle import flamingo_oracle as O  # noqa: F401
    sd = {k: v.clone().requires_grad_(True) for k, v in sd_cpu.items()}
    ins = [t.clone().requires_grad_(True) if t is not None and t.is_floating_point() else t for t in inputs]
    y, w = fn(sd, *ins)
    (y * w).sum().backward()
    return y.detach(), {k: v.grad for k, v in sd.items()}, [t.grad if t is not None and t.is_floating_point() else None for t in ins]


def test_perceiver_resampler_vs_golden_and_oracle():
    from open_flamingo_b200.src.helpers import PerceiverResampler
    from oracle import flamingo_oracle as O
    fx = load("perceiver")
    sd_cpu = seeded_state_dict(fx["shapes"], fx["seed"])
    m = PerceiverResampler(dim=fx["dim"], depth=fx["depth"]).cuda()
    m.load_state_dict(sd_cpu)
    x = seeded_tensor("perceiver/x", fx["x_shape"], 1)
    w = seeded_tensor("perceiver/w", fx["y"].shape, 1)
    y = m(x.cuda())
    cmp(y, fx["y"], OUT_TOL, "perceiver y vs golden")
    (y * w.cuda()).sum().backward()
    _, g_ref, _ = oracle_grads(lambda sd, xx: (O.perceiver_resampler(xx, sd), w), sd_cpu, x)
    for k, p in m.named_parameters():
        assert p.grad is not None, k
        cmp(p.grad, g_ref[k], GRAD_TOL, f"perceiver grad {k}")


def test_perceiver_with_embeddings_and_many_tokens():
    from open_flamingo_b200.src.helpers import PerceiverResampler
    from oracle import flamingo_oracle as O
    fx = load("perceiver_embs")
    sd_cpu = seeded_state_dict(fx["shapes"], fx["seed"])
    m = PerceiverResampler(dim=fx["dim"], depth=fx["depth"], max_num_media=3, max_num_frames=2).cuda()
    m.load_state_dict(sd_cpu)
    x = seeded_tensor("perceiver_embs/x", fx["x_shape"], 2)
    y = m(x.cuda())
    cmp(y, fx["y"], OUT_TOL, "perceiver+embs vs golden")
    # the embeddings are trainable in the reference (helpers.py:118-125): their gradients must flow through the
    # media rows of every layer's norm_media / to_kv
    w = seeded_tensor("perceiver_embs/w", tuple(y.shape), 2)
    (y * w.cuda()).sum().backward()
    sd_req = {k: v.clone().requires_grad_(True) for k, v in sd_cpu.items()}
    (O.perceiver_resampler(x, sd_req) * w).sum().backward()
    for name in ("frame_embs", "media_time_embs", "latents"):
        cmp(dict(m.named_parameters())[name].grad, sd_req[name].grad, GRAD_TOL, f"perceiver+embs d{name}")
    # longer media (ragged tile tail: v + n = 200 + 64 keys)
    torch.manual_seed(0)
    m2 = PerceiverResampler(dim=128, depth=1).cuda()
    x2 = torch.randn(1, 3, 1, 200, 128)
    ref = O.perceiver_resampler(x2, {k: v.detach().cpu() for k, v in m2.state_dict().items()})
    cmp(m2(x2.cuda()), ref, OUT_TOL, "perceiver v=200")


@pytest.mark.parametrize("idx", [0, 1, 2, 3])
def test_gated_xattn_block_vs_golden_and_oracle(idx):
    from open_flamingo_b200.src.helpers import GatedCrossAttentionBlock
    from oracle import flamingo_oracle as O
    fxs = load("xattn")
    c = fxs["cases"][idx]
    sd_cpu = seeded_state_dict(c["shapes"], c["seed"])
    blk = GatedCrossAttentionBlock(dim=fxs["D"], dim_visual=fxs["Dv"], only_attend_immediate_media=c["immediate"]).cuda()
    blk.load_state_dict(sd_cpu)
    x = seeded_tensor(f"xattn/{c['name']}/x", c["x_shape"], 3)
    media = seeded_tensor(f"xattn/{c['name']}/media", c["media_shape"], 3)
    w = seeded_tensor(f"xattn/{c['name']}/w", c["y"].shape, 3)
    xg = x.cuda().requires_grad_(True)
    mg = media.cuda().requires_grad_(True)
    loc = None if c["loc"] is None else c["loc"].cuda()
    y = blk(xg, mg, media_locations=loc, use_cached_media=c["cached"])
    cmp(y, c["y"], OUT_TOL, f"xattn[{c['name']}] y vs golden")
    (y * w.cuda()).sum().backward()
    cmp(xg.grad, c["dx"], GRAD_TOL, f"xattn[{c['name']}] dx vs golden")
    _, g_ref, in_ref = oracle_grads(
        lambda sd, xx, mm: (O.gated_cross_attention_block(xx, mm, sd, "", c["loc"], c["cached"],
                                                          only_attend_immediate_media=c["immediate"]), w),
        sd_cpu, x, media)
    cmp(mg.grad, in_ref[1], GRAD_TOL, f"xattn[{c['name']}] dmedia")
    for k, p in blk.named_parameters():
        assert p.grad is not None, k
        if not k.endswith("_gate"):
            cmp(p.grad, g_ref[k], GRAD_TOL, f"xattn[{c['name']}] grad {k}")
    check_gate_grads(f"xattn[{c['name']}]", blk, sd_cpu, x, media, c["loc"], c["cached"], c["immediate"], w, g_ref)

    def oracle_conditioned():
        sd = {k: v.clone().requires_grad_(True) for k, v in sd_cpu.items()}
        yo = O.gated_cross_attention_block(x, media, sd, "", c["loc"], c["cached"], only_attend_immediate_media=c["immediate"])
        (0.5 * yo.pow(2).sum()).backward()
        return {k: v.grad for k, v in sd.items()}

    check_gate_grads_conditioned(f"xattn[{c['name']}]", blk,
                                 lambda: blk(x.cuda(), media.cuda(), media_locations=loc, use_cached_media=c["cached"]),
                                 oracle_conditioned)
    if c["name"] == "eq":
        tt = c["loc"].cumsum(-1)
        # rows before the first <image>: block output == x + gated FFN only; attention branch contributes 0 exactly
        assert (tt == 0).any()


def test_xattn_zero_gate_is_identity():
    """Reference init: gates are 0 -> the block is the identity (helpers.py:255,258; SURVEY fact 1)."""
    from open_flamingo_b200.src.helpers import GatedCrossAttentionBlock
    blk = GatedCrossAttentionBlock(dim=128, dim_visual=128).cuda()
    x = torch.randn(2, 16, 128, device="cuda")
    media = torch.randn(2, 1, 64, 128, device="cuda")
    loc = torch.zeros(2, 16, dtype=torch.bool, device="cuda")
    loc[:, 0] = True
    assert torch.equal(blk(x, media, media_locations=loc), x)


def test_vit_tokens_vs_golden():
    from open_flamingo_b200.src.vit import VisionTransformer
    fx = load("vit")
    sd = seeded_state_dict(fx["shapes"], fx["seed"])
    sd["proj"] = torch.eye(fx["cfg"]["width"])
    vit = VisionTransformer(**fx["cfg"], output_tokens=True).cuda()
    vit.load_state_dict(sd)
    imgs = seeded_tensor("vit/images", fx["images_shape"], 20)
    _, tokens = vit(imgs.cuda())
    cmp(tokens, fx["tokens"], OUT_TOL, "vit tokens vs golden")


def build_product_model(fx, every):
    from open_flamingo_b200 import create_model_and_transforms
    from open_flamingo_b200.src.vit import CLIPVisionStandIn, VisionTransformer
    from open_flamingo_b200.testing import SimpleTokenizer
    lm = build_mpt(fx["mpt"], fx["lm_seed"], fx["lm_shapes"])
    vit = VisionTransformer(**fx["vit_cfg"])
    tok = SimpleTokenizer(fx["mpt"]["vocab_size"] - 3)
    model, _, tok = create_model_and_transforms(CLIPVisionStandIn(vit), None, lm, tok, cross_attn_every_n_layers=every,
                                                freeze_lm_embeddings=True)
    assert tok.encode("<image>")[-1] == fx["media_id"] and tok.encode("<|endofchunk|>")[-1] == fx["eoc_id"]
    missing, unexpected = model.load_state_dict(flamingo_state(fx), strict=False)
    assert not unexpected, unexpected
    # every trainable hot-path tensor must have been provided (the per-layer alias path
    # `transformer.blocks.{i}.gated_cross_attn_layer.*` shares storage with `gated_cross_attn_layers.{i}.*`)
    assert all(not k.startswith(("perceiver.", "lang_encoder.gated_cross_attn_layers.", "vision_encoder."))
               for k in missing), missing
    return model.cuda().eval()


@pytest.mark.parametrize("every", [1, 2])
def test_full_flamingo_vs_golden(every):
    fx = load(f"flamingo_every{every}")
    model = build_product_model(fx, every)
    vision_x = seeded_tensor("flamingo/vision_x", fx["vision_x_shape"], 33).cuda()
    lang_x, labels = fx["lang_x"].cuda(), fx["labels"].cuda()
    out = model(vision_x=vision_x, lang_x=lang_x, attention_mask=torch.ones_like(lang_x), labels=labels)
    cmp(out.logits, fx["logits"], OUT_TOL, "logits vs golden")
    assert abs(out.loss.item() - fx["loss"].item()) < 2e-2 * abs(fx["loss"].item())
    out.loss.backward()
    from golden_utils import check_digest
    named = dict(model.named_parameters())
    for k, d in fx["grads"].items():
        assert named[k].grad is not None, k
        check_digest(k, named[k].grad, d, GRAD_TOL, atol_scale=1.0)
    with torch.no_grad():
        gen = model.generate(vision_x=vision_x, lang_x=lang_x[:, :12], attention_mask=torch.ones_like(lang_x[:, :12]),
                             max_new_tokens=6, do_sample=False, pad_token_id=0)
        assert torch.equal(gen.cpu(), fx["generated"]), "greedy generate tokens differ from the reference"
        model.cache_media(input_ids=lang_x[:, :12], vision_x=vision_x)
        cached = model(vision_x=None, lang_x=lang_x[:, 12:15], attention_mask=None, clear_conditioned_layers=False).logits
        model.uncache_media()
        cmp(cached, fx["cached_logits"], OUT_TOL, "cached-media logits vs golden")


def test_error_behaviour_matches_reference():
    fx = load("flamingo_every1")
    model = build_product_model(fx, 1)
    lang_x = fx["lang_x"].cuda()
    with pytest.raises(AssertionError):
        model(vision_x=None, lang_x=lang_x)                                   # flamingo.py:94-96
    with pytest.raises(AssertionError):
        model(vision_x=torch.zeros(2, 2, 3, 56, 56, device="cuda"), lang_x=lang_x)  # ndim != 6 (flamingo.py:189)
    with pytest.raises(AssertionError):
        model(vision_x=torch.zeros(2, 2, 2, 3, 56, 56, device="cuda"), lang_x=lang_x)  # F != 1 (flamingo.py:191)
    layer = model.lang_encoder._get_decoder_layers()[0]
    with pytest.raises(ValueError):
        layer(torch.zeros(1, 4, 128, device="cuda"))                          # flamingo_lm.py:47-53
    with pytest.raises(RuntimeError):
        model.perceiver(torch.zeros(1, 1, 1, 4, 128))                         # CPU tensor: no fallback


def test_gated_xattn_block_of9b_width_vs_oracle():
    """BASELINE configs[3] shape class: D = 4096 (MPT-7B), media width 1024, 5 images -- fwd + input/param grads."""
    from open_flamingo_b200.src.helpers import GatedCrossAttentionBlock
    from oracle import flamingo_oracle as O
    torch.manual_seed(21)
    D, Dv, B, T, Ti, n = 4096, 1024, 2, 40, 5, 64
    blk = GatedCrossAttentionBlock(dim=D, dim_visual=Dv)
    with torch.no_grad():
        blk.attn_gate.fill_(0.6)
        blk.ff_gate.fill_(-0.4)
    sd_cpu = {k: v.detach().clone() for k, v in blk.state_dict().items()}
    blk = blk.cuda()
    x = torch.randn(B, T, D)
    media = torch.randn(B, Ti, n, Dv)
    loc = torch.zeros(B, T, dtype=torch.bool)
    loc[0, [2, 9, 17, 25, 33]] = True
    loc[1, [0, 8, 16, 24, 39]] = True
    w = torch.randn(B, T, D)
    xg, mg = x.cuda().requires_grad_(True), media.cuda().requires_grad_(True)
    y = blk(xg, mg, media_locations=loc.cuda())
    (y * w.cuda()).sum().backward()
    y_ref, g_ref, in_ref = oracle_grads(
        lambda sd, xx, mm: (O.gated_cross_attention_block(xx, mm, sd, "", loc), w), sd_cpu, x, media)
    cmp(y, y_ref, OUT_TOL, "9B-width y")
    cmp(xg.grad, in_ref[0], GRAD_TOL, "9B-width dx")
    cmp(mg.grad, in_ref[1], GRAD_TOL, "9B-width dmedia")
    for k, p in blk.named_parameters():
        if not k.endswith("_gate"):
            cmp(p.grad, g_ref[k], GRAD_TOL, f"9B-width grad {k}")
    check_gate_grads("9B-width", blk, sd_cpu, x, media, loc, False, True, w, g_ref)

    def oracle_conditioned():
        sd = {k: v.clone().requires_grad_(True) for k, v in sd_cpu.items()}
        yo = O.gated_cross_attention_block(x, media, sd, "", loc)
        (0.5 * yo.pow(2).sum()).backward()
        return {k: v.grad for k, v in sd.items()}

    check_gate_grads_conditioned("9B-width", blk, lambda: blk(x.cuda(), media.cuda(), media_locations=loc.cuda()),
                                 oracle_conditioned)


def test_perceiver_isolation_shape_vs_oracle():
    """BASELINE configs[4] shape: 64 latents x 4096 visual tokens x d=1024 (one image here; fwd + grads)."""
    from open_flamingo_b200.src.helpers import PerceiverResampler
    from oracle import flamingo_oracle as O
    torch.manual_seed(22)
    m = PerceiverResampler(dim=1024, depth=2)
    sd_cpu = {k: v.detach().clone() for k, v in m.state_dict().items()}
    m = m.cuda()
    x = torch.randn(1, 1, 1, 4096, 1024)
    w = torch.randn(1, 1, 64, 1024)
    y = m(x.cuda())
    (y * w.cuda()).sum().backward()
    y_ref, g_ref, _ = oracle_grads(lambda sd, xx: (O.perceiver_resampler(xx, sd), w), sd_cpu, x)
    cmp(y, y_ref, OUT_TOL, "C5 perceiver y")
    for k, p in m.named_parameters():
        cmp(p.grad, g_ref[k], GRAD_TOL, f"C5 perceiver grad {k}")


@pytest.mark.parametrize("v,dim,U", [(64, 128, 3), (192, 256, 2)])
def test_perceiver_folded_path_vs_oracle(v, dim, U):
    """v % 64 == 0 takes the folded path (norm_media folded into to_kv, media tokens normalised once): outputs and
    EVERY parameter gradient -- in particular norm_media.{weight,bias} and to_kv.weight, which are reconstructed
    from the folded wgrad -- against the fp32 oracle."""
    from open_flamingo_b200.src.helpers import PerceiverResampler
    from oracle import flamingo_oracle as O
    torch.manual_seed(31)
    m = PerceiverResampler(dim=dim, depth=2)
    with torch.no_grad():
        for name, p in m.named_parameters():
            if "norm" in name:   # make the affine terms non-trivial
                p.add_(0.2 * torch.randn_like(p))
    sd_cpu = {k: v_.detach().clone() for k, v_ in m.state_dict().items()}
    m = m.cuda()
    x = torch.randn(U, 1, 1, v, dim) * 1.5 + 0.3
    w = torch.randn(U, 1, 64, dim)
    y = m(x.cuda())
    (y * w.cuda()).sum().backward()
    y_ref, g_ref, _ = oracle_grads(lambda sd, xx: (O.perceiver_resampler(xx, sd), w), sd_cpu, x)
    cmp(y, y_ref, OUT_TOL, "folded perceiver y")
    for k, p in m.named_parameters():
        assert p.grad is not None, k
        cmp(p.grad, g_ref[k], GRAD_TOL, f"folded perceiver grad {k}")
