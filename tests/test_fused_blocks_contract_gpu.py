"""GPU: the fused blocks' forward and hand-written backward against float64 restatements that round where the kernels
round (tests/rounded_reference.py).

Blocks: fused.GatedXattnBlockFn, PerceiverLayerFn, PerceiverFoldedLayerFn, FinalNormFn (with _ffn_forward /
_ffn_backward inside) and lm_blocks.FrozenMptBlockFn, each called through the module that calls it in the model
(GatedCrossAttentionBlock, PerceiverResampler, FastMptBlock).  The output, the input gradients and every parameter
gradient are compared with two float64 evaluations on the same inputs and weights:
  ref_r   the restatement with bf16 rounding at the kernels' rounding points,
  ref_64  the same without rounding (the plain float64 block).
What remains between the kernels and ref_r is fp32-vs-fp64 arithmetic plus the one-ulp flips of bf16 roundings it
causes (and what those flips move downstream), so for every tensor
  (1) ||ours - ref_r||_2 <= L2 ||ref_r - ref_64||_2,
  (2) max |ours - ref_r| over a row <= ROW 2^-8 max |ref_r| over that row     (rows: the leading dimension; a vector is
      one row), so a row whose reference is exactly zero must come out exactly zero.
The gate gradients are dot products that cancel to far below their terms (DESIGN §2); they are bounded against the
cancelled mass instead:  |ours - ref_r| <= GATE_C (1 - tanh^2 g) sum |dout . branch|.

Measured on an H100 80GB HBM3 (700 W power limit), largest value over every tensor of every case, and the bound set:
  block family                  (1) measured / L2     (2) measured / ROW     gates measured / GATE_C
  gated block (10 cases)        0.18 / 0.25           1.50 / 3               9.6e-6 / 3e-5
  frozen MPT block (32 cases)   0.44 / 0.75           1.75 / 3               -
  Perceiver, depth 2 (4 cases)  0.83 / 1.5            5.1 / 8                -
One flip of a bf16 value costs up to 2^-7 of it (one ulp), so (2) sits at a few units.  The residue is larger than the
~1/10 of the rounding effect a sqrt(K) 2^-16 flip rate predicts: flips in the q / kv / LayerNorm outputs move every
score of their row or key, and the Perceiver's first-layer gradients pass through a second layer's backward, where the
residue reaches 0.5-0.8 of the rounding effect (largest for norm_media / norm_latents, to_kv and to_q of layer 0).
Each step alone (LayerNorm, GEMM epilogues, GELU, both attention families) agrees with its rounded restatement on
all but 0.01-0.14 % of its bf16 outputs.  Each of these wiring mutations fails this file: DGELU fed h instead of z,
the gated block's last LayerNorm backward adding dout instead of dx1, the two gates swapped in gate_bwd, the Perceiver's
second latent-row LayerNorm backward dropped, the folded dW_kv missing its colsum x beta term, the folded bias built
from gamma, the MPT backward attending causally without the saved mask, and its last LayerNorm backward adding dout.

A wiring mistake in a backward -- an operand swapped, a residual term dropped, gelu' taken of the wrong tensor, the
wrong mask -- moves a gradient by a sizeable fraction of the rounding effect or more, and fails (1) or (2).

Every LayerNorm weight and bias and every gate is drawn at random and distinct: at the default init (gamma = 1,
beta = 0, gates 0) a swapped or missing affine term would be invisible.  The gradient-sink tests cover frozen
parameters (None, the rest unchanged bit for bit), `_ofk_grad` buckets (prefill + fresh gradient, bit for bit where one
launch writes the parameter, one fp32 rounding per contribution where several add) and two backward passes.
"""
import math

import pytest
import torch

import rounded_reference as RR

pytestmark = pytest.mark.gpu
f32, f64, bf16 = torch.float32, torch.float64, torch.bfloat16
U32 = 2.0 ** -24
# (L2 ratio, per-row constant) per block family, from the measurements in the module docstring
BOUNDS = {"xattn": (0.25, 3.0), "mpt": (0.75, 3.0), "perceiver": (1.5, 8.0)}
GATE_C = 3e-5


# ------------------------------------------------------------------ the bounds
def check(errs, what, got, ref_r, ref_64):
    """Bounds (1) and (2) of the module docstring for one tensor; a violation is appended to errs.  (1) is skipped
    where rounding does not move the reference at all (the final norm's dbeta, a sum of the fp32 upstream gradient)."""
    l2_ratio, row_c = BOUNDS["perceiver" if "folded" in what else "mpt" if what.startswith("mpt") else "xattn"]
    if got is None:
        errs.append(f"{what}: no gradient")
        return
    got = got.detach().to(f64)
    if got.shape != ref_r.shape or not bool(torch.isfinite(got).all()):
        errs.append(f"{what}: shape {tuple(got.shape)} (reference {tuple(ref_r.shape)}) or non-finite values")
        return
    err = got - ref_r
    rnd = (ref_r - ref_64).norm().item()
    l2 = err.norm().item() / rnd if rnd > 0 else 0.0
    rows_e = err.reshape(err.shape[0], -1) if err.dim() > 1 else err.reshape(1, -1)
    rows_r = ref_r.reshape(rows_e.shape)
    unit = 2.0 ** -8 * rows_r.abs().amax(1)
    row_err = rows_e.abs().amax(1)
    row = (row_err / torch.where(unit > 0, unit, torch.ones_like(unit))).max().item()
    zero_rows_ok = bool((row_err[unit == 0] == 0).all())
    print(f"MEASURE {what}: l2 {l2:.4f} row {row:.4f}")
    if not zero_rows_ok:
        errs.append(f"{what}: rows whose reference is exactly zero are not")
    if l2 > l2_ratio:
        errs.append(f"{what}: ||ours - ref_r|| is {l2:.3f} x the rounding effect ||ref_r - ref_64||")
    if row > row_c:
        errs.append(f"{what}: a row is off by {row:.3f} x 2^-8 of its largest value")


def check_gate(errs, what, got, ref_r, g, dout, branch):
    t = math.tanh(g)
    mass = (1 - t * t) * (dout * branch).abs().sum().item()
    err = abs(got.item() - ref_r.item())
    print(f"MEASURE {what}: gate {err / mass if mass > 0 else 0.0:.3e}")
    if not err <= GATE_C * mass:
        errs.append(f"{what}: |err| {err:.3e} > {GATE_C} x the cancelled mass {mass:.3e}")


def reference_grads(fn, params64, inputs64, g64):
    """Run fn(params, *inputs) in float64 with autograd; returns (output, {name: grad}, [input grads])."""
    ps = {k: v.detach().clone().requires_grad_(True) for k, v in params64.items()}
    ins = [t.detach().clone().requires_grad_(t.is_floating_point()) if t is not None else None for t in inputs64]
    trace = {}
    y = fn(ps, *ins, trace)
    if "x1" in trace:
        trace["x1"].retain_grad()
    (y * g64).sum().backward()
    return y.detach(), {k: v.grad for k, v in ps.items()}, [t.grad if t is not None else None for t in ins], trace


def random_affine(module, seed):
    """Distinct random LayerNorm weights / biases (1 + 0.3 N, 0.3 N); Linear weights N / sqrt(fan_in)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in module.named_parameters():
            r = torch.randn(p.shape, generator=g)
            if name.endswith("_gate") or name in ("latents", "frame_embs", "media_time_embs"):
                p.copy_(r)
            elif p.dim() == 1:
                p.copy_(1.0 + 0.3 * r if name.endswith("weight") else 0.3 * r)
            else:
                p.copy_(r * p.shape[-1] ** -0.5)


# ------------------------------------------------------------------ gated cross-attention block
D, DV, HEADS = 128, 64, 2


def media_locations(B, T, T_img, pattern, seed):
    """b = 0: two text rows before the first <image>; b = 1: an <image> at row 0 ("late") or none at all
    ("surplus": text_time 0 everywhere); b >= 2 random.  "surplus" puts T_img + 2 <image> tokens in row 0: rows
    past the last media have no allowed key (mode eq)."""
    g = torch.Generator().manual_seed(seed)
    loc = torch.zeros(B, T, dtype=torch.bool)
    if T == 1:
        loc[::2, 0] = True
        return loc
    count = min(T - 2, T_img + (2 if pattern == "surplus" else 0))
    loc[0, 2 + torch.randperm(T - 2, generator=g)[:count]] = True
    if pattern == "late":
        loc[1, 0] = True
        loc[1, 1 + torch.randperm(T - 1, generator=g)[:T_img - 1]] = True
    for b in range(2, B):
        loc[b, torch.randperm(T, generator=g)[:T_img]] = True
    return loc


XATTN_CASES = {
    # id: (B, T, T_img, n, mode, cached, (attn_gate, ff_gate), x layout, location pattern)
    "eq-T129": (2, 129, 3, 64, "eq", False, (0.4, -0.4), "f32", "late"),
    "eq-surplus-T65": (2, 65, 2, 80, "eq", False, (-0.4, 3.0), "f32", "surplus"),
    "ge-T64-bf16": (2, 64, 5, 16, "ge", False, (3.0, 0.4), "bf16", "late"),
    "ge-surplus-T63-strided": (2, 63, 4, 64, "ge", False, (0.4, 0.4), "strided", "surplus"),
    "none-cached-T65": (2, 65, 5, 16, "none", True, (-0.4, -0.4), "f32", None),
    "eq-cached-T129-strided": (2, 129, 2, 80, "eq", True, (0.4, 3.0), "strided", "late"),
    "eq-cached-surplus-T64": (2, 64, 1, 16, "eq", True, (-0.4, 0.4), "f32", "surplus"),
    "eq-T1": (3, 1, 1, 80, "eq", False, (0.4, -0.4), "f32", "late"),
    "ge-T1-bf16": (3, 1, 3, 64, "ge", False, (-0.4, 3.0), "bf16", "late"),
    "zero-gates-eq-T65": (2, 65, 3, 64, "eq", False, (0.0, 0.0), "f32", "late"),
}


def make_xattn(mode, gates, seed):
    from open_flamingo_b200.src.helpers import GatedCrossAttentionBlock
    blk = GatedCrossAttentionBlock(dim=D, dim_visual=DV, heads=HEADS, only_attend_immediate_media=(mode != "ge"))
    random_affine(blk, seed)
    with torch.no_grad():
        blk.attn_gate.fill_(gates[0])
        blk.ff_gate.fill_(gates[1])
    return blk.cuda()


def xattn_inputs(B, T, T_img, n, layout, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if layout == "strided":   # views with a row stride of 2D / a column stride of 2, and an upstream gradient slice
        x = torch.randn(B, T, 2 * D, device="cuda", generator=g)[..., ::2]
        dout = torch.randn(B, T, D + 8, device="cuda", generator=g)[..., 3:3 + D]
        assert not x.is_contiguous() and not dout.is_contiguous()
    else:
        dt = bf16 if layout == "bf16" else f32
        x = torch.randn(B, T, D, device="cuda", generator=g).to(dt)
        dout = torch.randn(B, T, D, device="cuda", generator=g).to(dt)
    media = torch.randn(B, T_img, n, DV, device="cuda", generator=g)
    return x, media, dout


def run_xattn(blk, x, media, loc, cached, dout):
    """The model's call; returns (out, dx, dmedia, {name: grad})."""
    xg = x.detach().clone().requires_grad_(True) if x.is_contiguous() else x.detach().requires_grad_(True)
    mg = media.detach().clone().requires_grad_(True)
    blk.zero_grad(set_to_none=True)
    out = blk(xg, mg, media_locations=loc, use_cached_media=cached)
    out.backward(dout)
    return out.detach(), xg.grad, mg.grad, {k: p.grad for k, p in blk.named_parameters()}


def xattn_reference(blk, x, media, loc, cached, mode, dout, rounding):
    params = {k: p.detach().to(f64) for k, p in blk.named_parameters()}
    loc64 = None if loc is None else loc

    def fn(ps, xx, mm, trace):
        y = RR.gated_cross_attention_block(xx, mm, ps, "", loc64, cached, HEADS, mode != "ge", rounding=rounding,
                                           trace=trace)
        if rounding and x.dtype == bf16:   # the module hands back a bf16 output
            y = RR.rf(y)
        return y

    y, gp, (dx, dm), trace = reference_grads(fn, params, [x.to(f64), media.to(f64)], dout.to(f64))
    if rounding and x.dtype == bf16:       # and autograd rounds the gradient to the input's dtype
        dx = RR.to_bf16(dx)
    return y, gp, dx, dm, trace


@pytest.mark.parametrize("case", list(XATTN_CASES))
def test_gated_xattn_block_contract(case):
    B, T, T_img, n, mode, cached, gates, layout, pattern = XATTN_CASES[case]
    blk = make_xattn(mode, gates, seed=list(XATTN_CASES).index(case))
    x, media, dout = xattn_inputs(B, T, T_img, n, layout, seed=len(case))
    loc = None if pattern is None else media_locations(B, T, T_img, pattern, seed=T).cuda()
    out, dx, dmedia, grads = run_xattn(blk, x, media, loc, cached, dout)
    y_r, g_r, dx_r, dm_r, tr = xattn_reference(blk, x, media, loc, cached, mode, dout, True)
    y_6, g_6, dx_6, dm_6, _ = xattn_reference(blk, x, media, loc, cached, mode, dout, False)
    assert out.dtype == x.dtype and dx.dtype == x.dtype
    errs = []
    check(errs, f"{case} out", out, y_r, y_6)
    check(errs, f"{case} dx", dx, dx_r, dx_6)
    check(errs, f"{case} dmedia", dmedia, dm_r, dm_6)
    for k in grads:
        if k.endswith("_gate"):
            continue
        check(errs, f"{case} d{k}", grads[k], g_r[k], g_6[k])
    check_gate(errs, f"{case} dattn_gate", grads["attn_gate"], g_r["attn_gate"], gates[0], tr["x1"].grad, tr["attn_branch"])
    check_gate(errs, f"{case} dff_gate", grads["ff_gate"], g_r["ff_gate"], gates[1], dout.to(f64), tr["ff_branch"])
    assert not errs, "\n".join(errs)
    if gates == (0.0, 0.0):
        # the reference's init: both branches are cut off, so every branch parameter and the media get exactly zero
        # and the block passes dout straight through; the gates themselves still learn
        for k, gr in grads.items():
            if not k.endswith("_gate"):
                assert bool((gr == 0).all()), f"{case} d{k} is not exactly zero at zero gates"
        assert bool((dmedia == 0).all())
        assert torch.equal(dx, dout) and torch.equal(out, x)
        assert grads["attn_gate"].abs().item() > 0 and grads["ff_gate"].abs().item() > 0


# ------------------------------------------------------------------ Perceiver
PD, PN = 128, 16
PERCEIVER_CASES = {
    # id: (b, T, F, v, embs, expected path)
    "folded-v64-F2": (2, 2, 2, 32, False, "folded"),
    "folded-v128": (1, 3, 1, 128, False, "folded"),
    "unfolded-v40": (2, 2, 1, 40, False, "unfolded"),
    "unfolded-embs-v64-F2": (2, 2, 2, 32, True, "unfolded"),
}


def make_perceiver(embs, seed, depth=2):
    from open_flamingo_b200.src.helpers import PerceiverResampler
    kw = dict(max_num_media=3, max_num_frames=2) if embs else {}
    m = PerceiverResampler(dim=PD, depth=depth, heads=HEADS, num_latents=PN, **kw)
    random_affine(m, seed)
    return m.cuda()


def perceiver_inputs(b, T, Fr, v, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = 1.5 * torch.randn(b, T, Fr, v, PD, device="cuda", generator=g) + 0.3
    dout = torch.randn(b, T, PN, PD, device="cuda", generator=g)
    return x, dout


def run_perceiver(m, x, dout):
    m.zero_grad(set_to_none=True)
    y = m(x)
    y.backward(dout)
    return y.detach(), {k: p.grad for k, p in m.named_parameters()}


def perceiver_reference(m, x, dout, folded, rounding):
    params = {k: p.detach().to(f64) for k, p in m.named_parameters()}
    fn = lambda ps, xx, trace: RR.perceiver_resampler(xx, ps, heads=HEADS, folded=folded, rounding=rounding)  # noqa
    y, gp, _, _ = reference_grads(fn, params, [x.to(f64)], dout.to(f64))
    return y, gp


@pytest.mark.parametrize("case", list(PERCEIVER_CASES))
def test_perceiver_contract(case, monkeypatch):
    from open_flamingo_b200 import fused
    b, T, Fr, v, embs, path = PERCEIVER_CASES[case]
    m = make_perceiver(embs, seed=len(case))
    x, dout = perceiver_inputs(b, T, Fr, v, seed=v)
    calls = {"folded": 0, "unfolded": 0}
    for name, key in (("PerceiverFoldedLayerFn", "folded"), ("PerceiverLayerFn", "unfolded")):
        fn = getattr(fused, name)
        monkeypatch.setattr(fn, "apply", (lambda f, k: lambda *a: (calls.__setitem__(k, calls[k] + 1), f(*a))[1])(
            fn.apply, key))
    y, grads = run_perceiver(m, x, dout)
    assert calls[path] == 2 and sum(calls.values()) == 2, f"{case}: expected the {path} layer path, got {calls}"
    y_r, g_r = perceiver_reference(m, x, dout, path == "folded", True)
    y_6, g_6 = perceiver_reference(m, x, dout, path == "folded", False)
    errs = []
    check(errs, f"{case} out", y, y_r, y_6)
    for k, g in grads.items():
        check(errs, f"{case} d{k}", g, g_r[k], g_6[k])
    assert not errs, "\n".join(errs)


# ------------------------------------------------------------------ frozen MPT block
def make_mpt(d_model, n_heads, seed):
    from transformers import MptConfig
    from transformers.models.mpt.modeling_mpt import MptBlock, build_mpt_alibi_tensor
    torch.manual_seed(seed)
    cfg = MptConfig(d_model=d_model, n_heads=n_heads, n_layers=1, vocab_size=32, max_seq_len=256, expansion_ratio=4)
    blk = MptBlock(cfg, 0).eval().requires_grad_(False)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for _, p in blk.named_parameters():
            r = torch.randn(p.shape, generator=g)
            p.copy_(1.0 + 0.3 * r if p.dim() == 1 else r * p.shape[1] ** -0.5)
    return blk.cuda(), build_mpt_alibi_tensor(n_heads, cfg.max_seq_len, device="cuda")


def mpt_mask(B, T, kind):
    """HF's [B, 1, T, T] bool mask (True = masked) and the pure-causal flag, or (None, None) for kind "none"."""
    if kind == "none":
        return None, None
    att = torch.ones(B, T, dtype=torch.bool, device="cuda")
    if kind == "right_pad":
        att[0, T - min(7, T):] = False       # T = 1: the only row of batch 0 sees no key (uniform row)
    elif kind == "left_pad":
        att[1, :min(5, T)] = False
    causal = torch.ones(T, T, dtype=torch.bool, device="cuda").triu(1)
    m = causal.view(1, 1, T, T) | ~att.view(B, 1, 1, T)
    return m, att.all().to(torch.int32).reshape(1)


@pytest.mark.parametrize("head_dim", [64, 128])
@pytest.mark.parametrize("kind", ["none", "causal", "right_pad", "left_pad"])
@pytest.mark.parametrize("T", [1, 64, 65, 130])
def test_frozen_mpt_block_contract(head_dim, kind, T):
    from open_flamingo_b200 import lm_blocks
    d_model, B = 256, 2
    heads = d_model // head_dim
    blk, alibi = make_mpt(d_model, heads, seed=T + head_dim)
    fast = lm_blocks.accelerate(blk)
    mask, flag = mpt_mask(B, T, kind)
    g = torch.Generator(device="cuda").manual_seed(T)
    x = torch.randn(B, T, d_model, device="cuda", generator=g)
    dout = torch.randn(B, T, d_model, device="cuda", generator=g)
    xg = x.clone().requires_grad_(True)
    res = fast(xg, position_bias=alibi, attention_mask=mask, pure_causal_flag=flag)
    assert res is not None, "fast path declined"
    res[0].backward(dout)
    w = {k: v.detach().to(f64) for k, v in
         zip(("norm_1", "Wqkv", "out_proj", "norm_2", "up_proj", "down_proj"), fast.weights())}
    slopes = fast.slopes(x.device).to(f64)
    refs = []
    for rounding in (True, False):
        xr = x.to(f64).requires_grad_(True)
        y = RR.mpt_block(xr, w, heads, slopes, None if mask is None else mask[:, 0], blk.norm_1.eps, rounding=rounding)
        (y * dout.to(f64)).sum().backward()
        refs.append((y.detach(), xr.grad))
    what = f"mpt hd{head_dim} {kind} T{T}"
    errs = []
    check(errs, f"{what} out", res[0], refs[0][0], refs[1][0])
    check(errs, f"{what} dx", xg.grad, refs[0][1], refs[1][1])
    assert not errs, "\n".join(errs)


# ------------------------------------------------------------------ gradient sinks
def sink_models():
    """(name, module, run(): {param name: grad} after one forward + backward, params whose sink takes several
    contributions -> their count)."""
    B, T, T_img, n, mode, cached, gates, layout, pattern = XATTN_CASES["eq-T129"]
    blk = make_xattn(mode, gates, seed=5)
    x, media, dout = xattn_inputs(B, T, T_img, n, layout, seed=6)
    loc = media_locations(B, T, T_img, pattern, seed=7).cuda()

    def run_x():
        out = blk(x, media, media_locations=loc, use_cached_media=cached)
        out.backward(dout)

    m = make_perceiver(False, seed=8)
    px, pdout = perceiver_inputs(*PERCEIVER_CASES["folded-v64-F2"][:4], seed=9)

    def run_p():
        m(px).backward(pdout)

    multi = {}
    for i in range(2):
        multi[f"layers.{i}.0.to_kv.weight"] = 3              # latent-row wgrad, addcmul_ (W o gamma), addr_ (beta)
        multi[f"layers.{i}.0.norm_latents.weight"] = 2       # two layernorm_bwd calls (to_q and to_kv rows)
        multi[f"layers.{i}.0.norm_latents.bias"] = 2
        multi[f"layers.{i}.0.norm_media.weight"] = 1
        multi[f"layers.{i}.0.norm_media.bias"] = 1
    return [("xattn", blk, run_x, {}), ("perceiver-folded", m, run_p, multi)]


AUTOGRAD_ONLY = ("latents",)
ALIGN = 64   # the broadcast latents are a Function input: autograd reduces their gradient


def fresh_grads(module, run):
    module.zero_grad(set_to_none=True)
    run()
    return {k: (None if p.grad is None else p.grad.clone()) for k, p in module.named_parameters()}


def test_frozen_parameters_get_none_and_the_rest_is_unchanged():
    for name, module, run, _ in sink_models():
        full = fresh_grads(module, run)
        names = [k for k, _ in module.named_parameters()]
        frozen = set(names[1::3])
        for k, p in module.named_parameters():
            p.requires_grad_(k not in frozen)
        part = fresh_grads(module, run)
        for k in names:
            if k in frozen:
                assert part[k] is None, f"{name}: frozen {k} got a gradient"
            else:
                assert torch.equal(part[k], full[k]), f"{name}: {k} changed when other parameters were frozen"
        for _, p in module.named_parameters():
            p.requires_grad_(True)


def test_ofk_grad_buckets_accumulate_and_backward_passes_add():
    for name, module, run, multi in sink_models():
        fresh = fresh_grads(module, run)
        twice = fresh_grads(module, lambda: (run(), run()))
        for k, g in fresh.items():
            assert torch.equal(twice[k], g + g), f"{name}: two backward passes do not add for {k}"
        params = [(k, p) for k, p in module.named_parameters() if k not in AUTOGRAD_ONLY and
                  not k.endswith("_embs")]
        # one flat buffer with every view on a 64-element boundary, as train.FlatTrainer lays out its gradients
        flat = torch.empty(sum(-(-p.numel() // ALIGN) * ALIGN for _, p in params), device="cuda")
        gen = torch.Generator(device="cuda").manual_seed(3)
        views, off = {}, 0
        for k, p in params:
            v = flat[off:off + p.numel()].view(p.shape)
            v.copy_(torch.randn(p.shape, device="cuda", generator=gen) * fresh[k].abs().max().clamp_min(1e-3))
            views[k] = v
            off += -(-p.numel() // ALIGN) * ALIGN
        prefill = {k: v.clone() for k, v in views.items()}
        try:
            for k, p in params:
                p._ofk_grad = views[k]
            for passes in (1, 2):
                module.zero_grad(set_to_none=True)
                for k in views:
                    views[k].copy_(prefill[k])
                for _ in range(passes):
                    run()
                for k, p in params:
                    assert p.grad is None, f"{name}: {k} has an _ofk_grad bucket but autograd got a gradient"
                    want = prefill[k]
                    for _ in range(passes):
                        want = want + fresh[k]
                    got = views[k]
                    c = multi.get(k, 0)
                    if c == 0:
                        assert torch.equal(got, want), f"{name} ({passes} passes): bucket {k} != prefill + gradient"
                    else:
                        tol = passes * c * U32 * (want.abs() + prefill[k].abs() + fresh[k].abs()
                                                  + fresh[k].abs().max())
                        worst = ((got - want).abs() / tol).max().item()
                        print(f"MEASURE sink {name} {k} ({passes} passes): {worst:.3f} of {c} roundings")
                        assert worst <= 1.0, f"{name} ({passes} passes): bucket {k} off by {worst:.2f}x its bound"
        finally:
            for _, p in params:
                del p._ofk_grad
