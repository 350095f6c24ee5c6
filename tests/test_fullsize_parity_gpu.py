"""GPU: parity at the REAL model dimensions named by BASELINE.json -- not toy widths -- against the oracle.

  configs[0]  OF-3B (ViT-L/14 + MPT-1B-shaped LM, gated block before every layer), 1 image + 32 text tokens
  configs[1]  the same model at B = 4 x (2 images, 256 tokens): R = 1024 rows, so every projection runs the GEMM on
              many 128 x 128 tiles, as in the benchmark, and T_txt = 256 / head_dim 128 runs the
              LM attention exactly as in the benchmark
  configs[3]  OF-9B shape (ViT-L/14 + MPT-7B widths on 16 layers, head_dim 128, gated block before every 4th layer), small batch
  ViT-L/14    full depth, 257 tokens, against the oracle's vit_forward (flamingo.py:195 call site)

Three evaluations of the same weights and inputs (Flamingo.forward, flamingo.py:60-122; loss as train_utils.py:110-115):
  ref  = the oracle in fp32 (TF32 off) -- the restatement pinned to the unmodified reference by tests/test_oracle_golden.py;
         it is pure torch, so it is run on the GPU here only to make billion-parameter cases take seconds
  amp  = the same oracle under torch.autocast(bfloat16): the reference's OWN training numerics (train_utils.py:34-43)
  ours = open_flamingo_b200 under the same autocast context (what bench.py times)
Tolerance (SURVEY.md section 8c), err = ||x - ref||_2 / ||ref||_2:
  * logits, loss, the gradient of every trainable TENSOR and the hidden-state gradient arriving at every decoder
    position:  err(ours, ref) <= 2 x err(amp, ref) (+ a floor of 1e-3 for tensors both paths get essentially exactly)
    and cosine >= 0.999;
  * the two scalar tanh gates of a block (attn_gate, ff_gate; helpers.py:255-258): d gate = (1 - tanh^2) <dOut, branch> is
    a 10^5..10^6-term sum that cancels to ~1e-3 of its terms' scale at random init, so its bf16 rounding noise is of the
    order of the value itself in BOTH implementations and the per-tensor ratio ours / amp is a coin flip, in both
    directions across the 48 gates.  They are therefore tested as a
    population: the RMS over all gates of |g - g_ref| / ||dHidden_ref(layer)||_2 must satisfy ours <= 2.5 x amp, the
    median relative error ours <= 2 x amp, and the kernel that produces them is checked to be exact on its own
    inputs (fp64 dot product of the saved branch and the incoming gradient, 1e-5).
"""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu
bf16, f32 = torch.bfloat16, torch.float32
VIT_L14 = dict(image_size=224, patch_size=14, width=1024, layers=24, heads=16, output_dim=768)


from oracle.harness import PREFIXES as _PREFIXES  # noqa: E402


def _rel(a, ref):
    a, ref = a.detach().double().flatten(), ref.detach().double().flatten()
    return ((a - ref).norm() / (ref.norm() + 1e-30)).item()


def _cos(a, ref):
    a, ref = a.detach().double().flatten(), ref.detach().double().flatten()
    return torch.nn.functional.cosine_similarity(a, ref, dim=0).item()


class _NoTF32:
    def __enter__(self):
        self.prev = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
        torch.backends.cuda.matmul.allow_tf32 = False
        torch.backends.cudnn.allow_tf32 = False

    def __exit__(self, *exc):
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = self.prev
        return False


def _oracle_of(model, every):
    """The oracle around a private copy of the frozen LM and of every hot-path parameter (oracle/harness.py)."""
    from oracle.harness import oracle_from_model
    return oracle_from_model(model, every)


def _hidden_grad_hooks(layers, store):
    """Record the gradient arriving at the output of every decoder position (FlamingoLayer / HF block)."""
    handles = []
    for i, layer in enumerate(layers):
        def fwd_hook(mod, args, out, i=i):
            t = out[0] if isinstance(out, tuple) else out
            if t.requires_grad:
                t.register_hook(lambda g, i=i: store.__setitem__(i, g.detach().float().clone()))
        handles.append(layer.register_forward_hook(fwd_hook))
    return handles


def _run_oracle(orc, sd, trainable, batch, amp):
    hidden = {}
    handles = _hidden_grad_hooks(orc.blocks, hidden)
    from oracle.harness import oracle_train_step
    try:
        with _NoTF32():
            out = oracle_train_step(orc, sd, trainable, batch, amp_dtype=bf16 if amp else None)
    finally:
        for h in handles:
            h.remove()
    return (out.logits.detach().float(), out.loss.detach().float(), {k: sd[k].grad.detach().clone() for k in trainable},
            hidden)


def _run_ours(model, batch):
    model.zero_grad(set_to_none=True)
    hidden = {}
    handles = _hidden_grad_hooks(list(model.lang_encoder._get_decoder_layers()), hidden)
    try:
        with torch.autocast("cuda", dtype=bf16):
            out = model(vision_x=batch["vision_x"], lang_x=batch["lang_x"], attention_mask=batch["attention_mask"], labels=batch["labels"])
        out.loss.backward()
    finally:
        for h in handles:
            h.remove()
    grads = {k: p.grad.detach().clone() for k, p in model.named_parameters(remove_duplicate=False)
             if k.startswith(_PREFIXES) and p.requires_grad and p.grad is not None}
    return out.logits.detach().float(), out.loss.detach().float(), grads, hidden


def _is_gate(name):
    return name.endswith(".attn_gate") or name.endswith(".ff_gate")


def _compare(tag, runs, trainable):
    """runs: iterable of (ours, amp, ref) triples, one per batch, consumed one at a time so that only one batch's
    gradient copies are alive at once (each triple holds three copies of every trainable gradient)."""
    bad = []
    gate_z = {"ours": [], "amp": []}
    gate_rel = {"ours": [], "amp": []}
    summary = []
    for bi, (ours, amp, ref) in enumerate(runs):
        lo, so, go, ho = ours
        la, sa, ga, ha = amp
        lr, sr, gr, hr = ref
        rows = [("logits", _rel(lo, lr), _rel(la, lr), _cos(lo, lr)),
                ("loss", abs(so.item() - sr.item()) / abs(sr.item()), abs(sa.item() - sr.item()) / abs(sr.item()), 1.0)]
        for i in sorted(hr):
            rows.append((f"dHidden[{i}]", _rel(ho[i], hr[i]), _rel(ha[i], hr[i]), _cos(ho[i], hr[i])))
        for k in trainable:
            assert k in go, f"{tag}: no gradient for trainable parameter {k}"
            if _is_gate(k):
                layer = int(k.split(".")[2])
                scale = hr[layer].double().norm().item() + 1e-30
                for who, g in (("ours", go), ("amp", ga)):
                    gate_z[who].append(abs(g[k].item() - gr[k].item()) / scale)
                    gate_rel[who].append(abs(g[k].item() - gr[k].item()) / (abs(gr[k].item()) + 1e-30))
            else:
                rows.append((k, _rel(go[k], gr[k]), _rel(ga[k], gr[k]), _cos(go[k], gr[k])))
        for name, e_ours, e_amp, cos in rows:
            if not (e_ours <= 2.0 * e_amp + 1e-3):
                bad.append(f"batch {bi} {name}: err ours {e_ours:.3e} > 2 x amp {e_amp:.3e}")
            if name != "loss" and cos < 0.999:
                bad.append(f"batch {bi} {name}: cosine {cos:.5f}")
        worst = max(rows, key=lambda r: r[1] / max(r[2], 1e-3))
        summary.append(f"batch {bi}: {len(rows)} tensors, logits ours {rows[0][1]:.3e} / amp {rows[0][2]:.3e}, loss ours {rows[1][1]:.1e} / "
                       f"amp {rows[1][2]:.1e}, worst ratio {worst[0]} ours {worst[1]:.3e} / amp {worst[2]:.3e}")
        del ours, amp, ref, lo, go, ho, la, ga, ha, lr, gr, hr
    rms = {w: (sum(z * z for z in v) / len(v)) ** 0.5 for w, v in gate_z.items()}
    med = {w: sorted(v)[len(v) // 2] for w, v in gate_rel.items()}
    print(f"[{tag}] " + "; ".join(summary) + f"; gates ({len(gate_z['ours'])}): rms z ours {rms['ours']:.3e} / amp {rms['amp']:.3e}, "
          f"median rel err ours {med['ours']:.3e} / amp {med['amp']:.3e}")
    if not (rms["ours"] <= 2.5 * rms["amp"]):
        bad.append(f"gate gradients: rms normalised error ours {rms['ours']:.3e} > 2.5 x amp {rms['amp']:.3e}")
    if not (med["ours"] <= 2.0 * med["amp"] + 1e-3):
        bad.append(f"gate gradients: median relative error ours {med['ours']:.3e} > 2 x amp {med['amp']:.3e}")
    assert not bad, f"{tag}: " + "; ".join(bad[:8]) + (f" (+{len(bad) - 8} more)" if len(bad) > 8 else "")


def _three_ways(model, orc, sd, trainable, batch):
    return (_run_ours(model, batch), _run_oracle(orc, sd, trainable, batch, amp=True),
            _run_oracle(orc, sd, trainable, batch, amp=False))


def test_of9b_shape_every4_head_dim_128():
    """MPT-7B widths (d_model 4096, head_dim 128) with a gated block before every 4th layer, on 16 of the 32 decoder
    layers: the model and the oracle's fp32 copy of the frozen LM must fit one 80 GB GPU together.  Runs before the
    module-scoped OF-3B fixture is built, so the two models are never resident at the same time."""
    from open_flamingo_b200.testing import MPT_7B, build_flamingo
    model, _, tok = build_flamingo(VIT_L14, dict(MPT_7B, n_layers=16), cross_attn_every_n_layers=4, device="cuda",
                                   gate_init=1.0, seed=1)
    model.train()
    assert sum(l is not None for l in model.lang_encoder.gated_cross_attn_layers) == 4      # layers 3, 7, 11, 15
    orc, sd, trainable = _oracle_of(model, 4)
    runs = (_three_ways(model, orc, sd, trainable, _batch(tok, 2, 3, 192, MPT_7B["vocab_size"], seed=s, first_image_at=9))
            for s in (7, 17, 27))
    _compare("OF-9B shape 2x(3 img, 192 tok)", runs, trainable)
    del model, orc, sd
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def of3b():
    from open_flamingo_b200.testing import MPT_1B, build_flamingo
    model, _, tok = build_flamingo(VIT_L14, MPT_1B, cross_attn_every_n_layers=1, device="cuda", gate_init=1.0, seed=0)
    model.train()
    orc, sd, trainable = _oracle_of(model, 1)
    yield model, tok, orc, sd, trainable
    del model, orc, sd
    torch.cuda.empty_cache()


def _batch(tok, B, T_img, T_txt, vocab, seed, first_image_at=None):
    from open_flamingo_b200.testing import synthetic_batch
    media_id, eoc_id = tok.encode("<image>")[-1], tok.encode("<|endofchunk|>")[-1]
    b = synthetic_batch(B, T_img, T_txt, media_id, eoc_id, vocab, image_size=224, seed=seed)
    if first_image_at is not None:   # one row whose first <image> comes late: the zero-row rule (helpers.py:223-229)
        row = b["lang_x"][0]
        row[0] = 17
        row[first_image_at] = media_id
        b["labels"][0] = row
        b["labels"][0][row == media_id] = -100
    return {k: v.cuda() for k, v in b.items()}


def test_of3b_config0_one_image_32_tokens(of3b):
    from open_flamingo_b200.testing import MPT_1B
    model, tok, orc, sd, trainable = of3b
    runs = (_three_ways(model, orc, sd, trainable, _batch(tok, 1, 1, 32, MPT_1B["vocab_size"], seed=s)) for s in (5, 15, 25))
    _compare("OF-3B C1 1x(1 img, 32 tok)", runs, trainable)


def test_of3b_config1_shape_gemm2_path(of3b):
    from open_flamingo_b200 import _lib
    from open_flamingo_b200.testing import MPT_1B
    model, tok, orc, sd, trainable = of3b
    n0 = _lib.launch_count()
    runs = (_three_ways(model, orc, sd, trainable, _batch(tok, 4, 2, 256, MPT_1B["vocab_size"], seed=s, first_image_at=5))
            for s in (6, 16))
    _compare("OF-3B C2-shape 4x(2 img, 256 tok)", runs, trainable)
    assert _lib.launch_count() - n0 > 1000


def test_gate_backward_kernel_is_exact_on_its_inputs():
    """d gate from ofk_gate_bwd == (1 - tanh^2) <dOut, branch> evaluated in fp64 on the very same tensors."""
    from open_flamingo_b200 import ops
    torch.manual_seed(4)
    R, D = 1024, 2048
    dout = torch.randn(R, D, device="cuda")
    branch = torch.randn(R, D, device="cuda").to(bf16)
    gate = torch.tensor([0.37], device="cuda")
    dgate = torch.zeros(1, device="cuda")
    dbr = ops.gate_bwd(dout, branch, gate, dgate)
    t = torch.tanh(gate.double())
    want = ((1 - t * t) * (dout.double() * branch.double()).sum()).item()
    scale = ((1 - t * t) * (dout.double() * branch.double()).abs().sum()).item()   # size of the terms being cancelled
    assert abs(dgate.item() - want) <= 1e-6 * scale, (dgate.item(), want, scale)
    assert torch.equal(dbr, (dout * torch.tanh(gate)).to(bf16))


def test_vit_l14_full_depth_257_tokens():
    from open_flamingo_b200.src.vit import VisionTransformer
    from oracle import flamingo_oracle as O
    torch.manual_seed(2)
    with torch.device("cuda"):
        vit = VisionTransformer(**VIT_L14, output_tokens=True)
    x = torch.randn(4, 3, 224, 224, device="cuda")
    sd = {k: v.detach().float() for k, v in vit.state_dict().items()}
    with torch.no_grad(), _NoTF32():
        pooled_ref, tok_ref = O.vit_forward(x, sd, "", heads=16, patch=14, quick_gelu=True)
        with torch.autocast("cuda", dtype=bf16):
            pooled_amp, tok_amp = O.vit_forward(x, sd, "", heads=16, patch=14, quick_gelu=True)
        pooled, tok = vit(x)
    assert tok.shape == (4, 256, 1024)
    e_ours, e_amp = _rel(tok, tok_ref), _rel(tok_amp.float(), tok_ref)
    print(f"[ViT-L/14] tokens err ours {e_ours:.3e} / amp {e_amp:.3e}; cos {_cos(tok, tok_ref):.6f}")
    assert e_ours <= 2.0 * e_amp + 1e-3 and _cos(tok, tok_ref) >= 0.999
    assert _rel(pooled, pooled_ref) <= 2.0 * _rel(pooled_amp.float(), pooled_ref) + 1e-3
