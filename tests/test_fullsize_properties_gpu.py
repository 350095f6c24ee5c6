"""Size-independent properties checked at BASELINE.json's FULL sizes (configs[1]: OF-3B, 32 x (2 images, 256
tokens) per GPU), where the fp32 CPU oracle would take minutes per case:

  * wgmma GEMM at the FFN shapes: exact integer arithmetic (small-integer operands are exact in bf16 and their
    dot products exact in fp32, so the result must equal the integer product BIT FOR BIT), exact power-of-two
    homogeneity, split-K == single pass for exactly representable sums;
  * masked cross-attention at the OF-3B shape: rows of P sum to one (V = 1 gives O = 1), rows before the first
    <image> are exactly zero (helpers.py:223-229), keys of other images do not influence a row (helpers.py:210-218);
  * LayerNorm at [8192, 2048]: zero mean / unit variance rows, dx orthogonal to 1 and to x_hat;
  * the whole OF-3B training step: loss and gradient invariant under a permutation of the batch.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu
bf16, f32 = torch.bfloat16, torch.float32


@pytest.fixture(scope="module")
def ops():
    from open_flamingo_b200 import ops as _ops
    return _ops


@pytest.fixture(scope="module")
def L():
    from open_flamingo_b200 import _lib
    return _lib


def _ints(shape, lo, hi, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(lo, hi + 1, shape, device="cuda", generator=g).to(f32)


@pytest.mark.parametrize("M,N,K", [(8192, 8192, 2048), (8192, 2048, 8192), (16448, 4096, 1024)])
def test_gemm_full_size_is_exact_on_integers(ops, L, M, N, K):
    a = _ints((M, K), -3, 3, 1)
    b = _ints((N, K), -3, 3, 2)
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        ref = a @ b.t()                      # |sum| <= 9 * 8192 < 2^24: exact in fp32 in any summation order
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    out = ops.gemm(a.to(bf16), b.to(bf16), epi=L.EPI_STORE_F32)
    assert torch.equal(out, ref)
    # homogeneity under exact scaling: (4a) b^T == 4 (a b^T) bit for bit
    out4 = ops.gemm((4 * a).to(bf16), b.to(bf16), epi=L.EPI_STORE_F32)
    assert torch.equal(out4, 4 * ref)
    # MN-major operands (the dgrad / wgrad forms) read the same numbers through the other descriptor layout
    out_t = ops.gemm(a.t().contiguous().to(bf16), b.t().contiguous().to(bf16), a_mn=True, b_mn=True, epi=L.EPI_STORE_F32)
    assert torch.equal(out_t, ref)
    # split-K with the atomic epilogue accumulates the same exact integers on top of the existing contents
    acc = ref.clone()
    ops.gemm(a.to(bf16), b.to(bf16), epi=L.EPI_ATOMIC_F32, out=acc, splits=4)
    assert torch.equal(acc, 2 * ref)
    # bf16 store: the exact value rounded once
    outb = ops.gemm(a.to(bf16), b.to(bf16), epi=L.EPI_STORE_BF16)
    assert torch.equal(outb, ref.to(bf16))


def test_cross_attention_full_size_properties(ops):
    B, T, heads, n_media, n_lat = 32, 256, 8, 2, 64
    inner, nk = heads * 64, n_media * n_lat
    g = torch.Generator(device="cuda").manual_seed(3)
    q = torch.randn(B, T, inner, device="cuda", generator=g).to(bf16)
    k = torch.randn(B, nk, inner, device="cuda", generator=g).to(bf16)
    ones = torch.ones(B, nk, inner, device="cuda", dtype=bf16)
    # <image> at positions 5 and 130: text_time = 0 for t < 5, 1 for 5 <= t < 130, 2 afterwards
    loc = torch.zeros(B, T, dtype=torch.bool, device="cuda")
    loc[:, 5] = True
    loc[:, 130] = True
    tt = ops.text_time(media_locations=loc)
    o, lse = ops.attn_fwd(q, k, ones, heads, 0.125, mask_mode=1, text_time=tt, keys_per_media=n_lat)
    assert o[:, :5].abs().max().item() == 0.0                                  # exact zeros before the first image
    assert (o[:, 5:].float() - 1).abs().max().item() <= 2 ** -7               # P rounded to bf16 once, rows sum to 1
    # a row attending image 1 must not change when the keys / values of image 2 change (and vice versa)
    v = torch.randn(B, nk, inner, device="cuda", generator=g).to(bf16)
    o1, _ = ops.attn_fwd(q, k, v, heads, 0.125, mask_mode=1, text_time=tt, keys_per_media=n_lat)
    k2, v2 = k.clone(), v.clone()
    k2[:, n_lat:] = torch.randn(B, n_lat, inner, device="cuda", generator=g).to(bf16)
    v2[:, n_lat:] = 7.0
    o2, _ = ops.attn_fwd(q, k2, v2, heads, 0.125, mask_mode=1, text_time=tt, keys_per_media=n_lat)
    assert torch.equal(o1[:, :130], o2[:, :130])
    assert not torch.equal(o1[:, 130:], o2[:, 130:])
    # backward: dK / dV of image-2 keys receive nothing from rows that attend image 1 only
    d_o = torch.zeros(B, T, inner, device="cuda", dtype=bf16)
    d_o[:, 5:130] = torch.randn(B, 125, inner, device="cuda", generator=g).to(bf16)
    o1, lse1 = ops.attn_fwd(q, k, v, heads, 0.125, mask_mode=1, text_time=tt, keys_per_media=n_lat)
    dq, dk, dv = ops.attn_bwd(q, k, v, o1, d_o, lse1, heads, 0.125, mask_mode=1, text_time=tt, keys_per_media=n_lat)
    assert dk[:, n_lat:].abs().max().item() == 0.0 and dv[:, n_lat:].abs().max().item() == 0.0
    assert dq[:, :5].abs().max().item() == 0.0 and dq[:, 130:].abs().max().item() == 0.0
    assert dk[:, :n_lat].abs().max().item() > 0.0


def test_layernorm_full_size_properties(ops):
    rows, D = 8192, 2048
    g = torch.Generator(device="cuda").manual_seed(4)
    x = torch.randn(rows, D, device="cuda", generator=g) * 3 + 1.5
    ones, zeros = torch.ones(D, device="cuda"), torch.zeros(D, device="cuda")
    y, mean, rstd = ops.layernorm_fwd(x, ones, zeros, 1e-5, out_f32=True)
    assert y.mean(1).abs().max().item() <= 1e-5
    assert (y.var(1, unbiased=False) - 1).abs().max().item() <= 1e-4
    assert (mean - x.mean(1)).abs().max().item() <= 1e-5
    dy = torch.randn(rows, D, device="cuda", generator=g)
    dgamma, dbeta = torch.zeros(D, device="cuda"), torch.zeros(D, device="cuda")
    dx = ops.layernorm_bwd(dy, x, ones, mean, rstd, dgamma=dgamma, dbeta=dbeta)
    dx = dx[0] if isinstance(dx, tuple) else dx
    # the LayerNorm Jacobian projects out the constant and the x_hat directions
    assert dx.sum(1).abs().max().item() <= 2e-3
    assert (dx * y).sum(1).abs().max().item() <= 2e-2
    # parameter gradients are plain column sums
    assert (dbeta - dy.sum(0)).abs().max().item() <= 1e-3 * dy.sum(0).abs().max().item() + 1e-3
    assert (dgamma - (dy * y).sum(0)).abs().max().item() <= 1e-3 * (dy * y).sum(0).abs().max().item() + 1e-3
    # accumulate semantics: a second call adds on top
    ops.layernorm_bwd(dy, x, ones, mean, rstd, dgamma=dgamma, dbeta=dbeta)
    assert (dbeta - 2 * dy.sum(0)).abs().max().item() <= 2e-3 * dy.sum(0).abs().max().item() + 2e-3


def test_of3b_step_is_invariant_under_batch_permutation():
    """configs[1] at full size: mean-over-tokens loss and the summed gradient cannot depend on the order of the
    sequences in the batch (only fp32 / atomic summation order changes)."""
    from open_flamingo_b200.testing import MPT_1B, build_flamingo, synthetic_batch
    from open_flamingo_b200.train import FlatTrainer
    vit = dict(image_size=224, patch_size=14, width=1024, layers=24, heads=16, output_dim=768)
    torch.manual_seed(0)
    model, _, tok = build_flamingo(vit, MPT_1B, cross_attn_every_n_layers=1, device="cuda", gate_init=0.5, seed=0)
    model.train()
    trainer = FlatTrainer(model, lr=1e-4, weight_decay=0.1, max_grad_norm=1.0)
    media_id, eoc_id = tok.encode("<image>")[-1], tok.encode("<|endofchunk|>")[-1]
    batch = {k: v.cuda() for k, v in synthetic_batch(32, 2, 256, media_id, eoc_id, MPT_1B["vocab_size"], image_size=224,
                                                      seed=3).items()}
    perm = torch.randperm(32, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))

    def run(b):
        trainer.zero_grad()
        with torch.autocast("cuda", dtype=bf16):
            out = model(vision_x=b["vision_x"], lang_x=b["lang_x"], attention_mask=b["attention_mask"], labels=b["labels"])
        out.loss.backward()
        torch.cuda.synchronize()
        return out.loss.detach().float().item(), trainer.bucket.grads.detach().clone()

    l0, g0 = run(batch)
    l1, g1 = run({k: v[perm] for k, v in batch.items()})
    assert torch.isfinite(g0).all() and g0.norm().item() > 0
    rel = ((g0 - g1).norm() / g0.norm()).item()
    cos = torch.nn.functional.cosine_similarity(g0, g1, dim=0).item()
    print(f"permutation invariance: loss {l0:.6f} vs {l1:.6f}, grad rel diff {rel:.3e}, cos {cos:.6f}")
    # Not bit-identical: a sequence that moves to another row block can land in a tile whose k-reduction is
    # split differently (tail split, split-K wgrads), i.e. fp32 summation order changes, and a one-ulp bf16 flip
    # then propagates through 24 layers -- the same noise floor as any re-association under amp_bf16.
    assert abs(l0 - l1) <= 5e-4 * abs(l0), (l0, l1)
    assert rel <= 2e-2 and cos >= 0.9995, (rel, cos)
