"""Per-kernel numerics on the GPU: every libofk.so entry point against a plain torch fp32 reference of the
same op (tolerances are bf16-rounding sized and written next to each check)."""
import math

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


def close(got, ref, tol, what=""):
    err = (got.float() - ref.float()).abs().max().item()
    scale = ref.float().abs().max().item() + 1e-6
    assert err <= tol * scale, f"{what}: max_abs_err {err:.3e} vs ref_max {scale:.3e} (tol {tol})"


# ------------------------------------------------------------------ GEMM
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True), (True, False)])
@pytest.mark.parametrize("shape", [(256, 512, 512), (200, 272, 328), (32, 512, 2048), (1000, 768, 1096)])
def test_gemm_majors(ops, L, a_mn, b_mn, shape):
    M, N, K = shape
    torch.manual_seed(1)
    a = torch.randn((K, M) if a_mn else (M, K), device="cuda", dtype=bf16)
    b = torch.randn((K, N) if b_mn else (N, K), device="cuda", dtype=bf16)
    for bn in (128, 256, 512):  # every accepted tile-width hint
        out = ops.gemm(a, b, a_mn=a_mn, b_mn=b_mn, epi=L.EPI_STORE_F32, block_n=bn)
        A = a.float().t() if a_mn else a.float()
        B = b.float().t() if b_mn else b.float()
        close(out, A @ B.t(), 2e-3, f"gemm bn={bn}")  # fp32 accumulate; only summation-order noise


def test_gemm_epilogues(ops, L):
    torch.manual_seed(2)
    M, N, K = 512, 1024, 512
    a = torch.randn(M, K, device="cuda", dtype=bf16)
    b = torch.randn(N, K, device="cuda", dtype=bf16) * 0.05
    acc = a.float() @ b.float().t()
    bias = torch.randn(N, device="cuda")
    resid = torch.randn(M, N, device="cuda")
    gate = torch.tensor([0.7], device="cuda")
    tol = 1e-2  # one bf16 rounding (2^-8 relative) on O(1..6) values
    close(ops.gemm(a, b), acc.to(bf16), tol, "store_bf16")
    close(ops.gemm(a, b, epi=L.EPI_BIAS_BF16, bias=bias), (acc + bias).to(bf16), tol, "bias")
    t = (acc + bias).to(bf16).float()
    close(ops.gemm(a, b, epi=L.EPI_BIAS_QGELU_BF16, bias=bias), t * torch.sigmoid(1.702 * t), tol, "qgelu")
    z = torch.empty(M, N, device="cuda", dtype=bf16)
    h = torch.empty(M, N, device="cuda", dtype=bf16)
    ops.gemm(a, b, epi=L.EPI_GELU_DUAL, out=z, out2=h)
    close(z, acc.to(bf16), tol, "gelu z")
    close(h, torch.nn.functional.gelu(acc.to(bf16).float()), tol, "gelu h")
    br = torch.empty(M, N, device="cuda", dtype=bf16)
    o = ops.gemm(a, b, epi=L.EPI_GATE_RESID_F32, aux=resid, gate=gate, out2=br)
    close(o, acc.to(bf16).float() * math.tanh(0.7) + resid, tol, "gate_resid")
    close(br, acc.to(bf16), tol, "branch")
    close(ops.gemm(a, b, epi=L.EPI_GATE_RESID_F32, aux=resid), acc.to(bf16).float() + resid, tol, "resid")
    close(ops.gemm(a, b, epi=L.EPI_BIAS_RESID_F32, aux=resid, bias=bias), (acc + bias).to(bf16).float() + resid, tol, "bias_resid")
    zz = torch.randn(M, N, device="cuda", dtype=bf16)
    zf = zz.float().requires_grad_(True)
    torch.nn.functional.gelu(zf).sum().backward()
    close(ops.gemm(a, b, epi=L.EPI_DGELU_BF16, aux=zz), acc.to(bf16).float() * zf.grad, tol, "dgelu")
    for splits in (1, 4):
        for bn in (0, 512):
            o = torch.ones(M, N, device="cuda")
            ops.gemm(a, b, epi=L.EPI_ATOMIC_F32, out=o, splits=splits, block_n=bn)
            close(o, acc + 1.0, 2e-3, f"atomic splits={splits} bn={bn}")
    # the tile-width hint must not change the fused epilogues' results
    close(ops.gemm(a, b, block_n=512), acc.to(bf16), tol, "store_bf16 2cta")
    o = ops.gemm(a, b, epi=L.EPI_GATE_RESID_F32, aux=resid, gate=gate, out2=br, block_n=512)
    close(o, acc.to(bf16).float() * math.tanh(0.7) + resid, tol, "gate_resid 2cta")
    ops.gemm(a, b, epi=L.EPI_GELU_DUAL, out=z, out2=h, block_n=512)
    close(h, torch.nn.functional.gelu(acc.to(bf16).float()), tol, "gelu h 2cta")


@pytest.mark.parametrize("M,N,K", [(2560, 2048, 4096), (2496, 2048, 3072), (512, 2048, 8192), (8192, 2048, 3072)])
def test_gemm_tail_split_is_exact_and_epilogue_agnostic(ops, L, M, N, K):
    """Large-K shapes whose tile count leaves the last round of the persistent grid partly empty.  Integer operands
    make every partial sum exact, so the result must be bit-identical to the fp32 product whatever the tile hint or
    operand layout; the fused epilogues must see the completed sum; repeated launches give the same result."""
    g = torch.Generator(device="cuda").manual_seed(21)
    a = torch.randint(-3, 4, (M, K), device="cuda", generator=g).float()
    b = torch.randint(-3, 4, (N, K), device="cuda", generator=g).float()
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        ref = a @ b.t()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    a16, b16 = a.to(bf16), b.to(bf16)
    for _ in range(3):
        assert torch.equal(ops.gemm(a16, b16, epi=L.EPI_STORE_F32), ref)
    assert torch.equal(ops.gemm(a16, b16, epi=L.EPI_STORE_F32, block_n=256), ref)
    assert torch.equal(ops.gemm(a16.t().contiguous(), b16.t().contiguous(), a_mn=True, b_mn=True, epi=L.EPI_STORE_F32), ref)
    resid = torch.randint(-8, 9, (M, N), device="cuda", generator=g).float()
    bias = torch.randint(-8, 9, (N,), device="cuda", generator=g).float()
    o = ops.gemm(a16, b16, epi=L.EPI_BIAS_RESID_F32, aux=resid, bias=bias)
    assert torch.equal(o, (ref + bias).to(bf16).float() + resid)
    z = torch.empty(M, N, device="cuda", dtype=bf16)
    h = torch.empty(M, N, device="cuda", dtype=bf16)
    small = (a16 * 0.125).to(bf16), (b16 * 0.125).to(bf16)                              # keep GELU inputs O(1..10)
    ops.gemm(*small, epi=L.EPI_GELU_DUAL, out=z, out2=h)
    assert torch.equal(z, (ref / 64).to(bf16))
    close(h, torch.nn.functional.gelu((ref / 64).to(bf16).float()), 1e-2, "gelu after tail split")


def test_gemm_many_tiles_persistent(ops, L):
    """More tiles than SMs: exercises the persistent loop and the smem-ring phase wraps."""
    torch.manual_seed(12)
    for (M, N, K, a_mn, b_mn) in [(4096, 4096, 1024, False, False), (4096, 4096, 1024, False, True),
                                  (2048, 4096, 4096, True, True)]:
        a = torch.randn((K, M) if a_mn else (M, K), device="cuda", dtype=bf16)
        b = torch.randn((K, N) if b_mn else (N, K), device="cuda", dtype=bf16)
        A = a.float().t() if a_mn else a.float()
        B = b.float().t() if b_mn else b.float()
        ref = A @ B.t()
        for bn in (256, 512):
            close(ops.gemm(a, b, a_mn=a_mn, b_mn=b_mn, epi=L.EPI_STORE_F32, block_n=bn), ref, 3e-3, f"big bn={bn}")


def test_gemm_errors(ops, L):
    a = torch.randn(64, 64, device="cuda", dtype=bf16)
    with pytest.raises(ValueError):
        ops.gemm(a.float(), a)
    with pytest.raises(RuntimeError):
        ops.gemm(a, torch.randn(24, 64, device="cuda", dtype=bf16))  # N % 16 != 0
    with pytest.raises(RuntimeError):
        ops.gemm(a, a, epi=L.EPI_BIAS_BF16)  # missing bias


# ------------------------------------------------------------------ LayerNorm
@pytest.mark.parametrize("rows,D", [(37, 64), (513, 1024), (300, 2048), (129, 4096)])
def test_layernorm_fwd_bwd(ops, rows, D):
    torch.manual_seed(3)
    x = (torch.randn(rows, D, device="cuda") * 2 + 0.5)
    g = torch.randn(D, device="cuda")
    b = torch.randn(D, device="cuda")
    xr = x.clone().requires_grad_(True)
    gr = g.clone().requires_grad_(True)
    brr = b.clone().requires_grad_(True)
    ref = torch.nn.functional.layer_norm(xr, (D,), gr, brr, 1e-5)
    y32, mean, rstd = ops.layernorm_fwd(x, g, b, out_f32=True)
    close(y32, ref, 2e-5, "ln fwd f32")
    y16, _, _ = ops.layernorm_fwd(x, g, b)
    close(y16, ref.to(bf16), 1e-2, "ln fwd bf16")
    dy = torch.randn(rows, D, device="cuda")
    ref.backward(dy)
    dg = torch.zeros(D, device="cuda")
    db = torch.zeros(D, device="cuda")
    add = torch.randn(rows, D, device="cuda")
    dx = ops.layernorm_bwd(dy, x, g, mean, rstd, dgamma=dg, dbeta=db, dx_add=add)
    close(dx - add, xr.grad, 1e-4, "ln dx")
    close(dg, gr.grad, 1e-4, "ln dgamma")
    close(db, brr.grad, 1e-4, "ln dbeta")
    # bf16 dy path
    dx2 = ops.layernorm_bwd(dy.to(bf16), x, g, mean, rstd)
    close(dx2, xr.grad, 2e-2, "ln dx (bf16 dy)")


def test_layernorm_group_mapping(ops):
    """Two LayerNorms fill the halves of cat((x, latents), -2) in place (helpers.py:47-53)."""
    torch.manual_seed(4)
    U, v, n, D = 3, 20, 8, 128
    x = torch.randn(U * v, D, device="cuda")
    lat = torch.randn(U * n, D, device="cuda")
    g1, b1 = torch.randn(D, device="cuda"), torch.randn(D, device="cuda")
    g2, b2 = torch.randn(D, device="cuda"), torch.randn(D, device="cuda")
    buf = torch.zeros(U * (v + n), D, device="cuda", dtype=bf16)
    ops.layernorm_fwd(x, g1, b1, out=buf, rows_per_group=v, group_stride=v + n, group_offset=0)
    ops.layernorm_fwd(lat, g2, b2, out=buf, rows_per_group=n, group_stride=v + n, group_offset=v)
    ref = torch.cat([torch.nn.functional.layer_norm(x, (D,), g1, b1).view(U, v, D),
                     torch.nn.functional.layer_norm(lat, (D,), g2, b2).view(U, n, D)], dim=1).reshape(-1, D)
    close(buf, ref.to(bf16), 1e-2, "ln concat mapping")


# ------------------------------------------------------------------ attention
def ref_attention(q, k, v, heads, scale, mask_mode, tt, kpm):
    """Plain fp32 restatement (per helpers.py:190-232 semantics) on bf16-rounded inputs."""
    B, nq, _ = q.shape
    nk = k.shape[1]
    qh = q.float().view(B, nq, heads, 64).transpose(1, 2)
    kh = k.float().view(B, nk, heads, 64).transpose(1, 2)
    vh = v.float().view(B, nk, heads, 64).transpose(1, 2)
    sim = (qh * scale) @ kh.transpose(-1, -2)
    if mask_mode:
        media_time = (torch.arange(nk, device=q.device) // kpm + 1)[None, None, None, :]
        t = tt[:, None, :, None]
        allowed = (t == media_time) if mask_mode == 1 else (t >= media_time)
        sim = sim.masked_fill(~allowed, -torch.finfo(sim.dtype).max)
    sim = sim - sim.amax(dim=-1, keepdim=True).detach()
    attn = sim.softmax(dim=-1)
    if mask_mode == 1:
        attn = attn.masked_fill((tt == 0)[:, None, :, None], 0.0)
    out = attn @ vh
    return out.transpose(1, 2).reshape(B, nq, heads * 64)


CASES = [
    # B, heads, nq, nk, mask_mode, kpm
    (2, 8, 64, 320, 0, 64),      # perceiver, v=256
    (1, 8, 64, 1088, 0, 64),     # perceiver, longer media
    (3, 16, 257, 257, 0, 64),    # ViT: ragged q and k
    (4, 8, 256, 128, 1, 64),     # xattn eq, 2 images
    (2, 8, 100, 192, 1, 64),     # xattn eq, ragged q, 3 images
    (2, 8, 96, 192, 2, 64),      # xattn ge
    (2, 8, 1, 128, 1, 64),       # decode step
]


def make_tt(B, nq, n_media, mode, seed):
    gen = torch.Generator().manual_seed(seed)
    tt = torch.zeros(B, nq, dtype=torch.int32)
    for b in range(B):
        # random increasing media positions; row 0 of batch 0 starts with text before any image
        pos = sorted(torch.randperm(nq, generator=gen)[:n_media].tolist())
        if b == 0 and nq > 8:
            pos = [max(p, 5) for p in pos]
        loc = torch.zeros(nq, dtype=torch.int32)
        for p_ in pos:
            loc[p_] = 1
        tt[b] = loc.cumsum(0)
    return tt


@pytest.mark.parametrize("case", CASES)
def test_attention_fwd_bwd(ops, case):
    B, heads, nq, nk, mode, kpm = case
    torch.manual_seed(5)
    inner = heads * 64
    q = torch.randn(B, nq, inner, device="cuda").to(bf16)
    kv = torch.randn(B, nk, 2 * inner, device="cuda").to(bf16)
    k, v = kv[..., :inner], kv[..., inner:]  # strided views, as produced by the fused to_kv GEMM
    scale = 64 ** -0.5
    tt = None
    if mode:
        tt = make_tt(B, nq, nk // kpm, mode, 7).cuda()
        if nq == 1:
            tt[:] = nk // kpm
    o, lse = ops.attn_fwd(q, k, v, heads, scale, mask_mode=mode, text_time=tt, keys_per_media=kpm)
    qr = q.float().requires_grad_(True)
    kr = k.float().requires_grad_(True)
    vr = v.float().requires_grad_(True)
    ref = ref_attention(qr, kr, vr, heads, scale, mode, tt, kpm)
    assert torch.isfinite(o.float()).all()
    close(o, ref, 2e-2, "attn fwd")  # P and O are rounded to bf16 once each
    if mode == 1:
        zero_rows = (tt == 0)
        if zero_rows.any():
            assert o[zero_rows].abs().max().item() == 0.0  # exact zeros (helpers.py:223-229)
    d_o = torch.randn(B, nq, inner, device="cuda").to(bf16)
    ref.backward(d_o.float())
    dq, dk, dv = ops.attn_bwd(q, k, v, o, d_o, lse, heads, scale, mask_mode=mode, text_time=tt, keys_per_media=kpm)
    close(dq, qr.grad, 3e-2, "attn dq")
    close(dk, kr.grad, 3e-2, "attn dk")
    close(dv, vr.grad, 3e-2, "attn dv")


def test_attention_uniform_rows(ops):
    """ge-mode rows with text_time == 0 and eq-mode rows pointing past the last media: the reference's
    masked_fill(-max)+softmax gives a uniform row (helpers.py:218-221)."""
    torch.manual_seed(6)
    B, heads, nq, nk = 1, 8, 64, 128
    q = torch.randn(B, nq, 512, device="cuda").to(bf16)
    k = torch.randn(B, nk, 512, device="cuda").to(bf16)
    v = torch.randn(B, nk, 512, device="cuda").to(bf16)
    tt = torch.zeros(B, nq, dtype=torch.int32, device="cuda")
    tt[0, 10:] = 1
    tt[0, 40:] = 2
    o, _ = ops.attn_fwd(q, k, v, heads, 0.125, mask_mode=2, text_time=tt)
    close(o, ref_attention(q, k, v, heads, 0.125, 2, tt, 64), 2e-2, "ge uniform")
    tt2 = tt.clone()
    tt2[0, 50:] = 3  # more <image> tokens than media
    o, _ = ops.attn_fwd(q, k, v, heads, 0.125, mask_mode=1, text_time=tt2)
    close(o, ref_attention(q, k, v, heads, 0.125, 1, tt2, 64), 2e-2, "eq overflow uniform")


# ------------------------------------------------------------------ small kernels
def test_text_time(ops):
    torch.manual_seed(8)
    ids = torch.randint(0, 50, (5, 77), device="cuda")
    ids[0, :5] = 3
    tt = ops.text_time(input_ids=ids, media_token_id=7)
    ref = (ids == 7).cumsum(-1).int()
    assert torch.equal(tt, ref)
    loc = ids == 7
    assert torch.equal(ops.text_time(media_locations=loc), ref)
    cached = ops.text_time(media_locations=loc, use_cached_media=True, t_txt=3)
    assert torch.equal(cached, loc.sum(-1, keepdim=True).int().expand(-1, 3))


def test_gate_bwd_cast_add(ops):
    torch.manual_seed(9)
    n = 8 * 1000
    dout = torch.randn(n, device="cuda")
    branch = torch.randn(n, device="cuda").to(bf16)
    gate = torch.tensor([0.3], device="cuda")
    dgate = torch.zeros(1, device="cuda")
    dbr = ops.gate_bwd(dout, branch, gate, dgate)
    t = math.tanh(0.3)
    close(dbr, (dout * t).to(bf16), 1e-2, "dbranch")
    close(dgate, ((1 - t * t) * (dout * branch.float()).sum()).view(1), 1e-4, "dgate")
    close(ops.gate_bwd(dout, None, None, None), dout.to(bf16), 1e-2, "plain cast branch")
    x = torch.randn(1003, device="cuda")
    close(ops.cast_bf16(x), x.to(bf16), 0, "cast")
    y = torch.randn(1003, device="cuda")
    ref = x + y
    close(ops.add_(x, y), ref, 0, "add")


def test_patchify_assemble(ops):
    torch.manual_seed(10)
    n, H, P, D = 2, 28, 14, 64
    img = torch.randn(n, 3, H, H, device="cuda")
    ldp = 640
    pt = ops.patchify(img, P, ldp)
    w = torch.randn(D, 3, P, P, device="cuda")
    ref = torch.nn.functional.conv2d(img.to(bf16).float(), w.to(bf16).float(), stride=P)  # [n, D, 2, 2]
    ref = ref.flatten(2).transpose(1, 2).reshape(-1, D)
    wp = torch.zeros(D, ldp, device="cuda", dtype=bf16)
    wp[:, :3 * P * P] = w.reshape(D, -1).to(bf16)
    got = pt.float() @ wp.float().t()
    close(got, ref, 1e-4, "patchify == strided conv")
    assert pt[:, 3 * P * P:].abs().max().item() == 0
    g = (H // P) ** 2
    pe = torch.randn(n * g, D, device="cuda").to(bf16)
    cls = torch.randn(D, device="cuda")
    pos = torch.randn(g + 1, D, device="cuda")
    tok = ops.vit_assemble(pe, cls, pos, n, g, D).view(n, g + 1, D)
    ref = torch.cat([cls.expand(n, 1, D), pe.float().view(n, g, D)], 1) + pos
    close(tok, ref, 1e-6, "vit assemble")


def test_adamw_sumsq(ops):
    torch.manual_seed(11)
    n = 10007
    p = torch.randn(n, device="cuda")
    g = torch.randn(n, device="cuda")
    pr = p.clone().requires_grad_(True)
    opt = torch.optim.AdamW([pr], lr=1e-2, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.1)
    m = torch.zeros(n, device="cuda")
    v = torch.zeros(n, device="cuda")
    w16 = torch.empty(n, device="cuda", dtype=bf16)
    for step in (1, 2, 3):
        pr.grad = g.clone()
        opt.step()
        ops.adamw_(p, g, m, v, w16, 1e-2, 0.9, 0.999, 1e-8, 0.1, step)
    close(p, pr.detach(), 1e-5, "adamw")
    close(w16, p.to(bf16), 0, "adamw bf16 copy")
    out = torch.zeros(1, device="cuda")
    ops.sumsq_(g, out)
    close(out, (g * g).sum().view(1), 1e-5, "sumsq")


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("V", [50280, 61])
def test_causal_lm_loss_matches_hf(dtype, V):
    """Fused shifted cross-entropy vs transformers' ForCausalLMLoss (float logits, shift, mean over non-ignored)."""
    from transformers.loss.loss_utils import ForCausalLMLoss
    from open_flamingo_b200.fused import causal_lm_loss
    torch.manual_seed(13)
    B, T = 3, 17
    logits = (torch.randn(B, T, V, device="cuda") * 3).to(dtype)
    labels = torch.randint(0, V, (B, T), device="cuda")
    labels[0, 3] = -100
    labels[2, :5] = -100
    a = logits.clone().requires_grad_(True)
    b = logits.clone().requires_grad_(True)
    ref = ForCausalLMLoss(a, labels, V)
    got = causal_lm_loss(b, labels, V)
    assert abs(got.item() - ref.item()) <= 1e-4 * abs(ref.item()) + 1e-5
    (ref * 1.7).backward()
    (got * 1.7).backward()
    close(b.grad, a.grad, 1e-2 if dtype == torch.bfloat16 else 1e-5, "dlogits")
