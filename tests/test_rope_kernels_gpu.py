"""GPU: the GPT-NeoX kernels against float64.

ofk_rope_pack / ofk_rope_unpack_bwd (ops.rope_pack / rope_unpack_bwd).  Both compute in fp32 from bf16 inputs and round
once.  pack: y = x c + p s with |x|, |p| <= 1 * max and |c|, |s| <= 1; the two fp32 products and the fp32 sum add at most
3 * 2^-24 |y|-scale relative error before the bf16 rounding (2^-8 relative, half an ulp), so |y - y64| <= 2^-8 |y64|
+ 2^-22 max(|x| |c| + |p| |s|).  unpack: the same bound with one fused product.  Columns at or past rot are bit copies,
padding columns are exact zeros, and pack and unpack are adjoint: <pack(x), g> = <x, unpack(g)> up to the two
roundings.  Per-row cos/sin (left padding, as HF generate builds them) and one broadcast table are both covered.

ofk_gelu_bf16 after a BIAS_BF16 GEMM equals the BIAS_GELU_BF16 epilogue bit for bit.

ofk_attn_decode at head_dim 80 against float64, as test_kv_decode_gpu.py checks 64 and 128: within one bf16 rounding
per row; attn_decode_dev equals attn_decode bitwise at a smaller nk than the buffer holds."""
import pytest
import torch

from neox_reference import rotate
from test_kv_decode_gpu import _case, _check_rows, _in_cache, _reference

pytestmark = pytest.mark.gpu
bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64


def _tables(B, T, rot, per_row, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    inv = 1.0 / (10000 ** (torch.arange(0, rot, 2, device="cuda", dtype=f32) / rot))
    if per_row:   # left padding: positions start later in some rows (HF: cumsum(mask) - 1, padding at 1)
        pad = torch.randint(0, T // 2, (B,), device="cuda", generator=g)
        pos = (torch.arange(T, device="cuda")[None] - pad[:, None]).clamp(min=1).float()
    else:
        pos = torch.arange(T, device="cuda", dtype=f32)[None] + 7
    f = pos[..., None] * inv
    emb = torch.cat((f, f), -1)
    return emb.cos().contiguous(), emb.sin().contiguous()


@pytest.mark.parametrize("hd,rot", [(80, 80), (80, 20), (64, 64), (64, 16), (128, 32)])
@pytest.mark.parametrize("per_row", [False, True])
def test_rope_pack_and_unpack_against_float64(hd, rot, per_row):
    from open_flamingo_b200 import ops
    B, T, H = 3, 77, 4
    D = H * hd
    W = 128
    g = torch.Generator(device="cuda").manual_seed(hd + rot + per_row)
    # qkv as a column slice of a wider buffer, so strides differ from the width
    big = torch.randn(B, T, 3 * D + 16, device="cuda", generator=g).to(bf16)
    qkv = big[..., 8:8 + 3 * D]
    cos, sin = _tables(B if per_row else 1, T, rot, per_row, 3)
    q, k, v = ops.rope_pack(qkv, H, hd, cos, sin, q_width=W, kv_width=W)
    parts = qkv.view(B, T, H, 3, hd)
    x = [parts[..., i, :].reshape(B, T, D) for i in range(3)]
    for i, (got, name) in enumerate(((q, "q"), (k, "k"), (v, "v"))):
        g4 = got.view(B, T, H, W)
        assert torch.equal(g4[..., hd:], torch.zeros_like(g4[..., hd:])), f"{name}: padding not zero"
        src = x[i].view(B, T, H, hd)
        if i == 2:
            assert torch.equal(g4[..., :hd], src), "v is not a bit copy"
            continue
        assert torch.equal(g4[..., rot:hd], src[..., rot:]), f"{name}: pass-through columns are not bit copies"
        ref = rotate(x[i].double(), cos.double(), sin.double(), H).view(B, T, H, hd)
        mag = 2 * src.double().abs().amax(-1, keepdim=True)   # bounds |x c| + |p s| of every column of the head
        err = (g4[..., :hd].double() - ref).abs()
        assert (err <= 2.0 ** -8 * ref.abs() + 2.0 ** -22 * mag + 1e-30).all(), f"{name}: {err.max().item():.3e}"
        # with the same fp32 product and sum, the kernel equals torch's separate multiplies and add (HF's path)
        hf = rotate(x[i].float(), cos, sin, H).to(bf16).view(B, T, H, hd)
        assert torch.equal(g4[..., :hd], hf), f"{name}: differs from HF's rotation under autocast"
    assert torch.equal(q, ops.rope_pack(qkv, H, hd, cos, sin, q_width=W, kv_width=W)[0]), "not repeatable"

    # unpack: the transposed rotation of dq, dk and copies of dv, against float64
    dq, dk, dv = (torch.randn(B, T, H * W, device="cuda", generator=g).to(bf16) for _ in range(3))
    out = ops.rope_unpack_bwd(dq, dk, dv, H, hd, cos, sin)
    assert torch.equal(out, ops.rope_unpack_bwd(dq, dk, dv, H, hd, cos, sin)), "not repeatable"
    o5 = out.view(B, T, H, 3, hd)
    assert torch.equal(o5[..., 2, :], dv.view(B, T, H, W)[..., :hd]), "dv is not a bit copy"
    for i, dy in enumerate((dq, dk)):
        y = dy.view(B, T, H, W)[..., :hd].double().requires_grad_(True)
        xs = torch.zeros(B, T, H * hd, device="cuda", dtype=f64, requires_grad=True)
        rotate(xs, cos.double(), sin.double(), H).backward(y.reshape(B, T, H * hd))
        ref = xs.grad.view(B, T, H, hd)
        mag = 2 * y.detach().abs().amax(-1, keepdim=True)
        err = (o5[..., i, :].double() - ref).abs()
        assert (err <= 2.0 ** -8 * ref.abs() + 2.0 ** -22 * mag + 1e-30).all(), f"d{'qk'[i]}: {err.max().item():.3e}"
        assert torch.equal(o5[..., i, rot:], dy.view(B, T, H, W)[..., rot:hd]), "pass-through gradient not a copy"
    # adjointness on the data columns: <pack(x), g> = <x, unpack(g)>
    lhs = sum((p.view(B, T, H, W)[..., :hd].double() * d.view(B, T, H, W)[..., :hd].double()).sum()
              for p, d in ((q, dq), (k, dk), (v, dv)))
    rhs = (qkv.double() * out.double()).sum()
    mass = sum((p.double().abs() * d.double().abs()).sum() for p, d in ((q, dq), (k, dk), (v, dv)))
    assert (lhs - rhs).abs().item() <= 2 * 2.0 ** -8 * mass.item(), (lhs.item(), rhs.item())


def test_rope_pack_writes_into_cache_rows_and_pads_them():
    """The cached path: K and V land unpadded in rows [past, past + n) of a [B, cap, 2D] cache; rot = 0 pads them."""
    from open_flamingo_b200 import ops
    B, T, H, hd, cap, past = 2, 5, 4, 80, 32, 9
    D = H * hd
    qkv = torch.randn(B, T, 3 * D, device="cuda").to(bf16)
    cos, sin = _tables(1, T, hd, False, 1)
    buf = torch.full((B, cap, 2 * D), float("nan"), device="cuda", dtype=bf16)
    rows = buf[:, past:past + T]
    q, _, _ = ops.rope_pack(qkv, H, hd, cos, sin, q_width=hd, k=rows[..., :D], v=rows[..., D:])
    q2, k2, v2 = ops.rope_pack(qkv, H, hd, cos, sin)
    assert torch.equal(q, q2) and torch.equal(rows[..., :D], k2) and torch.equal(rows[..., D:], v2)
    assert torch.isnan(buf[:, :past]).all() and torch.isnan(buf[:, past + T:]).all(), "wrote outside the rows"
    _, kp, vp = ops.rope_pack(None, H, hd, kv_src=(rows[..., :D], rows[..., D:]), kv_width=128)
    for got, want in ((kp, k2), (vp, v2)):
        g4 = got.view(B, T, H, 128)
        assert torch.equal(g4[..., :hd], want.view(B, T, H, hd)) and not g4[..., hd:].any()


def test_gelu_bf16_equals_the_bias_gelu_epilogue():
    from open_flamingo_b200 import _lib as L
    from open_flamingo_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(5)
    a = (torch.randn(300, 320, device="cuda", generator=g) * 2).to(bf16)
    w = (torch.randn(1280, 320, device="cuda", generator=g) * 320 ** -0.5).to(bf16)
    b = torch.randn(1280, device="cuda", generator=g)
    z = ops.gemm(a, w, epi=L.EPI_BIAS_BF16, bias=b)
    h = ops.gemm(a, w, epi=L.EPI_BIAS_GELU_BF16, bias=b)
    assert torch.equal(ops.gelu_bf16(z), h)
    ref = torch.nn.functional.gelu(z.double())
    assert ((ops.gelu_bf16(z).double() - ref).abs() <= 2.0 ** -8 * ref.abs() + 1e-6).all()


@pytest.mark.parametrize("B,H", [(1, 32), (3, 32), (8, 4)])
@pytest.mark.parametrize("nk", [1, 63, 64, 65, 4097])
def test_decode_head_dim_80_against_float64(B, H, nk):
    from open_flamingo_b200 import ops
    hd = 80
    scale = hd ** -0.5
    for i, mask_kind in enumerate(("none", "pad", "full")):
        qkv, k, v, _, mask = _case(B, H, hd, nk, False, mask_kind, nk + 40, 100 * nk + 7 * i + B)
        q = qkv[:, :hd * H]
        kc, vc = _in_cache(k, v, nk + 40)
        what = f"B{B} H{H} nk{nk} mask={mask_kind}"
        o = ops.attn_decode(q, kc, vc, H, hd, scale, key_mask=mask)
        _check_rows(o, _reference(q, k, v, H, hd, scale, None, mask), what)
        assert torch.equal(o, ops.attn_decode(q, kc, vc, H, hd, scale, key_mask=mask)), what
        # the device-side key count over a larger buffer computes the same bits
        kc2, vc2 = _in_cache(k, v, nk + 300)
        kmax, vmax = (t.as_strided((B, nk + 300, H * hd), t.stride()) for t in (kc2, vc2))
        m2 = None
        if mask is not None:
            m2 = torch.ones((B, -(-(nk + 300) // 8) * 8), device="cuda", dtype=torch.uint8)
            m2[:, :nk] = mask[:, :nk]
        nk_dev = torch.tensor([nk], device="cuda", dtype=torch.int32)
        od = ops.attn_decode_dev(q, kmax, vmax, H, hd, scale, nk_dev, key_mask=m2)
        assert torch.equal(o, od), what + " (_dev)"
