"""GPU: the wgmma attention kernels behind ofk_attn_fwd / ofk_attn_bwd / ofk_attn_dense_fwd / ofk_attn_dense_bwd against
a plain fp32 torch restatement of the reference semantics (helpers.py:190-232 for the media rules; HF MptAttention for
the dense rules)."""
import pytest
import torch

from test_kernels_gpu import CASES, close, make_tt, ref_attention

pytestmark = pytest.mark.gpu
bf16, f32 = torch.bfloat16, torch.float32


@pytest.fixture(scope="module")
def ops():
    from open_flamingo_b200 import ops as _ops
    return _ops


def _media_run(ops, q, k, v, d_o, heads, scale, mode, tt, kpm):
    o, lse = ops.attn_fwd(q, k, v, heads, scale, mask_mode=mode, text_time=tt, keys_per_media=kpm)
    dq, dk, dv = ops.attn_bwd(q, k, v, o, d_o, lse, heads, scale, mask_mode=mode, text_time=tt, keys_per_media=kpm)
    torch.cuda.synchronize()
    return o, lse, dq, dk, dv


@pytest.mark.parametrize("case", CASES)
def test_media_attention_tc_vs_reference(ops, case):
    B, heads, nq, nk, mode, kpm = case
    torch.manual_seed(11)
    inner = heads * 64
    q = torch.randn(B, nq, inner, device="cuda").to(bf16)
    kv = torch.randn(B, nk, 2 * inner, device="cuda").to(bf16)
    k, v = kv[..., :inner], kv[..., inner:]
    d_o = torch.randn(B, nq, inner, device="cuda").to(bf16)
    scale = 64 ** -0.5
    tt = None
    if mode:
        tt = make_tt(B, nq, nk // kpm, mode, 7).cuda()
        if nq == 1:
            tt[:] = nk // kpm
    o, lse, dq, dk, dv = _media_run(ops, q, k, v, d_o, heads, scale, mode, tt, kpm)
    for t in (o, lse, dq, dk, dv):
        assert torch.isfinite(t.float()).all()
    # fp32 reference
    qr, kr, vr = (t.float().requires_grad_(True) for t in (q, k, v))
    ref = ref_attention(qr, kr, vr, heads, scale, mode, tt, kpm)
    ref.backward(d_o.float())
    close(o, ref, 2e-2, "o")
    close(dq, qr.grad, 3e-2, "dq")
    close(dk, kr.grad, 3e-2, "dk")
    close(dv, vr.grad, 3e-2, "dv")
    if mode == 1 and (tt == 0).any():
        assert o[(tt == 0)].abs().max().item() == 0.0 and dq[(tt == 0)].abs().max().item() == 0.0


def test_media_uniform_rows_tc(ops):
    """ge-mode rows before the first image and eq-mode rows pointing past the last media attend uniformly
    (masked_fill(-max) + softmax, helpers.py:218-221): forward and backward (no gradient to q / k from such rows)."""
    torch.manual_seed(6)
    B, heads, nq, nk = 1, 8, 64, 128
    q = torch.randn(B, nq, 512, device="cuda").to(bf16)
    k = torch.randn(B, nk, 512, device="cuda").to(bf16)
    v = torch.randn(B, nk, 512, device="cuda").to(bf16)
    d_o = torch.randn(B, nq, 512, device="cuda").to(bf16)
    tt = torch.zeros(B, nq, dtype=torch.int32, device="cuda")
    tt[0, 10:] = 1
    tt[0, 40:] = 2
    tt2 = tt.clone()
    tt2[0, 50:] = 3
    for mode, t in ((2, tt), (1, tt2)):
        o, lse, dq, dk, dv = _media_run(ops, q, k, v, d_o, heads, 0.125, mode, t, 64)
        qr, kr, vr = (x.float().requires_grad_(True) for x in (q, k, v))
        ref = ref_attention(qr, kr, vr, heads, 0.125, mode, t, 64)
        ref.backward(d_o.float())
        close(o, ref, 2e-2, f"uniform o mode {mode}")
        close(dq, qr.grad, 3e-2, f"uniform dq mode {mode}")
        close(dk, kr.grad, 3e-2, f"uniform dk mode {mode}")
        close(dv, vr.grad, 3e-2, f"uniform dv mode {mode}")


def test_vit_tail_rows_split(ops):
    """257 = 4 x 64 + 1 query rows (the ViT forward): the forward without an LSE writes the same bits as the one that
    also writes the LSE, overhanging row included, and matches fp32."""
    torch.manual_seed(19)
    B, heads, n = 3, 16, 257
    qkv = torch.randn(B, n, 3 * heads * 64, device="cuda").to(bf16)
    D = heads * 64
    q, k, v = qkv[..., :D], qkv[..., D:2 * D], qkv[..., 2 * D:]
    from open_flamingo_b200 import _lib
    n0 = _lib.launch_count()
    o_split, _ = ops.attn_fwd(q, k, v, heads, 0.125, want_lse=False)
    assert _lib.launch_count() - n0 == 1   # one forward-core launch, no separate LSE pass
    o_full, _ = ops.attn_fwd(q, k, v, heads, 0.125, want_lse=True)
    torch.cuda.synchronize()
    close(o_split, ref_attention(q, k, v, heads, 0.125, 0, None, 64), 2e-2, "vit split vs fp32")
    assert torch.equal(o_split, o_full)


# ------------------------------------------------------------------ dense (LM self-attention) rules
def ref_dense(q, k, v, heads, hd, scale, causal, mask, slopes):
    B, nq, _ = q.shape
    nk = k.shape[1]
    qh = q.view(B, nq, heads, hd).transpose(1, 2)
    kh = k.view(B, nk, heads, hd).transpose(1, 2)
    vh = v.view(B, nk, heads, hd).transpose(1, 2)
    s = (qh @ kh.transpose(-1, -2)) * scale
    if slopes is not None:
        s = s + slopes.view(1, heads, 1, 1) * torch.arange(nk, device=q.device, dtype=f32).view(1, 1, 1, nk)
    m = torch.zeros(B, 1, nq, nk, dtype=torch.bool, device=q.device)
    if causal:
        m = m | (torch.arange(nk, device=q.device)[None, :] > torch.arange(nq, device=q.device)[:, None] + (nk - nq))
    if mask is not None:
        m = m | mask.bool().view(B, 1, nq, nk)
    s = s.masked_fill(m, torch.finfo(f32).min)
    return (s.softmax(-1) @ vh).transpose(1, 2).reshape(B, nq, heads * hd)


def _dense_masks(B, T, kind):
    if kind == "causal":
        return None, True
    lens = [T, max(1, T - 37), max(1, T // 2), 3][:B] + [T] * max(0, B - 4)
    keep = torch.zeros(B, T, dtype=torch.bool)
    for b, n in enumerate(lens):
        if kind == "left_pad":
            keep[b, T - n:] = True
        else:
            keep[b, :n] = True
    causal = torch.arange(T)[None, :] > torch.arange(T)[:, None]
    m = causal[None] | ~keep[:, None, :]          # HF: masked = future key or padded key
    return m.to(torch.uint8).cuda().contiguous(), False


DENSE_CASES = [
    # B, heads, head_dim, T, mask kind, alibi
    (2, 4, 64, 96, "causal", True),
    (3, 2, 128, 200, "causal", True),
    (4, 16, 128, 256, "causal", True),       # MPT-1B block at configs[1]'s T_txt
    (2, 32, 128, 512, "causal", True),       # MPT-7B block at configs[3]'s T_txt
    (4, 4, 64, 130, "left_pad", True),
    (4, 2, 128, 256, "right_pad", True),
    (2, 2, 128, 257, "left_pad", False),
]


@pytest.mark.parametrize("case", DENSE_CASES)
def test_dense_attention_tc_vs_reference(ops, case):
    B, heads, hd, T, kind, alibi = case
    torch.manual_seed(13)
    D = heads * hd
    qkv = torch.randn(B, T, 3 * D, device="cuda").to(bf16)
    q, k, v = qkv[..., :D], qkv[..., D:2 * D], qkv[..., 2 * D:]
    d_o = torch.randn(B, T, D, device="cuda").to(bf16)
    scale = hd ** -0.5
    slopes = (2.0 ** (-8.0 * torch.arange(1, heads + 1, device="cuda", dtype=f32) / heads)) if alibi else None
    mask, causal = _dense_masks(B, T, kind)

    def run():
        o, lse = ops.attn_dense_fwd(q, k, v, heads, hd, scale, causal=causal, mask=mask, slopes=slopes)
        dqkv = torch.empty_like(qkv)
        ops.attn_dense_bwd(q, k, v, o, d_o, lse, heads, hd, scale, causal=causal, mask=mask, slopes=slopes,
                           dq=dqkv[..., :D], dk=dqkv[..., D:2 * D], dv=dqkv[..., 2 * D:])
        torch.cuda.synchronize()
        return o, lse, dqkv

    o, lse, dqkv = run()
    assert torch.isfinite(o.float()).all() and torch.isfinite(dqkv.float()).all()
    qr, kr, vr = (t.float().requires_grad_(True) for t in (q, k, v))
    ref = ref_dense(qr, kr, vr, heads, hd, scale, causal, mask, slopes)
    ref.backward(d_o.float())
    close(o, ref, 2e-2, "dense o")
    close(dqkv[..., :D], qr.grad, 3e-2, "dense dq")
    close(dqkv[..., D:2 * D], kr.grad, 3e-2, "dense dk")
    close(dqkv[..., 2 * D:], vr.grad, 3e-2, "dense dv")


def test_dense_pure_causal_device_flag(ops):
    """An all-ones HF attention_mask arrives as a full [B, T, T] byte mask plus a DEVICE flag saying it is exactly the
    causal rule: the kernel must ignore the bytes (tile skipping) and give the causal result."""
    torch.manual_seed(17)
    B, heads, hd, T = 2, 4, 128, 256
    D = heads * hd
    qkv = torch.randn(B, T, 3 * D, device="cuda").to(bf16)
    q, k, v = qkv[..., :D], qkv[..., D:2 * D], qkv[..., 2 * D:]
    causal_bytes = (torch.arange(T)[None, :] > torch.arange(T)[:, None]).to(torch.uint8)[None].expand(B, T, T).contiguous().cuda()
    flag = torch.ones(1, dtype=torch.int32, device="cuda")
    o1, _ = ops.attn_dense_fwd(q, k, v, heads, hd, hd ** -0.5, causal=False, mask=causal_bytes, pure_causal_flag=flag)
    o2, _ = ops.attn_dense_fwd(q, k, v, heads, hd, hd ** -0.5, causal=True)
    assert torch.equal(o1, o2)
