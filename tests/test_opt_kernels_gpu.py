"""GPU: the OPT block's new kernels -- the residual dropout pair (ofk_dropout_resid_fwd / _bwd), ReLU and its backward,
and the bf16 scale -- against their stated formulas, bit for bit.

Dropout: at p = 0 the forward is a gate-less GATE_RESID_F32 GEMM's result (and, with a bias, BIAS_RESID_F32's); kept
elements are x + bf16(branch * scale) and dropped ones x itself; the backward is nonzero exactly where the forward
kept, with bf16(bf16(dout) * scale); the keep fraction over 2^24 elements is within 6 sigma of 1 - p; the mask depends
on (seed, offset, row, column) only, not on strides; and captured-graph replays draw fresh masks that re-seeding the
device pair reproduces."""
import pytest
import torch

from opt_reference import dropout_scale

pytestmark = pytest.mark.gpu
bf16, f32 = torch.bfloat16, torch.float32


def _pair(seed, offset):
    return torch.tensor([seed, offset], dtype=torch.int64, device="cuda")


def _xb(R, C, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(R, C, device="cuda", generator=g),
            torch.randn(R, C, device="cuda", generator=g).to(bf16))


def test_p0_forward_is_the_gate_less_residual_epilogue():
    from open_flamingo_b200 import _lib as L, ops
    g = torch.Generator(device="cuda").manual_seed(1)
    M, N, K = 300, 512, 256
    a = torch.randn(M, K, device="cuda", generator=g).to(bf16)
    w = torch.randn(N, K, device="cuda", generator=g).to(bf16)
    bias = torch.randn(N, device="cuda", generator=g)
    x = torch.randn(M, N, device="cuda", generator=g)
    want = ops.gemm(a, w, epi=L.EPI_GATE_RESID_F32, aux=x)
    got = ops.dropout_resid_fwd(x, ops.gemm(a, w), 0.0, None)
    assert torch.equal(got, want)
    want_b = ops.gemm(a, w, epi=L.EPI_BIAS_RESID_F32, bias=bias, aux=x)
    got_b = ops.dropout_resid_fwd(x, ops.gemm(a, w, epi=L.EPI_BIAS_BF16, bias=bias), 0.0, _pair(5, 9))
    assert torch.equal(got_b, want_b)
    inplace = x.clone()
    ops.dropout_resid_fwd(inplace, ops.gemm(a, w), 0.0, None, out=inplace)
    assert torch.equal(inplace, want)


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_kept_and_dropped_elements_and_backward(p):
    from open_flamingo_b200 import ops
    R, C = 333, 1040
    x, b = _xb(R, C, 2)
    so = _pair(123456789012345, 77)
    out = ops.dropout_resid_fwd(x, b, p, so)
    keep = ops.dropout_resid_fwd(torch.zeros_like(x), torch.ones_like(b), p, so) != 0
    scale = dropout_scale(p)
    want = torch.where(keep, x + (b.float() * scale).to(bf16).float(), x)
    assert torch.equal(out, want)
    assert torch.equal(out[~keep], x[~keep])
    assert 0 < keep.sum().item() < keep.numel()
    dout = torch.randn(R, C, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    db = ops.dropout_resid_bwd(dout, p, so)
    want_db = torch.where(keep, (dout.to(bf16).float() * scale).to(bf16), torch.zeros_like(b))
    assert torch.equal(db, want_db)
    assert torch.equal(db != 0, keep & (want_db != 0))
    inplace = x.clone()
    ops.dropout_resid_fwd(inplace, b, p, so, out=inplace)
    assert torch.equal(inplace, out)


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_keep_fraction(p):
    from open_flamingo_b200 import ops
    R, C = 4096, 4096   # 2^24 elements
    keep = ops.dropout_resid_fwd(torch.zeros(R, C, device="cuda"), torch.ones(R, C, device="cuda", dtype=bf16), p,
                                 _pair(2024, 3)) != 0
    n = keep.numel()
    frac = keep.sum().item() / n
    sigma = (p * (1 - p) / n) ** 0.5
    assert abs(frac - (1 - p)) <= 6 * sigma, (frac, 1 - p, sigma)
    # columns and rows are not correlated with the draw: every column and row group keeps about 1 - p
    assert (keep.float().mean(0) - (1 - p)).abs().max().item() < 0.05
    assert (keep.float().mean(1) - (1 - p)).abs().max().item() < 0.05


def test_mask_depends_on_seed_offset_row_column_only():
    from open_flamingo_b200 import ops
    R, C, p = 200, 256, 0.3
    x, b = _xb(R, C, 4)
    so = _pair(99, 1000)
    base = ops.dropout_resid_fwd(x, b, p, so)
    assert torch.equal(ops.dropout_resid_fwd(x, b, p, so.clone()), base)
    # the same values in strided views: one more column group of padding per row
    xs = torch.zeros(R, C + 64, device="cuda")
    bs = torch.zeros(R, C + 128, device="cuda", dtype=bf16)
    os_ = torch.full((R, C + 32), float("nan"), device="cuda")
    xs[:, :C], bs[:, :C] = x, b
    ops.dropout_resid_fwd(xs[:, :C], bs[:, :C], p, so, out=os_[:, :C])
    assert torch.equal(os_[:, :C], base)
    assert torch.isnan(os_[:, C:]).all(), "wrote past the row"
    keep_full = ops.dropout_resid_fwd(torch.zeros_like(x), torch.ones_like(b), p, so) != 0
    for other in (_pair(99, 1001), _pair(100, 1000)):
        keep_o = ops.dropout_resid_fwd(torch.zeros_like(x), torch.ones_like(b), p, other) != 0
        assert not torch.equal(keep_o, keep_full)
        assert (keep_o != keep_full).float().mean().item() > 0.2


def test_graph_replays_draw_fresh_masks_and_reseeding_reproduces():
    from open_flamingo_b200 import lm_blocks, ops
    R, C, p = 64, 512, 0.25
    rng = lm_blocks.dropout_rng("cuda")
    zeros, ones = torch.zeros(R, C, device="cuda"), torch.ones(R, C, device="cuda", dtype=bf16)
    out = torch.empty(R, C, device="cuda")
    torch.manual_seed(11)
    rng.take()   # eager call: seeds the device pair from torch's generator
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.dropout_resid_fwd(zeros, ones, p, rng.take(), out=out)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.dropout_resid_fwd(zeros, ones, p, rng.take(), out=out)
    start = rng.state.clone()

    def replays(n):
        res = []
        for _ in range(n):
            graph.replay()
            res.append(out.clone())
        torch.cuda.synchronize()
        return res

    first = replays(3)
    assert not torch.equal(first[0], first[1]) and not torch.equal(first[1], first[2])
    rng.state.copy_(start)
    assert all(torch.equal(a, b) for a, b in zip(first, replays(3)))
    # torch.manual_seed re-draws the seed at the next eager call, and the same seed gives the same sequence
    torch.manual_seed(11)
    a = rng.take()
    torch.manual_seed(11)
    assert torch.equal(rng.take(), a)
    torch.manual_seed(12)
    assert not torch.equal(rng.take()[0], a[0])


def test_relu_relu_backward_and_scale_are_exact():
    from open_flamingo_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(6)
    z = torch.randn(513, 264, device="cuda", generator=g).to(bf16)
    z[0, :8] = torch.tensor([0.0, -0.0, float("inf"), -float("inf"), 1e-38, -1e-38, 3.0, -3.0])
    h = ops.relu_bf16(z)
    assert torch.equal(h, torch.relu(z))
    zz = z.clone()
    ops.relu_bf16(zz, out=zz)
    assert torch.equal(zz, h)
    dh = torch.randn(513, 264, device="cuda", generator=g).to(bf16)
    zr = z.float().requires_grad_(True)
    torch.relu(zr.to(bf16)).backward(dh)
    want = torch.where(h > 0, dh, torch.zeros_like(dh))
    assert torch.equal(ops.relu_bwd_bf16(dh, h), want)
    assert torch.equal(zr.grad.to(bf16), want)
    for hd in (64, 80, 128):
        s = hd ** -0.5
        q = torch.randn(3, 77, 4 * hd, device="cuda", generator=g).to(bf16)
        assert torch.equal(ops.scale_bf16(q, s), q * s), hd   # torch: bf16 tensor * Python float
        wide = torch.randn(50, 3 * 4 * hd, device="cuda", generator=g).to(bf16)
        before = wide.clone()
        ops.scale_bf16(wide[:, :4 * hd], s, out=wide[:, :4 * hd])
        assert torch.equal(wide[:, :4 * hd], before[:, :4 * hd] * s) and torch.equal(wide[:, 4 * hd:],
                                                                                     before[:, 4 * hd:])
