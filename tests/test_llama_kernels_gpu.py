"""GPU: ofk_rmsnorm_fwd / ofk_rmsnorm_bwd and ofk_swiglu_fwd / ofk_swiglu_bwd against float64 restatements of the same
f32 / bf16 inputs.

Bounds (u = 2^-24 per fp32 operation, one bf16 rounding = at most 2^-8 relative):
  RMSNorm forward.  mean(x^2) sums D fp32 products, so its relative error is at most delta = (D + 8) u (the +8 covers
  the product, the division, the eps add and rsqrtf's two ulps); rstd is within delta of float64's.  y is that fp32
  value rounded once:  |y - y64| <= (2^-8 (1 + delta) + delta) |y64|.
  RMSNorm backward.  dx = rstd (g dy - xhat m) + dx_add with m a mean of D fp32 products: every term of the sum is off
  by at most delta of its magnitude and rstd enters up to cubed (xhat m), so
  |dx - dx64| <= 4 delta rstd (|g dy| + |xhat| mean|g dy xhat|) + u |dx_add|.
  SwiGLU forward.  h = bf16(bf16(silu(g)) u): two roundings, silu in fp32 within 8 u:
  |h - silu64(g) u| <= (2 2^-8 + 2^-16 + 8 u) |silu64(g) u|.
  SwiGLU backward.  dg = bf16(dh u silu'(g)): one rounding of an fp32 value within 16 u,
  |dg - dg64| <= (2^-8 + 16 u) |dg64|;  du = bf16(dh bf16(silu(g))): two roundings as in the forward.
bf16 keeps 8 significant bits, so one round-to-nearest moves a value by at most 2^-8 of itself.  These bounds alone
would also admit an extra rounding, so each output is also compared with a float64 restatement that rounds to bf16
exactly where the kernel does: y = bf16(g (x rstd)) with the kernel's own fp32 rstd, h = bf16(bf16(silu(g)) u),
dg = bf16(dh u silu'(g)), du = bf16(dh bf16(silu(g))).  The fp32 evaluation sits within a few u of the float64 one, so
it lands on the other side of a bf16 rounding boundary for a fraction of elements of order 16 u / 2^-8 = 2^-16; all
but 0.1 % of the elements (and one) must match exactly.  An extra rounding (bf16(x rstd) before the gamma product, a rounded dh u) moves tens
of percent.  A tiny absolute term (2^-126) covers values that flush to zero.  Every output is also bitwise
repeatable."""
import pytest
import torch

pytestmark = pytest.mark.gpu
bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64
U = 2.0 ** -24
TINY = 2.0 ** -126


def _mostly_equal(got, want):
    """got equals want (bf16 values) on all but 0.1 % of the elements, and one."""
    miss = (got.double() != want.double()).sum().item()
    assert miss <= 1 + 1e-3 * got.numel(), f"{miss} of {got.numel()} elements off the restatement's rounding"


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _strided(t, extra):
    """t's values in the first columns of a wider buffer: a row stride above the width."""
    buf = torch.full((t.shape[0], t.shape[1] + extra), float("nan"), device=t.device, dtype=t.dtype)
    buf[:, :t.shape[1]] = t
    return buf[:, :t.shape[1]]


@pytest.mark.parametrize("D", [64, 4096, 5120, 8192])
@pytest.mark.parametrize("strided", [False, True])
def test_rmsnorm_forward_and_backward_against_float64(D, strided):
    from open_flamingo_b200 import ops
    rows, eps = 133, 1e-6                     # 133: not a multiple of any block or tile
    g = _gen(D)
    x = torch.randn(rows, D, device="cuda", generator=g) * 3 + 0.5
    x[5] *= 1e-3                              # a small row: eps matters
    gamma = 1 + 0.3 * torch.randn(D, device="cuda", generator=g)
    dy = torch.randn(rows, D, device="cuda", generator=g).to(bf16)
    add = torch.randn(rows, D, device="cuda", generator=g)
    if strided:
        x, dy, add = _strided(x, 64), _strided(dy, 72), _strided(add, 8)
    y, rstd = ops.rmsnorm_fwd(x, gamma, eps)
    delta = (D + 8) * U
    x64, g64 = x.double(), gamma.double()
    rstd64 = torch.rsqrt(x64.pow(2).mean(-1) + eps)
    assert ((rstd.double() - rstd64).abs() <= delta * rstd64).all()
    y64 = g64 * (x64 * rstd64[:, None])
    err = (y.double() - y64).abs()
    assert (err <= (2.0 ** -8 * (1 + delta) + delta) * y64.abs() + TINY).all(), err.max().item()
    _mostly_equal(y, (g64 * (x64 * rstd.double()[:, None])).to(bf16))

    out = torch.full((rows, D + 16), float("nan"), device="cuda", dtype=bf16)[:, :D] if strided else None
    dx = torch.full((rows, D + 4), float("nan"), device="cuda")[:, :D] if strided else None
    y2, rstd2 = ops.rmsnorm_fwd(x, gamma, eps, out=out)
    assert torch.equal(y2, y) and torch.equal(rstd2, rstd), "forward not bitwise repeatable"
    got = ops.rmsnorm_bwd(dy, x, gamma, rstd, dx=dx, dx_add=add)
    gd = g64 * dy.double()
    xh = x64 * rstd64[:, None]
    m = (gd * xh).mean(-1, keepdim=True)
    ref = rstd64[:, None] * (gd - xh * m) + add.double()
    bound = 4 * delta * rstd64[:, None] * (gd.abs() + xh.abs() * (gd * xh).abs().mean(-1, keepdim=True)) + \
        U * add.double().abs() + TINY
    err = (got.double() - ref).abs()
    assert (err <= bound).all(), (err / bound).max().item()
    again = ops.rmsnorm_bwd(dy, x, gamma, rstd, dx_add=add)
    assert torch.equal(again, got), "backward not bitwise repeatable"
    # dx_add aliasing dx: the gradient is added in place
    acc = add.clone()
    ops.rmsnorm_bwd(dy, x, gamma, rstd, dx=acc, dx_add=acc)
    assert torch.equal(acc, got)
    # without dx_add
    plain = ops.rmsnorm_bwd(dy, x, gamma, rstd)
    assert ((plain.double() - (ref - add.double())).abs() <= bound).all()


def _silu64(g):
    return g / (1 + torch.exp(-g))


@pytest.mark.parametrize("F", [8, 11008])
@pytest.mark.parametrize("strided", [False, True])
def test_swiglu_forward_and_backward_against_float64(F, strided):
    from open_flamingo_b200 import ops
    rows = 77
    gen = _gen(F)
    gu = (torch.randn(rows, 2 * F, device="cuda", generator=gen) * 3).to(bf16)
    # large and negative gates: silu(-100) is -0 (exp overflows to inf), silu(100) = 100; no NaN either way
    edge = torch.tensor([-100.0, -88.0, -30.0, -1e-3, 0.0, 1e-3, 30.0, 100.0], device="cuda").to(bf16)
    gu[3, :8] = edge
    dh = torch.randn(rows, F, device="cuda", generator=gen).to(bf16)
    if strided:
        gu, dh = _strided(gu, 24), _strided(dh, 8)
    h = ops.swiglu_fwd(gu)
    assert torch.isfinite(h.float()).all()
    g64, u64 = gu[:, :F].double(), gu[:, F:].double()
    s64 = _silu64(g64)
    ref = s64 * u64
    err = (h.double() - ref).abs()
    assert (err <= (2 * 2.0 ** -8 + 2.0 ** -16 + 8 * U) * ref.abs() + TINY).all(), err.max().item()
    # the restatement with the same two roundings agrees on nearly every element (fp32 silu may sit on the other side
    # of a bf16 rounding boundary)
    _mostly_equal(h, (s64.to(bf16).double() * u64).to(bf16))
    assert h[3, 0].item() == 0   # silu(-100) = -0
    out = torch.empty(rows, F + 8, device="cuda", dtype=bf16)[:, :F] if strided else None
    assert torch.equal(ops.swiglu_fwd(gu, out=out), h)

    dgu = ops.swiglu_bwd(dh, gu)
    assert torch.isfinite(dgu.float()).all()
    sg = torch.sigmoid(g64)
    dg64 = dh.double() * u64 * sg * (1 + g64 * (1 - sg))
    err = (dgu[:, :F].double() - dg64).abs()
    assert (err <= (2.0 ** -8 + 16 * U) * dg64.abs() + TINY).all(), err.max().item()
    _mostly_equal(dgu[:, :F], dg64.to(bf16))
    du64 = dh.double() * s64
    err = (dgu[:, F:].double() - du64).abs()
    assert (err <= (2 * 2.0 ** -8 + 2.0 ** -16 + 8 * U) * du64.abs() + TINY).all(), err.max().item()
    _mostly_equal(dgu[:, F:], (dh.double() * s64.to(bf16).double()).to(bf16))
    out = torch.empty(rows, 2 * F + 16, device="cuda", dtype=bf16)[:, :2 * F] if strided else None
    assert torch.equal(ops.swiglu_bwd(dh, gu, out=out), dgu), "backward not bitwise repeatable"


def test_zero_rows_make_empty_outputs_without_a_launch():
    from open_flamingo_b200 import _lib, ops
    n0 = _lib.launch_count()
    x = torch.empty(0, 64, device="cuda")
    y, rstd = ops.rmsnorm_fwd(x, torch.ones(64, device="cuda"), 1e-6)
    assert y.shape == (0, 64) and rstd.shape == (0,)
    dx = ops.rmsnorm_bwd(torch.empty(0, 64, device="cuda", dtype=bf16), x, torch.ones(64, device="cuda"), rstd)
    assert dx.shape == (0, 64)
    gu = torch.empty(0, 32, device="cuda", dtype=bf16)
    assert ops.swiglu_fwd(gu).shape == (0, 16)
    assert ops.swiglu_bwd(torch.empty(0, 16, device="cuda", dtype=bf16), gu).shape == (0, 32)
    assert _lib.launch_count() == n0
