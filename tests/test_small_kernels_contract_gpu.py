"""GPU: the LayerNorm, cross-entropy and elementwise kernels against float64 restatements, with per-element bounds.

Entry points: ofk_layernorm_fwd / _bwd (every LN of the ViT, the Perceiver, the gated blocks and the frozen MPT blocks),
ofk_ce_fwd / _bwd (the training loss, through fused.causal_lm_loss and called directly for the per-row LSE),
ofk_cast_f32_bf16, ofk_add_f32, ofk_patchify, ofk_vit_assemble, ofk_gate_bwd, ofk_sumsq and ofk_adamw.

The references are computed in float64 on the GPU from the exact values the kernel read (bf16 inputs as their float
values; the backward of LayerNorm from the forward's own f32 mean / rstd; each AdamW step from the kernel's own state).
Inputs are views inside NaN-filled buffers, so a read outside the view poisons the result.  Outputs are windows inside
NaN-filled buffers, and the bytes around each window must come back bit-identical.  Every reduction is run twice and
must give bitwise-equal results.

Exact operations, checked bit for bit: cast_bf16 (round to nearest even; NaN positions only, payloads may differ),
add_ (one fp32 add), patchify (a gather and one rounding), vit_assemble (bf16 -> f32 and one fp32 add), gate_bwd with
no gate (a cast), and AdamW's bf16 copy (= bf16(p) after every step).

Bounds (u = 2^-24, the fp32 unit roundoff; 2^-8 that of bf16, whose significand has 8 bits; a sum added in a chain of
depth k is off by at most k u sum|terms|):
  LayerNorm forward (one warp per row, lane sums of ceil(D/128) float4s, pairwise inside a float4, then a 5-level
  butterfly: depth k = ceil(D/128) + 8):
    mean:  dmu <= k u sum|x| / D + u |mu|
    var:   the second pass sums (x - mu_hat)^2 = var + (mu - mu_hat)^2, so dvar <= dmu^2 + (k + 3) u (var + dmu^2)
    rstd:  rsqrtf (2 ulp) of var + eps: eps_r <= dvar / (2 (var + eps)) + 4u
    y:     |y - Y| <= |g| r (|x - mu| (eps_r + 4u) + dmu (1 + eps_r)) + 3u (|Y| + |b|);  bf16 y adds 2^-8 (|Y| + that)
  LayerNorm backward (rows striped over <= 528 blocks of 256 threads; row sums: ceil(D/1024) + 2 per thread, 5 warp
  levels, 8 warps in order: k1 = ceil(D/1024) + 16):
    a = dy g, xh = (x - mean) rstd (2u), m1 = sum a / D, m2 = sum a xh / D,
    dm1 <= (k1 + 2) u sum|a| / D,  dm2 <= (k1 + 5) u sum|a xh| / D,
    |dx - ref| <= rstd (dm1 + |xh| dm2 + 5u (|a| + |m1| + |xh m2|)) + 2u (|ref| + |dx_add|)
    dgamma / dbeta: per thread a chain over the block's rows (ceil(rows / nblocks)), then per column 16 row groups of
    ceil(nblocks / 16) partials and the fixed 16-term sum: k2 = ceil(rows / nblocks) + ceil(nblocks / 16) + 18,
    |dgamma - ref| <= (k2 + 4) u sum|dy xh| + u |ref|,  |dbeta - ref| <= (k2 + 1) u sum|dy| + u |ref|.
  Cross-entropy (one 256-thread block per row, online (max, sum) per thread, then warp and block combines; every
  element is rescaled at most c = ceil(V/256) + 13 times, and each __expf of an argument t is off by 2^-21 + 3u|t|,
  the arguments of one element adding up to at most 3 (M - v)):
    lse:   |lse - ref| <= c (2^-21 + 6u) + 9u sum_j p_j (M - v_j) + 2u |log l| + 2u |lse| + 4u
    loss:  (sum over counted rows of the lse bound + (ceil(rows/256) + 14) u sum|lse - v_target|) / count + u |loss|
    dlogits: (p (|dlse| + 2^-21 + 3u |v - lse| + 4u) + 2^-126) |g| / count + 4u |ref|, dlse the measured LSE error
    and 2^-126 the flush of __expf results below FLT_MIN; bf16 adds 2^-8 (|ref| + that).
  gate_bwd: dbranch within (2^-8 + 8u) |dout tanh(g)|;  dgate: a chain of 8 products per grid-stride step, 5 + 8
    levels per block, then <= 2112 partials (9 per thread, 5 + 8 levels): k = 8 ceil(n / (8 grid 256)) + 40,
    |dgate - ref| <= (k + 2) u (1 - t^2) sum|dout branch| + 8u |sum dout branch| + u |ref|  (tanhf: 2 ulp).
  sumsq: k = ceil(n / (grid 256)) + 36,  |out - ref| <= (k + 1) u sum x^2 + u |ref|.
  AdamW, per step from the kernel's own state, with the f32 hyper-parameters the kernel received:
    dm <= 4u (b1 |m| + (1 - b1) |g'|),  dv <= 5u (b2 v + (1 - b2) g'^2),
    bias corrections: eps_bc = u from the host, or 8u b^step / bc + u from the device step (powf: 4 ulp),
    |p - ref| <= 4u |p_old| + |lr/bc1| (dm + |m| (eps_den + eps_step + 3u)) / denom + u |ref|,
    eps_den = 10u + eps_bc2 / 2 (sqrtf of v, rsqrtf of bc2, a product and + eps), eps_step = 2u + eps_bc1."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64
U = 2.0 ** -24
BF16_U = 2.0 ** -8                   # unit roundoff of bf16 (8-bit significand): one rounding is off by <= 2^-8 relative
FLUSH = 2.0 ** -126                  # __expf flushes results below FLT_MIN to zero
NAN = float("nan")


@pytest.fixture(scope="module")
def ops():
    from open_flamingo_b200 import ops as _ops
    return _ops


@pytest.fixture(scope="module")
def lib():
    from open_flamingo_b200 import _lib
    return _lib


# ------------------------------------------------------------------ NaN-surrounded views and canary windows
class Window:
    """A [rows, cols] window at (r0, c0) of a NaN-filled [r0 + rows + pad, ld] buffer (1-D: rows = None)."""

    def __init__(self, rows, cols, dtype, r0=1, c0=4, pad=2, ld=None):
        if rows is None:
            self.buf = torch.full((c0 + cols + pad,), NAN, device="cuda", dtype=dtype)
            self.view = self.buf[c0:c0 + cols]
        else:
            ld = c0 + cols + 8 if ld is None else ld
            self.buf = torch.full((r0 + rows + pad, ld), NAN, device="cuda", dtype=dtype)
            self.view = self.buf[r0:r0 + rows, c0:c0 + cols]
        self.inside = torch.zeros(self.buf.shape, dtype=torch.bool, device="cuda")
        if rows is None:
            self.inside[c0:c0 + cols] = True
        else:
            self.inside[r0:r0 + rows, c0:c0 + cols] = True
        self.before = self.buf.clone()

    def fill(self, t):
        self.view.copy_(t.reshape(self.view.shape))
        self.before = self.buf.clone()
        return self.view

    def outside_untouched(self, what):
        bits = {1: torch.uint8, 2: torch.int16, 4: torch.int32}[self.buf.element_size()]
        same = self.buf.view(bits) == self.before.view(bits)
        assert bool(same[~self.inside].all()), f"{what}: bytes outside the output window changed"

    def check(self, what):
        self.outside_untouched(what)
        assert not bool(torch.isnan(self.view.float()).any()), f"{what}: NaN left inside the output window"


def placed(t, c0=4):
    """t (2-D) as a view at row 1, column c0 of a NaN-filled buffer with 8 spare columns (row stride cols + c0 + 8)."""
    w = Window(t.shape[0], t.shape[1], t.dtype, c0=c0)
    return w.fill(t)


def within(err, bound, what):
    worst = (err / bound).max().item()
    assert worst <= 1.0, f"{what}: off by {worst:.3g}x its bound (max |err| {err.max().item():.3e})"


# ------------------------------------------------------------------ LayerNorm
LN_D = [4, 60, 1020, 1024, 1028, 2044, 2048, 2052, 2560, 4092, 4096]
LN_ROWS = [1, 3, 5, 527, 528, 529, 1057]
EPS = 1e-5


def ln_inputs(rows, D, seed):
    """x rows: N(0.5, 2) except row 0 = 1000 + 0.01 z (large mean, small spread), row 1 constant, row 2 one outlier
    column (its position moves with D); gamma / beta per-column N(0, 1)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(rows, D, device="cuda", generator=g) * 2 + 0.5
    if rows > 0:
        x[0] = 1000.0 + 0.01 * torch.randn(D, device="cuda", generator=g)
    if rows > 1:
        x[1] = 3.0
    if rows > 2:
        x[2] = 0.1 * torch.randn(D, device="cuda", generator=g)
        x[2, (D * 5) // 7] = 400.0
    gamma = torch.randn(D, device="cuda", generator=g)
    beta = torch.randn(D, device="cuda", generator=g)
    return x, gamma, beta


def ln_fwd_ref(x, gamma, beta):
    X = x.to(f64)
    D = X.shape[1]
    mu = X.mean(1, keepdim=True)
    var = ((X - mu) ** 2).mean(1, keepdim=True)
    r = 1.0 / torch.sqrt(var + EPS)
    Y = (X - mu) * r * gamma.to(f64) + beta.to(f64)
    k = math.ceil(D / 128) + 8
    dmu = k * U * X.abs().sum(1, keepdim=True) / D + U * mu.abs()
    dvar = dmu ** 2 + (k + 3) * U * (var + dmu ** 2)
    eps_r = dvar / (2 * (var + EPS)) + 4 * U
    bound = gamma.to(f64).abs() * r * ((X - mu).abs() * (eps_r + 4 * U) + dmu * (1 + eps_r)) + \
        3 * U * (Y.abs() + beta.to(f64).abs())
    return dict(Y=Y, mu=mu[:, 0], r=r[:, 0], dmu=dmu[:, 0], eps_r=eps_r[:, 0], bound=bound)


def check_ln_fwd(R, y, mean, rstd, what):
    b = R["bound"]
    if y.dtype == bf16:
        b = b + BF16_U * (R["Y"].abs() + b)
    within((y.to(f64) - R["Y"]).abs(), b + 1e-300, f"{what} y")
    if mean is not None:
        within((mean.to(f64) - R["mu"]).abs(), R["dmu"] + 1e-300, f"{what} mean")
        within((rstd.to(f64) - R["r"]).abs(), R["eps_r"] * R["r"], f"{what} rstd")


def ln_bwd_ref(dy, x, gamma, mean, rstd, dx_add=None, dgamma0=None, dbeta0=None):
    """The backward the kernel computes, from the kernel's own f32 mean / rstd."""
    X, DY, G = x.to(f64), dy.to(f64), gamma.to(f64)
    rows, D = X.shape
    r = rstd.to(f64)[:, None]
    xh = (X - mean.to(f64)[:, None]) * r
    a = DY * G
    m1 = a.mean(1, keepdim=True)
    m2 = (a * xh).mean(1, keepdim=True)
    dx = r * (a - m1 - xh * m2)
    add = torch.zeros_like(dx) if dx_add is None else dx_add.to(f64)
    dx = dx + add
    k1 = math.ceil(D / 1024) + 16
    dm1 = (k1 + 2) * U * a.abs().sum(1, keepdim=True) / D
    dm2 = (k1 + 5) * U * (a * xh).abs().sum(1, keepdim=True) / D
    bdx = r * (dm1 + xh.abs() * dm2 + 5 * U * (a.abs() + m1.abs() + (xh * m2).abs())) + 2 * U * (dx.abs() + add.abs())
    nblocks = min(rows, 528)
    k2 = math.ceil(rows / nblocks) + math.ceil(nblocks / 16) + 18
    dg = (DY * xh).sum(0) + (0 if dgamma0 is None else dgamma0.to(f64))
    db = DY.sum(0) + (0 if dbeta0 is None else dbeta0.to(f64))
    bdg = (k2 + 4) * U * (DY * xh).abs().sum(0) + U * dg.abs()
    bdb = (k2 + 1) * U * DY.abs().sum(0) + U * db.abs()
    return dict(dx=dx, bdx=bdx, dg=dg, bdg=bdg, db=db, bdb=bdb)


@pytest.mark.parametrize("rows", LN_ROWS)
@pytest.mark.parametrize("D", LN_D)
def test_layernorm_against_float64(ops, D, rows):
    x, gamma, beta = ln_inputs(rows, D, seed=rows * 7919 + D)
    xv, gv, bv = placed(x), Window(None, D, f32).fill(gamma), Window(None, D, f32).fill(beta)
    R = ln_fwd_ref(x, gamma, beta)
    for dt in (f32, bf16):
        w = Window(rows, D, dt)
        y, mean, rstd = ops.layernorm_fwd(xv, gv, bv, EPS, out=w.view)
        w.check(f"ln fwd {dt}")
        check_ln_fwd(R, y, mean, rstd, f"ln fwd {dt} D={D} rows={rows}")
        y2, mean2, rstd2 = ops.layernorm_fwd(xv, gv, bv, EPS, out=torch.empty_like(w.view))
        assert torch.equal(y2, y) and torch.equal(mean2, mean) and torch.equal(rstd2, rstd), "ln fwd not repeatable"
    g = torch.Generator(device="cuda").manual_seed(D + rows)
    dy32 = torch.randn(rows, D, device="cuda", generator=g)
    add = torch.randn(rows, D, device="cuda", generator=g)
    dg0 = torch.randn(D, device="cuda", generator=g)
    db0 = torch.randn(D, device="cuda", generator=g)
    for dyt in (f32, bf16):
        dy = placed(dy32.to(dyt))
        Rb = ln_bwd_ref(dy, x, gamma, mean, rstd, dx_add=add, dgamma0=dg0, dbeta0=db0)
        results = []
        for _ in range(2):
            dxw, dgw, dbw = Window(rows, D, f32), Window(None, D, f32), Window(None, D, f32)
            dgw.fill(dg0)
            dbw.fill(db0)
            out = ops.layernorm_bwd(dy, xv, gv, mean, rstd, dgamma=dgw.view, dbeta=dbw.view, dx=dxw.view,
                                    dx_add=placed(add))
            assert out.data_ptr() == dxw.view.data_ptr()
            for win, name in ((dxw, "dx"), (dgw, "dgamma"), (dbw, "dbeta")):
                win.check(f"ln bwd {name}")
            results.append((dxw.view.clone(), dgw.view.clone(), dbw.view.clone()))
        what = f"ln bwd dy={dyt} D={D} rows={rows}"
        within((results[0][0].to(f64) - Rb["dx"]).abs(), Rb["bdx"] + 1e-300, f"{what} dx")
        within((results[0][1].to(f64) - Rb["dg"]).abs(), Rb["bdg"] + 1e-300, f"{what} dgamma")
        within((results[0][2].to(f64) - Rb["db"]).abs(), Rb["bdb"] + 1e-300, f"{what} dbeta")
        assert all(torch.equal(p, q) for p, q in zip(*results)), f"{what}: not bitwise repeatable"


@pytest.mark.parametrize("D", [64, 1028, 2560])
def test_layernorm_backward_modes(ops, D):
    """want_dx=False with the affine gradients, dx / dbeta only, and dx is dx_add (in place), each against the full
    backward's reference; bf16 dy."""
    rows = 529
    x, gamma, beta = ln_inputs(rows, D, seed=D)
    _, mean, rstd = ops.layernorm_fwd(x, gamma, beta, EPS)
    g = torch.Generator(device="cuda").manual_seed(3 * D)
    dy = torch.randn(rows, D, device="cuda", generator=g).to(bf16)
    add = torch.randn(rows, D, device="cuda", generator=g)
    dg0, db0 = torch.randn(D, device="cuda", generator=g), torch.randn(D, device="cuda", generator=g)
    R = ln_bwd_ref(dy, x, gamma, mean, rstd, dgamma0=dg0, dbeta0=db0)
    Ra = ln_bwd_ref(dy, x, gamma, mean, rstd, dx_add=add)
    # parameter gradients only
    dgw, dbw = Window(None, D, f32), Window(None, D, f32)
    dgw.fill(dg0)
    dbw.fill(db0)
    assert ops.layernorm_bwd(dy, x, gamma, mean, rstd, dgamma=dgw.view, dbeta=dbw.view, want_dx=False) is None
    dgw.check("dgamma")
    dbw.check("dbeta")
    within((dgw.view.to(f64) - R["dg"]).abs(), R["bdg"], "want_dx=False dgamma")
    within((dbw.view.to(f64) - R["db"]).abs(), R["bdb"], "want_dx=False dbeta")
    # dx and dbeta, no dgamma
    dbw = Window(None, D, f32)
    dbw.fill(db0)
    dx = ops.layernorm_bwd(dy, x, gamma, mean, rstd, dbeta=dbw.view)
    within((dx.to(f64) - R["dx"]).abs(), R["bdx"] + 1e-300, "dx with dbeta only")
    within((dbw.view.to(f64) - R["db"]).abs(), R["bdb"], "dbeta only")
    # dx only, in place onto dx_add
    buf = Window(rows, D, f32)
    inplace = buf.fill(add)
    out = ops.layernorm_bwd(dy, x, gamma, mean, rstd, dx=inplace, dx_add=inplace)
    buf.check("dx is dx_add")
    assert out.data_ptr() == inplace.data_ptr()
    within((inplace.to(f64) - Ra["dx"]).abs(), Ra["bdx"] + 1e-300, "dx is dx_add")


@pytest.mark.parametrize("D", [64, 1028, 2560])
@pytest.mark.parametrize("U_,v,n", [(3, 20, 8), (2, 257, 64), (1, 5, 529)])
def test_layernorm_group_mapping_fwd_bwd(ops, D, U_, v, n):
    """Two LayerNorms fill the halves of cat((x, latents), -2) in place and read their gradients back through the same
    mapping (fused.PerceiverLayerFn: media rows -> parameter gradients only, latent rows -> dx accumulated in place)."""
    x, g1, b1 = ln_inputs(U_ * v, D, seed=11 + D)
    lat, g2, b2 = ln_inputs(U_ * n, D, seed=13 + D)
    w = Window(U_ * (v + n), D, bf16)
    _, xm, xr = ops.layernorm_fwd(x, g1, b1, EPS, out=w.view, rows_per_group=v, group_stride=v + n, group_offset=0)
    cat = w.view.view(U_, v + n, D)
    assert bool(torch.isnan(cat[:, v:].float()).all()), "the media LayerNorm wrote latent rows"
    _, lm, lr = ops.layernorm_fwd(lat, g2, b2, EPS, out=w.view, rows_per_group=n, group_stride=v + n, group_offset=v)
    w.check("grouped fwd")
    check_ln_fwd(ln_fwd_ref(x, g1, b1), cat[:, :v].reshape(-1, D), xm, xr, "grouped fwd media")
    check_ln_fwd(ln_fwd_ref(lat, g2, b2), cat[:, v:].reshape(-1, D), lm, lr, "grouped fwd latents")
    g = torch.Generator(device="cuda").manual_seed(D * 5 + v)
    dkv = placed(torch.randn(U_ * (v + n), D, device="cuda", generator=g).to(bf16))
    d3 = dkv.view(U_, v + n, D)
    dg0, db0 = torch.randn(D, device="cuda", generator=g), torch.randn(D, device="cuda", generator=g)
    Rm = ln_bwd_ref(d3[:, :v].reshape(-1, D), x, g1, xm, xr, dgamma0=dg0, dbeta0=db0)
    dg, db = dg0.clone(), db0.clone()
    assert ops.layernorm_bwd(dkv, x, g1, xm, xr, dgamma=dg, dbeta=db, want_dx=False, rows_per_group=v,
                             group_stride=v + n, group_offset=0) is None
    within((dg.to(f64) - Rm["dg"]).abs(), Rm["bdg"], "grouped bwd media dgamma")
    within((db.to(f64) - Rm["db"]).abs(), Rm["bdb"], "grouped bwd media dbeta")
    prev = torch.randn(U_ * n, D, device="cuda", generator=g)
    Rl = ln_bwd_ref(d3[:, v:].reshape(-1, D), lat, g2, lm, lr, dx_add=prev, dgamma0=dg0, dbeta0=db0)
    buf = Window(U_ * n, D, f32)
    dlat = buf.fill(prev)
    dg, db = dg0.clone(), db0.clone()
    ops.layernorm_bwd(dkv, lat, g2, lm, lr, dgamma=dg, dbeta=db, dx=dlat, dx_add=dlat, rows_per_group=n,
                      group_stride=v + n, group_offset=v)
    buf.check("grouped bwd latents dx")
    within((dlat.to(f64) - Rl["dx"]).abs(), Rl["bdx"] + 1e-300, "grouped bwd latents dx")
    within((dg.to(f64) - Rl["dg"]).abs(), Rl["bdg"], "grouped bwd latents dgamma")
    within((db.to(f64) - Rl["db"]).abs(), Rl["bdb"], "grouped bwd latents dbeta")


def test_layernorm_rejects_bad_operands(ops):
    D, rows = 256, 10
    x, g, b = ln_inputs(rows, D, seed=1)
    _, mean, rstd = ops.layernorm_fwd(x, g, b)
    dy = torch.randn(rows, D, device="cuda")
    bad_fwd = [dict(gamma=g.to(bf16)), dict(gamma=g[:-4]), dict(beta=torch.randn(2 * D, device="cuda")[::2]),
               dict(out=torch.empty(rows - 1, D, device="cuda", dtype=bf16)),
               dict(out=torch.empty(rows, D, device="cuda", dtype=torch.float16)),
               dict(out=torch.empty(13, D, device="cuda", dtype=bf16), rows_per_group=5, group_stride=7,
                    group_offset=2),                                       # row 9 -> 1 * 7 + 2 + 4: needs 14 rows
               dict(out=torch.empty(100, D, device="cuda", dtype=bf16), rows_per_group=5, group_stride=7,
                    group_offset=3)]                                       # 3 + 5 > 7
    for kw in bad_fwd:
        args = dict(gamma=g, beta=b)
        args.update(kw)
        with pytest.raises(ValueError):
            ops.layernorm_fwd(x, args.pop("gamma"), args.pop("beta"), **args)
    bad_bwd = [dict(mean=mean.double()), dict(mean=mean[:-1]), dict(rstd=rstd[:-1]),
               dict(dgamma=torch.zeros(D + 4, device="cuda")), dict(dbeta=torch.zeros(D, device="cuda", dtype=bf16)),
               dict(dx=torch.empty(rows, D - 4, device="cuda")), dict(dx_add=torch.zeros(rows, D, device="cuda",
                                                                                          dtype=bf16)),
               dict(gamma=g[:-4]), dict(dy=dy[:-1]),
               dict(dy=torch.randn(13, D, device="cuda"), rows_per_group=5, group_stride=7, group_offset=2),
               dict(dy=torch.randn(100, D, device="cuda"), rows_per_group=5, group_stride=7, group_offset=3)]
    for kw in bad_bwd:
        args = dict(dy=dy, gamma=g, mean=mean, rstd=rstd)
        args.update(kw)
        with pytest.raises(ValueError):
            ops.layernorm_bwd(args.pop("dy"), x, args.pop("gamma"), args.pop("mean"), args.pop("rstd"), **args)
    # aligned row stride, misaligned base pointer: rejected by the library before any launch
    xb = torch.randn(rows, D + 8, device="cuda")
    with pytest.raises(RuntimeError, match="aligned"):
        ops.layernorm_fwd(xb[:, 1:1 + D], g, b)
    with pytest.raises(RuntimeError, match="aligned"):
        ops.layernorm_bwd(dy, xb[:, 2:2 + D], g, mean, rstd)
    with pytest.raises(RuntimeError, match="aligned"):
        ops.layernorm_fwd(x, g, b, out=torch.empty(rows, D + 8, device="cuda", dtype=bf16)[:, 2:2 + D])


# ------------------------------------------------------------------ cross-entropy
CE_V = [8, 61, 2048, 2056, 50277, 50280]


def ce_reference(lg, labels, ignore_index):
    """lg: [rows, V] as the kernel reads it; labels [B, T].  Float64 LSE, shifted targets, per-row loss terms."""
    B, T = labels.shape
    X = lg.to(f64)
    rows, V = X.shape
    tgt = torch.full((B, T), ignore_index, dtype=torch.int64, device="cuda")
    tgt[:, :-1] = labels[:, 1:]
    tgt = tgt.reshape(-1)
    valid = (tgt != ignore_index) & (tgt >= 0) & (tgt < V)
    M = X.amax(1, keepdim=True)
    l = torch.exp(X - M).sum(1, keepdim=True)
    lse = (M + torch.log(l))[:, 0]
    P = torch.exp(X - lse[:, None])
    fin = torch.isfinite(X)
    gap = torch.where(fin, M - X, torch.zeros_like(X))
    c = math.ceil(V / 256) + 13
    blse = c * (2.0 ** -21 + 6 * U) + 9 * U * (P * gap).sum(1) + 2 * U * torch.log(l[:, 0]).abs() + \
        2 * U * lse.abs() + 4 * U
    safe = torch.where(valid, tgt, torch.zeros_like(tgt))
    vt = X.gather(1, safe[:, None])[:, 0]
    term = torch.where(valid, lse - vt, torch.zeros_like(lse))
    return dict(X=X, lse=lse, blse=blse, P=P, tgt=tgt, valid=valid, term=term, safe=safe)


def ce_direct(lib, lg, labels, ignore_index, gscale, dwin):
    """ofk_ce_fwd / ofk_ce_bwd on a [rows, V] view (row stride free), as fused.CausalLMLossFn calls them."""
    rows, V = lg.shape
    T = labels.shape[1]
    lab = labels.contiguous()
    lsew = Window(None, rows, f32)
    acc = torch.zeros(2, device="cuda")
    lib.check(lib.lib().ofk_ce_fwd(lg.data_ptr(), int(lg.dtype == f32), lg.stride(0), rows, V, lab.data_ptr(), T, 1,
                                   int(ignore_index), lsew.view.data_ptr(), acc[0:1].data_ptr(), acc[1:2].data_ptr(),
                                   lib.stream_ptr()))
    gs = torch.tensor([gscale], device="cuda")
    lib.check(lib.lib().ofk_ce_bwd(lg.data_ptr(), int(lg.dtype == f32), lg.stride(0), rows, V, lab.data_ptr(), T, 1,
                                   int(ignore_index), lsew.view.data_ptr(), gs.data_ptr(), acc[1:2].data_ptr(),
                                   dwin.view.data_ptr(), dwin.view.stride(0), lib.stream_ptr()))
    lsew.outside_untouched("lse")
    return lsew.view.clone(), acc


def check_ce(R, lse, loss, count, dlogits, gscale, what):
    lerr = (lse.to(f64) - R["lse"]).abs()
    within(lerr, R["blse"], f"{what} lse")
    valid = R["valid"]
    n = int(valid.sum().item())
    assert count == n, f"{what}: count {count} != {n}"
    if n == 0:
        assert math.isnan(loss), f"{what}: a batch with every target ignored must give NaN (0 / 0), got {loss}"
    else:
        ref = R["term"].sum().item() / n
        rows = R["X"].shape[0]
        ks = math.ceil(rows / 256) + 14
        b = ((R["blse"] * valid).sum().item() + ks * U * R["term"].abs().sum().item()) / n + 2 * U * abs(ref)
        assert abs(loss - ref) <= b, f"{what}: loss {loss!r} vs {ref!r} (bound {b:.3e})"
    sc = gscale / max(n, 1)
    onehot = torch.zeros_like(R["P"]).scatter_(1, R["safe"][:, None], 1.0)
    ref = torch.where(valid[:, None], (R["P"] - onehot) * sc, torch.zeros_like(R["P"]))
    gap = torch.where(torch.isfinite(R["X"]), (R["X"] - R["lse"][:, None]).abs(), torch.zeros_like(R["X"]))
    b = (R["P"] * (lerr[:, None] + 2.0 ** -21 + 3 * U * gap + 4 * U) + FLUSH) * abs(sc) + 4 * U * ref.abs()
    b = torch.where(valid[:, None], b, torch.zeros_like(b))
    if dlogits.dtype == bf16:
        b = b + BF16_U * (ref.abs() + b)
    within((dlogits.to(f64) - ref).abs(), b + 1e-300, f"{what} dlogits")


def ce_logits(B, T, V, dtype, seed, scale=3.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, T, V, device="cuda", generator=g) * scale
    return x.to(dtype).float(), g


def ce_labels(B, T, V, g, ignore_index):
    """Distinct labels at t = 0 of every row; targets at columns 0, 7, 8, 2047, 2048 and V - 1 (where they exist);
    a few ignored positions."""
    labels = torch.randint(0, V, (B, T), device="cuda", generator=g)
    labels[:, 0] = torch.arange(B, device="cuda") % V
    edges = [c for c in (0, 7, 8, 2047, 2048, V - 1) if c < V]
    for i, c in enumerate(edges):
        if T > 1:
            labels[i % B, 1 + (i * 3) % (T - 1)] = c
    if T > 4:
        labels[0, 3] = ignore_index
        labels[B - 1, T - 2] = ignore_index
    return labels


def run_ce(lib, x3, labels, ignore_index, dtype, col0, ld, what, gscale=1.7):
    """x3: [B, T, V] float values (dtype-representable).  The logits are a [B, T, V] column slice at column col0 of a
    NaN-filled [B, T, ld] buffer; checked through causal_lm_loss (loss and autograd gradient) and ofk_ce_* (LSE and a
    dlogits window)."""
    from open_flamingo_b200.fused import causal_lm_loss
    B, T, V = x3.shape
    buf = torch.full((B, T, ld), NAN, device="cuda", dtype=dtype)
    buf[..., col0:col0 + V] = x3.to(dtype)
    lg3 = buf[..., col0:col0 + V]
    R = ce_reference(lg3.reshape(B * T, V), labels, ignore_index)
    losses, grads = [], []
    for _ in range(2):
        leaf = lg3.detach().requires_grad_(True)
        loss = causal_lm_loss(leaf, labels, V, ignore_index=ignore_index)
        (loss * gscale).backward()
        losses.append(loss.detach())
        grads.append(leaf.grad.reshape(B * T, V))
    assert not bool(torch.isnan(grads[0].float()).any()), f"{what}: NaN in the gradient"
    assert torch.equal(losses[0], losses[1]) or (losses[0].isnan() and losses[1].isnan()), f"{what}: loss not repeatable"
    assert torch.equal(grads[0], grads[1]), f"{what}: gradient not repeatable"
    dwin = Window(B * T, V, dtype, c0=col0, ld=ld)
    lse, acc = ce_direct(lib, lg3.reshape(B * T, V), labels, ignore_index, gscale, dwin)
    dwin.outside_untouched(f"{what} dlogits")
    assert torch.equal(dwin.view, grads[0]), f"{what}: ofk_ce_bwd into a window differs from the autograd gradient"
    count = int(acc[1].item())
    check_ce(R, lse, losses[0].item(), count, grads[0], gscale, what)
    return R, losses[0], grads[0]


# (first column, row stride) of the [B, T, V] logits inside a wider buffer.  slice-col3: a row stride that is a multiple
# of 8 with rows starting 6 (bf16) or 12 (f32) bytes past a 16-byte boundary, which must take the scalar path.
LAYOUTS = {"dense": lambda V: (0, V), "slice-aligned": lambda V: (8, V + 24), "slice-col3": lambda V: (3, V + 24),
           "slice-odd-ld": lambda V: (1, V + 5)}


@pytest.mark.parametrize("dtype", [bf16, f32], ids=["bf16", "f32"])
@pytest.mark.parametrize("V", CE_V)
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_cross_entropy_against_float64(lib, layout, V, dtype):
    B, T = (2, 40) if V > 10000 else (3, 17)
    x3, g = ce_logits(B, T, V, dtype, seed=V + 3)
    # a target equal to its row's max
    x3[1, 4, 5 % V] = x3[1, 4].max() + 1.0
    labels = ce_labels(B, T, V, g, -100)
    labels[1, 5] = 5 % V
    col0, ld = LAYOUTS[layout](V)
    run_ce(lib, x3, labels, -100, dtype, col0, ld, f"ce {layout} V={V} {dtype}")


@pytest.mark.parametrize("dtype", [bf16, f32], ids=["bf16", "f32"])
@pytest.mark.parametrize("V", [61, 2048, 2056])
def test_cross_entropy_many_rows(lib, V, dtype):
    """>= 2048 rows: the one-block loss sum strides over rows; a custom ignore_index that is a real class, and a label
    of -100 that is then out of range (dropped from the sum and the count)."""
    B, T = 4, 520
    x3, g = ce_logits(B, T, V, dtype, seed=V)
    labels = ce_labels(B, T, V, g, 5)
    labels[2, 7] = -100
    labels[3, 100:110] = 5
    R, _, _ = run_ce(lib, x3, labels, 5, dtype, 0, V, f"ce rows={B * T} V={V} {dtype}")
    assert not bool(R["valid"].view(B, T)[3, 99:109].any())


@pytest.mark.parametrize("dtype", [bf16, f32], ids=["bf16", "f32"])
@pytest.mark.parametrize("V", [61, 2056, 50280])
def test_cross_entropy_every_target_ignored(lib, V, dtype):
    """Every label ignored (and 1 x 1, where the shift leaves nothing): the loss is NaN and the gradient zero, as HF's
    ForCausalLMLoss gives on CPU."""
    from transformers.loss.loss_utils import ForCausalLMLoss
    from open_flamingo_b200.fused import causal_lm_loss
    for B, T in ((1, 1), (2, 9)):
        x3, g = ce_logits(B, T, V, dtype, seed=V + T)
        labels = torch.randint(0, V, (B, T), device="cuda", generator=g)
        if T > 1:
            labels[:, 1:] = -100
        run_ce(lib, x3, labels, -100, dtype, 0, V, f"ce all ignored {B}x{T}")
        ref_leaf = x3.to(dtype).cpu().requires_grad_(True)
        ref = ForCausalLMLoss(ref_leaf, labels.cpu(), V)
        (ref * 1.7).backward()
        leaf = x3.to(dtype).requires_grad_(True)
        got = causal_lm_loss(leaf, labels, V)
        (got * 1.7).backward()
        assert math.isnan(ref.item()) and math.isnan(got.item())
        assert torch.equal(leaf.grad.cpu(), ref_leaf.grad)


@pytest.mark.parametrize("dtype", [bf16, f32], ids=["bf16", "f32"])
@pytest.mark.parametrize("V", [61, 2048, 2056, 50280])
@pytest.mark.parametrize("layout", ["dense", "slice-col3"])
def test_cross_entropy_large_and_infinite_logits(lib, layout, V, dtype):
    """fp32 logits of +-1e4, and rows with -inf entries (masked vocabulary): rows whose first 2048 columns are -inf
    (every thread of both read paths starts at -inf), rows with scattered -inf, and one row that is -inf but for its
    target.  The loss is finite, as HF's is."""
    B, T = 2, 33
    x3, g = ce_logits(B, T, V, dtype, seed=V * 3, scale=1e4 if dtype == f32 else 3.0)
    labels = ce_labels(B, T, V, g, -100)
    x3[0, 2:6, :min(2048, V - 1)] = -math.inf
    x3[1, 10:20] = torch.where(torch.rand(10, V, device="cuda", generator=g) < 0.3, -math.inf, x3[1, 10:20])
    x3[1, 25] = -math.inf
    x3[1, 25, labels[1, 26]] = 0.5
    tgt = torch.full((B, T), 0, dtype=torch.int64, device="cuda")
    tgt[:, :-1] = labels[:, 1:]
    ok = (tgt < 0) | (tgt >= V)
    hit = torch.isinf(x3.gather(2, tgt.clamp(0, V - 1)[..., None])[..., 0]) & ~ok
    x3[hit.nonzero(as_tuple=True) + (tgt[hit],)] = 1.0                   # keep every target finite
    col0, ld = LAYOUTS[layout](V)
    _, loss, grad = run_ce(lib, x3, labels, -100, dtype, col0, ld, f"ce inf {layout} V={V} {dtype}")
    assert math.isfinite(loss.item()) and bool(torch.isfinite(grad.float()).all())


# ------------------------------------------------------------------ exact elementwise kernels
def cast_inputs(n, seed):
    """Ties of bf16 rounding (odd and even), values one ulp either side, subnormals, +-0, +-inf, NaN, the overflow edge
    (the largest float that rounds to the largest bf16, the smallest that rounds to inf), and normal values."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    ints = torch.randint(0, 2 ** 16, (n,), device="cuda", generator=g, dtype=torch.int64)
    hi = torch.randint(0, 2 ** 15, (n,), device="cuda", generator=g, dtype=torch.int64)
    kind = torch.arange(n, device="cuda") % 8
    low = torch.where(kind == 0, torch.full_like(ints, 0x8000), ints)                  # exact ties
    low = torch.where(kind == 1, torch.full_like(ints, 0x7FFF), low)                   # just below a tie
    low = torch.where(kind == 2, torch.full_like(ints, 0x8001), low)                   # just above
    bits = (hi << 16) | low
    bits = torch.where(kind == 3, bits & 0x007FFFFF, bits)                             # subnormals
    x = (bits.to(torch.int32)).view(f32).clone()
    x = torch.where(torch.arange(n, device="cuda") % 16 == 9, -x, x)
    specials = torch.tensor([0.0, -0.0, math.inf, -math.inf, NAN, 3.3895313892515355e38, 3.3895314e38,
                             -3.3961775292304025e38, 1e-45, -1e-45, 1.0, -2.5], device="cuda")
    specials[5] = torch.tensor([0x7F7F7FFF], dtype=torch.int32).view(f32).item()      # rounds down to bf16 max
    specials[6] = torch.tensor([0x7F7F8000], dtype=torch.int32).view(f32).item()      # tie at the top: rounds to inf
    specials[7] = -torch.tensor([0x7F7FC000], dtype=torch.int32).view(f32).item()
    k = min(n, specials.numel())
    x[(torch.arange(k, device="cuda") * 7) % n] = specials[:k]
    return x


@pytest.mark.parametrize("n", list(range(1, 18)) + [1003, 4_325_376 * 2 + 13])
def test_cast_bf16_bitwise(ops, n):
    x = cast_inputs(n, seed=n)
    src = Window(None, n, f32).fill(x)
    w = Window(None, n, bf16, c0=8)
    ops.cast_bf16(src, out=w.view)
    w.outside_untouched("cast")
    ref = x.to(bf16)
    got_nan, ref_nan = torch.isnan(w.view), torch.isnan(ref)
    assert torch.equal(got_nan, ref_nan), "cast: NaN positions differ"
    assert torch.equal(w.view[~got_nan].view(torch.int16), ref[~ref_nan].view(torch.int16)), "cast: bits differ"


@pytest.mark.parametrize("n", [1, 3, 4, 5, 8, 9, 1003, 4096, 2_000_003])
def test_add_bitwise(ops, n):
    g = torch.Generator(device="cuda").manual_seed(n)
    a = torch.randn(n, device="cuda", generator=g) * torch.exp(4 * torch.randn(n, device="cuda", generator=g))
    b = torch.randn(n, device="cuda", generator=g)
    dst = Window(None, n, f32)
    dst.fill(a)
    ops.add_(dst.view, Window(None, n, f32).fill(b))
    dst.check("add")
    assert torch.equal(dst.view, a + b)


def test_add_cast_reject_bad_operands(ops):
    a = torch.randn(1000, device="cuda")
    for src in (a[:-4], a.to(bf16), torch.randn(2000, device="cuda")[::2]):
        with pytest.raises(ValueError):
            ops.add_(a, src)
    with pytest.raises(ValueError):
        ops.add_(torch.randn(2000, device="cuda")[::2], a)
    with pytest.raises(ValueError):
        ops.cast_bf16(a, out=torch.empty(999, device="cuda", dtype=bf16))
    with pytest.raises(ValueError):
        ops.cast_bf16(a.double())
    with pytest.raises(RuntimeError, match="aligned"):
        ops.add_(a[1:], torch.randn(999, device="cuda"))


@pytest.mark.parametrize("n,H,W,P", [(2, 28, 42, 14), (1, 48, 32, 16), (3, 14, 14, 14), (2, 224, 112, 14)])
@pytest.mark.parametrize("padded", [False, True])
def test_patchify_bitwise(ops, lib, n, H, W, P, padded):
    g = torch.Generator(device="cuda").manual_seed(H * W + P)
    img = torch.randn(n, 3, H, W, device="cuda", generator=g)
    kvalid = 3 * P * P
    ldp = (kvalid + 63) // 64 * 64 + (64 if kvalid % 64 == 0 else 0) if padded else kvalid
    rows = n * (H // P) * (W // P)
    ref = img.to(bf16).unfold(2, P, P).unfold(3, P, P).permute(0, 2, 3, 1, 4, 5).reshape(rows, kvalid)
    w = Window(None, rows * ldp, bf16, c0=5)                     # patch rows need no alignment (2-byte stores)
    lib.check(lib.lib().ofk_patchify(img.data_ptr(), n, H, W, P, w.view.data_ptr(), ldp, lib.stream_ptr()))
    w.check("patchify")
    out = w.view.view(rows, ldp)
    assert torch.equal(out[:, :kvalid].view(torch.int16), ref.view(torch.int16))
    assert torch.equal(out[:, kvalid:].view(torch.int16), torch.zeros_like(out[:, kvalid:]).view(torch.int16)), \
        "patchify padding is not exactly +0"
    if ldp == 640:
        assert torch.equal(ops.patchify(img, P, ldp), out)


@pytest.mark.parametrize("n,g,D", [(1, 0, 4), (2, 1, 4), (3, 4, 12), (2, 256, 64), (1, 16, 1028), (2, 49, 1024)])
def test_vit_assemble_bitwise(ops, lib, n, g, D):
    gen = torch.Generator(device="cuda").manual_seed(n * 1000 + g + D)
    pe = torch.randn(n * g, D, device="cuda", generator=gen).to(bf16)
    cls = torch.randn(D, device="cuda", generator=gen)
    pos = torch.randn(g + 1, D, device="cuda", generator=gen)
    pev = Window(None, n * g * D, bf16, c0=4).fill(pe).view(n * g, D)
    clsv = Window(None, D, f32).fill(cls)
    posv = Window(None, (g + 1) * D, f32).fill(pos).view(g + 1, D)
    tok = ops.vit_assemble(pev, clsv, posv, n, g, D).view(n, g + 1, D)
    ref = torch.cat([cls.expand(n, 1, D), pe.float().view(n, g, D)], 1) + pos
    assert torch.equal(tok, ref)
    w = Window(None, n * (g + 1) * D, f32)
    lib.check(lib.lib().ofk_vit_assemble(pev.data_ptr(), clsv.data_ptr(), posv.data_ptr(), n, g, D, w.view.data_ptr(),
                                         lib.stream_ptr()))
    w.check("vit_assemble")
    assert torch.equal(w.view.view(n, g + 1, D), ref)
    bads = [dict(pe=pe.float()), dict(cls=cls.to(bf16)), dict(cls=cls[:-4] if D > 4 else cls[:0]), dict(pos=pos[:-1]),
            dict(pe=torch.zeros(n * g + 1, D, device="cuda", dtype=bf16))]
    for bad in bads:
        a = dict(pe=pe, cls=cls, pos=pos)
        a.update(bad)
        with pytest.raises(ValueError):
            ops.vit_assemble(a["pe"], a["cls"], a["pos"], n, g, D)
    if g > 0:
        flat = torch.empty(n * g * D + 2, device="cuda", dtype=bf16)
        with pytest.raises(RuntimeError, match="aligned"):
            ops.vit_assemble(flat[2:].view(n * g, D), cls, pos, n, g, D)


# ------------------------------------------------------------------ gate backward and sumsq
GRID_SPAN = 132 * 16 * 256                  # threads of a full grid-stride pass


@pytest.mark.parametrize("n", [8, 8 * 1001, 3 * GRID_SPAN * 8 + 56])
@pytest.mark.parametrize("gate_value", [0.3, 0.0, -0.7, None])
def test_gate_bwd_against_float64(ops, n, gate_value):
    g = torch.Generator(device="cuda").manual_seed(n)
    dout = torch.randn(n, device="cuda", generator=g)
    branch = torch.randn(n, device="cuda", generator=g).to(bf16)
    doutv = Window(None, n, f32).fill(dout)
    branchv = Window(None, n, bf16, c0=8).fill(branch)
    if gate_value is None:
        db = ops.gate_bwd(doutv, None, None, None)
        assert torch.equal(db.view(torch.int16), dout.to(bf16).view(torch.int16)), "gate None: not a plain cast"
        return
    gate = torch.tensor([gate_value], device="cuda")
    t = math.tanh(float(gate.item()))
    dg0 = 0.625
    outs = []
    for _ in range(2):
        dgate = torch.full((1,), dg0, device="cuda")
        db = ops.gate_bwd(doutv, branchv, gate, dgate)
        outs.append((db, dgate))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1]), "gate_bwd not repeatable"
    db, dgate = outs[0]
    ref = dout.to(f64) * t
    within((db.to(f64) - ref).abs(), (BF16_U + 8 * U) * ref.abs() + 1e-300, "dbranch")
    prod = dout.to(f64) * branch.to(f64)
    dot = prod.sum().item()
    want = dg0 + (1 - t * t) * dot
    grid = min(math.ceil(n / 8 / 256), 132 * 16)
    k = 8 * math.ceil(n / (8 * grid * 256)) + 40
    b = (k + 2) * U * (1 - t * t) * prod.abs().sum().item() + 8 * U * abs(dot) + U * abs(want)
    assert abs(dgate.item() - want) <= b, f"dgate {dgate.item()!r} vs {want!r} (bound {b:.3e})"


def test_gate_bwd_rejects_bad_operands(ops):
    n = 8 * 100
    dout = torch.randn(n, device="cuda")
    br = torch.randn(n, device="cuda").to(bf16)
    gate, dgate = torch.tensor([0.2], device="cuda"), torch.zeros(1, device="cuda")
    for args in ((dout, br[:-8], gate, dgate), (dout, br, gate.double(), dgate), (dout, br.float(), gate, dgate),
                 (dout.to(bf16), br, gate, dgate), (dout, None, gate, dgate), (dout, br, gate, dgate.double())):
        with pytest.raises(ValueError):
            ops.gate_bwd(*args)
    t = torch.randn(n + 8, device="cuda")
    with pytest.raises(RuntimeError, match="aligned"):
        ops.gate_bwd(t[3:3 + n], br, gate, dgate)                       # contiguous, 12 bytes off
    with pytest.raises(RuntimeError, match="aligned"):
        ops.gate_bwd(dout, torch.randn(n + 8, device="cuda").to(bf16)[4:4 + n], gate, dgate)


@pytest.mark.parametrize("n", [1, 1001, 3 * GRID_SPAN + 17])
def test_sumsq_against_float64(ops, n):
    g = torch.Generator(device="cuda").manual_seed(n)
    x = torch.randn(n, device="cuda", generator=g) * torch.exp(2 * torch.randn(n, device="cuda", generator=g))
    xv = Window(None, n, f32, c0=1).fill(x)                          # read one float at a time: any 4-byte offset
    outs = []
    for _ in range(2):
        out = torch.full((1,), 2.5, device="cuda")
        ops.sumsq_(xv, out)
        outs.append(out)
    assert torch.equal(outs[0], outs[1]), "sumsq not repeatable"
    sq = x.to(f64) ** 2
    want = 2.5 + sq.sum().item()
    grid = min(math.ceil(n / 256), 132 * 16)
    k = math.ceil(n / (grid * 256)) + 36
    b = (k + 1) * U * sq.sum().item() + U * abs(want)
    assert abs(outs[0].item() - want) <= b, f"sumsq {outs[0].item()!r} vs {want!r} (bound {b:.3e})"
    with pytest.raises(ValueError):
        ops.sumsq_(x.to(bf16), out)
    with pytest.raises(ValueError):
        ops.sumsq_(x, out.double())


# ------------------------------------------------------------------ AdamW
def f32v(v):
    return float(torch.tensor(v, dtype=f32).item())


@pytest.mark.parametrize("start", [1, 10_000])
@pytest.mark.parametrize("wd", [0.1, 0.0])
@pytest.mark.parametrize("device_args", ["host", "clip", "step_dev", "lr_dev", "all"])
def test_adamw_against_float64(ops, device_args, wd, start):
    """Six steps, each checked against a float64 AdamW step (torch.optim.AdamW's update) from the kernel's own state.
    Device arguments replace the host values they override, so a kernel that ignored them would be caught."""
    n = 10007
    g = torch.Generator(device="cuda").manual_seed(n + start)
    p = torch.randn(n, device="cuda", generator=g)
    m = torch.zeros(n, device="cuda")
    v = torch.zeros(n, device="cuda")
    if start > 1:
        m = 0.01 * torch.randn(n, device="cuda", generator=g)
        v = 1e-4 * torch.rand(n, device="cuda", generator=g)
    w16 = Window(None, n, bf16, c0=8)
    lr, b1, b2, eps = 1e-2, 0.9, 0.999, 1e-8
    use_clip = device_args in ("clip", "all")
    use_step = device_args in ("step_dev", "all")
    use_lr = device_args in ("lr_dev", "all")
    clip = torch.tensor([0.37], device="cuda") if use_clip else None
    step_dev = torch.zeros(1, device="cuda") if use_step else None
    lr_dev = torch.tensor([3e-3], device="cuda") if use_lr else None
    F = f32v
    for i in range(6):
        step = start + i
        grad = torch.randn(n, device="cuda", generator=g)
        grad[::17] = 0.0                                                # g = 0: the denominator is sqrt(v) or eps
        P0, M0, V0 = p.to(f64), m.to(f64), v.to(f64)
        if use_step:
            step_dev.fill_(float(step))
        host_step = 1 if use_step else step                           # a wrong host value the device step overrides
        ops.adamw_(p, grad, m, v, w16.view, 1.0 if use_lr else lr, b1, b2, eps, wd, host_step, clip, step_dev, lr_dev)
        w16.check("w16")
        assert torch.equal(w16.view.view(torch.int16), p.to(bf16).view(torch.int16)), "w16 != bf16(p)"
        B1, B2, EPS, WD = F(b1), F(b2), F(eps), F(wd)
        LR = F(3e-3) if use_lr else F(lr)
        cs = F(0.37) if use_clip else 1.0
        G = grad.to(f64) * cs
        bc1, bc2 = 1 - B1 ** step, 1 - B2 ** step
        if use_step:
            e1 = 8 * U * B1 ** step / bc1 + U
            e2 = 8 * U * B2 ** step / bc2 + U
        else:
            bc1, bc2 = F(1 - b1 ** step), F(1 - b2 ** step)
            e1 = e2 = U
        Mr = B1 * M0 + (1 - B1) * G
        Vr = B2 * V0 + (1 - B2) * G * G
        den = torch.sqrt(Vr) / math.sqrt(bc2) + EPS
        Pr = P0 * (1 - LR * WD) - (LR / bc1) * Mr / den
        dm = 4 * U * (B1 * M0.abs() + (1 - B1) * G.abs())
        within((m.to(f64) - Mr).abs(), dm + 1e-300, f"exp_avg step {step}")
        within((v.to(f64) - Vr).abs(), 5 * U * Vr + 1e-300, f"exp_avg_sq step {step}")
        eps_den, eps_step = 10 * U + e2 / 2, 2 * U + e1
        bp = 4 * U * P0.abs() + (LR / bc1) * (dm + Mr.abs() * (eps_den + eps_step + 3 * U)) / den + U * Pr.abs()
        within((p.to(f64) - Pr).abs(), bp, f"param step {step} ({device_args}, wd {wd})")


def test_adamw_matches_torch_optim(ops):
    """Three steps from zero state against torch.optim.AdamW run in float64."""
    n = 10007
    g = torch.Generator(device="cuda").manual_seed(11)
    p = torch.randn(n, device="cuda", generator=g)
    grad = torch.randn(n, device="cuda", generator=g)
    pr = p.to(f64).clone().requires_grad_(True)
    opt = torch.optim.AdamW([pr], lr=1e-2, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.1)
    m, v = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    w16 = torch.empty(n, device="cuda", dtype=bf16)
    for step in (1, 2, 3):
        pr.grad = grad.to(f64)
        opt.step()
        ops.adamw_(p, grad, m, v, w16, 1e-2, 0.9, 0.999, 1e-8, 0.1, step)
    err = (p.to(f64) - pr.detach()).abs()
    # three steps of the per-step bound above, plus the f32 rounding of the hyper-parameters (lr, betas)
    assert err.max().item() <= 2e-6 * pr.detach().abs().max().item(), err.max().item()
    assert torch.equal(w16, p.to(bf16))


def test_adamw_rejects_bad_operands(ops):
    n = 1000
    t = [torch.zeros(n, device="cuda") for _ in range(4)]
    w16 = torch.empty(n, device="cuda", dtype=bf16)
    bad = [(0, t[0][:-1]), (1, t[1].to(bf16)), (2, t[2][:-1]), (3, torch.zeros(2 * n, device="cuda")[::2]),
           (4, torch.empty(n - 1, device="cuda", dtype=bf16)), (4, torch.empty(n, device="cuda"))]
    for i, b in bad:
        args = t + [w16]
        args[i] = b
        with pytest.raises(ValueError):
            ops.adamw_(*args, 1e-3, 0.9, 0.999, 1e-8, 0.0, 1)
    with pytest.raises(ValueError):
        ops.adamw_(*t, w16, 1e-3, 0.9, 0.999, 1e-8, 0.0, 1, clip_scale=torch.ones(1, device="cuda", dtype=f64))
    with pytest.raises(ValueError):
        ops.adamw_(*t, w16, 1e-3, 0.9, 0.999, 1e-8, 0.0, 1, step_dev=torch.ones(1, device="cuda", dtype=torch.int32))
