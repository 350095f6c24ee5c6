"""GPU: the contract of the wgmma GEMM (csrc/gemm.cu), checked exactly wherever the arithmetic allows.

Operands are small integers times one power of two, so every product and partial sum is exact in fp32 and the float64
product is what the kernel's accumulators hold, in any summation order.  Outputs that are a single rounding of that
sum (fp32 stores, atomics, bf16 stores, residual adds) must match bit for bit; the GELU / gate epilogues, whose
transcendental functions are approximations, are held to per-element bounds derived from those approximations.

Covered: all 40 instantiations (4 operand layouts x 10 epilogues) at tile edges, operands that are views with
poisoned neighbours, output windows inside canary buffers, in-place residual updates, the grouped row maps, the
streaming-store path, and independence of the result from the persistent grid's size."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64
LAYOUTS = [(False, False), (False, True), (True, True), (True, False)]
EPIS = ["STORE_BF16", "STORE_F32", "ATOMIC_F32", "BIAS_BF16", "BIAS_QGELU_BF16", "GELU_DUAL", "GATE_RESID_F32",
        "DGELU_BF16", "BIAS_RESID_F32", "BIAS_GELU_BF16"]
BIAS_EPIS = {"BIAS_BF16", "BIAS_QGELU_BF16", "BIAS_RESID_F32", "BIAS_GELU_BF16"}
GATE = 0.7


@pytest.fixture(scope="module")
def ops():
    from open_flamingo_b200 import ops as _ops
    return _ops


@pytest.fixture(scope="module")
def L():
    from open_flamingo_b200 import _lib
    return _lib


def _up8(x):
    return (x + 7) // 8 * 8


class Problem:
    """One GEMM problem: A [M, K] and B [N, K] (logical, float64) and the epilogue inputs.

    A and B are integers with |sum| <= K * lim^2 <= 2^23, A scaled by a power of two that puts the products in about
    [-6, 6], the range over which the GELU epilogues are checked.  bf16 rounding depends only on the significant bits,
    and the integer sums carry up to 23 of them, so bf16 outputs are genuinely rounded (ties included).  Bias,
    residual and atomic initial values are integers on the same grid, so the fp32 adds of the epilogues are exact."""

    def __init__(self, M, N, K, seed):
        self.M, self.N, self.K = M, N, K
        g = torch.Generator(device="cuda").manual_seed(seed)

        def ints(lim, *shape):
            return torch.randint(-lim, lim + 1, shape, generator=g, device="cuda", dtype=f64)

        lim = min(100, math.isqrt((1 << 23) // K))
        ai, bi = ints(lim, M, K), ints(lim, N, K)
        acc_i = ai @ bi.t()
        top = max(int(acc_i.abs().max().item()), 6)
        s = 2.0 ** -math.ceil(math.log2(top / 6))
        self.A, self.B, self.acc = ai * s, bi, acc_i * s
        self.bias = ints(max(1, top // 4), N) * s
        self.resid = ints(top, M, N) * s
        self.init = ints(top, M, N) * s
        self.z = (torch.rand(M, N, generator=g, device="cuda", dtype=f64) * 12 - 6).to(bf16)   # saved pre-activation


def operand(x, mn, pad=0, fill=0.0):
    """x: logical [rows, K] float64, exact in bf16.  Returns it as a bf16 view stored K-major ([rows, K]) or MN-major
    ([K, rows]) inside a buffer with `pad` extra rows and at least `pad` extra columns (row stride a multiple of 8
    elements), holding `fill` outside the view."""
    t = x.t() if mn else x
    r, c = t.shape
    buf = torch.full((r + pad, _up8(c + pad)), fill, device="cuda", dtype=bf16)
    view = buf[:r, :c]
    view.copy_(t)
    return view


def to_bf16(x):
    """Round-to-nearest-even to bf16 of a float64 tensor whose values are exact in fp32 (as the accumulators are)."""
    return x.float().to(bf16)


def gelu64(x):
    return 0.5 * x * (1.0 + torch.special.erf(x / math.sqrt(2.0)))


def gelu64_grad(x):
    return 0.5 * (1.0 + torch.special.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


def qgelu64(x):
    return x * torch.sigmoid(1.702 * x)


def exact(got, want, what):
    assert got.dtype == want.dtype and got.shape == want.shape, what
    if not torch.equal(got, want):
        bad = (got != want).nonzero()
        i = tuple(bad[0].tolist())
        raise AssertionError(f"{what}: {len(bad)} of {want.numel()} elements differ; first at {i}: "
                             f"got {got[i].item()!r}, want {want[i].item()!r}")


def within(got, ref, bound, what):
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)   # a NaN is out of bound
    if bad.any():
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError(f"{what}: {int(bad.sum())} of {ref.numel()} elements out of bound; first at {i}: "
                             f"got {got[i].item()!r}, ref {ref[i].item()!r}, bound {bound[i].item():.3e}")


def fresh(rows, cols, dtype):
    return torch.empty((rows, cols), device="cuda", dtype=dtype)


def run_epilogue(ops, L, name, p, a, b, a_mn, b_mn, alloc=fresh):
    """Run epilogue `name` on (a, b), which hold p.A and p.B, with outputs from `alloc`, and check every output
    against p's float64 reference."""
    M, N = p.M, p.N
    epi = getattr(L, "EPI_" + name)
    kw = dict(a_mn=a_mn, b_mn=b_mn, epi=epi)
    if name in BIAS_EPIS:
        kw["bias"] = p.bias.float()
    acc = p.acc
    accb = to_bf16(acc)
    what = f"{name} {(M, N, p.K)} a_mn={a_mn} b_mn={b_mn}"
    if name == "STORE_F32":
        exact(ops.gemm(a, b, out=alloc(M, N, f32), **kw), acc.float(), what)
    elif name == "ATOMIC_F32":
        for splits in (1, 3):   # split order cannot change an exact sum
            out = alloc(M, N, f32)
            out.copy_(p.init)
            ops.gemm(a, b, out=out, splits=splits, **kw)
            exact(out, (p.init + acc).float(), f"{what} splits={splits}")
    elif name == "STORE_BF16":
        exact(ops.gemm(a, b, out=alloc(M, N, bf16), **kw), accb, what)
    elif name == "BIAS_BF16":
        exact(ops.gemm(a, b, out=alloc(M, N, bf16), **kw), to_bf16(acc + p.bias), what)
    elif name in ("BIAS_GELU_BF16", "BIAS_QGELU_BF16"):
        t = to_bf16(acc + p.bias).double()
        ref = gelu64(t) if name == "BIAS_GELU_BF16" else qgelu64(t)
        within(ops.gemm(a, b, out=alloc(M, N, bf16), **kw), ref, 2.0 ** -8 * ref.abs() + 1e-6, what)
    elif name == "GELU_DUAL":
        z, h = alloc(M, N, bf16), alloc(M, N, bf16)
        ops.gemm(a, b, out=z, out2=h, **kw)
        exact(z, accb, what + " z")
        ref = gelu64(accb.double())
        within(h, ref, 2.0 ** -8 * ref.abs() + 1e-6, what + " h")
    elif name == "DGELU_BF16":
        ref = accb.double() * gelu64_grad(p.z.double())
        got = ops.gemm(a, b, out=alloc(M, N, bf16), aux=p.z, **kw)
        within(got, ref, 2.0 ** -8 * ref.abs() + 5e-7 * accb.double().abs(), what)
    elif name in ("GATE_RESID_F32", "BIAS_RESID_F32"):
        branch = to_bf16(acc + p.bias) if name == "BIAS_RESID_F32" else accb
        resid = p.resid.float()
        br = alloc(M, N, bf16)
        out = ops.gemm(a, b, out=alloc(M, N, f32), out2=br, aux=resid, **kw)   # gate NULL: multiplier 1
        exact(out, (branch.double() + p.resid).float(), what)
        exact(br, branch, what + " out2")
        if name == "GATE_RESID_F32":
            gate = torch.tensor([GATE], device="cuda", dtype=f32)
            tg = math.tanh(float(gate.item()))
            br2 = alloc(M, N, bf16)
            out = ops.gemm(a, b, out=alloc(M, N, f32), out2=br2, aux=resid, gate=gate, **kw)
            ref = accb.double() * tg + p.resid
            within(out, ref, 2.0 ** -21 * ((accb.double() * tg).abs() + p.resid.abs()), what + " gated")
            exact(br2, accb, what + " gated out2")
    else:
        raise AssertionError(name)


# ------------------------------------------------------------------ A. every instantiation at tile edges
EDGE_SHAPES = [
    (1, 16, 8),         # smallest legal sizes; a partial k-block
    (65, 144, 72),      # one row past a half-tile; one tile + 16 columns; one k-block + 8
    (200, 48, 64),      # N < 64: the second 64-column epilogue half is skipped, the second 32-column group half masked
    (129, 272, 328),    # M, N and K all past tile multiples
    (1153, 400, 136),   # 10 m-tiles: the last GROUP_M raster group is partial
    (33, 64, 5),        # K not a multiple of 8: K-major operands need a padded row stride
]


@pytest.mark.parametrize("name", EPIS)
@pytest.mark.parametrize("a_mn,b_mn", LAYOUTS)
@pytest.mark.parametrize("M,N,K", EDGE_SHAPES)
def test_every_instantiation_at_tile_edges(ops, L, M, N, K, a_mn, b_mn, name):
    p = Problem(M, N, K, seed=M * 7 + N * 3 + K)
    run_epilogue(ops, L, name, p, operand(p.A, a_mn), operand(p.B, b_mn), a_mn, b_mn)


@pytest.mark.parametrize("name", EPIS)
def test_streaming_stores_are_exact(ops, L, name):
    """Outputs of 16 Mi elements or more are written with evict-first stores (st.global.cs): a separate store path."""
    p = Problem(4096, 4096, 72, seed=41)
    run_epilogue(ops, L, name, p, operand(p.A, False), operand(p.B, True), False, True)


# ------------------------------------------------------------------ B. poisoned strided operands
@pytest.mark.parametrize("a_mn,b_mn", LAYOUTS)
@pytest.mark.parametrize("M,N,K", [(33, 64, 5), (65, 144, 72), (129, 272, 328)])
def test_operand_views_read_nothing_outside_the_view(ops, L, M, N, K, a_mn, b_mn):
    """A and B are views into buffers that are NaN everywhere else, with at least a whole TMA box (128 rows, 64 columns)
    of margin on every side that TMA could read from: past K (within the row stride for K-major operands, the next rows
    for MN-major ones) and past M / N.  One NaN read would spread through the sums."""
    p = Problem(M, N, K, seed=5)
    nan = float("nan")
    a, b = operand(p.A, a_mn, pad=128, fill=nan), operand(p.B, b_mn, pad=128, fill=nan)
    for name in ("STORE_F32", "STORE_BF16", "ATOMIC_F32"):
        run_epilogue(ops, L, name, p, a, b, a_mn, b_mn)


# ------------------------------------------------------------------ C. output canaries
class Canvas:
    """Hands out output windows inside larger buffers filled with a fixed bit pattern (a NaN): 5 rows and 8 columns in
    from the corner, a row stride != N, and a margin of more than one 128 x 128 tile below and to the right.  `check`
    asserts that everything outside the windows is bitwise unchanged."""
    PATTERN = {f32: (torch.int32, 0x7FA5A5A5), bf16: (torch.int16, 0x7FA5)}
    R0, C0 = 5, 8   # the window keeps 16-byte alignment for f32 and bf16

    def __init__(self):
        self.windows = []

    def __call__(self, rows, cols, dtype):
        buf = torch.empty((self.R0 + rows + 136, _up8(self.C0 + cols + 136)), device="cuda", dtype=dtype)
        it, pat = self.PATTERN[dtype]
        buf.view(it).fill_(pat)
        self.windows.append((buf, rows, cols))
        return buf[self.R0:self.R0 + rows, self.C0:self.C0 + cols]

    def check(self, what):
        for buf, rows, cols in self.windows:
            it, pat = self.PATTERN[buf.dtype]
            outside = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
            outside[self.R0:self.R0 + rows, self.C0:self.C0 + cols] = False
            bad = (buf.view(it) != pat) & outside
            assert not bad.any(), f"{what}: {int(bad.sum())} elements written outside the window, first at " \
                                  f"{tuple(bad.nonzero()[0].tolist())} (window at {(self.R0, self.C0)}, {rows} x {cols})"


@pytest.mark.parametrize("name", EPIS)
@pytest.mark.parametrize("M,N,K", [(129, 272, 328), (200, 48, 64)])
def test_outputs_write_only_inside_their_window(ops, L, M, N, K, name):
    p = Problem(M, N, K, seed=9)
    canvas = Canvas()
    for a_mn, b_mn in ((False, False), (True, True)):
        run_epilogue(ops, L, name, p, operand(p.A, a_mn), operand(p.B, b_mn), a_mn, b_mn, alloc=canvas)
    canvas.check(name)


# ------------------------------------------------------------------ D. residual aliasing
@pytest.mark.parametrize("name", ["BIAS_RESID_F32", "GATE_RESID_F32"])
def test_residual_epilogues_in_place_and_with_differently_strided_aux(ops, L, name):
    """x += branch in place (aux is out, as in the ViT blocks), and an aux whose row stride and offset differ from
    out's."""
    p = Problem(129, 272, 328, seed=13)
    M, N = p.M, p.N
    a, b = operand(p.A, False), operand(p.B, True)
    kw = dict(b_mn=True, epi=getattr(L, "EPI_" + name))
    if name in BIAS_EPIS:
        kw["bias"] = p.bias.float()
    branch = to_bf16(p.acc + p.bias) if name == "BIAS_RESID_F32" else to_bf16(p.acc)
    want = (branch.double() + p.resid).float()
    x = p.resid.float()
    assert ops.gemm(a, b, aux=x, out=x, **kw) is x
    exact(x, want, name + " in place")
    aux = torch.full((M + 3, N + 36), float("nan"), device="cuda")[3:, 4:4 + N]
    aux.copy_(p.resid)
    out = torch.full((M, N + 8), float("nan"), device="cuda")[:, :N]
    ops.gemm(a, b, aux=aux, out=out, **kw)
    exact(out, want, name + " strided aux")


# ------------------------------------------------------------------ E. grouped row maps
def plain_expected(p, name):
    return {"STORE_BF16": lambda: to_bf16(p.acc), "BIAS_BF16": lambda: to_bf16(p.acc + p.bias),
            "STORE_F32": lambda: p.acc.float()}[name]()


@pytest.mark.parametrize("name", ["STORE_BF16", "BIAS_BF16", "STORE_F32"])
@pytest.mark.parametrize("v,n", [(64, 8), (100, 28), (256, 64)])
def test_grouped_out_map_fills_the_halves_of_an_interleaved_buffer(ops, L, v, n, name):
    """Two GEMMs write the media rows and the latent rows of a [U*(v+n), N] buffer, as PerceiverAttention's k/v
    projection does: each writes only its own rows, and together they give cat((media, latents), rows)."""
    U, N, K = 3, 160, 72
    pm, pl = Problem(U * v, N, K, seed=17), Problem(U * n, N, K, seed=18)
    dtype = f32 if name == "STORE_F32" else bf16
    canvas = Canvas()
    kv = canvas(U * (v + n), N, dtype)
    kv3 = kv.view(U, v + n, N)
    epi = getattr(L, "EPI_" + name)
    ops.gemm_grouped(operand(pm.A, False), operand(pm.B, False), epi=epi, bias=pm.bias.float(), out=kv, M=U * v, N=N,
                     K=K, out_map=(v, v + n, 0))
    it, pat = Canvas.PATTERN[dtype]
    assert (kv3[:, v:].contiguous().view(it) == pat).all(), "the media GEMM wrote into latent rows"
    exact(kv3[:, :v].reshape(U * v, N), plain_expected(pm, name), "media rows")
    ops.gemm_grouped(operand(pl.A, False), operand(pl.B, False), epi=epi, bias=pl.bias.float(), out=kv, M=U * n, N=N,
                     K=K, out_map=(n, v + n, v))
    want = torch.cat([plain_expected(pm, name).view(U, v, N), plain_expected(pl, name).view(U, n, N)], 1)
    exact(kv3.contiguous(), want, "interleaved buffer")
    canvas.check("grouped out_map")


@pytest.mark.parametrize("name", ["ATOMIC_F32", "STORE_F32"])
@pytest.mark.parametrize("b_mn", [True, False])
@pytest.mark.parametrize("half", ["media", "latents"])
def test_grouped_ak_map_reduces_over_one_half(ops, L, half, b_mn, name):
    """Weight gradient over only the media (or only the latent) rows of a concatenated [U*(v+n), M] gradient, as the
    Perceiver backward does.  The rows that are not selected are NaN."""
    U, v, n, M, N = 3, 128, 64, 200, 80
    rows, go = (v, 0) if half == "media" else (n, v)
    K = U * rows
    p = Problem(M, N, K, seed=23)
    buf = torch.full((U * (v + n) + 64, _up8(M + 64)), float("nan"), device="cuda", dtype=bf16)
    buf[:U * (v + n)].view(U, v + n, -1)[:, go:go + rows, :M] = p.A.t().reshape(U, rows, M).to(bf16)
    a = buf[:U * (v + n), :M]
    b = operand(p.B, b_mn)
    epi = getattr(L, "EPI_" + name)
    out = fresh(M, N, f32)
    want = p.acc
    if name == "ATOMIC_F32":
        out.copy_(p.init)
        want = p.init + p.acc
    ops.gemm_grouped(a, b, a_mn=True, b_mn=b_mn, epi=epi, out=out, M=M, N=N, K=K, ak_map=(rows, v + n, go))
    exact(out, want.float(), f"ak_map {half}")


# ------------------------------------------------------------------ F. grid-size invariance
@pytest.mark.parametrize("a_mn,b_mn", LAYOUTS)
@pytest.mark.parametrize("M,N,K", [(2304, 2304, 256), (384, 640, 520)])
def test_result_does_not_depend_on_grid_size(ops, L, M, N, K, a_mn, b_mn):
    """Each output tile is reduced by one CTA in a fixed order, so neither the number of SMs the persistent grid leaves
    free (ofk_gemm_reserve_sms, used while all-reduces are in flight) nor the tile-width hint may change a bit.  The
    training step's run-to-run reproducibility rests on this.  One shape has more tiles (324) than SMs, one fewer."""
    g = torch.Generator(device="cuda").manual_seed(29)
    a = torch.randn((K, M) if a_mn else (M, K), generator=g, device="cuda").to(bf16)
    b = torch.randn((K, N) if b_mn else (N, K), generator=g, device="cuda").to(bf16)
    resid = torch.randn(M, N, generator=g, device="cuda")
    gate = torch.tensor([GATE], device="cuda")

    def run(block_n):
        o = ops.gemm(a, b, a_mn=a_mn, b_mn=b_mn, epi=L.EPI_STORE_F32, block_n=block_n)
        br = fresh(M, N, bf16)
        r = ops.gemm(a, b, a_mn=a_mn, b_mn=b_mn, epi=L.EPI_GATE_RESID_F32, aux=resid, gate=gate, out2=br,
                     block_n=block_n)
        return o.view(torch.int32), r.view(torch.int32), br.view(torch.int16)

    lib = L.lib()
    prev = lib.ofk_gemm_reserve_sms(0)
    try:
        base = run(0)
        for reserve in (0, 16, 64):
            lib.ofk_gemm_reserve_sms(reserve)
            for block_n in (0, 128, 256, 512):
                for rep in range(2):
                    for what, got, want in zip(("STORE_F32", "GATE_RESID", "out2"), run(block_n), base):
                        assert torch.equal(got, want), f"{what}: reserve={reserve} block_n={block_n} launch {rep}"
    finally:
        lib.ofk_gemm_reserve_sms(prev)
