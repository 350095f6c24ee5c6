"""GPU: the training attention kernels against a float64 restatement of their semantics, with per-element bounds.

Entry points: ofk_attn_fwd / ofk_attn_bwd (media rules: Perceiver, gated cross-attention, ViT) and ofk_attn_dense_fwd /
ofk_attn_dense_bwd (MPT blocks, including the chunked-prefill call with nq < nk over the KV cache).

Semantics restated (computed in float64 on the GPU from the same bf16 inputs):
  media  (helpers.py:190-232): key allowed when text_time == key // kpm + 1 (mode 1) or >= (mode 2); a row with no
         allowed key attends uniformly over all keys and passes no gradient to q or k; mode 1 with text_time == 0 is
         exactly zero.
  dense  (HF MptAttention): S = scale * Q K^T + slope[h] * key; key allowed when key <= row + nk - nq (causal) and its
         mask byte is 0; masked scores take finfo.min, so a fully masked row attends uniformly (no gradient to q, k).
  backward: dS = P o (dP - delta) * scale on allowed scores, dq = dS K, dk = dS^T Q, dv = P^T dO.

Bounds (u = 2^-24, the fp32 unit roundoff; every term is built in float64 from the reference, per element or per row):
  score error  dS_r = scale * hd*u * max_k (|q_r| . |k_k|)  [fp32 dot over hd]  + 4u (|slope| nk + max_k |S_rk|)
               [ALiBi bias and the fma/subtract of the log2-domain score].
  eps_rec_r = 2 dS_r + 2^-20: relative error of a recomputed P (its score and the row's max/LSE each move by dS_r;
               ex2.approx adds ~2^-22).
  o:   |o - ref| <= 2^-8 |ref| + (eps_P + eps_rec_r + nk u) (P |V|)
       2^-8 |ref| is the bf16 store (2^-9) with slack; eps_P is the rounding of P fed to the P.V product: 2^-8 for the
       media kernels (one bf16 rounding of P), 2^-16 for the dense kernels (P as bf16 hi + lo, lo = P - hi exact in fp32,
       so only lo's own rounding, 2^-9 |lo| <= 2^-18 P, is left); nk u covers the fp32 accumulation over nk keys.
  lse: |lse - ref| <= log2(e) dS_r + 2 log2(e) (n + 4) u + 4u |ref| + 1e-6  (log2 domain; l summed in fp32 over n keys).
  dq:  |dq - ref| <= 2^-8 |ref| + M |K| + nk u (|dS| |K|),   dk: 2^-8 |ref| + M^T |Q| + nq u (|dS|^T |Q|),  with
       M = scale P o (eps1 (|dP| + |delta|) + hd u (|dO| |V|^T) + d_delta_r),  eps1 = 2^-8 + eps_rec_r
       (dS rounded to bf16 once, P recomputed), d_delta_r = |sum dO (o - O_ref)| + hd u sum |dO| |o|: the kernel forms
       delta from its own bf16 o, whose deviation from the exact O is measured, not assumed.
  dv:  |dv - ref| <= 2^-8 |ref| + ((2^-8 + eps_rec_r) P)^T |dO| + nq u (P^T |dO|)   (P rounded to bf16 once).

Random N(0, 1) operands average predicate mistakes away, so most cases use planted inputs: every (row, head) puts one
key's score about 20 nats above the rest (q = a multiple of that key's row), picked among the keys where the row's
allowed set changes (the causal diagonal and the key after it, media block edges, mask holes) and keys 63/64, 127/128,
nk - 1.  A one-key mistake then moves the output by O(|v|).  Keys come in pairs 2i, 2i + 1 with nearly equal rows and
opposite values, so a row that sees both outputs a small difference whose bf16 rounding of P is visible.

Exact properties checked bit for bit: zero rows (o, lse, dq), dq of uniform rows, dk / dv of keys nothing reaches,
output with and without LSE, repeated launches, one (batch, head) alone, the pure-causal flag, and the bytes around every
output window (all inputs are views with NaN around them; outputs are windows inside NaN-filled buffers)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64
U = 2.0 ** -24
LOG2E = 1.0 / math.log(2.0)
MASKED_LOG2 = -30000.0           # the dense kernels' log2-domain stand-in for finfo.min


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
    """A [B, rows, cols] window at (r0, c0) of a NaN-filled [B, rows + pad, c0 + cols + extra] bf16 buffer."""

    def __init__(self, B, rows, cols, r0=0, c0=0, pad=0, extra=0, dtype=bf16):
        self.buf = torch.full((B, rows + r0 + pad, c0 + cols + extra), float("nan"), device="cuda", dtype=dtype)
        self.view = self.buf[:, r0:r0 + rows, c0:c0 + cols]
        self.inside = torch.zeros(self.buf.shape, dtype=torch.bool, device="cuda")
        self.inside[:, r0:r0 + rows, c0:c0 + cols] = True
        self.before = self.buf.clone()

    def fill(self, t):
        self.view.copy_(t)
        return self.view

    def check(self, what):
        bits = torch.int16 if self.buf.element_size() == 2 else torch.int32
        same = self.buf.view(bits) == self.before.view(bits)
        assert bool(same[~self.inside].all()), f"{what}: bytes outside the output window changed"
        assert not bool(torch.isnan(self.view.float()).any()), f"{what}: NaN left inside the output window"


def heads_split(t, heads, hd):
    B, n, _ = t.shape
    return t.to(f64).reshape(B, n, heads, hd).permute(0, 2, 1, 3)


# ------------------------------------------------------------------ inputs
def planted(B, heads, hd, nq, nk, scale, allowed, seed):
    """q, k, v, d_o (float32, bf16-representable) with one dominant key per (row, head); see the module docstring."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    K = torch.randn(B, nk, heads, hd, device="cuda", generator=g)
    V = torch.randn(B, nk, heads, hd, device="cuda", generator=g)
    npair = nk // 2
    K[:, 1:2 * npair:2] = K[:, 0:2 * npair:2] + 0.1 * torch.randn(B, npair, heads, hd, device="cuda", generator=g)
    V[:, 1:2 * npair:2] = -V[:, 0:2 * npair:2]
    K, V = K.to(bf16).float(), V.to(bf16).float()
    # candidate keys of each row: both sides of every change of the row's allowed set, plus fixed tile edges
    cand = torch.zeros(B, nq, nk, dtype=torch.bool, device="cuda")
    if nk > 1:
        flip = allowed[..., 1:] != allowed[..., :-1]
        cand[..., :-1] |= flip
        cand[..., 1:] |= flip
    for kk in (63, 64, 127, 128, nk - 1):
        if kk < nk:
            cand[..., kk] = True
    pick = torch.rand(B, heads, nq, nk, device="cuda", generator=g).masked_fill(~cand[:, None], -1.0)
    tgt = pick.argmax(-1)                                                          # [B, heads, nq]
    Kh = K.permute(0, 2, 1, 3)                                                     # [B, heads, nk, hd]
    Kt = torch.gather(Kh, 2, tgt[..., None].expand(B, heads, nq, hd))
    Q = Kt * (20.0 / (scale * (Kt * Kt).sum(-1, keepdim=True)))
    q = Q.permute(0, 2, 1, 3).reshape(B, nq, heads * hd)
    dO = torch.randn(B, nq, heads * hd, device="cuda", generator=g)
    return q, K.reshape(B, nk, heads * hd), V.reshape(B, nk, heads * hd), dO


def randn_inputs(B, heads, hd, nq, nk, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return tuple(torch.randn(B, n, heads * hd, device="cuda", generator=g) for n in (nq, nk, nk, nq))


def place_inputs(q, k, v, d_o, cap_extra=3):
    """q as a column slice of a [B, nq + 5, 3D] qkv-like buffer, k / v as the K / V halves of a [B, nk + cap_extra, 2D]
    KV-cache buffer (rows past nk stale = NaN), everything else NaN.  d_o is returned plain (it must share o's strides)."""
    B, nq, D = q.shape
    nk = k.shape[1]
    qw = Window(B, nq, D, r0=0, c0=D, pad=5, extra=D).fill(q.to(bf16))
    kv = torch.full((B, nk + cap_extra, 2 * D), float("nan"), device="cuda", dtype=bf16)
    kv[:, :nk, :D] = k.to(bf16)
    kv[:, :nk, D:] = v.to(bf16)
    return qw, kv[:, :nk, :D], kv[:, :nk, D:], d_o.to(bf16)


# ------------------------------------------------------------------ float64 reference and bounds
def reference(q, k, v, d_o, heads, hd, scale, allowed, zero=None, slopes=None, uniform_lse=None):
    """allowed: [B, nq, nk] bool; zero: [B, nq] rows that are exactly zero (media mode 1, text_time == 0).
    Rows with no allowed key that are not zero rows attend uniformly over all keys.  Returns float64 tensors in the
    [B, heads, n, hd] / [B, heads, nq] layout plus what the bounds need."""
    Q, K, V, dO = (heads_split(t, heads, hd) for t in (q, k, v, d_o))
    B, H, nq, _ = Q.shape
    nk = K.shape[2]
    S = scale * Q @ K.transpose(-1, -2)
    key = torch.arange(nk, device="cuda", dtype=f64)
    if slopes is not None:
        S = S + slopes.to(f64).view(1, H, 1, 1) * key
    A = allowed[:, None].expand(B, H, nq, nk)
    zero = torch.zeros(B, nq, dtype=torch.bool, device="cuda") if zero is None else zero
    Z = zero[:, None, :].expand(B, H, nq)
    unif = ~A.any(-1) & ~Z
    Sm = S.masked_fill(~A, -math.inf)
    m = Sm.amax(-1, keepdim=True)
    m = torch.where(torch.isfinite(m), m, torch.zeros_like(m))
    E = torch.exp(Sm - m)
    l = E.sum(-1, keepdim=True)
    P = E / torch.where(l > 0, l, torch.ones_like(l))
    P = torch.where(unif[..., None], torch.full_like(P, 1.0 / nk), P)
    P = torch.where(Z[..., None], torch.zeros_like(P), P)
    lse = LOG2E * (m[..., 0] + torch.log(torch.where(l[..., 0] > 0, l[..., 0], torch.ones_like(l[..., 0]))))
    lse = torch.where(unif, torch.full_like(lse, uniform_lse(nk)), lse)
    lse = torch.where(Z, torch.zeros_like(lse), lse)
    O = P @ V
    live = A & ~(unif | Z)[..., None]
    absQ, absK, absV, absdO = Q.abs(), K.abs(), V.abs(), dO.abs()
    dS_r = scale * hd * U * (absQ @ absK.transpose(-1, -2)).amax(-1)
    dS_r = dS_r + 4 * U * S.abs().amax(-1)
    if slopes is not None:
        dS_r = dS_r + 4 * U * slopes.abs().to(f64).view(1, H, 1) * nk
    eps_rec = 2 * dS_r + 2.0 ** -20
    n_live = torch.where(unif, torch.full_like(dS_r, nk), live.sum(-1).to(f64))
    return dict(Q=Q, K=K, V=V, dO=dO, S=S, P=P, O=O, lse=lse, live=live, unif=unif, zero=Z, dS_r=dS_r,
                eps_rec=eps_rec, n_live=n_live, absQ=absQ, absK=absK, absV=absV, absdO=absdO, scale=scale)


def check_fwd(R, o, lse, eps_P, what):
    """o: kernel output [B, nq, H*hd] bf16; lse: [B, H, nq] f32 (or None)."""
    P, nk = R["P"], R["K"].shape[2]
    PV = P @ R["absV"]
    eps = (eps_P + R["eps_rec"] + nk * U)[..., None]
    bound = 2.0 ** -8 * R["O"].abs() + eps * PV + 1e-30
    err = (heads_split(o, R["Q"].shape[1], R["Q"].shape[3]) - R["O"]).abs()
    worst = (err / bound).max().item()
    assert worst <= 1.0, f"{what}: o off by {worst:.2f}x its bound (max |err| {err.max().item():.3e})"
    zero = R["zero"]
    if zero.any():
        oz = heads_split(o, R["Q"].shape[1], R["Q"].shape[3])[zero]
        assert bool((oz == 0).all()), f"{what}: zero rows are not exactly zero"
    if lse is None:
        return
    lref = R["lse"]
    lb = LOG2E * R["dS_r"] + 2 * LOG2E * (R["n_live"] + 4) * U + 4 * U * lref.abs() + 1e-6
    lerr = (lse.to(f64) - lref).abs()
    worst = (lerr / lb).max().item()
    assert worst <= 1.0, f"{what}: lse off by {worst:.2f}x its bound (max |err| {lerr.max().item():.3e})"
    if zero.any():
        assert bool((lse[zero] == 0).all()), f"{what}: zero rows' LSE is not the sentinel 0"


def check_bwd(R, o, dq, dk, dv, what):
    H, hd = R["Q"].shape[1], R["Q"].shape[3]
    P, live, scale = R["P"], R["live"], R["scale"]
    nq, nk = P.shape[2], P.shape[3]
    Q, K, V, dO, O = R["Q"], R["K"], R["V"], R["dO"], R["O"]
    ok = heads_split(o, H, hd)
    dP = dO @ V.transpose(-1, -2)
    delta = (dO * O).sum(-1, keepdim=True)
    dS = torch.where(live, P * (dP - delta) * scale, torch.zeros_like(P))
    ref = dict(dq=dS @ K, dk=dS.transpose(-1, -2) @ Q, dv=P.transpose(-1, -2) @ dO)
    d_delta = (dO * (ok - O)).sum(-1, keepdim=True).abs() + hd * U * (R["absdO"] * ok.abs()).sum(-1, keepdim=True)
    eps1 = 2.0 ** -8 + R["eps_rec"][..., None]
    M = scale * P * (eps1 * (dP.abs() + delta.abs()) + hd * U * (R["absdO"] @ R["absV"].transpose(-1, -2)) + d_delta)
    M = torch.where(live, M, torch.zeros_like(M))
    aS = dS.abs()
    bounds = dict(
        dq=M @ R["absK"] + nk * U * (aS @ R["absK"]),
        dk=M.transpose(-1, -2) @ R["absQ"] + nq * U * (aS.transpose(-1, -2) @ R["absQ"]),
        dv=((2.0 ** -8 + R["eps_rec"][..., None]) * P).transpose(-1, -2) @ R["absdO"]
        + nq * U * (P.transpose(-1, -2) @ R["absdO"]))
    for name, got in (("dq", dq), ("dk", dk), ("dv", dv)):
        g = heads_split(got, H, hd)
        b = 2.0 ** -8 * ref[name].abs() + bounds[name] + 1e-30
        err = (g - ref[name]).abs()
        worst = (err / b).max().item()
        assert worst <= 1.0, f"{what}: {name} off by {worst:.2f}x its bound (max |err| {err.max().item():.3e})"
    gq = heads_split(dq, H, hd)
    nograd = R["unif"] | R["zero"]
    if nograd.any():
        assert bool((gq[nograd] == 0).all()), f"{what}: uniform / zero rows pass gradient to q"
    # keys that no row may attend to and that no uniform row reaches get exactly zero dk and dv
    dead = ~live.any(2) & ~R["unif"].any(2, keepdim=True).expand(-1, -1, nk)
    if dead.any():
        assert bool((heads_split(dk, H, hd)[dead] == 0).all()), f"{what}: unreachable keys have nonzero dk"
        assert bool((heads_split(dv, H, hd)[dead] == 0).all()), f"{what}: unreachable keys have nonzero dv"


# ------------------------------------------------------------------ media rules
def media_allowed(tt, nk, kpm, mode):
    B, nq = tt.shape
    if mode == 0:
        return torch.ones(B, nq, nk, dtype=torch.bool, device="cuda"), None
    media = torch.arange(nk, device="cuda") // kpm + 1
    t = tt[:, :, None]
    allowed = (t == media) if mode == 1 else (t >= media)
    zero = (tt == 0) if mode == 1 else None
    return allowed, zero


def text_time(B, nq, n_media, seed):
    """Monotone text_time rows (cumulative <image> counts) with every pattern the kernels branch on:
    b = 0: text before the first image, a change across rows 63/64 and inside a 64-row block, and more <image> tokens
           than media at the end (mode 1: uniform rows mixed with normal rows in one block);
    b = 1: the first two 64-row blocks all zero (mode 1: a block of zero rows, the nblk == 0 path), then steps;
    b = 2: random steps."""
    g = torch.Generator().manual_seed(seed)
    tt = torch.zeros(B, nq, dtype=torch.int32)
    if nq == 1:
        tt[:, 0] = torch.randint(0, n_media + 2, (B,), generator=g)
        return tt.cuda()
    for b in range(B):
        if b == 0:
            pos = [5, 30, 64, 70] + list(range(90, nq, 37))
            pos = pos[:n_media + 1]
            if nq > 60:
                pos.append(nq - 3)            # one more <image> than media near the end
        elif b == 1:
            pos = list(range(min(128, nq // 2), nq, 11))[:n_media]
        else:
            pos = sorted(torch.randperm(nq, generator=g)[:n_media].tolist())
        loc = torch.zeros(nq, dtype=torch.int32)
        for p in pos:
            if p < nq:
                loc[p] += 1
        tt[b] = loc.cumsum(0)
    return tt.cuda()


MEDIA_CASES = [
    # B, heads, nq, nk, mode, kpm, planted
    (1, 1, 1, 1, 0, 64, True),
    (3, 8, 63, 65, 0, 64, True),
    (1, 16, 64, 127, 0, 64, True),
    (3, 1, 65, 257, 0, 64, True),
    (1, 8, 129, 4160, 0, 64, True),
    (3, 16, 257, 257, 0, 64, False),          # ViT-L/14, random operands
    (3, 8, 129, 48, 1, 16, True),             # n_media 3
    (3, 1, 257, 240, 1, 48, True),            # n_media 5
    (1, 8, 65, 64, 1, 64, True),              # n_media 1
    (3, 8, 129, 240, 1, 80, True),            # n_media 3, media blocks straddle 64-key tiles
    (3, 16, 63, 640, 1, 128, True),           # n_media 5
    (3, 8, 1, 240, 1, 48, True),              # decode-like single row
    (3, 8, 257, 80, 2, 16, True),             # n_media 5
    (3, 1, 64, 48, 2, 48, True),              # n_media 1
    (3, 8, 129, 192, 2, 64, True),            # n_media 3
    (3, 16, 129, 400, 2, 80, True),           # n_media 5
    (3, 8, 65, 384, 2, 128, True),            # n_media 3
    (3, 8, 129, 240, 1, 80, False),           # random operands on the straddling path
    (2, 8, 96, 192, 2, 64, False),
]
BIG = [                                       # the real workload shapes, random operands
    (32, 8, 256, 128, 1, 64, False),          # gated cross-attention core, 2 images
    (8, 8, 512, 320, 1, 64, False),           # gated cross-attention core, 5 images
    (2, 8, 64, 4160, 0, 64, False),           # Perceiver core: 4096 visual tokens + 64 latents
    (2, 8, 192, 1088, 0, 64, False),          # several key tiles and several query tiles
    (4, 16, 257, 257, 0, 64, False),          # ViT-L/14
]


def _media_case(case, seed=0):
    B, heads, nq, nk, mode, kpm, plant = case
    scale = 64 ** -0.5
    tt = text_time(B, nq, nk // kpm, 7 + seed) if mode else None
    allowed, zero = media_allowed(tt, nk, kpm, mode) if mode else media_allowed(torch.zeros(B, nq), nk, kpm, 0)
    if plant:
        q, k, v, d_o = planted(B, heads, 64, nq, nk, scale, allowed, 100 + seed)
    else:
        q, k, v, d_o = randn_inputs(B, heads, 64, nq, nk, 100 + seed)
    return scale, tt, allowed, zero, q, k, v, d_o


@pytest.mark.parametrize("case", MEDIA_CASES + BIG, ids=lambda c: "-".join(map(str, c)))
def test_media_attention_against_float64(ops, case):
    B, heads, nq, nk, mode, kpm, _ = case
    D = heads * 64
    scale, tt, allowed, zero, q, k, v, d_o = _media_case(case)
    qw, kv_k, kv_v, d_o16 = place_inputs(q, k, v, d_o)
    ow = Window(B, nq, D, r0=1, c0=64, pad=2, extra=8)
    o, lse = ops.attn_fwd(qw, kv_k, kv_v, heads, scale, mask_mode=mode, text_time=tt, keys_per_media=kpm, out=ow.view)
    o2, none = ops.attn_fwd(qw, kv_k, kv_v, heads, scale, mask_mode=mode, text_time=tt, keys_per_media=kpm,
                            want_lse=False)
    # d_o shares o's strides: a window of the same shape of buffer
    dow = Window(B, nq, D, r0=1, c0=64, pad=2, extra=8)
    dow.fill(d_o16)
    dqw = Window(B, nq, D, r0=0, c0=2, pad=3, extra=6)       # dq/dk/dv only need 4-byte alignment
    dkw = Window(B, nk, D, r0=2, c0=0, pad=0, extra=2)
    dvw = Window(B, nk, D, r0=0, c0=8, pad=1, extra=0)
    ops.attn_bwd(qw, kv_k, kv_v, o, dow.view, lse, heads, scale, mask_mode=mode, text_time=tt, keys_per_media=kpm,
                 dq=dqw.view, dk=dkw.view, dv=dvw.view)
    torch.cuda.synchronize()
    assert none is None and torch.equal(o, o2), "output without the LSE differs from the output with it"
    for w, name in ((ow, "o"), (dqw, "dq"), (dkw, "dk"), (dvw, "dv")):
        w.check(name)
    R = reference(qw, kv_k, kv_v, d_o16, heads, 64, scale, allowed, zero, uniform_lse=lambda n: math.log2(n))
    what = f"media {case}"
    check_fwd(R, o, lse, 2.0 ** -8, what)
    check_bwd(R, o, dqw.view, dkw.view, dvw.view, what)


# ------------------------------------------------------------------ dense rules
def mpt_slopes(heads):
    return (2.0 ** (-8.0 * torch.arange(1, heads + 1, device="cuda", dtype=f32) / heads)).contiguous()


def dense_mask(B, nq, nk, kind, seed):
    """[B, nq, nk] bool, True = masked (None for kind 'causal'/'flag', which use the causal rule)."""
    off = nk - nq
    causal = torch.arange(nk, device="cuda")[None, :] > torch.arange(nq, device="cuda")[:, None] + off
    if kind in ("causal", "flag"):
        return None
    g = torch.Generator(device="cuda").manual_seed(seed)
    if kind in ("left_pad", "right_pad"):
        lens = [nk, max(1, nk - 37), max(1, nk // 2), 3][:B]
        keep = torch.zeros(B, nk, dtype=torch.bool, device="cuda")
        for b, n in enumerate(lens):
            if kind == "left_pad":
                keep[b, nk - n:] = True
            else:
                keep[b, :n] = True
        return causal[None] | ~keep[:, None, :]
    assert kind == "random"
    m = torch.rand(B, nq, nk, device="cuda", generator=g) < 0.3
    m[:, 0::5] = True                                    # fully masked rows
    rows = torch.arange(1, nq, 5, device="cuda")         # rows with a single hole
    m[:, rows] = True
    holes = torch.randint(0, nk, (B, rows.numel()), device="cuda", generator=g)
    m[torch.arange(B, device="cuda")[:, None], rows[None, :], holes] = False
    if nq >= 128:
        m[:, 64:128] = True                              # a fully masked 64-row block
    return m


def dense_fwd_ctypes(lib, q, k, v, heads, hd, scale, causal, mask, slopes, flag, out, lse):
    """ofk_attn_dense_fwd into caller-owned windows (ops.attn_dense_fwd allocates its output)."""
    B, nq, nk = q.shape[0], q.shape[1], k.shape[1]
    L = lib
    L.check(L.lib().ofk_attn_dense_fwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), L.ptr(lse), B, heads,
                                       hd, nq, nk, q.stride(0), q.stride(1), k.stride(0), k.stride(1), v.stride(0),
                                       v.stride(1), out.stride(0), out.stride(1), scale, int(causal), L.ptr(mask),
                                       L.ptr(slopes), L.ptr(flag), L.stream_ptr()))


DENSE_CASES = [
    # B, heads, hd, nq, nk, kind, alibi, planted, backward
    (1, 2, 64, 1, 1, "causal", False, True, True),
    (3, 2, 128, 63, 63, "causal", False, True, True),
    (2, 4, 64, 64, 64, "causal", True, False, True),
    (2, 2, 128, 65, 65, "causal", False, True, True),
    (3, 4, 64, 129, 129, "left_pad", False, True, True),
    (2, 2, 128, 257, 257, "right_pad", False, True, True),
    (2, 4, 128, 257, 257, "causal", True, False, True),
    (2, 2, 64, 512, 512, "causal", False, True, True),
    (3, 2, 128, 512, 512, "random", False, True, True),
    (2, 2, 64, 129, 129, "random", True, False, True),
    (1, 32, 128, 512, 512, "causal", True, False, True),      # MPT-7B block
    (2, 4, 128, 256, 2048, "causal", True, False, False),    # MPT-7B context, the largest ALiBi bias
]
for _nq, _nk, _hd in ((2, 65, 128), (63, 200, 64), (64, 128, 128), (65, 1000, 64)):   # chunked prefill: nq < nk
    for _kind in ("causal", "random", "flag"):
        DENSE_CASES.append((2, 2, _hd, _nq, _nk, _kind, False, True, True))
DENSE_CASES.append((3, 4, 128, 63, 200, "left_pad", True, False, True))


@pytest.mark.parametrize("case", DENSE_CASES, ids=lambda c: "-".join(map(str, c)))
def test_dense_attention_against_float64(ops, lib, case):
    B, heads, hd, nq, nk, kind, alibi, plant, bwd = case
    D = heads * hd
    scale = hd ** -0.5
    slopes = mpt_slopes(heads) if alibi else None
    mask = dense_mask(B, nq, nk, kind, 5)
    causal_rule = torch.arange(nk, device="cuda")[None, :] > torch.arange(nq, device="cuda")[:, None] + (nk - nq)
    masked = causal_rule[None].expand(B, nq, nk) if mask is None else mask
    if plant:
        q, k, v, d_o = planted(B, heads, hd, nq, nk, scale, ~masked, 200)
    else:
        q, k, v, d_o = randn_inputs(B, heads, hd, nq, nk, 200)
    qw, kv_k, kv_v, d_o16 = place_inputs(q, k, v, d_o)
    mask8 = None if mask is None else mask.to(torch.uint8).contiguous()
    flag = None
    if kind == "flag":
        # garbage bytes under the pure-causal flag: the kernel must ignore them
        mask8 = torch.randint(0, 256, (B, nq, nk), device="cuda", dtype=torch.uint8)
        flag = torch.ones(1, dtype=torch.int32, device="cuda")
    causal = mask is None and kind != "flag"
    ow = Window(B, nq, D, r0=2, c0=8, pad=1, extra=64)
    lsew = Window(1, 1, B * heads * nq, c0=4, extra=4, dtype=f32)
    dense_fwd_ctypes(lib, qw, kv_k, kv_v, heads, hd, scale, causal, mask8, slopes, flag, ow.view, lsew.view)
    o2, _ = ops.attn_dense_fwd(qw, kv_k, kv_v, heads, hd, scale, causal=causal, mask=mask8, slopes=slopes,
                               pure_causal_flag=flag, want_lse=False)
    o, lse = ow.view, lsew.view.reshape(B, heads, nq)
    if bwd:
        dow = Window(B, nq, D, r0=2, c0=8, pad=1, extra=64)
        dow.fill(d_o16)
        dqw = Window(B, nq, D, r0=1, c0=2, pad=0, extra=2)
        dkw = Window(B, nk, D, r0=0, c0=D + 2, pad=2, extra=0)
        dvw = Window(B, nk, D, r0=3, c0=0, pad=0, extra=8)
        ops.attn_dense_bwd(qw, kv_k, kv_v, o, dow.view, lse, heads, hd, scale, causal=causal, mask=mask8,
                           slopes=slopes, pure_causal_flag=flag, dq=dqw.view, dk=dkw.view, dv=dvw.view)
    torch.cuda.synchronize()
    assert torch.equal(o, o2), "output without the LSE differs from the output with it"
    ow.check("o")
    lsew.check("lse")
    R = reference(qw, kv_k, kv_v, d_o16, heads, hd, scale, ~masked, slopes=slopes,
                  uniform_lse=lambda n: MASKED_LOG2 + math.log2(n))
    what = f"dense {case}"
    check_fwd(R, o, lse, 2.0 ** -16, what)
    if bwd:
        for w, name in ((dqw, "dq"), (dkw, "dk"), (dvw, "dv")):
            w.check(name)
        check_bwd(R, o, dqw.view, dkw.view, dvw.view, what)


# ------------------------------------------------------------------ bitwise properties
def _media_all(ops, q, k, v, d_o, heads, scale, mode, tt, kpm):
    o, lse = ops.attn_fwd(q, k, v, heads, scale, mask_mode=mode, text_time=tt, keys_per_media=kpm)
    dq, dk, dv = ops.attn_bwd(q, k, v, o, d_o, lse, heads, scale, mask_mode=mode, text_time=tt, keys_per_media=kpm)
    return o, lse, dq, dk, dv


def _dense_all(ops, q, k, v, d_o, heads, hd, scale, causal, mask, slopes, flag):
    o, lse = ops.attn_dense_fwd(q, k, v, heads, hd, scale, causal=causal, mask=mask, slopes=slopes,
                                pure_causal_flag=flag)
    dq, dk, dv = ops.attn_dense_bwd(q, k, v, o, d_o, lse, heads, hd, scale, causal=causal, mask=mask, slopes=slopes,
                                    pure_causal_flag=flag)
    return o, lse, dq, dk, dv


def _assert_same(a, b, what):
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), f"{what}: output {i} differs bitwise"


@pytest.mark.parametrize("case", [(3, 8, 129, 240, 1, 80, True), (3, 4, 65, 257, 0, 64, False),
                                  (3, 4, 129, 192, 2, 64, True)], ids=lambda c: "-".join(map(str, c)))
def test_media_repeatable_and_independent_of_other_batches_and_heads(ops, case):
    B, heads, nq, nk, mode, kpm, _ = case
    scale, tt, _, _, q, k, v, d_o = _media_case(case, seed=1)
    q, k, v, d_o = (t.to(bf16) for t in (q, k, v, d_o))
    full = _media_all(ops, q, k, v, d_o, heads, scale, mode, tt, kpm)
    again = _media_all(ops, q, k, v, d_o, heads, scale, mode, tt, kpm)
    _assert_same(full, again, "repeated launch")
    for b, h in ((1, 0), (B - 1, heads - 1)):
        c = slice(h * 64, (h + 1) * 64)
        sub = [t[b:b + 1, :, c] for t in (q, k, v, d_o)]
        d_o1 = sub[3].contiguous()
        tt1 = None if tt is None else tt[b:b + 1]
        one = _media_all(ops, sub[0], sub[1], sub[2], d_o1, 1, scale, mode, tt1, kpm)
        want = (full[0][b:b + 1, :, c], full[1][b:b + 1, h:h + 1], full[2][b:b + 1, :, c], full[3][b:b + 1, :, c],
                full[4][b:b + 1, :, c])
        _assert_same(one, want, f"batch {b} head {h} alone")


@pytest.mark.parametrize("shape", [(2, 4, 128, 129, 129), (2, 2, 64, 63, 200), (3, 2, 128, 65, 1000)],
                         ids=lambda c: "-".join(map(str, c)))
def test_dense_flag_repeatable_and_independent(ops, shape):
    """pure_causal_flag = 1 over garbage mask bytes gives the bits of causal=True without a mask (nq <= nk); with the flag
    at 0 the same bytes are honoured; launches repeat bit for bit; one (batch, head) computed alone gives the same bits."""
    B, heads, hd, nq, nk = shape
    D = heads * hd
    scale = hd ** -0.5
    slopes = mpt_slopes(heads)
    q, k, v, d_o = (t.to(bf16) for t in randn_inputs(B, heads, hd, nq, nk, 300))
    garbage = torch.randint(0, 256, (B, nq, nk), device="cuda", dtype=torch.uint8)
    on = torch.ones(1, dtype=torch.int32, device="cuda")
    off = torch.zeros(1, dtype=torch.int32, device="cuda")
    causal = _dense_all(ops, q, k, v, d_o, heads, hd, scale, True, None, slopes, None)
    flagged = _dense_all(ops, q, k, v, d_o, heads, hd, scale, False, garbage, slopes, on)
    _assert_same(flagged, causal, "pure-causal flag over garbage bytes vs causal")
    _assert_same(_dense_all(ops, q, k, v, d_o, heads, hd, scale, True, None, slopes, None), causal, "repeated launch")
    honoured = _dense_all(ops, q, k, v, d_o, heads, hd, scale, False, garbage, slopes, off)
    plain = _dense_all(ops, q, k, v, d_o, heads, hd, scale, False, garbage, slopes, None)
    _assert_same(honoured, plain, "flag 0 vs no flag")
    assert not torch.equal(honoured[0], causal[0]), "flag 0 ignored the mask bytes"
    for b, h in ((0, heads - 1), (B - 1, 0)):
        c = slice(h * hd, (h + 1) * hd)
        sub = [t[b:b + 1, :, c] for t in (q, k, v)] + [d_o[b:b + 1, :, c].contiguous()]
        one = _dense_all(ops, *sub, 1, hd, scale, True, None, slopes[h:h + 1].contiguous(), None)
        want = (causal[0][b:b + 1, :, c], causal[1][b:b + 1, h:h + 1], causal[2][b:b + 1, :, c],
                causal[3][b:b + 1, :, c], causal[4][b:b + 1, :, c])
        _assert_same(one, want, f"batch {b} head {h} alone")


def test_lse_and_delta_windows(ops, lib):
    """lse and delta (f32 [B, heads, nq] arrays) written through the C entry points at an offset inside NaN buffers:
    the bytes around them stay untouched and no NaN is left inside."""
    L = lib
    B, heads, nq, nk = 2, 4, 65, 192
    D = heads * 64
    q, k, v, d_o = (t.to(bf16) for t in randn_inputs(B, heads, 64, nq, nk, 400))
    tt = text_time(B, nq, 3, 3)
    o = torch.empty(B, nq, D, device="cuda", dtype=bf16)
    dq = torch.empty_like(q)
    dk, dv = torch.empty_like(k), torch.empty_like(k)
    n = B * heads * nq
    lsew = Window(1, 1, n, c0=4, extra=3, dtype=f32)
    deltaw = Window(1, 1, n, c0=8, extra=5, dtype=f32)
    st = L.stream_ptr()
    s = (q.stride(0), q.stride(1))
    L.check(L.lib().ofk_attn_fwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lsew.view.data_ptr(), B, heads,
                                 nq, nk, *s, k.stride(0), k.stride(1), v.stride(0), v.stride(1), o.stride(0),
                                 o.stride(1), 0.125, 1, tt.data_ptr(), 64, st))
    L.check(L.lib().ofk_attn_bwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), d_o.data_ptr(),
                                 lsew.view.data_ptr(), deltaw.view.data_ptr(), dq.data_ptr(), dk.data_ptr(),
                                 dv.data_ptr(), B, heads, nq, nk, *s, k.stride(0), k.stride(1), v.stride(0), v.stride(1),
                                 o.stride(0), o.stride(1), dq.stride(0), dq.stride(1), dk.stride(0), dk.stride(1),
                                 dv.stride(0), dv.stride(1), 0.125, 1, tt.data_ptr(), 64, st))
    torch.cuda.synchronize()
    lsew.check("media lse")
    deltaw.check("media delta")
    O = heads_split(o, heads, 64)
    want = (heads_split(d_o, heads, 64) * O).sum(-1)
    got = deltaw.view.reshape(B, heads, nq).to(f64)
    assert bool(((got - want).abs() <= 64 * U * (heads_split(d_o, heads, 64).abs() * O.abs()).sum(-1) + 1e-30).all())
    # dense backward: delta for head_dim 128 sums all 128 columns
    hd = 128
    D = heads * hd
    q, k, v, d_o = (t.to(bf16) for t in randn_inputs(B, heads, hd, nq, nq, 401))
    o, lse = ops.attn_dense_fwd(q, k, v, heads, hd, hd ** -0.5, causal=True)
    dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    deltaw = Window(1, 1, n, c0=2, extra=1, dtype=f32)
    s = (q.stride(0), q.stride(1))
    L.check(L.lib().ofk_attn_dense_bwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), d_o.data_ptr(),
                                       lse.data_ptr(), deltaw.view.data_ptr(), dq.data_ptr(), dk.data_ptr(),
                                       dv.data_ptr(), B, heads, hd, nq, nq, *s, *s, *s, o.stride(0), o.stride(1), *s, *s,
                                       *s, hd ** -0.5, 1, None, None, None, st))
    torch.cuda.synchronize()
    deltaw.check("dense delta")
    O = heads_split(o, heads, hd)
    want = (heads_split(d_o, heads, hd) * O).sum(-1)
    got = deltaw.view.reshape(B, heads, nq).to(f64)
    assert bool(((got - want).abs() <= hd * U * (heads_split(d_o, heads, hd).abs() * O.abs()).sum(-1) + 1e-30).all())


# ------------------------------------------------------------------ ops-level argument checks (raise before launching)
def test_ops_rejects_bad_attention_arguments(ops, lib):
    B, heads, nq, nk = 2, 4, 65, 128
    D = heads * 64
    q, k, v, d_o = (t.to(bf16) for t in randn_inputs(B, heads, 64, nq, nk, 500))
    tt = text_time(B, nq, 2, 1)
    o, lse = ops.attn_fwd(q, k, v, heads, 0.125, mask_mode=1, text_time=tt)
    qd, kd, vd, dod = (t.to(bf16) for t in randn_inputs(B, 2, 128, nq, nk, 501))
    od, lsed = ops.attn_dense_fwd(qd, kd, vd, 2, 128, 128 ** -0.5, causal=True)
    torch.cuda.synchronize()
    n0 = lib.launch_count()
    bad = [
        lambda: ops.attn_fwd(q, k, v, heads + 1, 0.125),                                    # heads too large
        lambda: ops.attn_fwd(q, k[:, :-1], v, heads, 0.125),                                # k / v shapes differ
        lambda: ops.attn_fwd(q, k[:1], v[:1], heads, 0.125),                                # batch differs
        lambda: ops.attn_fwd(q.float(), k, v, heads, 0.125),
        lambda: ops.attn_fwd(q, k, v, heads, 0.125, out=torch.empty(B, nq + 1, D, device="cuda", dtype=bf16)),
        lambda: ops.attn_fwd(q, k, v, heads, 0.125, out=torch.empty(B, nq, D, device="cuda", dtype=f32)),
        lambda: ops.attn_fwd(q, k, v, heads, 0.125, mask_mode=1, text_time=tt.long()),
        lambda: ops.attn_bwd(q, k, v, o, d_o, lse, heads, 0.125, mask_mode=1, text_time=None),
        lambda: ops.attn_bwd(q, k, v, o, d_o, lse, heads, 0.125, mask_mode=2, text_time=tt[:, :-1]),
        lambda: ops.attn_bwd(q, k, v, o, d_o, lse.double(), heads, 0.125, mask_mode=1, text_time=tt),
        lambda: ops.attn_bwd(q, k, v, o, d_o, lse[:, :2], heads, 0.125, mask_mode=1, text_time=tt),
        lambda: ops.attn_bwd(q, k, v, o, d_o, lse, heads + 1, 0.125, mask_mode=1, text_time=tt),
        lambda: ops.attn_bwd(q, k, v[:, :-1], o, d_o, lse, heads, 0.125, mask_mode=1, text_time=tt),
        lambda: ops.attn_bwd(q, k, v, o, d_o, lse, heads, 0.125, mask_mode=1, text_time=tt, dq=torch.empty_like(k)),
        lambda: ops.attn_bwd(q, k, v, o, d_o, lse, heads, 0.125, mask_mode=1, text_time=tt, dk=torch.empty_like(q)),
        lambda: ops.attn_dense_fwd(qd, kd, vd, 3, 128, 0.1),                                # heads * head_dim too large
        lambda: ops.attn_dense_fwd(qd.float(), kd, vd, 2, 128, 0.1),
        lambda: ops.attn_dense_fwd(qd, kd, vd[:, :-1], 2, 128, 0.1),
        lambda: ops.attn_dense_fwd(qd, kd, vd, 2, 128, 0.1, slopes=torch.ones(1, device="cuda")),
        lambda: ops.attn_dense_fwd(qd, kd, vd, 2, 128, 0.1, slopes=torch.ones(2, device="cuda", dtype=f64)),
        lambda: ops.attn_dense_fwd(qd, kd, vd, 2, 128, 0.1,
                                   pure_causal_flag=torch.ones(1, device="cuda", dtype=torch.int64)),
        lambda: ops.attn_dense_bwd(qd, kd, vd, od, dod, lsed, 2, 128, 0.1,
                                   mask=torch.zeros(B, nq, nk + 1, device="cuda", dtype=torch.uint8)),
        lambda: ops.attn_dense_bwd(qd, kd, vd, od, dod, lsed, 2, 128, 0.1,
                                   mask=torch.zeros(B, nk, nq, device="cuda", dtype=torch.uint8).transpose(1, 2)),
        lambda: ops.attn_dense_bwd(qd, kd, vd, od, dod, lsed[:, :1], 2, 128, 0.1, causal=True),
        lambda: ops.attn_dense_bwd(qd, kd, vd, od, dod, lsed.to(bf16), 2, 128, 0.1, causal=True),
        lambda: ops.attn_dense_bwd(qd, kd, vd, od[:, :-1], dod[:, :-1], lsed, 2, 128, 0.1, causal=True),
        lambda: ops.attn_dense_bwd(qd, kd, vd, od, dod, lsed, 2, 128, 0.1, causal=True, slopes=torch.ones(1, device="cuda")),
        lambda: ops.attn_dense_bwd(qd, kd, vd, od, dod, lsed, 2, 128, 0.1, causal=True, dv=torch.empty_like(qd)),
    ]
    for i, fn in enumerate(bad):
        with pytest.raises(ValueError):
            fn()
        assert lib.launch_count() == n0, f"case {i} launched a kernel before raising"
