"""GPU: the 128 x 256 clustered GEMM tile (csrc/gemm.cu, "wide"), exactly, at its edges and across the tile choice.

The library runs the wide tile when its work items (pairs of m-tiles x 256-wide n-tiles x splits) fill every cluster
slot once, and the 128 x 128 tile otherwise.  Reserving SMs removes cluster slots, so one shape runs on both sides of
that rule: the shapes below have 45-47 wide work items, fewer than the 66 cluster slots of a 132-SM H100 with no SM
reserved and more than the 34 left with 64 reserved.  Both sides reduce over k in the same order, so every output
must match bit for bit, and the exact ones must match the float64 product (the contract suite's integer scheme).

Every shape has an odd number of m-tiles, so the last cluster's second CTA lies wholly past M, and more than
GROUP_M = 8 pairs, so the last pair-raster group is partial."""
import pytest
import torch

from test_gemm_contract_gpu import EPIS, LAYOUTS, Problem, fresh, operand, run_epilogue

pytestmark = pytest.mark.gpu

bf16, f32 = torch.bfloat16, torch.float32
K = 760                   # eleven whole k-blocks and a partial one: split-K 3 gives four k-blocks per slice, the
                          # fewest a wide tile runs with
# N: one 256-wide tile less / exactly / more than a tile, two tiles less / more.  M: 89, 45, 29 m-tiles.
SHAPES = [(11300, 240), (11300, 256), (5700, 272), (5700, 496), (3700, 528)]
RESERVES = (64, 63, 17, 1, 0)   # odd counts leave an odd number of SMs before rounding to whole clusters


@pytest.fixture(scope="module")
def ops():
    from open_flamingo_b200 import ops as _ops
    return _ops


@pytest.fixture(scope="module")
def L():
    from open_flamingo_b200 import _lib
    return _lib


class Recorder:
    """Allocates the outputs of one run_epilogue call and keeps them, to compare runs bit for bit."""

    def __init__(self):
        self.outs = []

    def __call__(self, rows, cols, dtype):
        t = fresh(rows, cols, dtype)
        self.outs.append(t)
        return t

    def bits(self):
        return [t.view(torch.int32 if t.dtype == f32 else torch.int16).clone() for t in self.outs]


def at_reserve(L, reserve, fn):
    lib = L.lib()
    prev = lib.ofk_gemm_reserve_sms(reserve)
    try:
        return fn()
    finally:
        lib.ofk_gemm_reserve_sms(prev)


@pytest.mark.parametrize("name", EPIS)
@pytest.mark.parametrize("a_mn,b_mn", LAYOUTS)
@pytest.mark.parametrize("M,N", SHAPES)
def test_wide_and_narrow_tiles_agree_exactly(ops, L, M, N, a_mn, b_mn, name):
    """Each reserve runs the epilogue against the float64 reference (split-K 1 and 3 for the atomic one), and all
    reserves produce the same bits."""
    p = Problem(M, N, K, seed=M + 3 * N)
    a, b = operand(p.A, a_mn), operand(p.B, b_mn)
    base = None
    for reserve in RESERVES:
        rec = Recorder()
        at_reserve(L, reserve, lambda: run_epilogue(ops, L, name, p, a, b, a_mn, b_mn, alloc=rec))
        bits = rec.bits()
        if base is None:
            base = bits
            continue
        for i, (got, want) in enumerate(zip(bits, base)):
            assert torch.equal(got, want), f"{name} output {i}: reserve {reserve} differs from reserve {RESERVES[0]}"


@pytest.mark.parametrize("name", ["STORE_BF16", "STORE_F32"])
def test_grouped_out_map_on_wide_tiles(ops, L, name):
    """The grouped out map (rows of a [U * (v + n), N] interleaved buffer) on both tile shapes."""
    U, v, n, N = 4, 2825, 7, 240    # U * v = 11300 rows: 89 m-tiles
    p = Problem(U * v, N, K, seed=31)
    dtype = f32 if name == "STORE_F32" else bf16
    want = p.acc.float() if name == "STORE_F32" else p.acc.float().to(bf16)
    epi = getattr(L, "EPI_" + name)
    for reserve in RESERVES:
        buf = torch.full((U * (v + n), N), float("nan"), device="cuda", dtype=dtype)
        at_reserve(L, reserve, lambda: ops.gemm_grouped(operand(p.A, False), operand(p.B, False), epi=epi, out=buf,
                                                        M=U * v, N=N, K=K, out_map=(v, v + n, 0)))
        b3 = buf.view(U, v + n, N)
        assert torch.equal(b3[:, :v].reshape(U * v, N), want), f"reserve {reserve}: media rows"
        assert b3[:, v:].isnan().all(), f"reserve {reserve}: wrote into the other group's rows"


@pytest.mark.parametrize("name", ["ATOMIC_F32", "STORE_F32"])
def test_grouped_ak_map_on_wide_tiles(ops, L, name):
    """Weight gradient over one half of a concatenated MN-major A (the ak map) on both tile shapes."""
    U, v, n, M, N = 3, 128, 64, 11300, 240
    K_ = U * v
    p = Problem(M, N, K_, seed=37)
    buf = torch.full((U * (v + n), M + 12), float("nan"), device="cuda", dtype=bf16)   # row stride 16-byte aligned
    buf[:, :M].view(U, v + n, M)[:, :v] = p.A.t().reshape(U, v, M).to(bf16)
    a = buf[:, :M]
    epi = getattr(L, "EPI_" + name)
    for splits in ((1, 3) if name == "ATOMIC_F32" else (1,)):
        for reserve in RESERVES:
            out = fresh(M, N, f32)
            want = p.acc
            if name == "ATOMIC_F32":
                out.copy_(p.init)
                want = p.init + p.acc
            at_reserve(L, reserve, lambda: ops.gemm_grouped(a, operand(p.B, True), a_mn=True, b_mn=True, epi=epi,
                                                            out=out, M=M, N=N, K=K_, splits=splits,
                                                            ak_map=(v, v + n, 0)))
            assert torch.equal(out, want.float()), f"reserve {reserve} splits {splits}"
