"""CPU: the GEMM entry points reject bad arguments with the documented error code, before they touch a device.

Every call runs in a child process with no CUDA device visible and with made-up device addresses that are never
dereferenced.  A call whose arguments pass validation reaches device discovery and returns OFK_ERR_CUDA (-3), so a
missing or late check shows up as a wrong code and can never launch a kernel."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ARG, ALIGN, NO_DEVICE = -1, -2, -3
STORE_BF16, STORE_F32, ATOMIC_F32, BIAS_BF16, BIAS_QGELU, GELU_DUAL, GATE_RESID, DGELU, BIAS_RESID, BIAS_GELU = range(10)
F32_OUT = (STORE_F32, ATOMIC_F32, GATE_RESID, BIAS_RESID)
BIAS_EPIS = (BIAS_BF16, BIAS_QGELU, BIAS_RESID, BIAS_GELU)
OUT2_EPIS = (GELU_DUAL, GATE_RESID, BIAS_RESID)
AUX_EPIS = (GATE_RESID, BIAS_RESID, DGELU)

# made-up, 16-byte-aligned device addresses (never dereferenced: no device is visible)
A_PTR, B_PTR, OUT_PTR, OUT2_PTR, AUX_PTR, BIAS_PTR, GATE_PTR = (k << 32 for k in range(1, 8))
M, N, K = 128, 128, 64


def gemm_args(epi, **kw):
    """ofk_gemm_bf16 arguments for a valid call of `epi` (row strides in elements), with `kw` overriding."""
    a = dict(epi=epi, a_mn=0, b_mn=0, A=A_PTR, lda=K, B=B_PTR, ldb=K, M=M, N=N, K=K, splits=1, block_n=0,
             out=OUT_PTR, ldo=N, out2=0, ldo2=0, aux=0, ldaux=0, bias=0, gate=0, stream=0)
    if epi in OUT2_EPIS:
        a.update(out2=OUT2_PTR, ldo2=N)
    if epi in AUX_EPIS:
        a.update(aux=AUX_PTR, ldaux=N)
    if epi in BIAS_EPIS:
        a.update(bias=BIAS_PTR)
    if epi == GATE_RESID:
        a.update(gate=GATE_PTR)
    a.update(kw)
    return ["ofk_gemm_bf16", list(a.values())]


def grouped_args(epi, **kw):
    a = dict(epi=epi, a_mn=0, b_mn=0, A=A_PTR, lda=K, B=B_PTR, ldb=K, M=M, N=N, K=K, splits=1, block_n=0,
             out=OUT_PTR, ldo=N, bias=BIAS_PTR if epi in BIAS_EPIS else 0, out_rpg=0, out_gs=0, out_go=0, ak_rpg=0,
             ak_gs=0, ak_go=0, stream=0)
    a.update(kw)
    return ["ofk_gemm_bf16_grouped", list(a.values())]


def _lib_cases():
    c = {}
    for epi in range(10):
        c[f"valid-epi{epi}"] = (gemm_args(epi), NO_DEVICE)
    # A / B operands (TMA): base and row stride
    c["A+8B"] = (gemm_args(STORE_F32, A=A_PTR + 8), ALIGN)
    c["B+2B"] = (gemm_args(STORE_F32, B=B_PTR + 2), ALIGN)
    c["lda%8"] = (gemm_args(STORE_F32, lda=K + 4), ALIGN)
    c["ldb%8"] = (gemm_args(STORE_F32, ldb=K + 2), ALIGN)
    c["mn-lda%8"] = (gemm_args(STORE_F32, a_mn=1, lda=M + 4), ALIGN)
    # out: 16-byte pieces of f32 or bf16, depending on the epilogue
    for epi in range(10):
        elem = 4 if epi in F32_OUT else 2
        c[f"out+{elem}B-epi{epi}"] = (gemm_args(epi, out=OUT_PTR + elem), ALIGN)
        c[f"ldo+{16 // elem // 2}-epi{epi}"] = (gemm_args(epi, ldo=N + 16 // elem // 2), ALIGN)
    c["ldo+4-f32-ok"] = (gemm_args(STORE_F32, ldo=N + 4), NO_DEVICE)
    # out2 (bf16)
    for epi in OUT2_EPIS:
        c[f"out2+2B-epi{epi}"] = (gemm_args(epi, out2=OUT2_PTR + 2), ALIGN)
        c[f"out2+8B-epi{epi}"] = (gemm_args(epi, out2=OUT2_PTR + 8), ALIGN)
        c[f"ldo2+4-epi{epi}"] = (gemm_args(epi, ldo2=N + 4), ALIGN)
    # aux: f32 residual or bf16 pre-activation
    for epi in AUX_EPIS:
        elem = 2 if epi == DGELU else 4
        c[f"aux+{elem}B-epi{epi}"] = (gemm_args(epi, aux=AUX_PTR + elem), ALIGN)
        c[f"ldaux+{8 // elem}-epi{epi}"] = (gemm_args(epi, ldaux=N + 8 // elem), ALIGN)
    c["ldaux+4-f32-ok"] = (gemm_args(GATE_RESID, ldaux=N + 4), NO_DEVICE)
    # bias (float4 loads)
    for epi in BIAS_EPIS:
        c[f"bias+4B-epi{epi}"] = (gemm_args(epi, bias=BIAS_PTR + 4), ALIGN)
        c[f"bias+8B-epi{epi}"] = (gemm_args(epi, bias=BIAS_PTR + 8), ALIGN)
    # grouped maps
    kv = dict(a_mn=1, b_mn=1, lda=M, ldb=N, K=256)
    c["grouped-valid-ak"] = (grouped_args(ATOMIC_F32, ak_rpg=64, ak_gs=72, ak_go=0, **kv), NO_DEVICE)
    c["grouped-ak-rpg%64"] = (grouped_args(ATOMIC_F32, ak_rpg=32, ak_gs=40, ak_go=0, **kv), ARG)
    c["grouped-ak-K%rpg"] = (grouped_args(ATOMIC_F32, ak_rpg=128, ak_gs=136, ak_go=0, **dict(kv, K=192)), ARG)
    c["grouped-ak-kmajor-A"] = (grouped_args(ATOMIC_F32, ak_rpg=64, ak_gs=72, ak_go=0, **dict(kv, a_mn=0, lda=256)), ARG)
    for epi in (STORE_BF16, BIAS_BF16, STORE_F32):
        c[f"grouped-valid-out-epi{epi}"] = (grouped_args(epi, out_rpg=64, out_gs=72, out_go=8), NO_DEVICE)
    for epi in set(range(10)) - {STORE_BF16, BIAS_BF16, STORE_F32}:
        c[f"grouped-out-epi{epi}"] = (grouped_args(epi, out_rpg=64, out_gs=72, out_go=8), ARG)
    c["grouped-out+2B"] = (grouped_args(STORE_BF16, out=OUT_PTR + 2, out_rpg=64, out_gs=72, out_go=8), ALIGN)
    c["grouped-bias+4B"] = (grouped_args(BIAS_BF16, bias=BIAS_PTR + 4, out_rpg=64, out_gs=72, out_go=8), ALIGN)
    return c


LIB_CASES = _lib_cases()

# ops.gemm: (epi, aux (shape, dtype) or None, out2 (shape, dtype) or None, expected outcome)
OPS_CASES = {
    "valid-gate-resid": (GATE_RESID, ((M, N), "float32"), ((M, N), "bfloat16"), "RuntimeError"),
    "valid-dgelu": (DGELU, ((M, N), "bfloat16"), None, "RuntimeError"),
    "valid-gelu-dual": (GELU_DUAL, None, ((M, N), "bfloat16"), "RuntimeError"),
    "valid-bias-resid-wide": (BIAS_RESID, ((M + 1, N + 16), "float32"), ((M, N + 8), "bfloat16"), "RuntimeError"),
    "gate-resid-aux-bf16": (GATE_RESID, ((M, N), "bfloat16"), None, "ValueError"),
    "gate-resid-aux-short-rows": (GATE_RESID, ((M - 1, N), "float32"), None, "ValueError"),
    "bias-resid-aux-f64": (BIAS_RESID, ((M, N), "float64"), None, "ValueError"),
    "bias-resid-aux-narrow": (BIAS_RESID, ((M, N - 16), "float32"), None, "ValueError"),
    "dgelu-aux-f32": (DGELU, ((M, N), "float32"), None, "ValueError"),
    "dgelu-aux-narrow": (DGELU, ((M, N - 8), "bfloat16"), None, "ValueError"),
    "gelu-dual-out2-f32": (GELU_DUAL, None, ((M, N), "float32"), "ValueError"),
    "gelu-dual-out2-short-rows": (GELU_DUAL, None, ((M - 1, N), "bfloat16"), "ValueError"),
    "gate-resid-out2-f32": (GATE_RESID, ((M, N), "float32"), ((M, N), "float32"), "ValueError"),
    "bias-resid-out2-narrow": (BIAS_RESID, ((M, N), "float32"), ((M, N - 16), "bfloat16"), "ValueError"),
}

CHILD = r"""
import ctypes, json, sys
sys.path.insert(0, sys.argv[1])
import torch
from open_flamingo_b200 import _lib, ops
cases = json.load(sys.stdin)
lib = _lib.lib()
res = {"lib": {}, "ops": {}}
for name, ((fn, args), _) in cases["lib"].items():
    res["lib"][name] = getattr(lib, fn)(*args)
# ops.gemm's own checks: CPU tensors stand in for device tensors (host addresses, never dereferenced -- a call that gets
# through reaches device discovery and fails there)
_lib.require_cuda = lambda *t: None
_lib.stream_ptr = lambda: 0
for name, (epi, aux, out2, _) in cases["ops"].items():
    M, N, K = cases["mnk"]
    kw = {}
    if aux is not None:
        kw["aux"] = torch.zeros(aux[0], dtype=getattr(torch, aux[1]))
    if out2 is not None:
        kw["out2"] = torch.zeros(out2[0], dtype=getattr(torch, out2[1]))
    if epi in cases["bias_epis"]:
        kw["bias"] = torch.zeros(N)
    try:
        ops.gemm(torch.zeros(M, K, dtype=torch.bfloat16), torch.zeros(N, K, dtype=torch.bfloat16), epi=epi, **kw)
        res["ops"][name] = "ok"
    except Exception as e:
        res["ops"][name] = type(e).__name__ + ": " + str(e)
print(json.dumps(res))
"""


@pytest.fixture(scope="module")
def results():
    import __graft_entry__ as g
    g.build()
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", CHILD, ROOT]
    payload = json.dumps({"lib": LIB_CASES, "ops": OPS_CASES, "mnk": [M, N, K], "bias_epis": BIAS_EPIS})
    r = subprocess.run(cmd, input=payload, capture_output=True, text=True, env=env, timeout=600)
    assert r.returncode == 0, r.stderr
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("case", sorted(LIB_CASES))
def test_gemm_entry_point_return_code(results, case):
    got, want = results["lib"][case], LIB_CASES[case][1]
    assert got == want, f"{case}: returned {got}, expected {want} (-3 = the check ran after device discovery or not at all)"


@pytest.mark.parametrize("case", sorted(OPS_CASES))
def test_ops_gemm_checks_epilogue_operands(results, case):
    got, want = results["ops"][case], OPS_CASES[case][3]
    assert got.startswith(want + ":"), f"{case}: {got}"
    if want == "RuntimeError":
        assert "libofk error -3" in got, got   # passed ops.gemm's checks and the library's, failed for want of a device
