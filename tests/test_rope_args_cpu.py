"""CPU: ofk_rope_pack, ofk_rope_unpack_bwd and ofk_gelu_bf16 reject bad arguments with the documented error code before
they touch a device; the decode workspace accepts head_dim 80 and still rejects 96; and the new kernels, and the decode
kernels at head_dim 80, keep everything in registers.

As in test_decode_args_cpu.py, every call runs in a child process with no CUDA device visible and with made-up device
addresses that are never dereferenced.  A call whose arguments pass validation reaches the launch and returns
OFK_ERR_CUDA (-3), so a missing or late check shows up as a wrong code."""
import json
import os
import subprocess
import sys

import pytest

from test_abi_cpu import _sass_by_kernel

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ARG, ALIGN, NO_DEVICE = -1, -2, -3
SRC, COS, SIN, Q, K, V, DQKV = (k << 32 for k in range(1, 8))
B, T, H, HD, ROT, W = 2, 77, 4, 80, 80, 128


def pack_args(**kw):
    a = dict(src_q=SRC, src_k=SRC + 2 * HD, src_v=SRC + 4 * HD, src_bs=T * 3 * H * HD, ld_src=3 * H * HD,
             src_hs=3 * HD, batch=B, rows=T, heads=H, head_dim=HD, rot=ROT, cos=COS, sin=SIN, cs_bs=0, ld_cs=ROT,
             q=Q, q_bs=T * H * W, ldq=H * W, q_w=W, k=K, k_bs=T * H * W, ldk=H * W, k_w=W,
             v=V, v_bs=T * H * W, ldv=H * W, v_w=W, stream=0)
    a.update(kw)
    return list(a.values())


def unpack_args(**kw):
    a = dict(dq=Q, dq_bs=T * H * W, lddq=H * W, dk=K, dk_bs=T * H * W, lddk=H * W, dv=V, dv_bs=T * H * W, lddv=H * W,
             width=W, batch=B, rows=T, heads=H, head_dim=HD, rot=ROT, cos=COS, sin=SIN, cs_bs=T * ROT, ld_cs=ROT,
             dqkv=DQKV, dqkv_bs=T * 3 * H * HD, lddqkv=3 * H * HD, stream=0)
    a.update(kw)
    return list(a.values())


def _cases():
    pack = {
        "valid": (pack_args(), NO_DEVICE),
        "valid-partial-rot": (pack_args(rot=20), NO_DEVICE),
        "valid-no-rotation": (pack_args(rot=0, cos=0, sin=0), NO_DEVICE),
        "valid-unpadded": (pack_args(q_w=HD, ldq=H * HD, k_w=HD, ldk=H * HD, v_w=HD, ldv=H * HD), NO_DEVICE),
        "valid-kv-only": (pack_args(src_q=0, q=0), NO_DEVICE),
        "valid-per-row-cos": (pack_args(cs_bs=T * ROT), NO_DEVICE),
        "rot-odd": (pack_args(rot=21), ARG),
        "rot-gt-hd": (pack_args(rot=HD + 2), ARG),
        "rot-neg": (pack_args(rot=-2), ARG),
        "cos-missing": (pack_args(cos=0), ARG),
        "sin-missing": (pack_args(sin=0), ARG),
        "ld-cs-below-rot": (pack_args(ld_cs=ROT - 2), ARG),
        "width-below-hd": (pack_args(q_w=72), ARG),
        "width-not-8": (pack_args(k_w=132, ldk=H * 132), ARG),
        "hd-not-8": (pack_args(head_dim=84, rot=84, ld_cs=84), ARG),
        "dst-missing": (pack_args(v=0), ARG),
        "no-source": (pack_args(src_q=0, src_k=0, src_v=0), ARG),
        "ldq-short": (pack_args(ldq=H * W - 8), ARG),
        "src-head-stride-short": (pack_args(src_hs=HD - 8), ARG),
        "batch0": (pack_args(batch=0), ARG),
        "rows0": (pack_args(rows=0), ARG),
        "heads0": (pack_args(heads=0), ARG),
        "cos+2B": (pack_args(cos=COS + 2), ALIGN),
    }
    for name, base in (("src_q", SRC), ("src_k", SRC + 2 * HD), ("q", Q), ("k", K), ("v", V)):
        for off in (2, 8):
            pack[f"{name}+{off}B"] = (pack_args(**{name: base + off}), ALIGN)
    for name, base in (("src_bs", T * 3 * H * HD), ("ld_src", 3 * H * HD), ("q_bs", T * H * W), ("ldk", H * W)):
        pack[f"{name}+4"] = (pack_args(**{name: base + 4}), ALIGN)
    pack["src_hs+4"] = (pack_args(src_hs=3 * HD + 4), ALIGN)

    unpack = {
        "valid": (unpack_args(), NO_DEVICE),
        "valid-no-rotation": (unpack_args(rot=0, cos=0, sin=0), NO_DEVICE),
        "valid-unpadded": (unpack_args(width=HD, lddq=H * HD, lddk=H * HD, lddv=H * HD), NO_DEVICE),
        "rot-odd": (unpack_args(rot=11), ARG),
        "rot-gt-hd": (unpack_args(rot=HD + 2), ARG),
        "cos-missing": (unpack_args(cos=0), ARG),
        "width-below-hd": (unpack_args(width=72), ARG),
        "width-not-8": (unpack_args(width=132, lddq=H * 132, lddk=H * 132, lddv=H * 132), ARG),
        "dv-null": (unpack_args(dv=0), ARG),
        "out-null": (unpack_args(dqkv=0), ARG),
        "out-ld-short": (unpack_args(lddqkv=3 * H * HD - 8), ARG),
        "cos+2B": (unpack_args(sin=SIN + 2), ALIGN),
    }
    for name, base in (("dq", Q), ("dk", K), ("dv", V), ("dqkv", DQKV)):
        unpack[f"{name}+8B"] = (unpack_args(**{name: base + 8}), ALIGN)
    for name, base in (("lddq", H * W), ("dk_bs", T * H * W), ("lddqkv", 3 * H * HD)):
        unpack[f"{name}+4"] = (unpack_args(**{name: base + 4}), ALIGN)

    gelu = {"valid": ([SRC, Q, 1024, 0], NO_DEVICE), "n-not-8": ([SRC, Q, 1020, 0], ARG),
            "z-null": ([0, Q, 1024, 0], ARG), "z+8B": ([SRC + 8, Q, 1024, 0], ALIGN), "h+2B": ([SRC, Q + 2, 1024, 0], ALIGN),
            "empty": ([SRC, Q, 0, 0], 0)}
    return {"pack": pack, "unpack": unpack, "gelu": gelu}


CASES = _cases()
WS_CASES = {"hd80": ((B, 32, 80, 4097), "pos"), "hd80-nk1": ((1, 32, 80, 1), "pos"), "hd96": ((B, H, 96, 300), ARG),
            "hd72": ((B, H, 72, 300), ARG)}

CHILD = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
from open_flamingo_b200 import _lib
cases = json.load(sys.stdin)
lib = _lib.lib()
fns = {"pack": lib.ofk_rope_pack, "unpack": lib.ofk_rope_unpack_bwd, "gelu": lib.ofk_gelu_bf16}
res = {k: {n: fns[k](*args) for n, (args, _) in cases[k].items()} for k in fns}
res["ws"] = {n: lib.ofk_attn_decode_workspace_bytes(*args) for n, (args, _) in cases["ws"].items()}
print(json.dumps(res))
"""


@pytest.fixture(scope="module")
def results():
    import __graft_entry__ as g
    g.build()
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", CHILD, ROOT]
    r = subprocess.run(cmd, input=json.dumps(dict(CASES, ws=WS_CASES)), capture_output=True, text=True, env=env,
                       timeout=600)
    assert r.returncode == 0, r.stderr
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("fn,case", [(f, c) for f in sorted(CASES) for c in sorted(CASES[f])])
def test_rope_and_gelu_return_codes(results, fn, case):
    got, want = results[fn][case], CASES[fn][case][1]
    assert got == want, f"{fn} {case}: returned {got}, expected {want} (-3 = the check ran after the launch or not at all)"


@pytest.mark.parametrize("case", sorted(WS_CASES))
def test_decode_workspace_bytes_head_dim_80(results, case):
    got, want = results["ws"][case], WS_CASES[case][1]
    if want == "pos":
        b, h, hd, nk = WS_CASES[case][0]
        assert got >= b * h * (hd + 2) * 4 and got % 4 == 0, got
    else:
        assert got == want, got


def test_new_kernels_use_no_local_memory():
    kernels = _sass_by_kernel()
    names = [k for k in kernels if "rope_pack_kernel" in k or "rope_unpack_bwd_kernel" in k or "gelu_bf16_kernel" in k
             or ("kv_decode" in k and "ILi80E" in k)]
    assert len(names) == 5, sorted(names)
    for k in names:
        assert not kernels[k] & {"LDL", "STL"}, f"{k}: local-memory traffic"
