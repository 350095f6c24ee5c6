"""CPU: ofk_attn_decode rejects bad arguments with the documented error code, before it touches a device.

As in test_gemm_args_cpu.py, every call runs in a child process with no CUDA device visible and with made-up device
addresses that are never dereferenced.  A call whose arguments pass validation reaches device discovery and returns
OFK_ERR_CUDA (-3), so a missing or late check shows up as a wrong code and can never launch a kernel."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ARG, ALIGN, NO_DEVICE = -1, -2, -3
Q_PTR, K_PTR, V_PTR, O_PTR, MASK_PTR, SLOPES_PTR, WS_PTR = (k << 32 for k in range(1, 8))
B, H, HD, NK = 3, 4, 128, 300
D = H * HD


def decode_args(**kw):
    a = dict(q=Q_PTR, q_bs=3 * D, k=K_PTR, v=V_PTR, kv_bs=512 * 2 * D, ldkv=2 * D, o=O_PTR, o_bs=D, batch=B, heads=H,
             head_dim=HD, nk=NK, scale=HD ** -0.5, mask=MASK_PTR, mask_bs=304, slopes=SLOPES_PTR, ws=WS_PTR, stream=0)
    a.update(kw)
    return list(a.values())


def _cases():
    c = {
        "valid": (decode_args(), NO_DEVICE),
        "valid-hd64": (decode_args(head_dim=64), NO_DEVICE),
        "valid-no-mask-no-slopes": (decode_args(mask=0, mask_bs=3, slopes=0), NO_DEVICE),
        "valid-nk1": (decode_args(nk=1), NO_DEVICE),
        "valid-slopes+4B": (decode_args(slopes=SLOPES_PTR + 4), NO_DEVICE),   # read as scalars
        "hd32": (decode_args(head_dim=32), ARG),
        "hd96": (decode_args(head_dim=96), ARG),
        "hd256": (decode_args(head_dim=256), ARG),
        "batch0": (decode_args(batch=0), ARG),
        "heads0": (decode_args(heads=0), ARG),
        "nk0": (decode_args(nk=0), ARG),
        "nk-neg": (decode_args(nk=-5), ARG),
        "q-null": (decode_args(q=0), ARG),
        "k-null": (decode_args(k=0), ARG),
        "o-null": (decode_args(o=0), ARG),
        "ws-null": (decode_args(ws=0), ARG),
    }
    for name, ptr in (("q", Q_PTR), ("k", K_PTR), ("v", V_PTR), ("o", O_PTR), ("mask", MASK_PTR), ("ws", WS_PTR)):
        for off in (2, 8):
            c[f"{name}+{off}B"] = (decode_args(**{name: ptr + off}), ALIGN)
    for name, base in (("q_bs", 3 * D), ("kv_bs", 512 * 2 * D), ("ldkv", 2 * D), ("o_bs", D), ("mask_bs", 304)):
        for off in (1, 4):
            c[f"{name}+{off}"] = (decode_args(**{name: base + off}), ALIGN)
    return c


CASES = _cases()
WS_CASES = {"hd128": ((B, H, 128, NK), "pos"), "hd64": ((B, H, 64, NK), "pos"), "hd96": ((B, H, 96, NK), ARG),
            "nk0": ((B, H, 128, 0), ARG), "batch0": ((0, H, 128, NK), ARG)}

CHILD = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
from open_flamingo_b200 import _lib
cases = json.load(sys.stdin)
lib = _lib.lib()
res = {"call": {n: lib.ofk_attn_decode(*args) for n, (args, _) in cases["call"].items()},
       "ws": {n: lib.ofk_attn_decode_workspace_bytes(*args) for n, (args, _) in cases["ws"].items()}}
print(json.dumps(res))
"""


@pytest.fixture(scope="module")
def results():
    import __graft_entry__ as g
    g.build()
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", CHILD, ROOT]
    r = subprocess.run(cmd, input=json.dumps({"call": CASES, "ws": WS_CASES}), capture_output=True, text=True, env=env,
                       timeout=600)
    assert r.returncode == 0, r.stderr
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("case", sorted(CASES))
def test_decode_entry_point_return_code(results, case):
    got, want = results["call"][case], CASES[case][1]
    assert got == want, f"{case}: returned {got}, expected {want} (-3 = the check ran after device discovery or not at all)"


@pytest.mark.parametrize("case", sorted(WS_CASES))
def test_decode_workspace_bytes(results, case):
    got, want = results["ws"][case], WS_CASES[case][1]
    if want == "pos":
        b, h, hd, nk = WS_CASES[case][0]
        assert got >= b * h * (hd + 2) * 4 and got % 4 == 0, got   # room for at least one split's partials
    else:
        assert got == want, got
