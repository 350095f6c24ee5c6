"""CPU: the four training attention entry points (ofk_attn_fwd / ofk_attn_bwd for the media rules, ofk_attn_dense_fwd /
ofk_attn_dense_bwd for the LM blocks) reject bad arguments with the documented error code, before they touch a device.

As in test_gemm_args_cpu.py, every call runs in a child process with no CUDA device visible and with made-up device
addresses that are never dereferenced.  A call whose arguments pass validation reaches the first CUDA call and returns
OFK_ERR_CUDA (-3), so a missing or late check shows up as a wrong code and can never launch a kernel."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ARG, ALIGN, NO_DEVICE = -1, -2, -3
(Q, K, V, O, DO, LSE, DELTA, DQ, DK, DV, TT, MASK, SLOPES, FLAG) = (k << 32 for k in range(1, 15))
B, H, NQ, NK, KPM = 3, 4, 100, 192, 64
D = H * 64


# Argument lists in the order of include/ofk.h.  Defaults are a valid problem: q a column slice of a qkv-like buffer,
# k/v column slices of one [B, nk, 2D] (media) or [B, capacity, 2D] / [B, T, 3D] (dense) buffer, and gradients as
# column slices of a [B, n, 3D] or [B, n, 2D] buffer.
MEDIA_FWD = dict(q=Q, k=K, v=V, o=O, lse=LSE, batch=B, heads=H, nq=NQ, nk=NK, q_bs=NQ * 3 * D, ldq=3 * D,
                 k_bs=NK * 2 * D, ldk=2 * D, v_bs=NK * 2 * D, ldv=2 * D, o_bs=NQ * D, ldo=D, scale=0.125, mask_mode=1,
                 text_time=TT, kpm=KPM, stream=0)
MEDIA_BWD = dict(q=Q, k=K, v=V, o=O, d_o=DO, lse=LSE, delta=DELTA, dq=DQ, dk=DK, dv=DV, batch=B, heads=H, nq=NQ, nk=NK,
                 q_bs=NQ * 3 * D, ldq=3 * D, k_bs=NK * 2 * D, ldk=2 * D, v_bs=NK * 2 * D, ldv=2 * D, o_bs=NQ * D, ldo=D,
                 dq_bs=NQ * 3 * D, lddq=3 * D, dk_bs=NK * 2 * D, lddk=2 * D, dv_bs=NK * 2 * D, lddv=2 * D,
                 scale=0.125, mask_mode=1, text_time=TT, kpm=KPM, stream=0)
HD = 128
DD = H * HD
DENSE_FWD = dict(q=Q, k=K, v=V, o=O, lse=LSE, batch=B, heads=H, head_dim=HD, nq=NQ, nk=NK, q_bs=NQ * DD, ldq=DD,
                 k_bs=512 * 2 * DD, ldk=2 * DD, v_bs=512 * 2 * DD, ldv=2 * DD, o_bs=NQ * DD, ldo=DD,
                 scale=HD ** -0.5, causal=1, mask=0, slopes=SLOPES, flag=0, stream=0)
DENSE_BWD = dict(q=Q, k=K, v=V, o=O, d_o=DO, lse=LSE, delta=DELTA, dq=DQ, dk=DK, dv=DV, batch=B, heads=H, head_dim=HD,
                 nq=NK, nk=NK, q_bs=NK * 3 * DD, ldq=3 * DD, k_bs=NK * 3 * DD, ldk=3 * DD, v_bs=NK * 3 * DD,
                 ldv=3 * DD, o_bs=NK * DD, ldo=DD, dq_bs=NK * 3 * DD, lddq=3 * DD, dk_bs=NK * 3 * DD, lddk=3 * DD,
                 dv_bs=NK * 3 * DD, lddv=3 * DD, scale=HD ** -0.5, causal=0, mask=MASK, slopes=SLOPES, flag=FLAG,
                 stream=0)
ENTRY = {"media_fwd": ("ofk_attn_fwd", MEDIA_FWD), "media_bwd": ("ofk_attn_bwd", MEDIA_BWD),
         "dense_fwd": ("ofk_attn_dense_fwd", DENSE_FWD), "dense_bwd": ("ofk_attn_dense_bwd", DENSE_BWD)}


def _cases():
    c = {}

    def add(entry, name, want, **kw):
        fn, defaults = ENTRY[entry]
        c[f"{entry}:{name}"] = (fn, list({**defaults, **kw}.values()), want)

    for e in ENTRY:
        bwd, dense = e.endswith("bwd"), e.startswith("dense")
        add(e, "valid", NO_DEVICE)
        add(e, "valid-nq1-nk1", NO_DEVICE, nq=1, nk=1, **({} if dense else {"mask_mode": 0}))
        add(e, "batch0", ARG, batch=0)
        add(e, "heads0", ARG, heads=0)
        add(e, "nq0", ARG, nq=0)
        add(e, "nk0", ARG, nk=0)
        add(e, "nk-neg", ARG, nk=-64)
        add(e, "batch65536", ARG, batch=65536)
        add(e, "heads65536", ARG, heads=65536)
        ptrs = ["q", "k", "v", "o"] + (["d_o", "lse", "delta", "dq", "dk", "dv"] if bwd else [])
        for p in ptrs:
            add(e, f"{p}-null", ARG, **{p: 0})
        # 16-byte operands at +2 and +8 bytes; 4-byte ones at +2 (and gradients written 32 bits at a time at +2)
        for p, base in (("q", Q), ("k", K), ("v", V), ("o", O)) + ((("d_o", DO),) if bwd else ()):
            for off in (2, 8):
                add(e, f"{p}+{off}B", ALIGN, **{p: base + off})
        four = [("lse", LSE)] + ([("delta", DELTA), ("dq", DQ), ("dk", DK), ("dv", DV)] if bwd else [])
        four += [("slopes", SLOPES), ("flag", FLAG)] if dense else [("text_time", TT)]
        for p, base in four:
            add(e, f"{p}+2B", ALIGN, **{p: base + 2})
        if bwd:
            for p, base in (("dq", DQ), ("dk", DK), ("dv", DV)):
                add(e, f"valid-{p}+4B", NO_DEVICE, **{p: base + 4})
        if dense:
            add(e, "valid-mask+1B", NO_DEVICE, mask=MASK + 1)               # read byte by byte
        # every batch and row stride of a 16-byte operand at +1 and +4 elements; gradient strides odd
        strides = ["q_bs", "ldq", "k_bs", "ldk", "v_bs", "ldv", "o_bs", "ldo"]
        for s in strides:
            base = ENTRY[e][1][s]
            for off in (1, 4):
                add(e, f"{s}+{off}", ALIGN, **{s: base + off})
        if bwd:
            for s in ("dq_bs", "lddq", "dk_bs", "lddk", "dv_bs", "lddv"):
                base = ENTRY[e][1][s]
                add(e, f"{s}+1", ALIGN, **{s: base + 1})
                add(e, f"valid-{s}+2", NO_DEVICE, **{s: base + 2})
        if dense:
            for hd in (32, 96, 256):
                add(e, f"hd{hd}", ARG, head_dim=hd)
            add(e, "valid-hd64", NO_DEVICE, head_dim=64)
            # the causal rule (or the pure-causal flag) with nq > nk
            add(e, "causal-nq>nk", ARG, nq=NK + 1, nk=NK, causal=1, mask=0, flag=0)
            add(e, "flag-nq>nk", ARG, nq=NK + 1, nk=NK, causal=0, mask=MASK, flag=FLAG)
            add(e, "valid-mask-nq>nk", NO_DEVICE, nq=NK + 1, nk=NK, causal=0, mask=MASK, flag=0)
            add(e, "valid-causal-nq<nk", NO_DEVICE, nq=65, nk=1000, causal=1, mask=0, flag=FLAG)
            add(e, "valid-causal-nq=nk=1", NO_DEVICE, nq=1, nk=1, causal=1)
        else:
            add(e, "mask_mode3", ARG, mask_mode=3)
            add(e, "mask_mode-1", ARG, mask_mode=-1)
            add(e, "text_time-null-mode1", ARG, text_time=0, mask_mode=1)
            add(e, "text_time-null-mode2", ARG, text_time=0, mask_mode=2)
            add(e, "valid-text_time-null-mode0", NO_DEVICE, text_time=0, mask_mode=0)
            for kpm in (0, 8, 24, -64):
                add(e, f"kpm{kpm}", ARG, kpm=kpm)
            add(e, "kpm-not-dividing-nk", ARG, kpm=80)            # 192 % 80 != 0
            add(e, "valid-kpm16", NO_DEVICE, kpm=16)
            add(e, "valid-kpm48", NO_DEVICE, kpm=48)
            add(e, "valid-kpm80", NO_DEVICE, kpm=80, nk=400, k_bs=400 * 2 * D, v_bs=400 * 2 * D,
                **({"dk_bs": 400 * 2 * D, "dv_bs": 400 * 2 * D} if bwd else {}))
            add(e, "valid-mode0-kpm0", NO_DEVICE, mask_mode=0, kpm=0, text_time=0)
            if not bwd:
                add(e, "valid-no-lse", NO_DEVICE, lse=0)
    return c


CASES = _cases()

CHILD = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
from open_flamingo_b200 import _lib
cases = json.load(sys.stdin)
lib = _lib.lib()
print(json.dumps({n: getattr(lib, fn)(*args) for n, (fn, args, _) in cases.items()}))
"""


@pytest.fixture(scope="module")
def results():
    import __graft_entry__ as g
    g.build()
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", CHILD, ROOT]
    r = subprocess.run(cmd, input=json.dumps(CASES), capture_output=True, text=True, env=env, timeout=600)
    assert r.returncode == 0, r.stderr
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_builders_match_the_abi():
    """The argument lists above have exactly the arity the ctypes signatures declare."""
    from open_flamingo_b200 import _lib
    for fn, args, _ in CASES.values():
        assert len(args) == len(_lib._SIGNATURES[fn][1]), fn


@pytest.mark.parametrize("case", sorted(CASES))
def test_attention_entry_point_return_code(results, case):
    got, want = results[case], CASES[case][2]
    assert got == want, f"{case}: returned {got}, expected {want} (-3 = the check ran after device discovery or not at all)"
