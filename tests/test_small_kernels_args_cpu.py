"""CPU: the LayerNorm, gate-backward, ViT token-assembly and cross-entropy entry points reject bad arguments with the
documented error code, before they touch a device.

As in test_attention_args_cpu.py, every call runs in a child process with no CUDA device visible and with made-up device
addresses that are never dereferenced.  A call whose arguments pass validation reaches the first CUDA call and returns
OFK_ERR_CUDA (-3), so a missing or late check shows up as a wrong code and can never launch a kernel.

The cross-entropy kernels reject no pointer: a bf16 row that is not 16-byte aligned is read by the scalar path, so those
cases must reach the device."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ARG, ALIGN, NO_DEVICE = -1, -2, -3
(X, GAMMA, BETA, Y, MEAN, RSTD, DY, DX, DXADD, DGAMMA, DBETA, WS, DOUT, BRANCH, GATE, DBRANCH, DGATE, PE, CLS, POS, TOK,
 LOGITS, LABELS, LSE, LOSS, COUNT, GSCALE, DLOGITS) = (k << 32 for k in range(1, 29))
ROWS, D = 300, 1028
U_, V_, N_ = 3, 20, 8                        # Perceiver group mapping: U images of v media rows and n latent rows

# Argument lists in the order of include/ofk.h.  Defaults are valid problems.
LN_FWD = dict(x=X, ldx=D, gamma=GAMMA, beta=BETA, eps=1e-5, rows=ROWS, D=D, y=Y, y_is_f32=0, ldy=D, rpg=0, gstride=0,
              goff=0, mean=MEAN, rstd=RSTD, stream=0)
LN_BWD = dict(dy=DY, dy_is_f32=0, lddy=D, rpg=0, gstride=0, goff=0, x=X, ldx=D, gamma=GAMMA, mean=MEAN, rstd=RSTD,
              rows=ROWS, D=D, dx=DX, lddx=D, dx_add=DXADD, ldadd=D, dgamma=DGAMMA, dbeta=DBETA, workspace=WS, stream=0)
GATE_BWD = dict(dout=DOUT, branch=BRANCH, gate=GATE, dbranch=DBRANCH, dgate=DGATE, n=8 * 1000, workspace=WS, stream=0)
VIT = dict(patch_emb=PE, class_emb=CLS, pos_emb=POS, n=2, g=256, D=1024, tokens=TOK, stream=0)
CE_FWD = dict(logits=LOGITS, is_f32=0, ld=50280, rows=4 * 17, vocab=50280, labels=LABELS, T=17, shift=1,
              ignore_index=-100, lse=LSE, loss_sum=LOSS, count=COUNT, stream=0)
CE_BWD = dict(logits=LOGITS, is_f32=0, ld=50280, rows=4 * 17, vocab=50280, labels=LABELS, T=17, shift=1,
              ignore_index=-100, lse=LSE, grad_scale=GSCALE, count=COUNT, dlogits=DLOGITS, ldd=50280, stream=0)
ENTRY = {"ln_fwd": ("ofk_layernorm_fwd", LN_FWD), "ln_bwd": ("ofk_layernorm_bwd", LN_BWD),
         "gate_bwd": ("ofk_gate_bwd", GATE_BWD), "vit": ("ofk_vit_assemble", VIT), "ce_fwd": ("ofk_ce_fwd", CE_FWD),
         "ce_bwd": ("ofk_ce_bwd", CE_BWD)}


def _cases():
    c = {}

    def add(entry, name, want, **kw):
        fn, defaults = ENTRY[entry]
        c[f"{entry}:{name}"] = (fn, list({**defaults, **kw}.values()), want)

    group_v = dict(rows=U_ * V_, rpg=V_, gstride=V_ + N_, goff=0)          # media rows of cat((x, latents))
    group_n = dict(rows=U_ * N_, rpg=N_, gstride=V_ + N_, goff=V_)         # latent rows
    for e in ("ln_fwd", "ln_bwd"):
        bwd = e == "ln_bwd"
        ymat, yf32 = ("dy", "dy_is_f32") if bwd else ("y", "y_is_f32")
        ybase = DY if bwd else Y
        add(e, "valid", NO_DEVICE)
        add(e, "valid-f32", NO_DEVICE, **{yf32: 1})
        add(e, "valid-group-media", NO_DEVICE, **group_v)
        add(e, "valid-group-latents", NO_DEVICE, **group_n)
        add(e, "valid-D4", NO_DEVICE, D=4, ldx=4, **({"lddy": 4, "lddx": 4, "ldadd": 4} if bwd else {"ldy": 4}))
        add(e, "valid-D4096", NO_DEVICE, D=4096, ldx=4096,
            **({"lddy": 4096, "lddx": 4096, "ldadd": 4096} if bwd else {"ldy": 4096}))
        add(e, "rows0", 0, rows=0)
        add(e, "D0", ARG, D=0)
        add(e, "D6", ARG, D=6)
        add(e, "D4100", ARG, D=4100)
        add(e, "x-null", ARG, x=0)
        add(e, "gamma-null", ARG, gamma=0)
        add(e, f"{ymat}-null", ARG, **{ymat: 0})
        add(e, "ldx+1", ALIGN, ldx=D + 1)
        # the group mapping: the groups of rows_per_group rows at group_offset must fit inside group_stride rows
        add(e, "group-offset-past-stride", ARG, **{**group_n, "goff": V_ + 1})
        add(e, "group-stride-short", ARG, **{**group_v, "gstride": V_ - 1})
        add(e, "group-offset-neg", ARG, **{**group_v, "goff": -1})
        add(e, "valid-group-offset-fills-stride", NO_DEVICE, **{**group_n, "goff": V_, "gstride": V_ + N_})
        # base pointers of float4 accesses at +4 and +8 bytes
        for p, base in (("x", X), ("gamma", GAMMA)) + ((("dx", DX), ("dx_add", DXADD), ("workspace", WS)) if bwd
                                                        else (("beta", BETA),)):
            for off in (4, 8):
                add(e, f"{p}+{off}B", ALIGN, **{p: base + off})
        # y / dy: 16 bytes as f32, 8 bytes as bf16 (read or written 4 elements at a time)
        for off in (4, 8):
            add(e, f"{ymat}-f32+{off}B", ALIGN, **{ymat: ybase + off, yf32: 1})
        add(e, f"{ymat}-bf16+2B", ALIGN, **{ymat: ybase + 2})
        add(e, f"{ymat}-bf16+4B", ALIGN, **{ymat: ybase + 4})
        add(e, f"valid-{ymat}-bf16+8B", NO_DEVICE, **{ymat: ybase + 8})
        add(e, "valid-mean+4B", NO_DEVICE, mean=MEAN + 4)               # per-row scalars
        if bwd:
            add(e, "valid-no-dx", NO_DEVICE, dx=0, lddx=0, dx_add=0, ldadd=0)
            add(e, "valid-dx-only", NO_DEVICE, dgamma=0, dbeta=0)
            add(e, "valid-dbeta-only", NO_DEVICE, dx=0, lddx=0, dx_add=0, ldadd=0, dgamma=0)
            add(e, "valid-dx-is-dx_add", NO_DEVICE, dx_add=DX)
            add(e, "nothing-wanted", 0, dx=0, dgamma=0, dbeta=0)
            add(e, "valid-dgamma+4B", NO_DEVICE, dgamma=DGAMMA + 4)       # summed one column at a time
            add(e, "workspace-null", ARG, workspace=0)
            add(e, "ldadd+2", ALIGN, ldadd=D + 2)
        else:
            add(e, "beta-null", ARG, beta=0)
            add(e, "valid-no-stats", NO_DEVICE, mean=0, rstd=0)
            add(e, "ldy+2", ALIGN, ldy=D + 2)

    e = "gate_bwd"
    add(e, "valid", NO_DEVICE)
    add(e, "valid-n8", NO_DEVICE, n=8)
    add(e, "valid-no-dgate", NO_DEVICE, dgate=0, workspace=0)
    add(e, "valid-plain-cast", NO_DEVICE, branch=0, gate=0, dgate=0, workspace=0)
    add(e, "valid-plain-cast-branch+8B", NO_DEVICE, branch=BRANCH + 8, gate=0, dgate=0, workspace=0)   # branch unused
    add(e, "valid-gate+4B", NO_DEVICE, gate=GATE + 4)
    add(e, "valid-workspace+4B", NO_DEVICE, workspace=WS + 4)
    add(e, "n0", 0, n=0)
    add(e, "n12", ARG, n=12)
    add(e, "dout-null", ARG, dout=0)
    add(e, "dbranch-null", ARG, dbranch=0)
    add(e, "branch-null-with-gate", ARG, branch=0)
    add(e, "workspace-null-with-dgate", ARG, workspace=0)
    for p, base in (("dout", DOUT), ("branch", BRANCH), ("dbranch", DBRANCH)):
        for off in (4, 8):
            add(e, f"{p}+{off}B", ALIGN, **{p: base + off})

    e = "vit"
    add(e, "valid", NO_DEVICE)
    add(e, "valid-g0", NO_DEVICE, g=0)                                      # class token only
    add(e, "valid-g0-patch_emb-null", NO_DEVICE, g=0, patch_emb=0)          # (an empty tensor's address may be 0)
    add(e, "valid-D4", NO_DEVICE, D=4)
    add(e, "valid-pe+8B", NO_DEVICE, patch_emb=PE + 8)
    add(e, "n0", 0, n=0)
    add(e, "g-neg", ARG, g=-1)
    add(e, "D0", ARG, D=0)
    add(e, "D-neg", ARG, D=-4)
    add(e, "D6", ARG, D=6)
    for p in ("patch_emb", "class_emb", "pos_emb", "tokens"):
        add(e, f"{p}-null", ARG, **{p: 0})
    add(e, "patch_emb+2B", ALIGN, patch_emb=PE + 2)
    add(e, "patch_emb+4B", ALIGN, patch_emb=PE + 4)
    for p, base in (("class_emb", CLS), ("pos_emb", POS), ("tokens", TOK)):
        for off in (4, 8):
            add(e, f"{p}+{off}B", ALIGN, **{p: base + off})

    for e in ("ce_fwd", "ce_bwd"):
        bwd = e == "ce_bwd"
        add(e, "valid", NO_DEVICE)
        add(e, "valid-f32", NO_DEVICE, is_f32=1)
        add(e, "valid-V61", NO_DEVICE, vocab=61, ld=61, **({"ldd": 61} if bwd else {}))
        add(e, "valid-column-slice", NO_DEVICE, ld=50304)
        add(e, "valid-1x1", NO_DEVICE, rows=1, T=1)
        # unaligned rows are read by the scalar path: accepted
        for off in (2, 4, 8):
            add(e, f"valid-logits+{off}B", NO_DEVICE, logits=LOGITS + off)
        add(e, "valid-f32-logits+4B", NO_DEVICE, logits=LOGITS + 4, is_f32=1)
        if bwd:
            add(e, "valid-dlogits+2B", NO_DEVICE, dlogits=DLOGITS + 2)
            add(e, "valid-dlogits+8B", NO_DEVICE, dlogits=DLOGITS + 8)
        add(e, "rows0", 0, rows=0)
        add(e, "rows-not-multiple-of-T", ARG, rows=4 * 17 + 1)
        add(e, "T0", ARG, T=0)
        add(e, "vocab0", ARG, vocab=0)
        for p in ("logits", "labels", "lse", "count") + (("grad_scale", "dlogits") if bwd else ("loss_sum",)):
            add(e, f"{p}-null", ARG, **{p: 0})
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
def test_small_kernel_entry_point_return_code(results, case):
    got, want = results[case], CASES[case][2]
    assert got == want, f"{case}: returned {got}, expected {want} (-3 = the check ran after device discovery or not at all)"
