"""CPU: the RMSNorm and SwiGLU entry points reject bad arguments with the documented error code before they touch a
device; their ops wrappers raise ValueError on shapes and dtypes; the new kernels keep everything in registers; and the
host logic of lm_blocks.FastLlamaBlock -- accelerate() returns it for a LlamaDecoderLayer, it declines every call the
kernels do not evaluate, and its packed QKV weight has the per-head (q | k | v) row order the rotary kernels read.

As in test_small_kernels_args_cpu.py, every call runs in a child process with no CUDA device visible and with made-up
device addresses that are never dereferenced.  A call whose arguments pass validation reaches the launch and returns
OFK_ERR_CUDA (-3), so a missing or late check shows up as a wrong code.  The host-logic checks read only
hidden_states.is_cuda, so a stand-in with is_cuda = True reaches every other check without a device."""
import json
import os
import subprocess
import sys
import types

import pytest
import torch

from test_abi_cpu import _sass_by_kernel

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ARG, ALIGN, NO_DEVICE = -1, -2, -3
X, GAMMA, Y, RSTD, DY, DX, DXADD, GU, H, DH, DGU = (k << 32 for k in range(1, 12))
ROWS, D, F = 300, 4096, 11008

# Argument lists in the order of include/ofk.h.  Defaults are valid problems.
FWD = dict(x=X, ldx=D, gamma=GAMMA, eps=1e-6, rows=ROWS, D=D, y=Y, ldy=D, rstd=RSTD, stream=0)
BWD = dict(dy=DY, lddy=D, x=X, ldx=D, gamma=GAMMA, rstd=RSTD, rows=ROWS, D=D, dx=DX, lddx=D, dx_add=DXADD, ldadd=D,
           stream=0)
SW_FWD = dict(gu=GU, ldgu=2 * F, rows=ROWS, F=F, h=H, ldh=F, stream=0)
SW_BWD = dict(dh=DH, lddh=F, gu=GU, ldgu=2 * F, rows=ROWS, F=F, dgu=DGU, lddgu=2 * F, stream=0)
ENTRY = {"rms_fwd": ("ofk_rmsnorm_fwd", FWD), "rms_bwd": ("ofk_rmsnorm_bwd", BWD),
         "swiglu_fwd": ("ofk_swiglu_fwd", SW_FWD), "swiglu_bwd": ("ofk_swiglu_bwd", SW_BWD)}


def _cases():
    c = {}

    def add(entry, name, want, **kw):
        fn, defaults = ENTRY[entry]
        c[f"{entry}:{name}"] = (fn, list({**defaults, **kw}.values()), want)

    for e in ("rms_fwd", "rms_bwd"):
        bwd = e == "rms_bwd"
        lds = ("lddy", "ldx", "lddx", "ldadd") if bwd else ("ldx", "ldy")

        def widths(d):
            return {k: d for k in lds}
        add(e, "valid", NO_DEVICE)
        for d in (8, 64, 5120, 8192):
            add(e, f"valid-D{d}", NO_DEVICE, D=d, **widths(d))
        add(e, "valid-rows1", NO_DEVICE, rows=1)
        add(e, "valid-strided", NO_DEVICE, **{k: D + 64 for k in lds})
        add(e, "rows0", ARG, rows=0)
        add(e, "rows-neg", ARG, rows=-1)
        add(e, "D0", ARG, D=0)
        add(e, "D12", ARG, D=12, **widths(12))
        add(e, "D8200", ARG, D=8200, **widths(8200))
        for k in lds:
            add(e, f"{k}-below-D", ARG, **{k: D - 8})
        for p in ("x", "gamma") + (("dy", "rstd", "dx") if bwd else ("y",)):
            add(e, f"{p}-null", ARG, **{p: 0})
        bases = {"x": X, "gamma": GAMMA, "y": Y, "dy": DY, "dx": DX, "dx_add": DXADD}
        for p in ("x", "gamma") + (("dy", "dx", "dx_add") if bwd else ("y",)):
            for off in (4, 8):
                add(e, f"{p}+{off}B", ALIGN, **{p: bases[p] + off})
        add(e, "rstd+2B", ALIGN, rstd=RSTD + 2)
        add(e, "valid-rstd+4B", NO_DEVICE, rstd=RSTD + 4)
        add(e, "ldx+2", ALIGN, ldx=D + 2)
        if bwd:
            add(e, "lddy+4", ALIGN, lddy=D + 4)            # bf16 rows are read 8 columns at a time
            add(e, "lddx+2", ALIGN, lddx=D + 2)
            add(e, "ldadd+2", ALIGN, ldadd=D + 2)
            add(e, "valid-no-dx_add", NO_DEVICE, dx_add=0, ldadd=0)
            add(e, "valid-dx_add-is-dx", NO_DEVICE, dx_add=DX)
        else:
            add(e, "ldy+4", ALIGN, ldy=D + 4)
            add(e, "valid-no-rstd", NO_DEVICE, rstd=0)

    for e in ("swiglu_fwd", "swiglu_bwd"):
        bwd = e == "swiglu_bwd"
        wide = ("ldgu", "lddgu") if bwd else ("ldgu",)
        narrow = ("lddh",) if bwd else ("ldh",)
        ptrs = {"gu": GU, **({"dh": DH, "dgu": DGU} if bwd else {"h": H})}
        add(e, "valid", NO_DEVICE)
        add(e, "valid-F8", NO_DEVICE, F=8, **{k: 16 for k in wide}, **{k: 8 for k in narrow})
        add(e, "valid-strided", NO_DEVICE, **{k: 2 * F + 64 for k in wide}, **{k: F + 8 for k in narrow})
        add(e, "rows0", ARG, rows=0)
        add(e, "F0", ARG, F=0)
        add(e, "F12", ARG, F=12, **{k: 24 for k in wide}, **{k: 16 for k in narrow})
        for k in wide:
            add(e, f"{k}-below-2F", ARG, **{k: 2 * F - 8})
        for k in narrow:
            add(e, f"{k}-below-F", ARG, **{k: F - 8})
        for k in wide + narrow:
            add(e, f"{k}+4", ALIGN, **{k: (2 * F if k in wide else F) + 4})
        for p, base in ptrs.items():
            add(e, f"{p}-null", ARG, **{p: 0})
            for off in (2, 8):
                add(e, f"{p}+{off}B", ALIGN, **{p: base + off})
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
    from open_flamingo_b200 import _lib
    for fn, args, _ in CASES.values():
        assert len(args) == len(_lib._SIGNATURES[fn][1]), fn


@pytest.mark.parametrize("case", sorted(CASES))
def test_rmsnorm_and_swiglu_return_codes(results, case):
    got, want = results[case], CASES[case][2]
    assert got == want, f"{case}: returned {got}, expected {want} (-3 = the check ran after the launch or not at all)"


def test_new_kernels_use_no_local_memory():
    kernels = _sass_by_kernel()
    names = [k for k in kernels if "rmsnorm_fwd_kernel" in k or "rmsnorm_bwd_kernel" in k or "swiglu_fwd_kernel" in k
             or "swiglu_bwd_kernel" in k]
    assert len(names) == 3 + 3 + 1 + 1, sorted(names)
    for k in names:
        assert not kernels[k] & {"LDL", "STL"}, f"{k}: local-memory traffic"


# ---------------------------------------------------------------------------------------------- ops wrappers
class _FakeCuda:
    """Passes L.require_cuda without a device: the wrappers' shape and dtype checks run before any library call."""

    def __enter__(self):
        from open_flamingo_b200 import _lib
        self.prev = _lib.require_cuda
        _lib.require_cuda = lambda *t: None
        return self

    def __exit__(self, *exc):
        from open_flamingo_b200 import _lib
        _lib.require_cuda = self.prev


@pytest.mark.parametrize("case", ["x-bf16", "x-1d", "x-strided-cols", "gamma-len", "gamma-f64", "out-f32",
                                  "out-short", "dy-f32", "dy-narrow", "rstd-len", "dx-bf16", "dx_add-short",
                                  "gu-odd", "gu-f32", "h-short", "dh-f32", "dh-narrow", "dgu-short"])
def test_ops_wrappers_reject_shapes_and_dtypes(case):
    from open_flamingo_b200 import ops
    b16 = torch.bfloat16
    R, Dm, Fm = 6, 64, 32
    x, g, rstd = torch.zeros(R, Dm), torch.ones(Dm), torch.ones(R)
    dy = torch.zeros(R, Dm, dtype=b16)
    gu, dh = torch.zeros(R, 2 * Fm, dtype=b16), torch.zeros(R, Fm, dtype=b16)
    calls = {
        "x-bf16": lambda: ops.rmsnorm_fwd(x.to(b16), g, 1e-6),
        "x-1d": lambda: ops.rmsnorm_fwd(x.view(-1), g, 1e-6),
        "x-strided-cols": lambda: ops.rmsnorm_fwd(torch.zeros(R, 2 * Dm)[:, ::2], g, 1e-6),
        "gamma-len": lambda: ops.rmsnorm_fwd(x, torch.ones(Dm + 8), 1e-6),
        "gamma-f64": lambda: ops.rmsnorm_fwd(x, g.double(), 1e-6),
        "out-f32": lambda: ops.rmsnorm_fwd(x, g, 1e-6, out=torch.zeros(R, Dm)),
        "out-short": lambda: ops.rmsnorm_fwd(x, g, 1e-6, out=torch.zeros(R - 1, Dm, dtype=b16)),
        "dy-f32": lambda: ops.rmsnorm_bwd(dy.float(), x, g, rstd),
        "dy-narrow": lambda: ops.rmsnorm_bwd(dy[:, :Dm - 8], x, g, rstd),
        "rstd-len": lambda: ops.rmsnorm_bwd(dy, x, g, torch.ones(R - 1)),
        "dx-bf16": lambda: ops.rmsnorm_bwd(dy, x, g, rstd, dx=torch.zeros(R, Dm, dtype=b16)),
        "dx_add-short": lambda: ops.rmsnorm_bwd(dy, x, g, rstd, dx_add=torch.zeros(R, Dm - 8)),
        "gu-odd": lambda: ops.swiglu_fwd(torch.zeros(R, 2 * Fm + 1, dtype=b16)),
        "gu-f32": lambda: ops.swiglu_fwd(gu.float()),
        "h-short": lambda: ops.swiglu_fwd(gu, out=torch.zeros(R, Fm - 8, dtype=b16)),
        "dh-f32": lambda: ops.swiglu_bwd(dh.float(), gu),
        "dh-narrow": lambda: ops.swiglu_bwd(dh[:, :Fm - 8], gu),
        "dgu-short": lambda: ops.swiglu_bwd(dh, gu, out=torch.zeros(R, 2 * Fm - 8, dtype=b16)),
    }
    with _FakeCuda(), pytest.raises(ValueError):
        calls[case]()


# ---------------------------------------------------------------------------------------------- host logic
CUDA_LIKE = types.SimpleNamespace(is_cuda=True)


def _layer(hd=128, heads=2, kv_heads=None, act="silu", attn_bias=False, mlp_bias=False, rope=None):
    from transformers import LlamaConfig
    from transformers.models.llama.modeling_llama import LlamaDecoderLayer
    kw = dict(hidden_size=hd * heads, num_attention_heads=heads, num_key_value_heads=kv_heads or heads,
              num_hidden_layers=1, intermediate_size=2 * hd * heads, vocab_size=32, hidden_act=act,
              attention_bias=attn_bias, mlp_bias=mlp_bias, attn_implementation="sdpa")
    if rope is not None:
        kw["rope_parameters"] = rope
    return LlamaDecoderLayer(LlamaConfig(**kw), 0).eval().requires_grad_(False)


def _pe(T=5, rot=128, B=1, dtype=torch.float32):
    return torch.zeros(B, T, rot, dtype=dtype), torch.zeros(B, T, rot, dtype=dtype)


def test_accelerate_returns_the_llama_block():
    from open_flamingo_b200 import lm_blocks
    layer = _layer()
    fast = lm_blocks.accelerate(layer)
    assert isinstance(fast, lm_blocks.FastLlamaBlock) and fast.block is layer
    assert fast.supported(CUDA_LIKE, _pe(), False)
    assert fast.applicable(CUDA_LIKE, _pe(), None, False, False)
    assert lm_blocks.FastLlamaBlock(_layer(hd=64)).supported(CUDA_LIKE, _pe(rot=64), False)
    assert lm_blocks.FastLlamaBlock(_layer().train()).supported(CUDA_LIKE, _pe(), False)   # no dropout configured
    llama3 = dict(rope_type="llama3", rope_theta=500000.0, factor=8.0, low_freq_factor=1.0, high_freq_factor=4.0,
                  original_max_position_embeddings=64)
    assert lm_blocks.FastLlamaBlock(_layer(rope=llama3)).supported(CUDA_LIKE, _pe(), False)


@pytest.mark.parametrize("case", ["cpu", "disabled", "output_attentions", "no_position_embeddings", "bf16_cos",
                                  "odd_rot", "rot_gt_hd", "head_dim_96", "hidden_act", "attention_bias", "mlp_bias",
                                  "gqa", "requires_grad", "dropout_training", "bad_scale", "bf16_weights"])
def test_declines(case):
    from open_flamingo_b200 import lm_blocks
    hd = 96 if case == "head_dim_96" else 128
    layer = _layer(hd=hd, heads=4 if case == "gqa" else 2, kv_heads=2 if case == "gqa" else None,
                   act="gelu" if case == "hidden_act" else "silu", attn_bias=case == "attention_bias",
                   mlp_bias=case == "mlp_bias")
    fast = lm_blocks.FastLlamaBlock(layer)
    hs, pe, oa = CUDA_LIKE, _pe(rot=hd), False
    prev = lm_blocks.ENABLED
    try:
        if case == "cpu":
            hs = torch.zeros(1, 5, 2 * hd)
        elif case == "disabled":
            lm_blocks.ENABLED = False
        elif case == "output_attentions":
            oa = True
        elif case == "no_position_embeddings":
            pe = None
        elif case == "bf16_cos":
            pe = _pe(dtype=torch.bfloat16)
        elif case == "odd_rot":
            pe = _pe(rot=21)
        elif case == "rot_gt_hd":
            pe = _pe(rot=hd + 2)
        elif case == "requires_grad":
            layer.mlp.gate_proj.weight.requires_grad_(True)   # not frozen: needs a wgrad this path lacks
        elif case == "dropout_training":
            layer.train()
            layer.self_attn.attention_dropout = 0.1
        elif case == "bad_scale":
            layer.self_attn.scaling = 64 ** -0.5
        elif case == "bf16_weights":
            layer.to(torch.bfloat16)
        assert not fast.supported(hs, pe, oa), case
        assert not fast.applicable(hs, pe, None, False, oa), case
        if case == "cpu":
            assert fast(hs, position_embeddings=pe) is None
    finally:
        lm_blocks.ENABLED = prev


def test_caches_other_than_kvcache_and_grad_mode_decline():
    from transformers import DynamicCache
    from open_flamingo_b200 import lm_blocks
    from open_flamingo_b200.kv_cache import KVCache
    fast = lm_blocks.FastLlamaBlock(_layer())
    assert not fast.applicable(CUDA_LIKE, _pe(), DynamicCache(), True, False)
    with torch.no_grad():
        assert fast.cache_layer(CUDA_LIKE, _pe(), DynamicCache(), False) is None
        assert fast.cache_layer(CUDA_LIKE, _pe(), KVCache(1), False) is not None
        assert fast.cache_layer(CUDA_LIKE, _pe(), KVCache(1), True) is None
    assert fast.cache_layer(CUDA_LIKE, _pe(), KVCache(1), False) is None   # gradient recorded


@pytest.mark.parametrize("case", ["kwarg_hidden_states", "kwarg_attentions", "config_hidden_states",
                                  "config_attentions"])
def test_declines_when_hf_records_layer_outputs(case):
    """LlamaModel collects output_hidden_states / output_attentions with hooks on the LlamaDecoderLayer and
    LlamaAttention modules, which the fast path bypasses."""
    from open_flamingo_b200 import lm_blocks
    from open_flamingo_b200.kv_cache import KVCache
    layer = _layer()
    fast = lm_blocks.FastLlamaBlock(layer)
    kw = {}
    if case.startswith("kwarg"):
        kw["output_" + case[len("kwarg_"):]] = True
    else:
        if case == "config_attentions":   # HF allows the attentions default only with eager attention
            layer.self_attn.config._attn_implementation = "eager"
        setattr(layer.self_attn.config, "output_" + case[len("config_"):], True)
    assert fast.records_outputs(kw.get("output_attentions"), kw.get("output_hidden_states"))
    assert fast(CUDA_LIKE, position_embeddings=_pe(), **kw) is None
    with torch.no_grad():   # LLaMA passes its cache as past_key_values=
        assert fast(CUDA_LIKE, position_embeddings=_pe(), past_key_values=KVCache(1), use_cache=True, **kw) is None
    if case.startswith("config"):
        assert not fast.records_outputs(False, False)


def test_float_mask_is_declined_before_any_kernel():
    from open_flamingo_b200 import lm_blocks
    B, T = 1, 5
    fast = lm_blocks.FastLlamaBlock(_layer())
    hs = types.SimpleNamespace(is_cuda=True, shape=(B, T, 256))
    assert fast(hs, attention_mask=torch.zeros(B, 1, T, T), position_embeddings=_pe(T)) is None


def test_packed_qkv_rows_are_the_per_head_interleave():
    """Packed row (h * 3 + p) * hd + j is row j of head h of part p (q, k, v): the layout ofk_rope_pack splits, as an
    index map on an exactly representable weight."""
    from open_flamingo_b200 import lm_blocks
    heads, hd, D = 4, 8, 32
    src = torch.arange(3 * D, dtype=torch.float32)[:, None].expand(3 * D, 16).contiguous()   # row index in each row
    wq, wk, wv = (src[i * D:(i + 1) * D].clone() for i in range(3))
    packed = lm_blocks._qkv16(wq, wk, wv, heads)
    assert packed.shape == (3 * D, 16) and packed.dtype == torch.bfloat16
    for h in range(heads):
        for p in range(3):
            for j in range(hd):
                assert packed[(h * 3 + p) * hd + j, 0].item() == p * D + h * hd + j
    gu = lm_blocks._gu16(wq, wk)
    assert torch.equal(gu.float(), torch.cat([wq, wk]))


def test_packed_weights_follow_in_place_edits():
    from open_flamingo_b200 import lm_blocks
    w = [torch.nn.Parameter(torch.full((16, 8), float(i)), requires_grad=False) for i in range(3)]
    first = lm_blocks._qkv16(*w, 2)
    assert lm_blocks._qkv16(*w, 2) is first
    with torch.no_grad():
        w[1].mul_(2)
    again = lm_blocks._qkv16(*w, 2)
    assert again is not first and again[8:16, 0].eq(2).all()
    # the head count is part of the layout: the same weights packed for 4 heads are another copy
    four = lm_blocks._qkv16(*w, 4)
    assert four is not again and four[4:8, 0].eq(2).all() and four[12:16, 0].eq(0).all()
