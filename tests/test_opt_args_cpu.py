"""CPU: the OPT block's entry points (ofk_dropout_resid_fwd / _bwd, ofk_relu_bf16, ofk_relu_bwd_bf16, ofk_scale_bf16)
reject bad arguments with the documented error code before they touch a device; their ops wrappers raise ValueError on
shapes and dtypes; the new kernels keep everything in registers; and the host logic of lm_blocks.FastOptBlock --
accelerate() returns it for an OPTDecoderLayer, it declines every call the kernels do not evaluate, and its packed QKV
weight and bias have the per-head (q | k | v) order the packing kernel reads.

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
X, BR, OUT, SO, DOUT, DBR, Z, H, DH, DZ = (k << 32 for k in range(1, 11))
ROWS, C = 300, 2560

# Argument lists in the order of include/ofk.h.  Defaults are valid problems.
DFWD = dict(x=X, ldx=C, branch=BR, ldb=C, rows=ROWS, cols=C, p=0.1, seed_offset=SO, out=OUT, ldo=C, stream=0)
DBWD = dict(dout=DOUT, ldd=C, rows=ROWS, cols=C, p=0.1, seed_offset=SO, dbranch=DBR, lddb=C, stream=0)
RELU = dict(z=Z, h=H, n=ROWS * C, stream=0)
RELU_BWD = dict(dh=DH, h=H, dz=DZ, n=ROWS * C, stream=0)
SCALE = dict(x=X, ldx=3 * C, rows=ROWS, cols=C, s=0.125, y=OUT, ldy=C, stream=0)
ENTRY = {"drop_fwd": ("ofk_dropout_resid_fwd", DFWD), "drop_bwd": ("ofk_dropout_resid_bwd", DBWD),
         "relu": ("ofk_relu_bf16", RELU), "relu_bwd": ("ofk_relu_bwd_bf16", RELU_BWD),
         "scale": ("ofk_scale_bf16", SCALE)}


def _cases():
    c = {}

    def add(entry, name, want, **kw):
        fn, defaults = ENTRY[entry]
        c[f"{entry}:{name}"] = (fn, list({**defaults, **kw}.values()), want)

    for e in ("drop_fwd", "drop_bwd"):
        fwd = e == "drop_fwd"
        f32_lds = ("ldx", "ldo") if fwd else ("ldd",)
        bf_lds = ("ldb",) if fwd else ("lddb",)
        ptrs = {"x": X, "branch": BR, "out": OUT} if fwd else {"dout": DOUT, "dbranch": DBR}
        add(e, "valid", NO_DEVICE)
        add(e, "valid-p0-no-seed", NO_DEVICE, p=0.0, seed_offset=0)
        add(e, "valid-p0.999", NO_DEVICE, p=0.999)
        add(e, "valid-cols8", NO_DEVICE, cols=8, **{k: 8 for k in f32_lds + bf_lds})
        add(e, "valid-strided", NO_DEVICE, **{k: C + 64 for k in f32_lds + bf_lds})
        add(e, "p-neg", ARG, p=-0.1)
        add(e, "p1", ARG, p=1.0)
        add(e, "p-nan", ARG, p=float("nan"))
        add(e, "no-seed", ARG, seed_offset=0)
        add(e, "rows0", ARG, rows=0)
        add(e, "cols0", ARG, cols=0)
        add(e, "cols12", ARG, cols=12, **{k: 16 for k in f32_lds + bf_lds})
        for k in f32_lds + bf_lds:
            add(e, f"{k}-below-cols", ARG, **{k: C - 8})
        for k in f32_lds:
            add(e, f"{k}+2", ALIGN, **{k: C + 2})
        for k in bf_lds:
            add(e, f"{k}+4", ALIGN, **{k: C + 4})
        add(e, "seed+4B", ALIGN, seed_offset=SO + 4)
        for p, base in ptrs.items():
            add(e, f"{p}-null", ARG, **{p: 0})
            for off in (4, 8):
                add(e, f"{p}+{off}B", ALIGN, **{p: base + off})
        # an argument error wins over an alignment error
        add(e, "p1-and-misaligned", ARG, p=1.0, **{list(ptrs)[0]: list(ptrs.values())[0] + 4})
        if fwd:
            add(e, "valid-out-is-x", NO_DEVICE, out=X)

    for e, ptrs in (("relu", {"z": Z, "h": H}), ("relu_bwd", {"dh": DH, "h": H, "dz": DZ})):
        add(e, "valid", NO_DEVICE)
        add(e, "valid-n0", 0, n=0)
        add(e, "n12", ARG, n=12)
        for p, base in ptrs.items():
            add(e, f"{p}-null", ARG, **{p: 0})
            add(e, f"{p}+8B", ALIGN, **{p: base + 8})
        add(e, "n12-and-misaligned", ARG, n=12, h=H + 8)
    add("relu", "valid-in-place", NO_DEVICE, h=Z)
    add("relu_bwd", "valid-in-place", NO_DEVICE, dz=DH)

    add("scale", "valid", NO_DEVICE)
    add("scale", "valid-in-place", NO_DEVICE, y=X, ldy=3 * C)
    add("scale", "rows0", ARG, rows=0)
    add("scale", "cols0", ARG, cols=0)
    add("scale", "cols12", ARG, cols=12)
    add("scale", "ldx-below-cols", ARG, ldx=C - 8)
    add("scale", "ldy-below-cols", ARG, ldy=C - 8)
    add("scale", "ldx+4", ALIGN, ldx=3 * C + 4)
    add("scale", "ldy+4", ALIGN, ldy=C + 4)
    for p, base in (("x", X), ("y", OUT)):
        add("scale", f"{p}-null", ARG, **{p: 0})
        add("scale", f"{p}+8B", ALIGN, **{p: base + 8})
    add("scale", "cols12-and-misaligned", ARG, cols=12, x=X + 8)
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
def test_opt_kernels_return_codes(results, case):
    got, want = results[case], CASES[case][2]
    assert got == want, f"{case}: returned {got}, expected {want} (-3 = the check ran after the launch or not at all)"


def test_new_kernels_use_no_local_memory():
    kernels = _sass_by_kernel()
    pats = ("dropout_resid_fwd_kernel", "dropout_resid_bwd_kernel", "relu_bf16_kernel", "relu_bwd_bf16_kernel",
            "scale_bf16_kernel")
    names = [k for k in kernels if any(p in k for p in pats)]
    assert len(names) == len(pats), sorted(names)
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


@pytest.mark.parametrize("case", ["x-bf16", "branch-f32", "branch-shape", "no-seed", "seed-int32", "seed-len",
                                  "out-bf16", "dout-bf16", "dbranch-f32", "z-f32", "h-len", "dh-strided", "scale-f32",
                                  "scale-1d", "scale-out-shape", "scale-ragged-batch"])
def test_ops_wrappers_reject_shapes_and_dtypes(case):
    from open_flamingo_b200 import ops
    b16 = torch.bfloat16
    R, Cm = 6, 64
    x, br = torch.zeros(R, Cm), torch.zeros(R, Cm, dtype=b16)
    so = torch.zeros(2, dtype=torch.int64)
    calls = {
        "x-bf16": lambda: ops.dropout_resid_fwd(x.to(b16), br, 0.1, so),
        "branch-f32": lambda: ops.dropout_resid_fwd(x, br.float(), 0.1, so),
        "branch-shape": lambda: ops.dropout_resid_fwd(x, br[:, :Cm - 8], 0.1, so),
        "no-seed": lambda: ops.dropout_resid_fwd(x, br, 0.1, None),
        "seed-int32": lambda: ops.dropout_resid_fwd(x, br, 0.1, so.int()),
        "seed-len": lambda: ops.dropout_resid_bwd(x, 0.1, torch.zeros(3, dtype=torch.int64)),
        "out-bf16": lambda: ops.dropout_resid_fwd(x, br, 0.1, so, out=br),
        "dout-bf16": lambda: ops.dropout_resid_bwd(br, 0.1, so),
        "dbranch-f32": lambda: ops.dropout_resid_bwd(x, 0.1, so, out=x),
        "z-f32": lambda: ops.relu_bf16(x),
        "h-len": lambda: ops.relu_bwd_bf16(br, br[:, :Cm - 8]),
        "dh-strided": lambda: ops.relu_bwd_bf16(torch.zeros(R, 2 * Cm, dtype=b16)[:, ::2], br),
        "scale-f32": lambda: ops.scale_bf16(x, 0.5),
        "scale-1d": lambda: ops.scale_bf16(br.view(-1), 0.5),
        "scale-out-shape": lambda: ops.scale_bf16(br, 0.5, out=br[:R - 1]),
        "scale-ragged-batch": lambda: ops.scale_bf16(torch.zeros(2, 4, 2 * Cm, dtype=b16)[:, :3, :Cm], 0.5),
    }
    with _FakeCuda(), pytest.raises(ValueError):
        calls[case]()


# ---------------------------------------------------------------------------------------------- host logic
CUDA_LIKE = types.SimpleNamespace(is_cuda=True)


def _layer(hd=64, heads=2, ffn=None, **kw):
    from transformers import OPTConfig
    from transformers.models.opt.modeling_opt import OPTDecoderLayer
    D = hd * heads
    args = dict(hidden_size=D, num_attention_heads=heads, num_hidden_layers=1, ffn_dim=ffn or 4 * D, vocab_size=32,
                word_embed_proj_dim=D, dropout=0.1, attention_dropout=0.0, attn_implementation="sdpa")
    args.update(kw)
    return OPTDecoderLayer(OPTConfig(**args), 0).eval().requires_grad_(False)


def test_accelerate_returns_the_opt_block():
    from open_flamingo_b200 import lm_blocks
    layer = _layer()
    fast = lm_blocks.accelerate(layer)
    assert isinstance(fast, lm_blocks.FastOptBlock) and fast.block is layer
    for hd in (64, 80, 128):
        f = lm_blocks.FastOptBlock(_layer(hd=hd))
        assert f.supported(CUDA_LIKE, False) and f.applicable(CUDA_LIKE, None, False, False), hd
    assert lm_blocks.FastOptBlock(_layer(hd=128, heads=32)).supported(CUDA_LIKE, False)   # D 4096 (OPT-6.7B)
    train = lm_blocks.FastOptBlock(_layer().train())     # residual dropout runs on the kernels
    assert train.supported(CUDA_LIKE, False) and train.dropout_p() == pytest.approx(0.1)
    assert lm_blocks.FastOptBlock(_layer()).dropout_p() == 0.0   # eval: no dropout


@pytest.mark.parametrize("case", ["cpu", "disabled", "record_outputs", "post_ln", "gelu", "no_bias", "non_affine_ln",
                                  "head_dim_96", "D_5120", "ffn_not_16", "attention_dropout_training",
                                  "requires_grad", "bf16_weights", "bad_scale"])
def test_declines(case):
    from open_flamingo_b200 import lm_blocks
    kw = {"post_ln": dict(do_layer_norm_before=False), "gelu": dict(activation_function="gelu"),
          "no_bias": dict(enable_bias=False), "non_affine_ln": dict(layer_norm_elementwise_affine=False),
          "head_dim_96": dict(hd=96), "D_5120": dict(hd=128, heads=40), "ffn_not_16": dict(ffn=520),
          "attention_dropout_training": dict(attention_dropout=0.1)}.get(case, {})
    layer = _layer(**kw)
    fast = lm_blocks.FastOptBlock(layer)
    hs, rec = CUDA_LIKE, False
    prev = lm_blocks.ENABLED
    try:
        if case == "cpu":
            hs = torch.zeros(1, 5, 128)
        elif case == "disabled":
            lm_blocks.ENABLED = False
        elif case == "record_outputs":
            rec = True
        elif case == "attention_dropout_training":
            layer.train()
        elif case == "requires_grad":
            layer.fc1.weight.requires_grad_(True)
        elif case == "bf16_weights":
            layer.to(torch.bfloat16)
        elif case == "bad_scale":
            layer.self_attn.scaling = 0.1
        assert not fast.supported(hs, rec), case
        assert not fast.applicable(hs, None, False, rec), case
        if case == "cpu":
            assert fast(hs) is None
    finally:
        lm_blocks.ENABLED = prev
    if case == "attention_dropout_training":   # attention dropout is only applied in training
        assert fast.supported(CUDA_LIKE, False) is False and lm_blocks.FastOptBlock(layer.eval()).supported(CUDA_LIKE,
                                                                                                          False)


def test_caches_other_than_kvcache_and_grad_mode_decline():
    from transformers import DynamicCache
    from open_flamingo_b200 import lm_blocks
    from open_flamingo_b200.kv_cache import KVCache
    fast = lm_blocks.FastOptBlock(_layer())
    assert not fast.applicable(CUDA_LIKE, DynamicCache(), True, False)
    with torch.no_grad():
        assert fast.cache_layer(CUDA_LIKE, DynamicCache(), False) is None
        assert fast.cache_layer(CUDA_LIKE, KVCache(1), False) is not None
        assert fast.cache_layer(CUDA_LIKE, KVCache(1), True) is None
    assert fast.cache_layer(CUDA_LIKE, KVCache(1), False) is None   # gradient recorded
    assert fast(CUDA_LIKE, past_key_values=DynamicCache(), use_cache=True) is None


@pytest.mark.parametrize("case", ["kwarg_hidden_states", "kwarg_attentions", "config_hidden_states",
                                  "config_attentions"])
def test_declines_when_hf_records_layer_outputs(case):
    """OPTDecoder collects output_hidden_states / output_attentions with hooks on the OPTDecoderLayer and
    OPTAttention modules, which the fast path bypasses."""
    from open_flamingo_b200 import lm_blocks
    from open_flamingo_b200.kv_cache import KVCache
    layer = _layer()
    fast = lm_blocks.FastOptBlock(layer)
    kw = {}
    if case.startswith("kwarg"):
        kw["output_" + case[len("kwarg_"):]] = True
    else:
        if case == "config_attentions":
            layer.self_attn.config._attn_implementation = "eager"
        setattr(layer.self_attn.config, "output_" + case[len("config_"):], True)
    assert fast.records_outputs(kw.get("output_attentions"), kw.get("output_hidden_states"))
    assert fast(CUDA_LIKE, **kw) is None
    with torch.no_grad():
        assert fast(CUDA_LIKE, past_key_values=KVCache(1), use_cache=True, **kw) is None
    if case.startswith("config"):
        assert not fast.records_outputs(False, False)


def test_float_mask_is_declined_before_any_kernel():
    from open_flamingo_b200 import lm_blocks
    B, T = 1, 5
    fast = lm_blocks.FastOptBlock(_layer())
    hs = types.SimpleNamespace(is_cuda=True, shape=(B, T, 128))
    assert fast(hs, attention_mask=torch.zeros(B, 1, T, T)) is None


def test_packed_qkv_weight_and_bias_are_the_per_head_interleave():
    """Packed row (h * 3 + p) * hd + j is row j of head h of part p (q, k, v), and the packed bias follows the same
    map: index maps on exactly representable values."""
    from open_flamingo_b200 import lm_blocks
    heads, hd, D = 4, 8, 32
    src = torch.arange(3 * D, dtype=torch.float32)[:, None].expand(3 * D, 16).contiguous()
    wq, wk, wv = (src[i * D:(i + 1) * D].clone() for i in range(3))
    bq, bk, bv = (torch.arange(D, dtype=torch.float32) + i * D for i in range(3))
    packed = lm_blocks._qkv16(wq, wk, wv, heads)
    bias = lm_blocks._qkv_bias(bq, bk, bv, heads)
    assert bias.shape == (3 * D,) and bias.dtype == torch.float32 and bias.is_contiguous()
    for h in range(heads):
        for p in range(3):
            for j in range(hd):
                r = (h * 3 + p) * hd + j
                assert packed[r, 0].item() == p * D + h * hd + j
                assert bias[r].item() == p * D + h * hd + j


def test_packed_bias_follows_in_place_edits_and_keys_on_the_head_count():
    from open_flamingo_b200 import lm_blocks
    b = [torch.nn.Parameter(torch.full((16,), float(i)), requires_grad=False) for i in range(3)]
    first = lm_blocks._qkv_bias(*b, 2)
    assert lm_blocks._qkv_bias(*b, 2) is first
    with torch.no_grad():
        b[1].add_(5)
    again = lm_blocks._qkv_bias(*b, 2)
    assert again is not first and again[8:16].eq(6).all()
    four = lm_blocks._qkv_bias(*b, 4)
    assert four is not again and four[4:8].eq(6).all() and four[12:16].eq(0).all()
    # the weight and the bias of the same parameters are separate entries
    w = [torch.nn.Parameter(torch.full((16, 8), float(i)), requires_grad=False) for i in range(3)]
    assert lm_blocks._qkv16(*w, 2).dtype == torch.bfloat16


def test_make_kv_cache_covers_an_opt_lm():
    """make_kv_cache returns a KVCache when every decoder block of the LM is an OPT block (the checks before it need
    CUDA weights, so the rule is read from FlamingoLayer's recognition here)."""
    from open_flamingo_b200.src.flamingo_lm import FlamingoLayer
    layer = FlamingoLayer(None, _layer())
    from open_flamingo_b200 import lm_blocks
    assert isinstance(layer._fast_block, lm_blocks.FastOptBlock)
