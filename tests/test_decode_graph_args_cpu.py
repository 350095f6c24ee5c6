"""CPU: the entry points of graph-replayed decoding and the fixed-capacity cache's host logic.

- ofk_attn_decode_dev and ofk_kv_append reject bad arguments with the documented error code before they touch a device
  (as in test_decode_args_cpu.py: a child process with no CUDA device and made-up device addresses; a call whose
  arguments pass validation reaches device discovery or the launch and returns OFK_ERR_CUDA, -3).
- The workspace ofk_attn_decode_workspace_bytes gives at nk_max holds the split partials of every nk <= nk_max.
- kv_cache.KVCache(capacity=...): overflow, in-place beam reorder, crop, reset, mask sizes, capacity buckets and the
  capacity generate(cache_implementation="static") asks for; HF's generate over it matches DynamicCache bitwise, with
  the batch x beams rows HF expands to."""
import json
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ARG, ALIGN, NO_DEVICE = -1, -2, -3
Q_PTR, K_PTR, V_PTR, O_PTR, MASK_PTR, SLOPES_PTR, WS_PTR, NK_PTR = (k << 32 for k in range(1, 9))
SRC_PTR, CACHE_PTR, POS_PTR, NEWM_PTR = (k << 32 for k in range(9, 13))
B, H, HD, NK_MAX = 3, 4, 128, 512
D = H * HD


def dev_args(**kw):
    a = dict(q=Q_PTR, q_bs=3 * D, k=K_PTR, v=V_PTR, kv_bs=NK_MAX * 2 * D, ldkv=2 * D, o=O_PTR, o_bs=D, batch=B, heads=H,
             head_dim=HD, nk_max=NK_MAX, nk_dev=NK_PTR, scale=HD ** -0.5, mask=MASK_PTR, mask_bs=NK_MAX,
             slopes=SLOPES_PTR, ws=WS_PTR, stream=0)
    a.update(kw)
    return list(a.values())


def append_args(**kw):
    a = dict(src=SRC_PTR, src_bs=2 * D, cache=CACHE_PTR, cache_bs=NK_MAX * 2 * D, ld=2 * D, batch=B, width=2 * D,
             capacity=NK_MAX, pos=POS_PTR, mask=MASK_PTR, mask_bs=NK_MAX, new_masked=NEWM_PTR, stream=0)
    a.update(kw)
    return list(a.values())


def _dev_cases():
    c = {
        "valid": (dev_args(), NO_DEVICE),
        "valid-hd64": (dev_args(head_dim=64), NO_DEVICE),
        "valid-no-mask-no-slopes": (dev_args(mask=0, mask_bs=3, slopes=0), NO_DEVICE),
        "valid-nk_max1": (dev_args(nk_max=1), NO_DEVICE),
        "valid-nk_dev+4B": (dev_args(nk_dev=NK_PTR + 4), NO_DEVICE),
        "hd32": (dev_args(head_dim=32), ARG),
        "hd96": (dev_args(head_dim=96), ARG),
        "hd256": (dev_args(head_dim=256), ARG),
        "batch0": (dev_args(batch=0), ARG),
        "heads0": (dev_args(heads=0), ARG),
        "batch65536": (dev_args(batch=65536), ARG),
        "nk_max0": (dev_args(nk_max=0), ARG),
        "nk_max-neg": (dev_args(nk_max=-5), ARG),
        "nk_dev-null": (dev_args(nk_dev=0), ARG),
        "nk_dev+2B": (dev_args(nk_dev=NK_PTR + 2), ALIGN),
        "q-null": (dev_args(q=0), ARG),
        "k-null": (dev_args(k=0), ARG),
        "v-null": (dev_args(v=0), ARG),
        "o-null": (dev_args(o=0), ARG),
        "ws-null": (dev_args(ws=0), ARG),
    }
    for name, ptr in (("q", Q_PTR), ("k", K_PTR), ("v", V_PTR), ("o", O_PTR), ("mask", MASK_PTR), ("ws", WS_PTR)):
        for off in (2, 8):
            c[f"{name}+{off}B"] = (dev_args(**{name: ptr + off}), ALIGN)
    for name, base in (("q_bs", 3 * D), ("kv_bs", NK_MAX * 2 * D), ("ldkv", 2 * D), ("o_bs", D), ("mask_bs", NK_MAX)):
        for off in (1, 4):
            c[f"{name}+{off}"] = (dev_args(**{name: base + off}), ALIGN)
    return c


def _append_cases():
    c = {
        "valid": (append_args(), NO_DEVICE),
        "valid-no-mask": (append_args(mask=0, mask_bs=0, new_masked=0), NO_DEVICE),
        "valid-no-new-masked": (append_args(new_masked=0), NO_DEVICE),
        "valid-capacity1": (append_args(capacity=1, mask_bs=8), NO_DEVICE),
        "valid-odd-mask": (append_args(mask=MASK_PTR + 3, mask_bs=NK_MAX + 1), NO_DEVICE),   # bytes: no alignment
        "src-null": (append_args(src=0), ARG),
        "cache-null": (append_args(cache=0), ARG),
        "pos-null": (append_args(pos=0), ARG),
        "batch0": (append_args(batch=0), ARG),
        "batch65536": (append_args(batch=65536), ARG),
        "width0": (append_args(width=0), ARG),
        "capacity0": (append_args(capacity=0), ARG),
        "capacity-neg": (append_args(capacity=-1), ARG),
        "ld<width": (append_args(ld=D), ARG),
        "mask_bs<capacity": (append_args(mask_bs=NK_MAX - 1), ARG),
        "pos+2B": (append_args(pos=POS_PTR + 2), ALIGN),
        "width+4": (append_args(width=2 * D - 4, ld=2 * D), ALIGN),
    }
    for name, ptr in (("src", SRC_PTR), ("cache", CACHE_PTR)):
        for off in (2, 8):
            c[f"{name}+{off}B"] = (append_args(**{name: ptr + off}), ALIGN)
    for name, base in (("src_bs", 2 * D), ("cache_bs", NK_MAX * 2 * D), ("ld", 2 * D)):
        for off in (1, 4):
            c[f"{name}+{off}"] = (append_args(**{name: base + off}), ALIGN)
    return c


DEV_CASES = _dev_cases()
APPEND_CASES = _append_cases()

CHILD = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
from open_flamingo_b200 import _lib
cases = json.load(sys.stdin)
lib = _lib.lib()
res = {"dev": {n: lib.ofk_attn_decode_dev(*args) for n, (args, _) in cases["dev"].items()},
       "append": {n: lib.ofk_kv_append(*args) for n, (args, _) in cases["append"].items()},
       "ws": {str(k): lib.ofk_attn_decode_workspace_bytes(*k) for k in map(tuple, cases["ws"])}}
print(json.dumps(res))
"""

WS_POINTS = [(b, h, hd, n) for b, h in ((1, 2), (1, 16), (3, 32), (24, 16)) for hd in (64, 128)
             for n in (1, 63, 64, 65, 300, 2049, 4097, 8192)]


@pytest.fixture(scope="module")
def results():
    import __graft_entry__ as g
    g.build()
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", CHILD, ROOT]
    r = subprocess.run(cmd, input=json.dumps({"dev": DEV_CASES, "append": APPEND_CASES, "ws": WS_POINTS}),
                       capture_output=True, text=True, env=env, timeout=600)
    assert r.returncode == 0, r.stderr
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("case", sorted(DEV_CASES))
def test_decode_dev_return_code(results, case):
    got, want = results["dev"][case], DEV_CASES[case][1]
    assert got == want, f"{case}: returned {got}, expected {want} (-3 = the check ran after device discovery or not at all)"


@pytest.mark.parametrize("case", sorted(APPEND_CASES))
def test_kv_append_return_code(results, case):
    got, want = results["append"][case], APPEND_CASES[case][1]
    assert got == want, f"{case}: returned {got}, expected {want} (-3 = the check ran after the launch or not at all)"


def _split_count(bh, nk, sms):
    """attention_decode.cu's split_count, restated."""
    s = min(64, (nk + 63) // 64)
    s = max(1, min(s, (2 * sms + bh - 1) // bh))
    c = -(-nk // s)
    c = -(-c // 32) * 32
    return -(-nk // c)


def _grid_splits(bh, nk_max, sms):
    """attention_decode.cu's max_split_count: the split count before the chunk rounding at nk_max."""
    return max(1, min(64, (nk_max + 63) // 64, (2 * sms + bh - 1) // bh))


@pytest.mark.parametrize("sms", [1, 66, 132, 144])
def test_workspace_at_nk_max_bounds_every_device_plan(results, sms):
    """The split plan at any nk <= nk_max fits both the grid and the workspace sized at nk_max.  The rounded split
    count itself is not monotone in nk (at B*H = 2 it is 64 at nk = 4096 and 43 at 4097), so the grid is sized by the
    count before rounding, which is."""
    dips = 0
    for b, h, hd, nk_max in WS_POINTS:
        ws = results["ws"][str((b, h, hd, nk_max))]
        grid = _grid_splits(b * h, nk_max, sms)
        assert ws >= b * h * grid * (hd + 2) * 4, (b, h, hd, nk_max, sms, ws)
        prev = 0
        for nk in range(1, nk_max + 1):
            s = _split_count(b * h, nk, sms)
            assert s <= grid, (b, h, nk, nk_max, sms)
            dips += s < prev
            prev = s
    assert sms != 66 or dips > 0   # the case the bound exists for does occur


# --------------------------------------------------------------------------------------------- fixed-capacity cache
from open_flamingo_b200.kv_cache import CAPACITY_BUCKET, KVCache, bucket_capacity  # noqa: E402


def test_capacity_buckets_and_static_plan():
    from open_flamingo_b200.decode_graph import static_cache_capacity
    assert CAPACITY_BUCKET == 64
    assert [bucket_capacity(n) for n in (1, 63, 64, 65, 200, 256, 257)] == [64, 64, 64, 128, 256, 256, 320]
    with pytest.raises(ValueError):
        bucket_capacity(0)
    assert KVCache(2, capacity=100).capacity == 128
    assert KVCache(2).capacity is None
    # rows = prompt + new tokens (or max_length, which counts the prompt), bucketed
    assert static_cache_capacity(24, max_new_tokens=8) == 64
    assert static_cache_capacity(200, max_new_tokens=20) == 256
    assert static_cache_capacity(200, max_new_tokens=64) == 320
    assert static_cache_capacity(30, max_length=80) == 128
    assert static_cache_capacity(30, max_new_tokens=8, max_length=500) == 64   # max_new_tokens wins, as in HF
    with pytest.raises(ValueError):
        static_cache_capacity(10)


def _allocate(cache, batch, heads, hd):
    for layer in cache.layers:
        layer.init_storage(batch, heads, hd, torch.float32, "cpu")
    cache.ensure_key_mask(batch, "cpu")


def _filled(capacity=64, batch=3, heads=2, hd=4, length=5):
    cache = KVCache(2, capacity=capacity)
    _allocate(cache, batch, heads, hd)
    for i, layer in enumerate(cache.layers):
        layer.buf.copy_(torch.arange(layer.buf.numel(), dtype=torch.float32).view_as(layer.buf) + 1000 * i)
        layer.length = length
    cache.key_mask.copy_(torch.randint(0, 2, cache.key_mask.shape, generator=torch.Generator().manual_seed(0)))
    return cache


def test_allocation_overflow_and_host_length():
    cache = _filled(capacity=50, length=0)
    assert cache.capacity == 64
    assert all(tuple(layer.buf.shape) == (3, 64, 16) for layer in cache.layers)
    assert tuple(cache.key_mask.shape) == (3, 64)
    ptrs = [layer.buf.data_ptr() for layer in cache.layers]
    layer = cache.layers[0]
    layer.length = 60
    assert layer.reserve(4) is layer.buf and layer.buf.data_ptr() == ptrs[0]
    with pytest.raises(ValueError):
        layer.reserve(5)
    for lay in cache.layers:
        lay.length = 63
    cache.check_room(1)
    with pytest.raises(ValueError):
        cache.check_room(2)
    assert [lay.buf.data_ptr() for lay in cache.layers] == ptrs
    assert cache.get_mask_sizes(1, 0) == (64, 0) and cache.get_mask_sizes(3, 1) == (66, 0)
    cache.crop(40)
    assert cache.get_seq_length() == 40 and cache.get_mask_sizes(2, 0) == (42, 0)
    cache.crop(-10)
    assert cache.get_seq_length() == 30
    w = cache.eager_writes
    cache.crop(35)
    assert cache.eager_writes == w + 1, "a crop ends a run of replayed steps"
    cache.key_mask_known = False
    cache.reset()
    assert cache.eager_writes == w + 2
    assert cache.get_seq_length() == 0 and cache.get_mask_sizes(4, 0) == (4, 0) and cache.key_mask_known
    assert [lay.buf.data_ptr() for lay in cache.layers] == ptrs


def test_reorder_cache_permutes_rows_in_place():
    cache = _filled(length=5)
    before = [layer.buf.clone() for layer in cache.layers]
    mask_before = cache.key_mask.clone()
    ptrs = [layer.buf.data_ptr() for layer in cache.layers] + [cache.key_mask.data_ptr()]
    idx = torch.tensor([2, 0, 0])
    cache.reorder_cache(idx)
    assert [layer.buf.data_ptr() for layer in cache.layers] + [cache.key_mask.data_ptr()] == ptrs
    for layer, b in zip(cache.layers, before):
        assert torch.equal(layer.buf[:, :5], b[idx, :5])
        assert torch.equal(layer.buf[:, 5:], b[:, 5:])     # rows past the length are not part of the state
    assert torch.equal(cache.key_mask, mask_before[idx])


def test_key_padding_from_2d_mask():
    cache = KVCache(1, capacity=16)
    _allocate(cache, 2, 1, 8)
    att = torch.tensor([[0, 0, 1, 1], [1, 1, 1, 1]])
    cache.note_key_padding(att, 2, 4, "cpu")
    assert cache.key_mask[:, :4].tolist() == [[1, 1, 0, 0], [0, 0, 0, 0]]
    cache.layers[0].length = 4
    cache.note_key_padding(torch.cat([att, torch.tensor([[1], [0]])], 1), 2, 1, "cpu")
    cache.note_key_padding(None, 2, 1, "cpu")   # same row again: no padding
    assert cache.key_mask[:, 4].tolist() == [0, 0]
    assert cache.key_mask_known
    cache.note_key_padding(torch.ones(2, 1, 1, 5, dtype=torch.bool), 2, 1, "cpu")
    assert not cache.key_mask_known


@pytest.fixture(scope="module")
def lm():
    from transformers import MptConfig, MptForCausalLM
    torch.manual_seed(0)
    cfg = MptConfig(d_model=64, n_heads=4, n_layers=2, vocab_size=97, max_seq_len=256, expansion_ratio=2)
    model = MptForCausalLM(cfg).eval()
    with torch.no_grad():
        for p in model.parameters():
            p.normal_(0.0, 0.5 if p.dim() > 1 else 0.1).add_(1.0 if p.dim() == 1 else 0.0)
    return model


@pytest.mark.parametrize("mode", ["greedy", "beam"])
def test_fixed_capacity_generate_matches_dynamic_cache_bitwise(lm, mode):
    from transformers import DynamicCache
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(3, 97, (3, 11), generator=g)
    att = torch.ones_like(ids)
    att[0, :4] = 0
    ids = ids.masked_fill(att == 0, 0)
    kw = dict(do_sample=False) if mode == "greedy" else dict(do_sample=False, num_beams=3, length_penalty=0.0)

    def run(cache):
        with torch.no_grad():
            return lm.generate(ids, attention_mask=att, past_key_values=cache, use_cache=True, output_scores=True,
                               return_dict_in_generate=True, pad_token_id=0, eos_token_id=None, max_new_tokens=12, **kw)
    cache = KVCache(2, capacity=11 + 12)
    got, ref = run(cache), run(DynamicCache())
    assert torch.equal(got.sequences, ref.sequences)
    assert all(torch.equal(x, y) for x, y in zip(got.scores, ref.scores))
    assert cache.layers[0].buf.shape[1] == 64
    assert cache.layers[0].buf.shape[0] == 3 * kw.get("num_beams", 1)   # HF's expanded batch, fixed at the prefill
    with pytest.raises(ValueError), torch.no_grad():   # 11 + 60 rows do not fit 64
        lm.generate(ids, attention_mask=att, past_key_values=KVCache(2, capacity=23), use_cache=True, pad_token_id=0,
                    eos_token_id=None, max_new_tokens=60, min_new_tokens=60, **kw)
