"""CPU: the LaION vision towers (open_clip ViT-H-14, ViT-g-14, ViT-bigG-14; head widths 80, 88, 104) are built by the
factory, from its own config table and through the open_clip branch; VisionTransformer's one head-width rule accepts
64 and the multiples of 8 in (64, 128] and rejects everything else before any kernel is reached; a forward on CPU
tensors still raises (there is no CPU path); and ops.rope_pack hands ofk_rope_pack the column-block (q | k | v) source
of an in_proj output with the right pointers and strides."""
import sys
import types

import pytest
import torch

from open_flamingo_b200 import _lib as L
from open_flamingo_b200 import ops
from open_flamingo_b200.src import factory
from open_flamingo_b200.src.vit import VisionTransformer
from open_flamingo_b200 import testing as T

# name: (width, layers, heads, MLP hidden, output_dim, testing preset)
LAION = {
    "ViT-H-14": (1280, 32, 16, 5120, 1024, T.VIT_H14),
    "ViT-g-14": (1408, 40, 16, 6144, 1024, T.VIT_G14),
    "ViT-bigG-14": (1664, 48, 16, 8192, 1280, T.VIT_BIGG14),
}


@pytest.fixture
def no_library(monkeypatch):
    """Any attempt to load libofk.so fails the test: the checks under test come before every kernel call."""
    def refuse():
        raise AssertionError("libofk was reached")
    monkeypatch.setattr(L, "lib", refuse)


@pytest.mark.parametrize("name", sorted(LAION))
def test_builtin_laion_tower_dims(name, no_library):
    width, layers, heads, hidden, out_dim, preset = LAION[name]
    with torch.device("meta"):
        wrapped, _, vis_dim = factory._build_vision(name, None, None)
    vit = wrapped.visual
    assert (vit.width, len(vit.transformer.resblocks), vit.heads) == (width, layers, heads)
    assert width // heads in (80, 88, 104)
    blk = vit.transformer.resblocks[0]
    assert blk.mlp.c_fc.out_features == hidden and blk.mlp.c_proj.in_features == hidden
    assert tuple(blk.attn.in_proj_weight.shape) == (3 * width, width)
    assert vit.output_dim == out_dim and tuple(vit.proj.shape) == (width, out_dim)
    assert vit.quick_gelu is False
    assert vis_dim == width
    assert vit.positional_embedding.shape[0] == 16 * 16 + 1
    with torch.device("meta"):
        from_preset = VisionTransformer(**preset)
    assert {k: v.shape for k, v in from_preset.state_dict().items()} == \
        {k: v.shape for k, v in vit.state_dict().items()}


def test_builtin_openai_towers_keep_quick_gelu(no_library):
    with torch.device("meta"):
        for name in ("ViT-L-14", "ViT-L-14-336", "ViT-B-16", "ViT-B-32"):
            assert factory._build_vision(name, None, None)[0].visual.quick_gelu is True


def _fake_open_clip(vision_cfg, visual):
    calls = []
    mod = types.ModuleType("open_clip")

    def create_model_and_transforms(name, pretrained=None, cache_dir=None):
        calls.append((name, pretrained, cache_dir))
        return types.SimpleNamespace(visual=visual), None, "image-processor"

    mod.create_model_and_transforms = create_model_and_transforms
    mod.get_model_config = lambda name: {"embed_dim": visual.output_dim, "vision_cfg": dict(vision_cfg)}
    return mod, calls


@pytest.mark.parametrize("pretrained,quick", [("laion2b_s32b_b79k", False), ("openai", True)])
def test_open_clip_branch_loads_a_head_width_80_tower(monkeypatch, no_library, pretrained, quick):
    cfg = dict(image_size=56, patch_size=14, width=160, layers=2, head_width=80, mlp_ratio=4.0)
    torch.manual_seed(0)
    theirs = VisionTransformer(image_size=56, patch_size=14, width=160, layers=2, heads=2, output_dim=48)
    with torch.no_grad():
        for p in theirs.parameters():
            p.normal_()
    mod, calls = _fake_open_clip(cfg, theirs)
    monkeypatch.setitem(sys.modules, "open_clip", mod)
    wrapped, proc, vis_dim = factory._build_vision("ViT-tiny-14", pretrained, "/cache")
    ours = wrapped.visual
    assert calls == [("ViT-tiny-14", pretrained, "/cache")]
    assert proc == "image-processor" and vis_dim == 160
    assert ours.heads == cfg["width"] // cfg["head_width"] == 2
    assert ours.output_dim == 48 and ours.quick_gelu is quick
    mine, ref = ours.state_dict(), theirs.state_dict()
    assert mine.keys() == ref.keys()
    for k in ref:
        assert torch.equal(mine[k], ref[k]), k


def test_open_clip_branch_rejects_an_unsupported_head_width(monkeypatch, no_library):
    # 192 / 48 = 4 heads of 48: no attention core runs them, padded or not
    cfg = dict(image_size=56, patch_size=14, width=192, layers=1, head_width=48, mlp_ratio=4.0)
    theirs = types.SimpleNamespace(output_dim=32, proj=torch.zeros(192, 32))
    mod, _ = _fake_open_clip(cfg, theirs)
    monkeypatch.setitem(sys.modules, "open_clip", mod)
    with pytest.raises(ValueError, match="head widths 64"):
        factory._build_vision("ViT-odd", "laion", None)


@pytest.mark.parametrize("width,heads", [(1000, 16), (64, 2), (120, 2), (200, 2), (272, 2), (64, 0)],
                         ids=["indivisible", "hd32", "hd60", "hd100", "hd136", "no-heads"])
def test_rejected_head_widths(width, heads, no_library):
    with pytest.raises(ValueError, match="head widths 64"):
        VisionTransformer(image_size=28, patch_size=14, width=width, layers=1, heads=heads, output_dim=16)


@pytest.mark.parametrize("hd", [64, 72, 80, 88, 96, 104, 112, 120, 128])
def test_accepted_head_widths(hd, no_library):
    with torch.device("meta"):
        vit = VisionTransformer(image_size=28, patch_size=14, width=2 * hd, layers=1, heads=2, output_dim=16)
    assert vit.width // vit.heads == hd


@pytest.mark.parametrize("hd", [64, 80])
def test_forward_on_cpu_raises(hd):
    vit = VisionTransformer(image_size=28, patch_size=14, width=2 * hd, layers=1, heads=2, output_dim=16,
                            output_tokens=True)
    with pytest.raises(RuntimeError, match="CUDA"):
        vit(torch.zeros(1, 3, 28, 28))


class _RecordingLib:
    def __init__(self):
        self.args = None

    def ofk_rope_pack(self, *args):
        self.args = args
        return 0


def _pack_args(monkeypatch, src, heads, hd, **kw):
    rec = _RecordingLib()
    monkeypatch.setattr(L, "require_cuda", lambda *t: None)
    monkeypatch.setattr(L, "lib", lambda: rec)
    monkeypatch.setattr(L, "stream_ptr", lambda: 0)
    q, k, v = ops.rope_pack(src, heads, hd, q_width=128, kv_width=128, **kw)
    return rec.args, (q, k, v)


@pytest.mark.parametrize("blocks", [False, True])
def test_rope_pack_source_layouts(monkeypatch, blocks):
    B, T_, heads, hd = 2, 5, 3, 80
    D = heads * hd
    src = torch.zeros(B, T_, 3 * D, dtype=torch.bfloat16)
    args, (q, k, v) = _pack_args(monkeypatch, src, heads, hd, blocks=blocks)
    base, es = src.data_ptr(), src.element_size()
    part = D if blocks else hd
    assert args[:3] == (base, base + part * es, base + 2 * part * es)
    assert args[3:6] == (T_ * 3 * D, 3 * D, hd if blocks else 3 * hd)   # batch stride, row stride, head stride
    assert args[6:11] == (B, T_, heads, hd, 0)                          # batch, rows, heads, head_dim, rot
    dests = args[15:27]
    for i, t in enumerate((q, k, v)):
        assert tuple(t.shape) == (B, T_, heads * 128)
        assert dests[4 * i:4 * i + 4] == (t.data_ptr(), T_ * heads * 128, heads * 128, 128)


def test_rope_pack_blocks_needs_src(monkeypatch):
    kc = torch.zeros(1, 4, 160, dtype=torch.bfloat16)
    monkeypatch.setattr(L, "require_cuda", lambda *t: None)
    with pytest.raises(ValueError, match="blocks"):
        ops.rope_pack(None, 2, 80, kv_src=(kc, kc), kv_width=128, blocks=True)
