"""GPU: CLIPImageProcessor equals, bit for bit, the CLIP eval transform computed by torchvision and Pillow on the host.

The reference transform is restated here as open_clip's image_transform(is_train=False) builds it (factory.py:42 of
the reference; open_clip transform.py): Resize(S, BICUBIC) -> CenterCrop(S) -> _convert_to_rgb -> ToTensor() ->
Normalize(mean, std), on the PIL image.  open_clip is not a dependency of this project, so the restatement is not
checked against open_clip itself."""
import numpy as np
import pytest
import torch
from PIL import Image

pytestmark = pytest.mark.gpu

MEAN = (0.48145466, 0.4578275, 0.40821073)
STD = (0.26862954, 0.26130258, 0.27577711)
SIZES = [(375, 500), (500, 375), (480, 640), (768, 1024), (3000, 4000), (17, 23), (1, 1), (1, 9), (9, 1), (224, 224),
         (224, 300), (225, 224), (303, 224), (100, 1000), (30000, 250)]     # (h, w); the last resizes vertically first


def reference(img, S):
    from torchvision import transforms as T
    tf = T.Compose([T.Resize(S, interpolation=T.InterpolationMode.BICUBIC), T.CenterCrop(S),
                    lambda im: im.convert("RGB"), T.ToTensor(), T.Normalize(MEAN, STD)])
    return tf(img)


def content(kind, h, w, c, seed):
    if kind == "random":
        a = np.random.default_rng(seed).integers(0, 256, (h, w, c), dtype=np.uint8)
    elif kind == "checker":
        a = ((np.indices((h, w)).sum(0) % 2) * 255).astype(np.uint8)[..., None].repeat(c, 2)
    else:
        a = np.full((h, w, c), 0 if kind == "zeros" else 255, np.uint8)
    return Image.fromarray(a if c == 3 else a[..., 0], "RGB" if c == 3 else "L")


def _proc(S):
    from open_flamingo_b200 import CLIPImageProcessor
    return CLIPImageProcessor(S, MEAN, STD)


def _same(got, want, what):
    got = got.cpu()
    assert got.dtype == torch.float32 and got.shape == want.shape, what
    bad = (got.view(torch.int32) != want.view(torch.int32)).sum().item()
    assert bad == 0, f"{what}: {bad} elements differ, max |d| {(got - want).abs().max().item():.3e}"


@pytest.mark.parametrize("S", [224, 336])
@pytest.mark.parametrize("mode", ["RGB", "L"])
@pytest.mark.parametrize("kind", ["random", "checker", "zeros", "ones"])
def test_single_image_equals_torchvision(S, mode, kind):
    torch.cuda.set_device(0)
    proc = _proc(S)
    c = 3 if mode == "RGB" else 1
    for i, (h, w) in enumerate(SIZES):
        if kind != "random" and h * w > 2_000_000:
            continue
        img = content(kind, h, w, c, seed=i)
        _same(proc(img), reference(img, S), f"{h}x{w} {mode} {kind} S={S}")


def _mixed(S):
    imgs = []
    for i, (h, w) in enumerate(SIZES):
        for c in (3, 1):
            imgs.append(content("random" if i % 2 else "checker", h, w, c, seed=100 + i))
    return imgs


@pytest.mark.parametrize("S", [224, 336])
def test_ragged_batch_equals_stacked_singles(S):
    torch.cuda.set_device(0)
    proc = _proc(S)
    imgs = _mixed(S)
    out = proc.batch(imgs)
    assert out.shape == (len(imgs), 3, S, S) and out.is_cuda
    singles = torch.stack([proc(im) for im in imgs])
    assert torch.equal(out.view(torch.int32), singles.view(torch.int32))
    for im, o in zip(imgs, out):
        _same(o, reference(im, S), f"{im.size} {im.mode}")


def test_host_pinned_and_device_inputs_give_the_same_bits():
    torch.cuda.set_device(0)
    proc = _proc(224)
    rng = np.random.default_rng(5)
    a = rng.integers(0, 256, (375, 500, 3), dtype=np.uint8)
    want = reference(Image.fromarray(a, "RGB"), 224)
    cpu = torch.from_numpy(a)
    pinned = cpu.pin_memory()
    dev = cpu.cuda()
    wide = torch.zeros(375, 512 * 3 + 16, dtype=torch.uint8, device="cuda")
    wide[:, :1500] = dev.view(375, 1500)
    strided = wide[:, :1500].view(375, 500, 3)          # rows 1552 bytes apart
    assert strided.stride() == (1552, 3, 1)
    cpu_strided = torch.zeros(375, 700, 3, dtype=torch.uint8)[:, 100:600]
    cpu_strided.copy_(cpu)
    for x, what in ((cpu, "cpu"), (pinned, "pinned"), (dev, "cuda"), (strided, "cuda row-strided"),
                    (cpu_strided, "cpu row-strided")):
        _same(proc(x), want, what)
    gray = rng.integers(0, 256, (77, 130), dtype=np.uint8)
    want = reference(Image.fromarray(gray, "L"), 224)
    for x in (torch.from_numpy(gray)[..., None], torch.from_numpy(gray)[..., None].cuda()):
        _same(proc(x), want, "L tensor")
    out = proc.batch([cpu, dev, Image.fromarray(a, "RGB"), strided])
    assert all(torch.equal(out[0], out[i]) for i in range(1, 4))


def test_output_window_leaves_neighbours_untouched():
    torch.cuda.set_device(0)
    S = 224
    proc = _proc(S)
    imgs = _mixed(S)[:5]
    buf = torch.full((4, 5, 2, 3, S, S), float("nan"), device="cuda")      # [B, T_img, F, C, H, W]
    window = buf[1, :, 1]
    proc.batch(imgs, out=window)
    torch.cuda.synchronize()
    want = torch.stack([reference(im, S) for im in imgs])
    _same(window, want, "window")
    canary = torch.ones_like(buf, dtype=torch.bool)
    canary[1, :, 1] = False
    assert torch.isnan(buf[canary]).all(), "a write outside the window"


def test_repeatable_and_two_launches_per_batch():
    torch.cuda.set_device(0)
    from open_flamingo_b200 import _lib
    proc = _proc(224)
    imgs = _mixed(224)
    a = proc.batch(imgs)
    b = proc.batch(imgs)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    rng = np.random.default_rng(3)
    counts = []
    for n in (1, 256):
        batch = [torch.from_numpy(rng.integers(0, 256, (int(rng.integers(40, 700)), int(rng.integers(40, 700)), 3),
                                               dtype=np.uint8)) for _ in range(n)]
        proc.batch(batch)                      # warm
        before = _lib.launch_count()
        proc.batch(batch)
        counts.append(_lib.launch_count() - before)
    assert counts == [2, 2], counts


def test_pinned_staging_is_reused_safely():
    """Back-to-back batches reuse one pinned buffer; each result still equals its own images."""
    torch.cuda.set_device(0)
    proc = _proc(224)
    rng = np.random.default_rng(11)
    batches = [[torch.from_numpy(rng.integers(0, 256, (480, 640, 3), dtype=np.uint8)) for _ in range(8)]
               for _ in range(4)]
    outs = [proc.batch(b) for b in batches]
    torch.cuda.synchronize()
    for b, o in zip(batches, outs):
        for x, y in zip(b, o):
            _same(y, reference(Image.fromarray(x.numpy(), "RGB"), 224), "reused staging")


def test_drop_in_for_the_model_input():
    """model(vision_x=...) logits from the processor's vision_x equal those from the host transform's, bit for bit."""
    torch.cuda.set_device(0)
    from open_flamingo_b200.testing import build_flamingo, synthetic_batch
    S = 56
    vit_cfg = dict(image_size=S, patch_size=14, width=128, layers=2, heads=2, output_dim=128)
    mpt_kw = dict(d_model=128, n_heads=2, n_layers=2, vocab_size=61, max_seq_len=64, expansion_ratio=2)
    model, _, tok = build_flamingo(vit_cfg, mpt_kw, device="cuda", gate_init=1.0, seed=3)
    media_id, eoc_id = tok.encode("<image>")[-1], tok.encode("<|endofchunk|>")[-1]
    batch = synthetic_batch(2, 2, 16, media_id, eoc_id, 61, image_size=S, seed=5)
    rng = np.random.default_rng(9)
    imgs = [Image.fromarray(rng.integers(0, 256, (int(rng.integers(30, 300)), int(rng.integers(30, 300)), 3),
                                         dtype=np.uint8), "RGB") for _ in range(4)]
    proc = _proc(S)
    vx_gpu = torch.empty(2, 2, 1, 3, S, S, device="cuda")
    proc.batch(imgs, out=vx_gpu.view(4, 3, S, S))
    vx_host = torch.stack([reference(im, S) for im in imgs]).view(2, 2, 1, 3, S, S).cuda()
    assert torch.equal(vx_gpu.view(torch.int32), vx_host.view(torch.int32))
    with torch.no_grad():
        kw = dict(lang_x=batch["lang_x"].cuda(), attention_mask=batch["attention_mask"].cuda())
        a = model(vision_x=vx_gpu, **kw).logits
        b = model(vision_x=vx_host, **kw).logits
    assert torch.equal(a, b)
