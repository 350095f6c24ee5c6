"""CPU: the host side of the GPU CLIP image processor.

- ofk_image_plan's bounds and int32 taps equal the integer restatement in image_reference.py bit for bit, and that
  restatement equals PIL.Image.resize(..., BICUBIC), so the tables pin Pillow's algorithm without a device;
- the plan's output size and crop offsets equal torchvision's Resize(S) / CenterCrop(S);
- every argument rejection of the three entry points returns its code without a device (ofk_clip_preprocess runs in
  a child process with no CUDA device visible and made-up device addresses that are never dereferenced: a call whose
  arguments pass validation reaches the plan copy and returns OFK_ERR_CUDA (-3));
- neither kernel uses local memory;
- CLIPImageProcessor's input validation, and its RuntimeError off the GPU."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from PIL import Image

import image_reference as R
from test_abi_cpu import _sass_by_kernel

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARG, ALIGN, NO_DEVICE = -1, -2, -3
MEAN = (0.48145466, 0.4578275, 0.40821073)
STD = (0.26862954, 0.26130258, 0.27577711)

HEADER = np.dtype([("magic", "<u4"), ("n", "<i4"), ("S", "<i4"), ("blocks1", "<i4"), ("bytes", "<i8"), ("tmp", "<i8"),
                   ("ws_bytes", "<i8"), ("mean", "<f4", 3), ("std", "<f4", 3)])
DESC = np.dtype([("src", "<u8"), ("ld", "<i8"), ("h", "<i4"), ("w", "<i4"), ("c", "<i4"), ("vfirst", "<i4"),
                 ("th", "<i4"), ("tw", "<i4"), ("origin", "<i4"), ("blk0", "<i4"), ("tmp", "<i8"), ("ts1", "<i8"),
                 ("os1", "<i8"), ("ts2", "<i8"), ("os2", "<i8"), ("tab1", "<i4"), ("k1", "<i4"), ("tab2", "<i4"),
                 ("k2", "<i4"), ("oh", "<i4"), ("ow", "<i4"), ("top", "<i4"), ("left", "<i4"), ("pad", "<i4", 2)])


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from open_flamingo_b200 import _lib
    return _lib.lib()


def _shape(dims):
    return np.ascontiguousarray(np.array(dims, dtype=np.int64).reshape(-1, 4))


def make_plan(lib, dims, S, mean=MEAN, std=STD):
    """(header, descriptors, int32 view of the plan, workspace bytes) of ofk_image_plan for images (h, w, c, ld)."""
    shape = _shape(dims)
    n = len(shape)
    pb, wb = ctypes.c_longlong(), ctypes.c_longlong()
    assert lib.ofk_image_plan_size(n, shape.ctypes.data, S, ctypes.byref(pb), ctypes.byref(wb)) == 0
    plan = np.zeros(pb.value // 4 + 4, np.int32)      # numpy buffers are 16-byte aligned
    src = np.arange(1, n + 1, dtype=np.uint64) << np.uint64(32)
    f3 = ctypes.c_float * 3
    rc = lib.ofk_image_plan(n, src.ctypes.data, shape.ctypes.data, S, f3(*mean), f3(*std), plan.ctypes.data, pb.value)
    assert rc == 0, lib.ofk_last_error()
    raw = plan.view(np.uint8)[:pb.value]
    hd = np.frombuffer(raw[:HEADER.itemsize].tobytes(), HEADER)[0]
    ds = np.frombuffer(raw[HEADER.itemsize:HEADER.itemsize + n * DESC.itemsize].tobytes(), DESC)
    return hd, ds, plan, wb.value


def _table(plan, at, k, S):
    t = plan[at:at + S * (k + 2)].reshape(S, k + 2)
    return t[:, :2], t[:, 2:]


def _expected_tables(h, w, S):
    """Restated (table1, table2) as (bounds, taps) for the crop window, positions as the plan stores them."""
    oh, ow = R.output_size(h, w, S)
    top, left = R.crop_offsets(oh, ow, S)
    bx, kx = R.taps(w, ow)
    by, ky = R.taps(h, oh)
    bx, kx, by, ky = bx[left:left + S].copy(), kx[left:left + S], by[top:top + S].copy(), ky[top:top + S]
    if R.vertical_first(h, w, oh):
        bx[:, 0] -= bx[0, 0]
        return (by, ky), (bx, kx)
    by[:, 0] -= by[0, 0]
    return (bx, kx), (by, ky)


def _check_image_tables(lib, h, w, S, c=3):
    hd, ds, plan, _ = make_plan(lib, [(h, w, c, w * c)], S)
    d = ds[0]
    (b1, k1), (b2, k2) = _expected_tables(h, w, S)
    gb1, gk1 = _table(plan, d["tab1"], d["k1"], S)
    gb2, gk2 = _table(plan, d["tab2"], d["k2"], S)
    for got, want, name in ((gb1, b1, "bounds1"), (gk1, k1, "taps1"), (gb2, b2, "bounds2"), (gk2, k2, "taps2")):
        assert got.shape == want.shape and np.array_equal(got, want), f"{h}x{w} S={S}: {name} differ"
    return d


# ---------------------------------------------------------------------------------------------- taps and bounds
def _pairs():
    rng = np.random.default_rng(7)
    pairs = [(224, 224), (1, 224), (7, 224), (2, 224), (1, 336), (7, 336), (4000, 224), (3000, 224), (9000, 224),
             (4000, 336), (225, 224), (223, 224), (600, 1), (17, 3), (3, 17)]
    pairs += [tuple(int(v) for v in rng.integers(1, 601, 2)) for _ in range(60)]
    return pairs


@pytest.mark.parametrize("n_in,n_out", _pairs())
def test_plan_taps_equal_the_restatement(lib, n_in, n_out):
    """A square n_in image at S = n_out resamples both axes n_in -> n_out over the full window."""
    d = _check_image_tables(lib, n_in, n_in, n_out)
    assert d["k1"] == d["k2"] == R.taps(n_in, n_out)[1].shape[1]


@pytest.mark.parametrize("h,w", [(375, 500), (500, 375), (480, 640), (17, 23), (1, 9), (9, 1), (303, 224),
                                 (100, 1000), (3000, 4000), (281, 2), (30000, 250), (1000, 2)])
@pytest.mark.parametrize("S", [224, 336])
def test_plan_tables_of_the_crop_window(lib, h, w, S):
    d = _check_image_tables(lib, h, w, S)
    oh, ow = R.output_size(h, w, S)
    vf = R.vertical_first(h, w, oh)
    assert d["vfirst"] == vf
    assert (d["th"], d["tw"]) == ((S, d["tw"]) if vf else (d["th"], S))


def test_identity_taps_copy_each_pixel():
    """An axis whose size does not change runs with taps (.., 0, 2^22, 0, ..): the pass returns its input."""
    for n in (1, 2, 5, 224):
        b, k = R.taps(n, n)
        for i in range(n):
            assert (k[i] != 0).sum() == 1 and k[i, i - b[i, 0]] == 1 << 22
    img = np.random.default_rng(0).integers(0, 256, (9, 224, 3), dtype=np.uint8)
    assert np.array_equal(R._pass(img, *R.taps(224, 224), axis=1), img)


# ---------------------------------------------------------------------------------------------- restatement vs PIL
def _pil(a):
    return Image.fromarray(a if a.shape[2] == 3 else a[..., 0], "RGB" if a.shape[2] == 3 else "L")


RESIZE_SIZES = [(375, 500, 224, 298), (480, 640, 224, 298), (17, 23, 224, 303), (1, 9, 224, 2016), (9, 1, 2016, 224),
                (3000, 1333, 504, 224), (225, 224, 225, 224), (100, 1000, 224, 2240), (901, 37, 5454, 224),
                (224, 300, 224, 300), (1, 1, 224, 224), (281, 2, 269, 263), (1000, 2, 224, 5), (37, 41, 12, 9),
                (250, 3, 250, 224)]


@pytest.mark.parametrize("h,w,oh,ow", RESIZE_SIZES)
@pytest.mark.parametrize("c", [3, 1])
def test_restatement_equals_pil_resize(h, w, oh, ow, c):
    rng = np.random.default_rng(h * 7919 + w * 31 + c)
    a = rng.integers(0, 256, (h, w, c), dtype=np.uint8)
    checker = ((np.indices((h, w)).sum(0) % 2) * 255).astype(np.uint8)[..., None].repeat(c, 2)
    for img in (a, checker):
        want = np.asarray(_pil(img).resize((ow, oh), Image.BICUBIC)).reshape(oh, ow, c)
        assert np.array_equal(R.resize(img, oh, ow), want)


# ---------------------------------------------------------------------------------------------- size and crop
SIZE_CASES = [(375, 500), (500, 375), (480, 640), (17, 23), (1, 1), (1, 9), (9, 1), (224, 224), (224, 300),
              (225, 224), (303, 224), (301, 224), (224, 303), (224, 301), (100, 1000), (768, 1024), (3000, 4000),
              (449, 224), (224, 451), (673, 336), (337, 336), (336, 339)]


@pytest.mark.parametrize("h,w", SIZE_CASES)
@pytest.mark.parametrize("S", [224, 336])
def test_size_and_crop_equal_torchvision(lib, h, w, S):
    from torchvision.transforms import CenterCrop, Resize
    from torchvision.transforms import functional as TF
    oh, ow = Resize(S, interpolation=TF.InterpolationMode.BICUBIC)(Image.new("L", (w, h))).size[::-1]
    idx = torch.arange(oh * ow, dtype=torch.int64).view(1, oh, ow)
    corner = int(CenterCrop(S)(idx)[0, 0, 0])
    _, ds, _, _ = make_plan(lib, [(h, w, 1, w)], S)
    assert (ds[0]["oh"], ds[0]["ow"]) == (oh, ow) == R.output_size(h, w, S)
    assert (ds[0]["top"], ds[0]["left"]) == divmod(corner, ow) == R.crop_offsets(oh, ow, S)


def test_crop_ties_round_half_to_even():
    assert R.crop_offsets(303, 224, 224) == (40, 0)    # 79 / 2 = 39.5 -> 40
    assert R.crop_offsets(301, 224, 224) == (38, 0)    # 77 / 2 = 38.5 -> 38


def test_plan_layout_is_consistent(lib):
    dims = [(375, 500, 3, 1500), (500, 375, 1, 400), (9, 1, 3, 3), (30000, 250, 1, 256)]
    hd, ds, plan, ws = make_plan(lib, dims, 224)
    assert hd["n"] == 4 and hd["S"] == 224 and hd["ws_bytes"] == ws
    assert np.array_equal(hd["mean"], np.float32(MEAN)) and np.array_equal(hd["std"], np.float32(STD))
    blk = 0
    for d, (h, w, c, ld) in zip(ds, dims):
        assert (d["h"], d["w"], d["c"], d["ld"]) == (h, w, c, ld)
        assert d["blk0"] == blk and d["tmp"] >= hd["tmp"] and d["tmp"] % 16 == 0
        assert d["tmp"] + d["th"] * d["tw"] * c <= ws
        blk += -(-int(d["th"]) * int(d["tw"]) // 256)
    assert hd["blocks1"] == blk
    assert ds[3]["vfirst"] == 1 and ds[0]["vfirst"] == 0


# ---------------------------------------------------------------------------------------------- argument rejection
def _plan_cases():
    S = 224
    good = [(375, 500, 3, 1500), (480, 640, 1, 640)]
    cases = {"valid": (good, S, NO_DEVICE)}
    for name, dims in {"h0": (0, 500, 3, 1500), "w0": (375, 0, 3, 1500), "c2": (375, 500, 2, 1500),
                       "c4": (375, 500, 4, 2000), "ld-short": (375, 500, 3, 1499), "h-neg": (-1, 500, 3, 1500),
                       "too-long": (1, 10_000_000, 3, 30_000_000)}.items():
        cases[name] = ([good[0], dims], S, ARG)
    cases["valid-ld-wide"] = ([(375, 500, 3, 1600)], S, NO_DEVICE)
    cases["valid-1x1"] = ([(1, 1, 1, 1)], S, NO_DEVICE)
    cases["S0"] = (good, 0, ARG)
    cases["S4097"] = (good, 4097, ARG)
    cases["valid-S4096"] = (good, 4096, NO_DEVICE)
    return cases


@pytest.mark.parametrize("case", sorted(_plan_cases()))
def test_plan_rejects_bad_images(lib, case):
    dims, S, want = _plan_cases()[case]
    shape = _shape(dims)
    pb, wb = ctypes.c_longlong(), ctypes.c_longlong()
    rc = lib.ofk_image_plan_size(len(shape), shape.ctypes.data, S, ctypes.byref(pb), ctypes.byref(wb))
    assert rc == (0 if want == NO_DEVICE else want), (case, lib.ofk_last_error())
    buf = np.zeros(max(pb.value, 64) // 4 + 4, np.int32)
    src = np.arange(1, len(shape) + 1, dtype=np.uint64) << np.uint64(32)
    f3 = ctypes.c_float * 3
    rc = lib.ofk_image_plan(len(shape), src.ctypes.data, shape.ctypes.data, S, f3(*MEAN), f3(*STD), buf.ctypes.data,
                            pb.value)
    assert rc == (0 if want == NO_DEVICE else want), (case, lib.ofk_last_error())


def test_plan_rejects_bad_arguments(lib):
    shape = _shape([(375, 500, 3, 1500)])
    pb, wb = ctypes.c_longlong(), ctypes.c_longlong()
    assert lib.ofk_image_plan_size(1, shape.ctypes.data, 224, ctypes.byref(pb), ctypes.byref(wb)) == 0
    assert lib.ofk_image_plan_size(1, None, 224, ctypes.byref(pb), ctypes.byref(wb)) == ARG
    assert lib.ofk_image_plan_size(1, shape.ctypes.data, 224, None, ctypes.byref(wb)) == ARG
    assert lib.ofk_image_plan_size(0, shape.ctypes.data, 224, ctypes.byref(pb), ctypes.byref(wb)) == ARG
    assert lib.ofk_image_plan_size(65536, shape.ctypes.data, 224, ctypes.byref(pb), ctypes.byref(wb)) == ARG
    buf = np.zeros(pb.value // 4 + 8, np.int32)
    src = np.array([1 << 32], np.uint64)
    zero = np.array([0], np.uint64)
    f3 = ctypes.c_float * 3
    m, s = f3(*MEAN), f3(*STD)

    def plan(**kw):
        a = dict(n=1, src=src.ctypes.data, shape=shape.ctypes.data, S=224, mean=m, std=s, plan=buf.ctypes.data,
                 bytes=pb.value)
        a.update(kw)
        return lib.ofk_image_plan(*a.values())
    assert plan() == 0
    assert plan(src=None) == ARG
    assert plan(src=zero.ctypes.data) == ARG
    assert plan(mean=None) == ARG
    assert plan(std=None) == ARG
    assert plan(plan=None) == ARG
    assert plan(std=f3(0.5, 0.0, 0.5)) == ARG
    assert plan(mean=f3(float("nan"), 0.0, 0.0)) == ARG
    assert plan(std=f3(float("inf"), 1.0, 1.0)) == ARG
    assert plan(bytes=pb.value + 4) == ARG
    assert plan(bytes=pb.value - 4) == ARG
    assert plan(plan=buf.ctypes.data + 4) == ALIGN


CHILD = r"""
import ctypes, json, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, sys.argv[2])
from open_flamingo_b200 import _lib
import test_image_preprocess_cpu as T
lib = _lib.lib()
hd, ds, plan, ws = T.make_plan(lib, [(375, 500, 3, 1500), (30000, 250, 1, 256)], 224)
WS, OUT = 1 << 40, 2 << 40
nbytes = int(hd["bytes"])
raw = plan.view(np.uint8)
res = {}
def call(name, mutate=None, **kw):
    p = plan.copy()
    if mutate:
        mutate(p.view(np.uint8))
    a = dict(plan=p.ctypes.data, bytes=nbytes, ws=WS, ws_bytes=ws, out=OUT, stride=3 * 224 * 224, stream=None)
    a.update(kw)
    res[name] = lib.ofk_clip_preprocess(*a.values())
def field(name, i, value, dtype=np.int32):
    off = T.HEADER.itemsize + i * T.DESC.itemsize + T.DESC.fields[name][1]
    def m(b):
        b[off:off + np.dtype(dtype).itemsize] = np.frombuffer(np.array([value], dtype).tobytes(), np.uint8)
    return m
def hfield(name, value, dtype):
    off = T.HEADER.fields[name][1]
    def m(b):
        b[off:off + np.dtype(dtype).itemsize] = np.frombuffer(np.array([value], dtype).tobytes(), np.uint8)
    return m
call("valid")
call("valid-wide-stride", stride=3 * 224 * 224 + 1)
call("valid-big-workspace", ws_bytes=ws + 1000)
call("plan-null", plan=None)
call("ws-null", ws=None)
call("out-null", out=None)
call("plan+4B", plan=plan.ctypes.data + 4)
call("ws+8B", ws=WS + 8)
call("out+2B", out=OUT + 2)
call("valid-out+4B", out=OUT + 4)
call("stride-short", stride=3 * 224 * 224 - 1)
call("ws-short", ws_bytes=ws - 1)
call("bytes-short", bytes=nbytes - 4)
call("bytes-tiny", bytes=8)
call("magic", mutate=hfield("magic", 0, np.uint32))
call("header-n", mutate=hfield("n", 3, np.int32))
call("header-S", mutate=hfield("S", 0, np.int32))
call("header-blocks", mutate=hfield("blocks1", 1, np.int32))
call("header-ws", mutate=hfield("ws_bytes", 1 << 50, np.int64))
call("desc-src-null", mutate=field("src", 0, 0, np.uint64))
call("desc-c", mutate=field("c", 1, 3))
call("desc-ld", mutate=field("ld", 0, 100, np.int64))
call("desc-th", mutate=field("th", 0, 10 ** 6))
call("desc-origin", mutate=field("origin", 0, 400))
call("desc-tmp", mutate=field("tmp", 1, 1 << 40, np.int64))
call("desc-blk0", mutate=field("blk0", 1, 0))
call("desc-ts1", mutate=field("ts1", 0, 1, np.int64))
call("desc-tab1", mutate=field("tab1", 0, 1 << 30))
call("desc-k2", mutate=field("k2", 0, 1000))
tab1 = int(ds[0]["tab1"])
def bad_pos(b):
    p = b.view(np.int32); p[tab1 + 223 * (int(ds[0]["k1"]) + 2)] = 498
call("tap-past-edge", mutate=bad_pos)
def bad_n(b):
    p = b.view(np.int32); p[tab1 + 1] = int(ds[0]["k1"]) + 1
call("tap-count", mutate=bad_n)
print(json.dumps(res))
"""

PREPROCESS_WANT = {"valid": NO_DEVICE, "valid-wide-stride": NO_DEVICE, "valid-big-workspace": NO_DEVICE,
                   "valid-out+4B": NO_DEVICE, "plan-null": ARG, "ws-null": ARG, "out-null": ARG, "plan+4B": ALIGN,
                   "ws+8B": ALIGN, "out+2B": ALIGN, "stride-short": ARG, "ws-short": ARG, "bytes-short": ARG,
                   "bytes-tiny": ARG, "magic": ARG, "header-n": ARG, "header-S": ARG, "header-blocks": ARG,
                   "header-ws": ARG, "desc-src-null": ARG, "desc-c": ARG, "desc-ld": ARG, "desc-th": ARG,
                   "desc-origin": ARG, "desc-tmp": ARG, "desc-blk0": ARG, "desc-ts1": ARG, "desc-tab1": ARG,
                   "desc-k2": ARG, "tap-past-edge": ARG, "tap-count": ARG}


@pytest.fixture(scope="module")
def preprocess_results(lib):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", CHILD, ROOT, os.path.join(ROOT, "tests")]
    r = subprocess.run(cmd, capture_output=True, text=True, env=env, timeout=600)
    assert r.returncode == 0, r.stderr
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("case", sorted(PREPROCESS_WANT))
def test_clip_preprocess_return_codes(preprocess_results, case):
    got, want = preprocess_results[case], PREPROCESS_WANT[case]
    assert got == want, f"{case}: returned {got}, expected {want} (-3 = the check ran after the CUDA call or not at all)"


def test_kernels_use_no_local_memory(lib):
    kernels = _sass_by_kernel()
    names = [k for k in kernels if "image_resample_first_kernel" in k or "image_resample_second_kernel" in k]
    assert len(names) == 2, sorted(names)
    for k in names:
        assert not kernels[k] & {"LDL", "STL"}, f"{k}: local-memory traffic"


# ---------------------------------------------------------------------------------------------- Python surface
@pytest.mark.parametrize("mode", ["RGBA", "P", "1", "CMYK", "LA", "I;16", "F"])
def test_processor_rejects_pil_modes_by_name(mode):
    from open_flamingo_b200 import CLIPImageProcessor
    with pytest.raises(ValueError, match=mode.replace(";", ".")):
        CLIPImageProcessor()(Image.new(mode, (8, 6)))


@pytest.mark.parametrize("case", ["float", "int16", "rank2", "rank4", "two-channels", "four-channels", "chw-numpy",
                                  "empty"])
def test_processor_rejects_other_inputs(case):
    from open_flamingo_b200 import CLIPImageProcessor
    bad = {"float": torch.zeros(6, 8, 3), "int16": torch.zeros(6, 8, 3, dtype=torch.int16),
           "rank2": torch.zeros(6, 8, dtype=torch.uint8), "rank4": torch.zeros(1, 6, 8, 3, dtype=torch.uint8),
           "two-channels": torch.zeros(6, 8, 2, dtype=torch.uint8),
           "four-channels": torch.zeros(6, 8, 4, dtype=torch.uint8),
           "chw-numpy": np.zeros((6, 8, 3), np.uint8), "empty": None}[case]
    with pytest.raises(ValueError):
        CLIPImageProcessor().batch([] if bad is None else [bad])


def test_ops_wrapper_rejects_shapes_and_dtypes():
    from open_flamingo_b200 import _lib, ops
    prev = _lib.require_cuda
    _lib.require_cuda = lambda *t: None
    try:
        img = torch.zeros(6, 8, 3, dtype=torch.uint8)
        for call in (lambda: ops.clip_preprocess([], 224, MEAN, STD),
                     lambda: ops.clip_preprocess([img.float()], 224, MEAN, STD),
                     lambda: ops.clip_preprocess([img[..., :2]], 224, MEAN, STD),
                     lambda: ops.clip_preprocess([img.permute(1, 0, 2)], 224, MEAN, STD),
                     lambda: ops.clip_preprocess([img[:, ::2]], 224, MEAN, STD),
                     lambda: ops.clip_preprocess([img], 0, MEAN, STD),
                     lambda: ops.clip_preprocess([img], 224, MEAN[:2], STD),
                     lambda: ops.clip_preprocess([img], 4, MEAN, STD, out=torch.zeros(1, 3, 4, 4, dtype=torch.float64)),
                     lambda: ops.clip_preprocess([img], 4, MEAN, STD, out=torch.zeros(1, 3, 4, 5)),
                     lambda: ops.clip_preprocess([img, img], 4, MEAN, STD, out=torch.zeros(3, 2, 4, 4)[:, :, 0]),
                     lambda: ops.clip_preprocess([img], 4, MEAN, STD, out=torch.zeros(1, 4, 4, 3).permute(0, 3, 1, 2))):
            with pytest.raises(ValueError):
                call()
    finally:
        _lib.require_cuda = prev


OFF_GPU = r"""
import sys
sys.path.insert(0, sys.argv[1])
import torch
from PIL import Image
from open_flamingo_b200 import CLIPImageProcessor, ops
for call in (lambda: CLIPImageProcessor()(Image.new("RGB", (8, 6))),
             lambda: CLIPImageProcessor().batch([torch.zeros(6, 8, 3, dtype=torch.uint8)]),
             lambda: ops.clip_preprocess([torch.zeros(6, 8, 3, dtype=torch.uint8)], 224, (0, 0, 0), (1, 1, 1))):
    try:
        call()
    except RuntimeError:
        continue
    raise SystemExit("no RuntimeError off the GPU")
print("ok")
"""


def test_processor_raises_off_the_gpu(lib):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", OFF_GPU, ROOT]
    r = subprocess.run(cmd, capture_output=True, text=True, env=env, timeout=600)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr


def test_image_module_does_not_import_torchvision():
    import re
    src = open(os.path.join(ROOT, "open_flamingo_b200", "image.py")).read()
    assert not re.search(r"^\s*(import|from)\s+torchvision", src, flags=re.M)
