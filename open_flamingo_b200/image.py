"""CLIPImageProcessor: open_clip's eval transform on the GPU, a drop-in for the `image_processor` that
create_model_and_transforms returns (open_clip image_transform(is_train=False), factory.py:42).

For a decoded PIL image in mode RGB or L its output equals, bit for bit, the fp32 tensor of
    Resize(S, BICUBIC) -> CenterCrop(S) -> convert("RGB") -> ToTensor() -> Normalize(mean, std)
computed by torchvision and Pillow on the host (see ofk_clip_preprocess in include/ofk.h for the rounding contract).
Other PIL modes are refused: Pillow resizes RGBA premultiplied and P and 1 with nearest, so converting them is the
caller's choice.  There is no host fallback: without libofk.so or a CUDA device the processor raises RuntimeError.
"""
import numpy as np
import torch

from . import ops

OPENAI_MEAN = (0.48145466, 0.4578275, 0.40821073)
OPENAI_STD = (0.26862954, 0.26130258, 0.27577711)


class CLIPImageProcessor:
    """proc(img) -> f32 [3, S, S] and proc.batch(images) -> f32 [N, 3, S, S] on the current CUDA device.

    Accepted images: PIL images in mode RGB or L, and uint8 [h, w, c] tensors (c = 1 or 3) on the CPU or on the
    current CUDA device; a row stride larger than w * c is allowed.  A batch stages every host image in one pinned
    buffer, copies it to the device once and runs two kernels for the whole batch."""

    def __init__(self, image_size=224, mean=OPENAI_MEAN, std=OPENAI_STD):
        self.image_size = int(image_size)
        self.mean = tuple(float(m) for m in mean)
        self.std = tuple(float(s) for s in std)
        if len(self.mean) != 3 or len(self.std) != 3:
            raise ValueError("mean and std must have 3 entries")
        self._pinned = None
        self._pinned_free = None  # event recorded after the last copy out of the pinned buffer

    def __call__(self, img):
        return self.batch([img])[0]

    @staticmethod
    def _host_pixels(img, i):
        """A host image as a uint8 [h, w, c] numpy array or CPU tensor; a CUDA tensor as itself."""
        if isinstance(img, torch.Tensor):
            if img.dtype != torch.uint8 or img.dim() != 3 or img.shape[2] not in (1, 3):
                raise ValueError(f"image {i}: tensors must be uint8 [h, w, 1 or 3] (HWC), got {tuple(img.shape)} "
                                 f"{img.dtype}")
            return img
        from PIL import Image
        if not isinstance(img, Image.Image):
            raise ValueError(f"image {i}: expected a PIL image or a uint8 HWC tensor, got {type(img).__name__}")
        if img.mode not in ("RGB", "L"):
            raise ValueError(f"image {i}: PIL mode {img.mode!r} is not supported; convert it to 'RGB' or 'L' first")
        a = np.asarray(img)
        return a.reshape(a.shape[0], a.shape[1], -1)

    def batch(self, images, out=None):
        """f32 [N, 3, S, S] on the current CUDA device (`out`, allocated when None; each image contiguous, images at any
        stride, so it may be a window of a vision_x buffer), image i the transform of images[i]."""
        images = list(images)
        if not images:
            raise ValueError("batch needs at least one image")
        pix = [self._host_pixels(img, i) for i, img in enumerate(images)]
        if not torch.cuda.is_available():
            raise RuntimeError("CLIPImageProcessor runs on the GPU (libofk.so, sm_90a); there is no CPU path")
        device = torch.device("cuda", torch.cuda.current_device())
        host = [i for i, p in enumerate(pix) if not (isinstance(p, torch.Tensor) and p.is_cuda)]
        offsets, total = {}, 0
        for i in host:
            offsets[i] = total
            total += -(-pix[i].shape[0] * pix[i].shape[1] * pix[i].shape[2] // 16) * 16
        if host:
            if self._pinned_free is not None:
                self._pinned_free.synchronize()  # the previous batch's copy may still be reading the buffer
            if self._pinned is None or self._pinned.numel() < total:
                self._pinned = torch.empty(total, dtype=torch.uint8, pin_memory=True)
            staged = self._pinned.numpy()
            for i in host:
                p, o = pix[i], offsets[i]
                view = staged[o:o + p.shape[0] * p.shape[1] * p.shape[2]].reshape(p.shape)
                view[...] = p.numpy() if isinstance(p, torch.Tensor) else p
            dev = torch.empty(total, dtype=torch.uint8, device=device)
            dev.copy_(self._pinned[:total], non_blocking=True)
            self._pinned_free = torch.cuda.Event()
            self._pinned_free.record()
            for i in host:
                h, w, c = pix[i].shape
                pix[i] = dev[offsets[i]:offsets[i] + h * w * c].view(h, w, c)
        return ops.clip_preprocess(pix, self.image_size, self.mean, self.std, out=out)
