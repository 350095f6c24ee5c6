"""Integer restatement of the CLIP eval transform the GPU image processor computes (test code only):
Resize(S, BICUBIC) + CenterCrop(S) on a PIL image, then ToTensor + Normalize.

Resize is Pillow's two-pass fixed-point bicubic (Image.resize(size, BICUBIC)):
  per axis, scale = in / out, fs = max(scale, 1), support = 2 fs; output i takes the source span
  [xmin, xmin + n) around center = (i + 0.5) scale with float64 weights bicubic((t + xmin - center + 0.5) / fs),
  a = -0.5, normalised by their left-to-right sum and rounded to int32 at 22 fractional bits;
  the horizontal pass runs first and rounds to uint8, then the vertical pass -- except that Image.resize runs the
  vertical pass first when the image is more than 100 times taller than wide and its height shrinks; each output is
  clip8(2^21 + sum pixel * tap) in int32.  An axis whose size does not change is not resampled.
Python floats are IEEE doubles with no contraction, so the taps here are the ones the contract names."""
import math

import numpy as np

PRECISION_BITS = 22
A = -0.5


def output_size(h, w, S):
    """torchvision Resize(S) on a PIL image: the shorter side becomes S, the longer int(S * long / short)."""
    if w <= h:
        return int(S * h / w), S
    return S, int(S * w / h)


def crop_offsets(h, w, S):
    """torchvision CenterCrop(S): (top, left), rounded half to even as Python's round."""
    return int(round((h - S) / 2.0)), int(round((w - S) / 2.0))


def _bicubic(x):
    if x < 0.0:
        x = -x
    if x < 1.0:
        return ((A + 2.0) * x - (A + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * A
    return 0.0


def taps(n_in, n_out):
    """(bounds [n_out, 2] int32 of (xmin, n), taps [n_out, ksize] int32) of one axis."""
    scale = n_in / n_out
    fs = max(scale, 1.0)
    support = 2.0 * fs
    ksize = 2 * int(math.ceil(support)) + 1
    bounds = np.zeros((n_out, 2), np.int32)
    k = np.zeros((n_out, ksize), np.int32)
    for i in range(n_out):
        center = (i + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        n = min(int(center + support + 0.5), n_in) - xmin
        w = [_bicubic((t + xmin - center + 0.5) / fs) for t in range(n)]
        ww = 0.0
        for v in w:
            ww += v
        if ww != 0.0:
            w = [v / ww for v in w]
        k[i, :n] = [int(v * (1 << PRECISION_BITS) + (0.5 if v >= 0 else -0.5)) for v in w]
        bounds[i] = (xmin, n)
    return bounds, k


def _clip8(acc):
    return np.where(acc >= 1 << (PRECISION_BITS + 8), 255, np.where(acc <= 0, 0, acc >> PRECISION_BITS)).astype(np.uint8)


def _pass(img, bounds, k, axis):
    """One resampling pass of uint8 img [H, W, C] along axis 0 or 1 in int32."""
    src = np.moveaxis(img, axis, 0).astype(np.int64)
    out = np.empty((len(bounds),) + src.shape[1:], np.uint8)
    for i, (xmin, n) in enumerate(bounds):
        acc = (1 << (PRECISION_BITS - 1)) + np.tensordot(k[i, :n].astype(np.int64), src[xmin:xmin + n], axes=(0, 0))
        acc = ((acc + 2 ** 31) % 2 ** 32) - 2 ** 31        # int32 wrap-around, as Pillow's int accumulator
        out[i] = _clip8(acc)
    return np.moveaxis(out, 0, axis)


def vertical_first(h, w, out_h):
    """Image.resize's pass order: vertical first for an image over 100 times taller than wide whose height shrinks."""
    return h > w * 100 and out_h < h


def resize(img, out_h, out_w):
    """Image.resize((out_w, out_h), BICUBIC) of uint8 img [H, W, C]."""
    h, w = img.shape[:2]
    order = (0, 1) if vertical_first(h, w, out_h) else (1, 0)
    for axis in order:
        n_in, n_out = (h, out_h) if axis == 0 else (w, out_w)
        if n_in != n_out:
            img = _pass(img, *taps(n_in, n_out), axis=axis)
    return img


def clip_uint8(img, S):
    """Resize(S, BICUBIC) + CenterCrop(S) of uint8 img [H, W, C] -> [S, S, C] uint8."""
    h, w = img.shape[:2]
    oh, ow = output_size(h, w, S)
    top, left = crop_offsets(oh, ow, S)
    if (oh, ow) == (h, w):
        return img[top:top + S, left:left + S]
    return resize(img, oh, ow)[top:top + S, left:left + S]
