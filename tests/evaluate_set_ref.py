"""numpy restatement (CPU) of EvaluateSet's page resize (Dataloader.py:290-291) as ops.page_resize_bicubic computes it:
``to_tensor(to_pil_image(page).resize((rw, rh), Image.BICUBIC))``, with Pillow's integer resampler (libImaging/Resample.c)
written out:

  * the bytes: ``page * 255`` in fp32, clamped to [0, 255] (NaN to 0) and truncated, as to_pil_image's ``mul(255).byte()``;
  * the weights: precompute_coeffs with the bicubic filter (a = -0.5, support 2 * max(scale, 1)) in double, then
    normalize_coeffs_8bpc's 22-bit integers;
  * the passes: horizontal first, into a clipped uint8 image, then vertical; each output is ``clip8((1 << 21) + sum)``.
    An axis whose size does not change is not resampled (Pillow skips that pass);
  * to_tensor: the byte / 255 in fp32.

Shared by the CPU golden test and the GPU tests."""
import math

import numpy as np

PRECISION_BITS = 22


def _bicubic(x: float) -> float:
    a = -0.5
    if x < 0.0:
        x = -x
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def coeffs(insize: int, outsize: int):
    """(first tap int64 [outsize], integer weights int64 [outsize, ksize]; zero past each output's window)."""
    scale = insize / outsize
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    ss = 1.0 / filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    first = np.zeros(outsize, np.int64)
    kk = np.zeros((outsize, ksize), np.int64)
    for xx in range(outsize):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), insize) - xmin
        w = [_bicubic((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for v in w:
            ww += v
        for x, v in enumerate(w):
            if ww != 0.0:
                v /= ww
            kk[xx, x] = int(-0.5 + v * (1 << PRECISION_BITS)) if v < 0 else int(0.5 + v * (1 << PRECISION_BITS))
        first[xx] = xmin
    return first, kk


def _pass(img: np.ndarray, outsize: int, axis: int) -> np.ndarray:
    """one resampling pass of a uint8 array along `axis` to `outsize`."""
    insize = img.shape[axis]
    if insize == outsize:
        return img
    first, kk = coeffs(insize, outsize)
    src = np.moveaxis(img, axis, -1).astype(np.int64)
    acc = np.full(src.shape[:-1] + (outsize,), 1 << (PRECISION_BITS - 1), np.int64)
    for t in range(kk.shape[1]):
        idx = np.minimum(first + t, insize - 1)           # past the window the weight is zero
        acc += src[..., idx] * kk[:, t]
    out = np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)
    return np.moveaxis(out, -1, axis)


def resize_bytes(img: np.ndarray, rh: int, rw: int) -> np.ndarray:
    """Image.resize((rw, rh), Image.BICUBIC) of uint8 images [..., h, w] (any leading axes, channels among them)."""
    return _pass(_pass(img, rw, img.ndim - 1), rh, img.ndim - 2)


def page_bytes(page: np.ndarray) -> np.ndarray:
    """to_pil_image's bytes of fp32 pages in [0, 1]: mul(255) in fp32, clamped to [0, 255], NaN to 0, truncated."""
    v = np.asarray(page, np.float32) * np.float32(255)
    return np.nan_to_num(np.clip(v, 0, 255), nan=0.0).astype(np.uint8)


def to_tensor(img: np.ndarray) -> np.ndarray:
    return img.astype(np.float32) / np.float32(255)


def page_resize(page: np.ndarray, rh: int, rw: int) -> np.ndarray:
    """fp32 [n, 3, h, w] pages -> fp32 [n, 3, rh, rw], as ops.page_resize_bicubic."""
    return to_tensor(resize_bytes(page_bytes(page), rh, rw))


def normalize_pad(x: np.ndarray, mean, std, hs: int, ws: int) -> np.ndarray:
    """torchvision's Normalize (sub_, then div_, in fp32) of fp32 [n, 3, h, w], zero-padded on the right and bottom."""
    m = np.asarray(mean, np.float32)[:, None, None]
    s = np.asarray(std, np.float32)[:, None, None]
    y = (np.asarray(x, np.float32) - m) / s
    n, c, h, w = y.shape
    out = np.zeros((n, c, hs, ws), np.float32)
    out[:, :, :h, :w] = y
    return out
