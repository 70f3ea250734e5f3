"""Restatement of PIL's 8-bit LANCZOS resize, `Image.resize((W2, H2), Image.LANCZOS)` on an RGB image (default box, no
reducing_gap), written from the algorithm's description: the reference the GPU resample passes are pinned to.

Coefficients are computed per output index in double with Python's `math.sin` (the C library's sin, which PIL calls too),
normalised by their plain left-to-right sum, and rounded to 22-bit fixed point.  Each pass accumulates in int32 from
1 << 21 and clips `acc >> 22` to [0, 255]; the intermediate image is uint8.  Horizontal pass first, then vertical; a pass
runs only if its dimension changes."""
import math

import numpy as np

PRECISION_BITS = 22


def _sinc(x):
    if x == 0.0:
        return 1.0
    x = x * math.pi
    return math.sin(x) / x


def _lanczos(x):
    return _sinc(x) * _sinc(x / 3) if -3.0 <= x < 3.0 else 0.0


def coeffs(in_size, out_size):
    """(ksize, bounds int32 [out, 2] = (first input index, taps), coefficients int32 [out, ksize], zero past the taps)."""
    scale = in_size / out_size
    fs = max(scale, 1.0)
    support = 3.0 * fs
    ss = 1.0 / fs
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((out_size, 2), np.int32)
    kk = np.zeros((out_size, ksize), np.int32)
    one = float(1 << PRECISION_BITS)
    for i in range(out_size):
        center = (i + 0.5) * scale
        xmin = max(0, int(center - support + 0.5))
        n = min(in_size, int(center + support + 0.5)) - xmin
        w = [_lanczos((x + xmin - center + 0.5) * ss) for x in range(n)]
        ww = 0.0
        for v in w:
            ww += v
        if ww != 0.0:
            w = [v / ww for v in w]
        kk[i, :n] = [int(v * one + 0.5) if v >= 0 else int(v * one - 0.5) for v in w]
        bounds[i] = (xmin, n)
    return ksize, bounds, kk


def _pass(img, axis, out_size):
    """One pass along `axis` (1: rows / height, 2: columns / width) of uint8 [B, H, W, 3]."""
    _, bounds, kk = coeffs(img.shape[axis], out_size)
    x = np.moveaxis(img, axis, 0).astype(np.int64)           # [in, ...]
    acc = np.full((out_size,) + x.shape[1:], 1 << (PRECISION_BITS - 1), np.int64)
    for t in range(kk.shape[1]):
        idx = np.minimum(bounds[:, 0] + t, x.shape[0] - 1)   # taps past n have coefficient 0
        k = kk[:, t].astype(np.int64).reshape((-1,) + (1,) * (x.ndim - 1))
        acc += k * x[idx]
    assert np.abs(acc).max() < 2 ** 31                       # the int32 accumulator of the real passes never overflows
    out = np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)
    return np.ascontiguousarray(np.moveaxis(out, 0, axis))


def resize(img, out_hw):
    """uint8 [H, W, 3] or [B, H, W, 3] -> [(B,) H2, W2, 3], equal to PIL's LANCZOS resize of each image."""
    a = np.asarray(img, np.uint8)
    single = a.ndim == 3
    if single:
        a = a[None]
    H2, W2 = out_hw
    if a.shape[2] != W2:
        a = _pass(a, 2, W2)
    if a.shape[1] != H2:
        a = _pass(a, 1, H2)
    return a[0] if single else a


def pil_resize(img, out_hw):
    """PIL itself, for comparison: uint8 [H, W, 3] -> [H2, W2, 3]."""
    from PIL import Image
    return np.asarray(Image.fromarray(np.asarray(img, np.uint8), "RGB").resize((out_hw[1], out_hw[0]), Image.LANCZOS))


def stripe_image(h, w, seed=0, b=None):
    """Random bytes with full-range 0/255 stripes (exercise overshoot and clipping): [h, w, 3], or [b, h, w, 3]."""
    rng = np.random.default_rng(seed)
    shape = (h, w, 3) if b is None else (b, h, w, 3)
    a = rng.integers(0, 256, shape, dtype=np.uint8)
    v = a[None] if b is None else a
    v[:, :, 3::11] = 255
    v[:, :, 5::11] = 0
    v[:, 7::13] = 0
    v[:, 8::13] = 255
    return a
