"""Pillow 12.2's ``Image.thumbnail(size)`` of an RGB image in memory, restated in numpy (the statement of
``se_resize_reducing_u8``, ``engine.thumbnail_u8`` and ``EditSession.image/jpeg/png(size=...)``).

``thumbnail`` is the size rule (``engine.thumbnail_size``), then ``resize(size, BICUBIC, reducing_gap=2.0)`` of the whole
image (``draft`` does nothing for an image in memory):

1. Reduce. ``fx = int(w / tw / 2) or 1`` and ``fy`` likewise. If either is > 1 the image becomes ``Image.reduce((fx, fy))``:
   ``ceil(w / fx) x ceil(h / fy)`` cells, each the average of the pixels it covers (right and bottom cells may be partial),
   per channel ``((s + n // 2) * m mod 2^32) >> 24`` with ``s`` the cell's byte sum, ``n`` its pixel count and
   ``m = uint32(float32(2^32) / float32(256 n mod 2^32))`` (Pillow's uint32 arithmetic; plain rounding differs).
2. Bicubic resize of the reduced image to ``(tw, th)`` with the box ``(0, 0, w / fx, h / fy)`` in C floats: the coefficient
   table of an axis of ``n_in`` samples is Pillow's with ``scale = in1 / out`` and ``center = (i + 0.5) scale`` (in double),
   its taps clamped to ``[0, n_in)``.
3. An axis is resampled when its length changes or its box end is not its length. A reduced image more than 100 times
   taller than wide whose height shrinks is resampled vertically first; any other horizontally first.
"""
import math

import numpy as np

from sketchedit_b200.engine import thumbnail_size  # noqa: F401  (the size rule, one place for the device flow and the tests)

PREC = 22


def factors(src_hw, dst_hw):
    """Pillow's reduce factors (fx, fy) of resize(dst, reducing_gap=2.0) of a whole src_hw = (h, w) image."""
    (h, w), (th, tw) = src_hw, dst_hw
    return int(w / tw / 2.0) or 1, int(h / th / 2.0) or 1


def reduce(a, fx, fy):
    """Image.reduce((fx, fy)) of a uint8 [h, w, c] array, Pillow's arithmetic on every cell."""
    h, w, c = a.shape
    oh, ow = -(-h // fy), -(-w // fx)
    pad = np.zeros((oh * fy, ow * fx, c), np.uint64)
    pad[:h, :w] = a
    s = pad.reshape(oh, fy, ow, fx, c).sum(axis=(1, 3)) % 2 ** 32
    cw = np.minimum(fx, w - np.arange(ow) * fx)
    ch = np.minimum(fy, h - np.arange(oh) * fy)
    n = (ch[:, None] * cw[None, :]).astype(np.uint64)
    m = (np.float32(2 ** 32) / ((256 * n) % 2 ** 32).astype(np.float32)).astype(np.uint64)
    return ((((s + (n // 2)[..., None]) * m[..., None]) % 2 ** 32) >> 24).astype(np.uint8)


def _bicubic(x):
    a = -0.5
    x = np.abs(x)
    near = ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    far = (((x - 5) * x + 8) * x - 4) * a
    return np.where(x < 1.0, near, np.where(x < 2.0, far, 0.0))


def coeff_table(n_in, in1, n_out):
    """Pillow's 8-bit coefficient table of one axis: n_in samples, box (0, in1) with in1 a C float, n_out outputs.
    Returns (bounds [n_out, 2] = (first sample, taps), coeffs [n_out, ksize] with 22 fractional bits, zero past the taps)."""
    in1 = float(np.float32(in1))
    scale = in1 / n_out
    fs = max(scale, 1.0)
    support = 2.0 * fs
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((n_out, 2), np.int64)
    coeffs = np.zeros((n_out, ksize), np.int64)
    for i in range(n_out):
        center = (i + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), n_in) - xmin
        k = _bicubic((np.arange(xmax) + xmin - center + 0.5) * (1.0 / fs))
        ww = 0.0
        for v in k:                      # summed in order, as the C loop does
            ww += v
        w = k / ww if ww != 0.0 else k
        coeffs[i, :xmax] = np.where(w < 0, np.trunc(-0.5 + w * (1 << PREC)), np.trunc(0.5 + w * (1 << PREC)))
        bounds[i] = xmin, xmax
    return bounds, coeffs


def resample(a, axis, in1, n_out):
    """One fixed-point bicubic pass of a uint8 [h, w, c] array along axis (0 rows, 1 columns) with the box end in1."""
    n_in = a.shape[axis]
    bounds, coeffs = coeff_table(n_in, in1, n_out)
    taps = np.arange(coeffs.shape[1])
    idx = np.minimum(bounds[:, :1] + taps[None, :], n_in - 1)        # taps past the bounds carry weight 0
    src = np.moveaxis(a, axis, 0).astype(np.int64)
    acc = (1 << (PREC - 1)) + np.einsum("okxc,ok->oxc", src[idx], coeffs)
    assert np.abs(acc).max() < 2 ** 31                                 # the kernels accumulate in int32
    return np.moveaxis(np.clip(acc >> PREC, 0, 255).astype(np.uint8), 0, axis)


def resize_reducing(a, dst_hw):
    """Image.fromarray(a).resize((tw, th), reducing_gap=2.0) of a uint8 [h, w, 3] array (steps 1 to 3 above)."""
    h, w = a.shape[:2]
    th, tw = dst_hw
    if (h, w) == (th, tw):
        return a.copy()
    fx, fy = factors((h, w), (th, tw))
    in1_w, in1_h = float(np.float32(w / fx)), float(np.float32(h / fy))
    if fx > 1 or fy > 1:
        a = reduce(a, fx, fy)
    rh, rw = a.shape[:2]
    need_h = tw != rw or in1_w != rw
    need_v = th != rh or in1_h != rh
    if rh > rw * 100 and th < rh:
        a = resample(a, 0, in1_h, th)
        return resample(a, 1, in1_w, tw) if need_h else a
    if need_h:
        a = resample(a, 1, in1_w, tw)
    if need_v:
        a = resample(a, 0, in1_h, th)
    return np.ascontiguousarray(a)


def thumbnail(a, size):
    """Image.thumbnail(size) of a uint8 [h, w, 3] array, as a new array (the array itself when it already fits)."""
    h, w = a.shape[:2]
    ts = thumbnail_size(w, h, size)
    if ts is None:
        return a
    return resize_reducing(a, (ts[1], ts[0]))


def photo_like(h, w, seed):
    """A smooth RGB image with edges and noise, like a photo (gradients, a disc, a stripe band, grain)."""
    rs = np.random.RandomState(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    r = 128 + 100 * np.sin(x / max(w, 1) * 6.1 + y / max(h, 1) * 2.3)
    g = 60 + 150 * (y / max(h - 1, 1))
    b = np.where((x - w / 2) ** 2 + (y - h / 3) ** 2 < (min(h, w) / 4) ** 2, 230.0, 40.0)
    b = b + 40 * ((x // 7 + y // 5) % 2)
    img = np.stack([r, g, b], -1) + rs.normal(0, 6, (h, w, 3))
    return np.clip(img, 0, 255).astype(np.uint8)
