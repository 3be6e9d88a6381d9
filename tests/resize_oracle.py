"""Numpy restatement of Pillow's 8-bit bilinear resampling (`Image.resize(size, Image.BILINEAR)` on an RGB image),
the resize of the reference's inference data loader (odtk/data.py:55-60), and of the resize ratio it uses.

Pillow resamples separably: a horizontal pass into a uint8 image, then a vertical pass.  Per output position it takes
the triangle filter over a window whose support grows with the downscale factor, computes the tap weights in IEEE
double, normalises them by their sum, converts them to fixed point with 22 fractional bits (rounding half away from
zero) and accumulates uint8 x weight in integers from 1 << 21, then shifts right by 22 and clamps to [0, 255].  A pass
whose input and output lengths are equal is the identity (its weights are 1 and 0).  numpy's float64 element-wise
operations round like the C code (no contraction), so this is bit-exact; tests/test_resize_host.py pins it to Pillow
through tests/golden/resize_pil.npz.  The CUDA kernel (odtk_preprocess_resize_u8) restates the same operations."""
import hashlib
import math

import numpy as np

PRECISION_BITS = 22


def resize_ratio(h, w, resize, max_size):
    """odtk/data.py:55-60 with the same Python float expressions: (ratio, dst_h, dst_w)."""
    ratio = resize / min(h, w)
    if ratio * max(h, w) > max_size:
        ratio = max_size / max(h, w)
    return ratio, int(ratio * h), int(ratio * w)


def coeffs(in_size, out_size):
    """Triangle-filter taps of one axis: (first input index [out], fixed-point weights [out, ksize] int64).  Taps past
    an output position's window have weight 0."""
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    support = 1.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    center = 0.0 + (np.arange(out_size, dtype=np.float64) + 0.5) * scale
    ss = 1.0 / filterscale
    lo = np.maximum(np.trunc(center - support + 0.5).astype(np.int64), 0)
    hi = np.minimum(np.trunc(center + support + 0.5).astype(np.int64), in_size)
    count = hi - lo
    j = np.arange(ksize)
    arg = ((lo[:, None] + j[None, :]).astype(np.float64) - center[:, None] + 0.5) * ss
    a = np.abs(arg)
    w = np.where(a < 1.0, 1.0 - a, 0.0)
    w[j[None, :] >= count[:, None]] = 0.0
    ww = np.zeros(out_size, np.float64)
    for t in range(ksize):                                  # the C loop's summation order
        ww = ww + w[:, t]
    k = np.where(ww[:, None] != 0.0, w / np.where(ww == 0.0, 1.0, ww)[:, None], w)
    one = float(1 << PRECISION_BITS)
    fixed = np.where(k < 0, np.trunc(-0.5 + k * one), np.trunc(0.5 + k * one)).astype(np.int64)
    return lo, fixed


def _pass(img, axis, out_size):
    """One resampling pass of a uint8 [H, W, 3] image along `axis` (1: horizontal, 0: vertical)."""
    in_size = img.shape[axis]
    lo, k = coeffs(in_size, out_size)
    acc = np.full((out_size,) + tuple(s for i, s in enumerate(img.shape) if i != axis), 1 << (PRECISION_BITS - 1), np.int64)
    src = np.moveaxis(img.astype(np.int64), axis, 0)
    for t in range(k.shape[1]):
        idx = np.minimum(lo + t, in_size - 1)               # weight 0 wherever the index had to be clamped
        acc += src[idx] * k[:, t].reshape((-1,) + (1,) * (src.ndim - 1))
    out = np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)
    return np.moveaxis(out, 0, axis)


def resize_bilinear(img, dst_h, dst_w):
    """uint8 [H, W, 3] -> uint8 [dst_h, dst_w, 3], bit-identical to PIL Image.resize((dst_w, dst_h), BILINEAR)."""
    img = np.ascontiguousarray(img, dtype=np.uint8)
    out = img if img.shape[1] == dst_w else _pass(img, 1, dst_w)
    return out if img.shape[0] == dst_h else _pass(out, 0, dst_h)


def digest(img):
    """SHA-256 of a uint8 image's bytes (C order): how tests/golden/resize_pil.npz stores Pillow's outputs."""
    return hashlib.sha256(np.ascontiguousarray(img, dtype=np.uint8).tobytes()).hexdigest()


def fixture_output(g, name):
    """Pillow's BILINEAR output of fixture case `name` (g: the loaded resize_pil.npz): rebuilt with resize_bilinear and
    checked against the stored digest of Pillow's own bytes, so what is returned IS Pillow's output, bit for bit."""
    dh, dw = (int(v) for v in g[name + "_dst"])
    out = resize_bilinear(g[name + "_img"], dh, dw)
    if digest(out) != str(g[name + "_pil_sha256"]):
        raise AssertionError("%s: the numpy resampler differs from Pillow %s's output" % (name, g["pillow_version"]))
    return out
