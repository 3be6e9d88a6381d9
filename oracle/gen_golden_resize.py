"""Writes tests/golden/resize_pil.npz: seeded uint8 RGB images, their resize ratio and destination size from the
reference's formula (odtk/data.py:55-60: ratio = resize / min side, capped so that ratio * max side <= max_size), and
the SHA-256 of Pillow's Image.BILINEAR result at that size (its uint8 [dst_h, dst_w, 3] bytes; the full-resolution
outputs would make the file megabytes large, and a digest pins them bit for bit just as well -- tests/resize_oracle.py
rebuilds each output and checks it against the digest).  The Pillow version is recorded.

    python oracle/gen_golden_resize.py

Cases: non-integer downscales (one capped by max_size), an upscale, portrait and landscape, odd sizes, a tiny image, a
same-size pass, and images with saturated 0 / 255 edges that exercise both clamps."""
import hashlib
import os

import numpy as np
import PIL
from PIL import Image

RESIZE, MAX_SIZE = 800, 1333
# (name, src_h, src_w, pattern)
CASES = [
    ("down_1500x2000", 1500, 2000, "big_blocks"), # downscale 1.875x, landscape
    ("down_cap_100x1400", 100, 1400, "blocks"),    # ratio capped by max_size: 1333 / 1400
    ("up_480x640", 480, 640, "blocks"),           # COCO-like upscale to 800x1066
    ("portrait_640x427", 640, 427, "blocks"),     # portrait upscale
    ("odd_333x517", 333, 517, "blocks"),
    ("tiny_3x5", 3, 5, "noise"),
    ("same_800x1333", 800, 1333, "blocks"),       # no resampling
    ("edges_150x100", 150, 100, "edges"),         # 0 / 255 stripes: overshoot clamps at both ends
    ("edges_1050x850", 1050, 850, "big_edges"),   # same, downscaling
]


def _image(rng, h, w, pattern):
    """Random blocks of 5x7 pixels (20x28 for the large downscales; every block edge is a step the filter has to
    interpolate and the file stays small), per-pixel noise for the small images, and for "edges" 0 / 255 stripes over the
    image (a 48-pixel band along the top and left for the large one)."""
    if pattern == "noise":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    bh, bw = (20, 28) if pattern.startswith("big") else (5, 7)
    img = rng.integers(0, 256, (-(-h // bh), -(-w // bw), 3), dtype=np.uint8).repeat(bh, 0).repeat(bw, 1)[:h, :w].copy()
    if pattern.endswith("edges"):
        band = 48 if pattern.startswith("big") else max(h, w)
        img[:, 0:band:4] = 255
        img[:, 1:band:4] = 0
        img[0:band:5] = 0
        img[1:band:5] = 255
    return img


def _resize_ratio(h, w):
    size = (w, h)                                             # PIL's im.size order
    ratio = RESIZE / min(size)
    if ratio * max(size) > MAX_SIZE:
        ratio = MAX_SIZE / max(size)
    dw, dh = (int(ratio * d) for d in size)
    return ratio, dh, dw


def main():
    rng = np.random.default_rng(20261015)
    out = {"pillow_version": np.array(PIL.__version__), "resize": np.int64(RESIZE), "max_size": np.int64(MAX_SIZE),
           "names": np.array([c[0] for c in CASES])}
    for name, h, w, pattern in CASES:
        img = _image(rng, h, w, pattern)
        ratio, dh, dw = _resize_ratio(h, w)
        res = np.asarray(Image.fromarray(img, "RGB").resize((dw, dh), Image.BILINEAR))
        out[name + "_img"] = img
        out[name + "_ratio"] = np.float64(ratio)
        out[name + "_dst"] = np.array([dh, dw], np.int64)
        out[name + "_pil_sha256"] = np.array(hashlib.sha256(np.ascontiguousarray(res).tobytes()).hexdigest())
        print("%-20s %4dx%-4d -> %4dx%-4d ratio %.6f" % (name, h, w, dh, dw, ratio))
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "resize_pil.npz")
    np.savez_compressed(path, **out)
    print("wrote", os.path.normpath(path), "with Pillow", PIL.__version__)


if __name__ == "__main__":
    main()
