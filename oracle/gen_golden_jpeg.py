"""Writes tests/golden/jpeg_pil.npz: baseline JPEG streams written by Pillow, with the shape and the SHA-256 of
`np.asarray(Image.open(f).convert("RGB"))` for each (the decode of odtk/data.py:50).  The Pillow and libjpeg-turbo
versions are recorded.  It also stores streams the GPU decoder must reject (progressive, CMYK) and one truncated
stream.

    python oracle/gen_golden_jpeg.py

Cases: 4:2:0 / 4:2:2 / 4:4:4 and grayscale; qualities 10 / 50 / 95 / 100; optimised Huffman tables; restart markers
every 3 MCUs and every MCU row; sizes 1x1, 8x8, 17x9, 37x53, 33x47 (partial MCUs on both axes), 7x4, 5x3, 12x5
(chroma planes 2 or 3 samples wide); two 640x480 images;
40 seeded random cases (size 1-300 px, sampling, quality, restart markers)."""
import hashlib
import io
import os

import numpy as np
import PIL
from PIL import Image, features

SUB = {"420": 2, "422": 1, "444": 0}


def _image(rng, h, w):
    """Smooth colour gradients, a few flat rectangles with sharp edges and mild noise: content a camera could produce
    (it keeps the streams small at high quality) with enough edges to exercise large AC coefficients."""
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.empty((h, w, 3), np.float64)
    for c in range(3):
        a, b, p = rng.uniform(-1, 1, 3)
        img[..., c] = 128 + 80 * np.sin(a * xx / 23.0 + b * yy / 17.0 + 6 * p)
    for _ in range(4):
        y0, x0 = rng.integers(0, h), rng.integers(0, w)
        img[y0:y0 + rng.integers(1, h + 1), x0:x0 + rng.integers(1, w + 1)] = rng.integers(0, 256, 3)
    img += rng.normal(0, 2.5, img.shape)
    return np.clip(img, 0, 255).round().astype(np.uint8)


def _encode(img, mode, **kw):
    f = io.BytesIO()
    im = Image.fromarray(img, "RGB")
    if mode == "gray":
        im = im.convert("L")
    else:
        kw["subsampling"] = SUB[mode]
    im.save(f, "JPEG", **kw)
    return f.getvalue()


def _cases(rng):
    out = []
    for mode in ("420", "422", "444", "gray"):
        out.append(("%s_q75" % mode, _encode(_image(rng, 61, 90), mode, quality=75)))
    for q in (10, 50, 95, 100):
        out.append(("420_q%d" % q, _encode(_image(rng, 72, 100), "420", quality=q)))
    out.append(("444_q100", _encode(_image(rng, 40, 56), "444", quality=100)))
    out.append(("gray_q100", _encode(_image(rng, 40, 56), "gray", quality=100)))
    out.append(("420_optimize", _encode(_image(rng, 64, 96), "420", quality=85, optimize=True)))
    out.append(("422_optimize", _encode(_image(rng, 50, 70), "422", quality=60, optimize=True)))
    out.append(("420_restart3", _encode(_image(rng, 70, 90), "420", quality=80, restart_marker_blocks=3)))
    out.append(("444_restart3", _encode(_image(rng, 30, 41), "444", quality=80, restart_marker_blocks=3)))
    out.append(("422_restart_rows", _encode(_image(rng, 45, 77), "422", quality=80, restart_marker_rows=1)))
    out.append(("gray_restart_rows", _encode(_image(rng, 33, 40), "gray", quality=80, restart_marker_rows=1)))
    for h, w in ((1, 1), (8, 8), (17, 9), (37, 53), (33, 47), (7, 4), (5, 3), (12, 5)):
        for mode in ("420", "422", "444", "gray"):
            out.append(("%s_%dx%d" % (mode, h, w), _encode(_image(rng, h, w), mode, quality=90)))
    out.append(("420_640x480", _encode(_image(rng, 480, 640), "420", quality=90)))
    out.append(("444_480x640", _encode(_image(rng, 640, 480), "444", quality=90, restart_marker_rows=2)))
    for k in range(40):
        h, w = (int(v) for v in rng.integers(1, 301, 2))
        mode = ("420", "422", "444", "gray")[k % 4]
        kw = {"quality": int(rng.integers(5, 101))}
        if k % 5 == 1:
            kw["optimize"] = True
        if k % 7 == 2:
            kw["restart_marker_blocks"] = int(rng.integers(1, 9))
        out.append(("rand%02d_%s_%dx%d" % (k, mode, h, w), _encode(_image(rng, h, w), mode, **kw)))
    return out


def _rejects(rng):
    img = _image(rng, 24, 32)
    prog = _encode(img, "420", quality=80, progressive=True)
    f = io.BytesIO()
    Image.fromarray(img, "RGB").convert("CMYK").save(f, "JPEG", quality=80)
    return [("progressive", prog), ("cmyk", f.getvalue())]


def main():
    rng = np.random.default_rng(20261016)
    out = {"pillow_version": np.array(PIL.__version__), "libjpeg_turbo_version": np.array(features.version("libjpeg_turbo"))}
    names = []
    for name, data in _cases(rng):
        rgb = np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))
        out[name + "_jpeg"] = np.frombuffer(data, np.uint8)
        out[name + "_shape"] = np.array(rgb.shape, np.int64)
        out[name + "_pil_sha256"] = np.array(hashlib.sha256(np.ascontiguousarray(rgb).tobytes()).hexdigest())
        names.append(name)
    out["names"] = np.array(names)
    rejects = _rejects(rng)
    for name, data in rejects:
        out["reject_" + name] = np.frombuffer(data, np.uint8)
    out["reject_names"] = np.array([r[0] for r in rejects])
    # a stream cut inside its entropy-coded data: Pillow refuses it ("image file is truncated")
    full = _encode(_image(rng, 61, 90), "420", quality=75)
    out["truncated_jpeg"] = np.frombuffer(full[:len(full) * 2 // 3], np.uint8)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "jpeg_pil.npz")
    np.savez_compressed(path, **out)
    print("wrote %s: %d cases, %d bytes of JPEG, Pillow %s, libjpeg-turbo %s" % (
        os.path.normpath(path), len(names), sum(out[n + "_jpeg"].size for n in names), PIL.__version__,
        features.version("libjpeg_turbo")))


if __name__ == "__main__":
    main()
