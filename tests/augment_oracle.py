"""numpy restatement of the training input path of odtk/data.py (CocoDataset / RotatedCocoDataset.__getitem__ with
training=True, :64-123, and collate_fn): rotation by quarter turns, horizontal flip, Pillow's ImageEnhance blends, the
uint8 HSV round trip of torchvision's PIL adjust_hue, normalisation, padding; and the target transforms.  Written from
Pillow's C arithmetic (Blend.c, Convert.c, Geometry.c) with numpy float32 / float64 standing for C float / double.
Independent of the CUDA kernels; the tests hold it against Pillow itself where Pillow is importable."""
import numpy as np

MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
F32 = np.float32


def rotate(im, rot, expand):
    """Image.rotate(90 * rot[, expand]) on uint8 [h, w, 3] (numpy, counter-clockwise).  90 / 270 on a non-square image
    without expand: NEAREST about the centre, same size, black fill (the floor of Pillow's half-integer coordinates)."""
    h, w = im.shape[:2]
    if rot == 0:
        return im.copy()
    if rot == 2:
        return im[::-1, ::-1].copy()
    if expand or h == w:
        return np.ascontiguousarray(np.rot90(im, rot))
    r = np.arange(h)[:, None]
    c = np.arange(w)[None, :]
    if rot == 1:
        sc, sr = (w + h - 1 - 2 * r) >> 1, (h - w + 1 + 2 * c) >> 1
    else:
        sc, sr = (w - h + 1 + 2 * r) >> 1, (w + h - 1 - 2 * c) >> 1
    sc, sr = np.broadcast_to(sc, (h, w)), np.broadcast_to(sr, (h, w))
    ok = (sr >= 0) & (sr < h) & (sc >= 0) & (sc < w)
    out = np.zeros_like(im)
    out[ok] = im[sr[ok], sc[ok]]
    return out


def blend(a, b, alpha):
    """Image.blend(a, b, alpha) per uint8 channel (Blend.c): a + alpha * (b - a) in C float; truncated for alpha in
    [0, 1], otherwise clamped to [0, 255] first."""
    alpha = F32(alpha)
    t = np.asarray(a, np.int32).astype(F32) + alpha * (np.asarray(b, np.int32) - np.asarray(a, np.int32)).astype(F32)
    if 0.0 <= alpha <= 1.0:
        return t.astype(np.uint8)
    return np.clip(t, 0.0, 255.0).astype(np.uint8)


def luma(im):
    """convert("L") of uint8 RGB (Convert.c L24): (r * 19595 + g * 38470 + b * 7471 + 0x8000) >> 16."""
    im = im.astype(np.int64)
    return ((im[..., 0] * 19595 + im[..., 1] * 38470 + im[..., 2] * 7471 + 0x8000) >> 16).astype(np.uint8)


def rgb_to_hsv(im):
    """convert("HSV") of uint8 RGB (Convert.c rgb2hsv_row)."""
    r, g, b = (im[..., k].astype(np.int32) for k in range(3))
    maxc, minc = np.maximum(r, np.maximum(g, b)), np.minimum(r, np.minimum(g, b))
    grey = maxc == minc
    cr = np.where(grey, 1, maxc - minc).astype(F32)
    s = cr / np.where(maxc == 0, 1, maxc).astype(F32)
    rc, gc, bc = ((maxc - x).astype(F32) / cr for x in (r, g, b))
    h = np.where(r == maxc, bc - gc,
                 np.where(g == maxc, (2.0 + rc.astype(np.float64) - bc).astype(F32),
                          (4.0 + gc.astype(np.float64) - rc).astype(F32)))
    h = np.fmod(h.astype(np.float64) / 6.0 + 1.0, 1.0).astype(F32)
    uh = np.clip((h.astype(np.float64) * 255.0).astype(np.int32), 0, 255)
    us = np.clip((s.astype(np.float64) * 255.0).astype(np.int32), 0, 255)
    uh, us = np.where(grey, 0, uh), np.where(grey, 0, us)
    return np.stack([uh, us, maxc], -1).astype(np.uint8)


def _round(x):
    """C round(): half away from zero."""
    return np.sign(x) * np.floor(np.abs(x) + 0.5)


def hsv_to_rgb(hsv):
    """convert("RGB") of uint8 HSV (Convert.c hsv2rgb)."""
    h, s, v = (hsv[..., k].astype(F32) for k in range(3))
    hd = h.astype(np.float64) * 6.0 / 255.0
    i = np.floor(hd).astype(np.int32)
    f = (hd - i.astype(F32)).astype(F32)
    fs = (s.astype(np.float64) / 255.0).astype(F32)
    vd = v.astype(np.float64)
    p = np.clip(_round(vd * (1.0 - fs.astype(np.float64))), 0, 255).astype(np.int32)
    q = np.clip(_round(vd * (1.0 - (fs * f).astype(np.float64))), 0, 255).astype(np.int32)
    t = np.clip(_round(vd * (1.0 - fs.astype(np.float64) * (1.0 - f.astype(np.float64)))), 0, 255).astype(np.int32)
    vi = hsv[..., 2].astype(np.int32)
    k = i % 6
    sel = [(vi, t, p), (q, vi, p), (p, vi, t), (p, q, vi), (t, p, vi), (vi, p, q)]
    out = np.zeros(hsv.shape, np.int32)
    for j, (a, b, c) in enumerate(sel):
        m = k == j
        out[..., 0] = np.where(m, a, out[..., 0])
        out[..., 1] = np.where(m, b, out[..., 1])
        out[..., 2] = np.where(m, c, out[..., 2])
    grey = hsv[..., 1] == 0
    out = np.where(grey[..., None], vi[..., None], out)
    return out.astype(np.uint8)


def hue_shift_u8(hue_factor):
    """The uint8 shift torchvision's PIL adjust_hue adds to H: np.int32(hue_factor * 255).astype(np.uint8)."""
    return int(np.int32(hue_factor * 255).astype(np.uint8))


def adjust_hue(im, shift):
    hsv = rgb_to_hsv(im)
    hsv[..., 0] = (hsv[..., 0].astype(np.int32) + shift) & 255
    return hsv_to_rgb(hsv)


def augment(im, rot=0, expand=False, flip=False, brightness=None, contrast=None, hue_shift=None, saturation=None):
    """Steps 1-6 on uint8 [h, w, 3]: an adjustment given as None is disabled (its factor is the clipped draw)."""
    im = rotate(im, rot, expand)
    if flip:
        im = im[:, ::-1].copy()
    if brightness is not None:
        im = blend(np.zeros_like(im), im, brightness)
    if contrast is not None:
        mean = int(float(int(luma(im).astype(np.int64).sum())) / float(im.shape[0] * im.shape[1]) + 0.5)
        im = blend(np.full_like(im, mean), im, contrast)
    if hue_shift is not None:
        im = adjust_hue(im, hue_shift)
    if saturation is not None:
        im = blend(np.repeat(luma(im)[..., None], 3, -1), im, saturation)
    return im


def normalize(im, mean=MEAN, std=STD):
    """uint8 [h, w, 3] -> float32 [3, h, w]: float(u8) / 255, - mean, / std, in float32 as the reference's tensors."""
    x = im.astype(F32).transpose(2, 0, 1) / F32(255)
    return np.stack([(x[k] - F32(mean[k])) / F32(std[k]) for k in range(3)])


def collate(datas, stride):
    """Pad each [3, h, w] to the stride, then to the batch maximum, with zeros: float32 [n, 3, H, W]."""
    hs = max(-(-d.shape[1] // stride) * stride for d in datas)
    ws = max(-(-d.shape[2] // stride) * stride for d in datas)
    out = np.zeros((len(datas), 3, hs, ws), F32)
    for i, d in enumerate(datas):
        out[i, :, :d.shape[1], :d.shape[2]] = d
    return out


# ---- the augment_ref.npz fixture -------------------------------------------------------------------------------------
def fixture_configs(g):
    import json
    return json.loads(str(g["configs_json"]))


def fixture_dir(g, d, rotated):
    """Write the fixture's files and its annotation JSON into directory d; returns the JSON path."""
    import os
    for k in g.files:
        if k.startswith("file:"):
            with open(os.path.join(d, k[5:]), "wb") as f:
                f.write(g[k].tobytes())
    path = os.path.join(d, "rotated.json" if rotated else "axis.json")
    with open(path, "w") as f:
        f.write(str(g["annotations_rotated_json" if rotated else "annotations_json"]))
    return path


def make_iterator(cfg, d, ann, rng, world=1):
    from retinanet_examples_b200 import data
    cls = data.RotatedDataIterator if cfg["rotated"] else data.DataIterator
    return cls(d, cfg["resize"], cfg["max_size"], 8, 32, world, ann, training=cfg["training"], rng=rng, **cfg["kwargs"])


def decode_file(path):
    """uint8 [h, w, 3] of a fixture file: the numpy JPEG decoder, or Pillow for what it does not take."""
    import jpeg_oracle
    with open(path, "rb") as f:
        data = f.read()
    try:
        return jpeg_oracle.decode(data)
    except ValueError:
        import io
        from PIL import Image
        return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


def oracle_batch(it, indices):
    """What the iterator's batch(indices) computes, with the package's draws and target transforms and this module's
    pixels: (data float32 [n, 3, H, W], target float32 [n, max_det, 5 or 6] or None)."""
    import torch
    import resize_oracle
    datas, targets = [], []
    for i in indices:
        id = it.ids[i]
        im = decode_file("{}/{}".format(it.path, it.coco.imgs[id]["file_name"]))
        h, w = im.shape[:2]
        ratio, dh, dw, angle, flip, (fb, fc, fh, fs) = it._draw(h, w)
        im = resize_oracle.resize_bilinear(im, dh, dw)
        im = augment(im, angle // 90 if it.rotate_augment else 0, it.rotated, flip, fb, fc,
                     None if fh is None else hue_shift_u8(fh), fs)
        datas.append(normalize(im))
        if it.training:
            boxes, cats = it._target(id)
            targets.append(torch.cat([it._transform(boxes, ratio, angle, flip, dh, dw), cats], dim=1))
    target = None
    if it.training:
        m = max(t.size(0) for t in targets)
        target = torch.stack([torch.cat([t, torch.ones([m - t.size(0), t.size(1)]) * -1]) for t in targets], 0)
    return collate(datas, it.stride), target


def sha256(a):
    import hashlib
    return hashlib.sha256(np.ascontiguousarray(a, np.float32).tobytes()).hexdigest()
