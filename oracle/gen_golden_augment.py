"""Writes tests/golden/augment_ref.npz: the training batches of the UNMODIFIED reference odtk/data.py (CocoDataset /
RotatedCocoDataset.__getitem__ + collate_fn, imported through oracle/ref_import.py) over a dozen small Pillow-encoded
JPEGs (baseline 4:2:0, 4:4:4, grayscale and one progressive file), for several augmentation configurations.

    python oracle/gen_golden_augment.py

pycocotools is not a dependency: a stand-in `pycocotools.coco.COCO` over the JSON (image order, each image's
annotations in file order, category ids in file order) is put in sys.modules before odtk.data is imported.  For each
configuration the generator seeds a random.Random, routes the reference's `random` calls to it (and logs every draw),
indexes the dataset batch by batch and collates.  Stored: the files, the JSON, seeds, batches, draws, the SHA-256 of
each batch's contiguous NCHW float32 `data` bytes and every `target` in full, plus the Pillow / torchvision versions."""
import hashlib
import io
import json
import os
import random
import sys
import types

import numpy as np
import PIL
import torch
import torchvision
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_import  # noqa: E402

# (name, h, w, kind)
FILES = [("a_420_37x53.jpg", 37, 53, "420"), ("b_444_61x29.jpg", 61, 29, "444"), ("c_gray_45x45.jpg", 45, 45, "gray"),
         ("d_420_80x51.jpg", 80, 51, "420"), ("e_prog_33x70.jpg", 33, 70, "progressive"),
         ("f_444_50x77.jpg", 50, 77, "444"), ("g_420_23x31.jpg", 23, 31, "420"), ("h_gray_70x41.jpg", 70, 41, "gray"),
         ("i_420_64x64.jpg", 64, 64, "420"), ("j_444_39x96.jpg", 39, 96, "444"), ("k_420_99x58.jpg", 99, 58, "420"),
         ("l_420_480x640.jpg", 480, 640, "420")]
SMALL = list(range(11))
BIG = [11]
DEFAULT = dict(augment_brightness=0.002, augment_contrast=0.002, augment_hue=0.0002, augment_saturation=0.002)
LARGE = dict(augment_brightness=0.8, augment_contrast=0.9, augment_hue=0.4, augment_saturation=1.2)
JIT = dict(resize=[96, 160], max_size=256)
# (name, rotated, kwargs, seed, batches)
CONFIGS = [
    ("axis_default", False, dict(JIT, **DEFAULT), 1, [SMALL[:4], SMALL[4:8], SMALL[8:]]),
    ("axis_rotate_default", False, dict(JIT, rotate_augment=True, **DEFAULT), 2, [SMALL[:6], SMALL[6:]]),
    ("axis_rotate_large", False, dict(JIT, rotate_augment=True, **LARGE), 3, [SMALL[:5], SMALL[5:]] * 2),
    ("axis_rotate_plain", False, dict(JIT, rotate_augment=True), 4, [SMALL]),
    ("rotated_rotate_default", True, dict(JIT, rotate_augment=True, **DEFAULT), 5, [SMALL[:6], SMALL[6:]]),
    ("rotated_rotate_large", True, dict(JIT, rotate_augment=True, **LARGE), 6, [SMALL[:5], SMALL[5:]] * 2),
    ("rotated_absolute", True, dict(JIT, rotate_augment=True, absolute_angle=True, **LARGE), 7, [SMALL[:6], SMALL[6:]] * 2),
    ("rotated_plain", True, dict(JIT, **DEFAULT), 8, [SMALL]),
    ("axis_default_640x480", False, dict(resize=[640, 1024], max_size=1333, **DEFAULT), 9, [BIG]),
    ("axis_eval", False, dict(resize=120, max_size=256, training=False), 10, [SMALL[:6]]),
]
STRIDE = 32


def _image(rng, h, w, gray):
    blocks = rng.integers(0, 256, (-(-h // 6), -(-w // 6), 1 if gray else 3), dtype=np.uint8).repeat(6, 0).repeat(6, 1)
    img = blocks[:h, :w].astype(np.int32) + rng.integers(-20, 21, (h, w, 1 if gray else 3))
    img = np.clip(img, 0, 255).astype(np.uint8)
    return Image.fromarray(img[..., 0] if gray else img)


def make_files(rng):
    out = {}
    for name, h, w, kind in FILES:
        im = _image(rng, h, w, kind == "gray")
        b = io.BytesIO()
        if kind == "444":
            im.save(b, "JPEG", quality=85, subsampling=0)
        elif kind == "progressive":
            im.save(b, "JPEG", quality=80, progressive=True)
        else:
            im.save(b, "JPEG", quality=80 if h < 400 else 60)
        out[name] = b.getvalue()
    return out


def make_annotations(rng):
    cats = [{"id": 7, "name": "c7"}, {"id": 3, "name": "c3"}, {"id": 11, "name": "c11"}]
    images, anns = [], []
    aid = 1
    for i, (name, h, w, _) in enumerate(FILES):
        images.append({"id": 100 + 3 * i, "file_name": name, "height": h, "width": w})
        nbox = 0 if i == 2 else int(rng.integers(1, 5))
        for j in range(nbox):
            bw, bh = float(rng.uniform(2, w / 2)), float(rng.uniform(2, h / 2))
            if i == 5 and j == 0:
                bw, bh = 0.5, 0.75                     # under 1 px both ways: skipped by _get_target
            box = [round(float(rng.uniform(0, w - bw)), 2), round(float(rng.uniform(0, h - bh)), 2), round(bw, 2), round(bh, 2)]
            if j % 2:
                box.append(round(float(rng.uniform(-1.5, 1.5)), 3))   # a theta: RotatedCocoDataset reads it
            ann = {"id": aid, "image_id": 100 + 3 * i, "category_id": cats[int(rng.integers(0, 3))]["id"], "bbox": box,
                   "area": bw * bh, "iscrowd": 0}
            anns.append(ann)
            aid += 1
    rng.shuffle(anns)                                  # per-image order = file order, not id order
    return {"images": images, "annotations": anns, "categories": cats}


def _coco_standin():
    mod = types.ModuleType("pycocotools.coco")

    class COCO:
        def __init__(self, path):
            with open(path) as f:
                self.dataset = json.load(f)
            self.imgs = {im["id"]: im for im in self.dataset["images"]}
            self.anns = {a["id"]: a for a in self.dataset["annotations"]}
            self.img_to_anns = {}
            for a in self.dataset["annotations"]:
                self.img_to_anns.setdefault(a["image_id"], []).append(a)

        def getCatIds(self):
            return [c["id"] for c in self.dataset["categories"]]

        def getAnnIds(self, imgIds):
            return [a["id"] for a in self.img_to_anns.get(imgIds, [])]

        def loadAnns(self, ids):
            return [self.anns[i] for i in ids]

        def loadImgs(self, id):
            return [self.imgs[id]]

    mod.COCO = COCO
    pkg = types.ModuleType("pycocotools")
    pkg.coco = mod
    sys.modules["pycocotools"] = pkg
    sys.modules["pycocotools.coco"] = mod


class LoggedRandom:
    """The two `random` functions odtk/data.py calls, from one seeded generator, logging every value drawn."""

    def __init__(self, seed):
        self.r, self.log = random.Random(seed), []

    def randint(self, a, b):
        v = self.r.randint(a, b)
        self.log.append(float(v))
        return v

    def normalvariate(self, mu, sigma):
        v = self.r.normalvariate(mu, sigma)
        self.log.append(v)
        return v


def main():
    rng = np.random.default_rng(2024)
    files = make_files(rng)
    ann = make_annotations(rng)
    _coco_standin()
    ref_import.import_reference()
    import odtk.data as D
    import tempfile
    # the axis-aligned datasets take [x, y, w, h] only
    ann_axis = dict(ann, annotations=[dict(a, bbox=a["bbox"][:4]) for a in ann["annotations"]])
    out = {"pillow_version": np.array(PIL.__version__), "torchvision_version": np.array(torchvision.__version__),
           "annotations_json": np.array(json.dumps(ann_axis)), "annotations_rotated_json": np.array(json.dumps(ann)),
           "stride": np.array(STRIDE)}
    for name, data in files.items():
        out["file:" + name] = np.frombuffer(data, np.uint8)
    meta = []
    with tempfile.TemporaryDirectory() as d:
        for name, data in files.items():
            with open(os.path.join(d, name), "wb") as f:
                f.write(data)
        ann_path = os.path.join(d, "ann.json")
        for ci, (cname, rotated, kw, seed, batches) in enumerate(CONFIGS):
            with open(ann_path, "w") as f:      # fresh JSON: RotatedCocoDataset appends theta to the loaded boxes
                json.dump(ann if rotated else ann_axis, f)
            kw = dict(kw)
            resize, max_size = kw.pop("resize"), kw.pop("max_size")
            training = kw.pop("training", True)
            cls = D.RotatedCocoDataset if rotated else D.CocoDataset
            ds = cls(d, resize=resize, max_size=max_size, stride=STRIDE, annotations=ann_path, training=training, **kw)
            lr = LoggedRandom(seed)
            D.random = lr
            digests = []
            for bi, idx in enumerate(batches):
                res = ds.collate_fn([ds[i] for i in idx])
                data = res[0]
                digests.append(hashlib.sha256(data.contiguous().numpy().tobytes()).hexdigest())
                out["cfg%d_b%d_shape" % (ci, bi)] = np.array(data.shape)
                if training:
                    out["cfg%d_b%d_target" % (ci, bi)] = res[1].numpy()
                else:
                    out["cfg%d_b%d_ids" % (ci, bi)] = res[1].numpy()
                    out["cfg%d_b%d_ratios" % (ci, bi)] = res[2].numpy()
            D.random = random
            out["cfg%d_draws" % ci] = np.array(lr.log, np.float64)
            meta.append({"name": cname, "rotated": rotated, "resize": resize, "max_size": max_size, "training": training,
                         "kwargs": kw, "seed": seed, "batches": batches, "sha256": digests})
    out["configs_json"] = np.array(json.dumps(meta))
    path = os.path.join(os.path.dirname(HERE), "tests", "golden", "augment_ref.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
