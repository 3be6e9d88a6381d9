"""CPU tests of the training input path (retinanet_examples_b200/data.py, tests/augment_oracle.py): the oracle plus the
iterator's host work (draws, targets) reproduce every batch of tests/golden/augment_ref.npz, which the unmodified
reference CocoDataset / RotatedCocoDataset wrote; the oracle matches Pillow and torchvision exhaustively where that is
cheap; odtk_augment_image_t's ctypes layout matches the header."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest
import torch

import augment_oracle as O
from retinanet_examples_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def fixture(golden_dir):
    return np.load(os.path.join(golden_dir, "augment_ref.npz"))


def _pillow():
    try:
        from PIL import Image  # noqa: F401
        return True
    except ImportError:
        return False


def _progressive_ok(it, indices):
    """The progressive fixture file needs Pillow on the host; skip the batches that hold it without Pillow."""
    return _pillow() or all("prog" not in it.coco.imgs[it.ids[i]]["file_name"] for i in indices)


class _LoggedRandom(random.Random):
    def __init__(self, seed):
        super().__init__(seed)
        self.log = []

    def randint(self, a, b):
        v = super().randint(a, b)
        self.log.append(float(v))
        return v

    def normalvariate(self, mu, sigma):
        v = super().normalvariate(mu, sigma)
        self.log.append(v)
        return v


def test_oracle_reproduces_fixture(fixture, tmp_path):
    checked = 0
    for ci, cfg in enumerate(O.fixture_configs(fixture)):
        ann = O.fixture_dir(fixture, str(tmp_path), cfg["rotated"])
        rng = _LoggedRandom(cfg["seed"])
        it = O.make_iterator(cfg, str(tmp_path), ann, rng)
        for bi, idx in enumerate(cfg["batches"]):
            if not _progressive_ok(it, idx):
                pytest.skip("Pillow is not installed: the progressive file has no host decoder")
            data, target = O.oracle_batch(it, idx)
            assert tuple(data.shape) == tuple(fixture["cfg%d_b%d_shape" % (ci, bi)]), cfg["name"]
            assert O.sha256(data) == cfg["sha256"][bi], (cfg["name"], bi)
            if cfg["training"]:
                assert torch.equal(target, torch.from_numpy(fixture["cfg%d_b%d_target" % (ci, bi)])), (cfg["name"], bi)
            checked += 1
        np.testing.assert_array_equal(np.array(rng.log), fixture["cfg%d_draws" % ci], err_msg=cfg["name"])
    assert checked == sum(len(c["batches"]) for c in O.fixture_configs(fixture))


def test_coco_standin_order(fixture, tmp_path):
    import json
    ann = O.fixture_dir(fixture, str(tmp_path), False)
    from retinanet_examples_b200.data import Coco
    c = Coco(ann)
    d = json.loads(str(fixture["annotations_json"]))
    assert list(c.imgs) == [im["id"] for im in d["images"]]
    assert c.cat_ids == [x["id"] for x in d["categories"]]
    for id, anns in c.img_to_anns.items():
        assert anns == [a for a in d["annotations"] if a["image_id"] == id]


def test_augment_image_layout():
    """odtk_augment_image_t: the ctypes struct has the header's field offsets and size."""
    fields = [f for f, _ in _lib.AugmentImage._fields_]
    src = ['#include <stddef.h>', '#include <stdio.h>', '#include "odtk_b200.h"', 'int main(void) {',
           '  printf("%zu\\n", sizeof(odtk_augment_image_t));']
    src += ['  printf("%%zu\\n", offsetof(odtk_augment_image_t, %s));' % f for f in fields]
    src += ['  return 0;', '}']
    d = os.environ.get("TMPDIR", "/tmp")
    c, exe = os.path.join(d, "augment_layout_%d.c" % os.getpid()), os.path.join(d, "augment_layout_%d" % os.getpid())
    with open(c, "w") as f:
        f.write("\n".join(src))
    try:
        subprocess.run(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), c, "-o", exe], check=True)
        got = [int(x) for x in subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split()]
    finally:
        for p in (c, exe):
            if os.path.exists(p):
                os.remove(p)
    assert got == [ctypes.sizeof(_lib.AugmentImage)] + [getattr(_lib.AugmentImage, f).offset for f in fields]


def _all_colours():
    c = np.arange(1 << 24, dtype=np.uint32)
    return np.stack([(c >> 16) & 255, (c >> 8) & 255, c & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)


@pytest.mark.skipif(not _pillow(), reason="Pillow is not installed")
def test_hsv_round_trip_all_colours():
    from PIL import Image
    img = _all_colours()
    hsv = np.asarray(Image.fromarray(img).convert("HSV")).copy()
    assert np.array_equal(hsv, O.rgb_to_hsv(img))
    for shift in (0, 1, 128, 255):
        x = hsv.copy()
        x[..., 0] = (x[..., 0].astype(np.int32) + shift) & 255
        assert np.array_equal(np.asarray(Image.fromarray(x, "HSV").convert("RGB")), O.adjust_hue(img, shift)), shift


@pytest.mark.skipif(not _pillow(), reason="Pillow is not installed")
def test_adjust_hue_matches_torchvision():
    from PIL import Image
    tf = pytest.importorskip("torchvision.transforms.functional")
    img = _all_colours()[::7, ::5].copy()
    for f in (0.0, 0.0002, -0.0002, 0.003, -0.004, 0.25, -0.37, 0.5, -0.5):
        ref = np.asarray(tf.adjust_hue(Image.fromarray(img), f))
        assert np.array_equal(ref, O.adjust_hue(img, O.hue_shift_u8(f))), f


@pytest.mark.skipif(not _pillow(), reason="Pillow is not installed")
def test_blend_every_pair():
    from PIL import Image
    a = np.repeat(np.arange(256, dtype=np.uint8), 256).reshape(256, 256)
    b = np.tile(np.arange(256, dtype=np.uint8), 256).reshape(256, 256)
    A, B = Image.fromarray(a), Image.fromarray(b)
    factors = list(np.linspace(0.0, 2.5, 180)) + [1e-7, 0.002, 0.998, 0.999999, 1.0, 1.0000001, 1.002, 254.9, 255.0, 300.5]
    for f in factors:
        f = float(np.float32(f))
        assert np.array_equal(np.asarray(Image.blend(A, B, f)), O.blend(a, b, f)), f


@pytest.mark.skipif(not _pillow(), reason="Pillow is not installed")
def test_luma_all_colours():
    from PIL import Image
    img = _all_colours()
    assert np.array_equal(np.asarray(Image.fromarray(img).convert("L")), O.luma(img))


@pytest.mark.skipif(not _pillow(), reason="Pillow is not installed")
def test_rotate_every_small_size():
    from PIL import Image
    rng = np.random.default_rng(0)
    for h in range(1, 25):
        for w in range(1, 25):
            a = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            im = Image.fromarray(a)
            for rot in (1, 2, 3):
                for expand in (False, True):
                    ref = np.asarray(im.rotate(rot * 90, expand=expand))
                    got = O.rotate(a, rot, expand)
                    assert ref.shape == got.shape and np.array_equal(ref, got), (h, w, rot, expand)


def test_augment_size_query_checks():
    """The host checks of odtk_augment_u8's size query."""
    L = _lib.lib()
    t = (_lib.AugmentImage * 1)()
    t[0].h, t[0].w = 5, 8
    q = lambda ch, cw, xb=120: L.odtk_augment_u8(None, xb, ctypes.byref(t), None, 1, ch, cw, None, 0, None, None, None, None)
    assert q(5, 8) > 0
    assert q(4, 8) == -1                      # larger than the canvas
    assert q(5, 8, 119) == -1                 # outside x
    t[0].rot, t[0].expand = 1, 1
    assert q(5, 8) == -1 and q(8, 5) > 0      # expand turns it to 8 x 5
    t[0].rot = 4
    assert q(8, 8) == -1
    t[0].rot, t[0].flags = 0, 16
    assert q(8, 8) == -1
    t[0].flags, t[0].contrast = 2, -1.0
    assert q(8, 8) == -1
    t[0].contrast, t[0].hue_shift = 1.0, 256
    assert q(8, 8) == -1


@pytest.mark.parametrize("world,rank", [(2, 0), (2, 1), (3, 2)])
def test_distributed_sharding_matches_the_reference(fixture, tmp_path, monkeypatch, world, rank):
    """world > 1: the images are sharded as the reference's DataLoader does, by torch's DistributedSampler over the
    dataset's len(ids) images, then batched by batch_size // world with the last partial batch kept."""
    import torch.distributed as dist
    from torch.utils.data.distributed import DistributedSampler
    monkeypatch.setattr(dist, "is_available", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda *a, **k: world)
    monkeypatch.setattr(dist, "get_rank", lambda *a, **k: rank)
    ann = O.fixture_dir(fixture, str(tmp_path), False)
    from retinanet_examples_b200 import data
    it = data.DataIterator(str(tmp_path), [96, 160], 256, 8, 32, world, ann, training=True, rng=random.Random(0))
    n = len(it.ids)
    want = list(DistributedSampler(range(n), num_replicas=world, rank=rank))
    assert it._indices() == want
    assert it.batch_size == 8 // world
    assert len(it) == -(-len(want) // (8 // world))
    single = data.DataIterator(str(tmp_path), [96, 160], 256, 8, 32, 1, ann, training=True, rng=random.Random(0))
    assert single._indices() == list(range(n)) and len(single) == -(-n // 8)
